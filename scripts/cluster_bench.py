"""Stage B's per-cluster kernels on a bench.py workload (config 2, full size, by default).  Prints one JSON line: the card, its power
limit and top SM clock; the `cluster_call` interval of ctx.timings() (mean, median, min and max over --steps timed steps after --warmup,
inputs resident as bench.py loads them) with the step's device time; and, from a separate torch.profiler run of --prof-steps steps, the
device time per step of each kernel of that interval (k_cluster_warp<48>, k_cluster_warp<128>, k_cluster_block) on its own.

    python scripts/cluster_bench.py [--config 2] [--scale 1.0] [--steps 30] [--warmup 5] [--prof-steps 3] [--out FILE]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, power, sm = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": sm}


def kernel_label(name):
    """stable label of a stage-B cluster kernel from its demangled name, None for every other kernel"""
    m = re.search(r"k_cluster_warp<(\d+)", name)
    if m:
        return f"k_cluster_warp<{m.group(1)}>"
    return "k_cluster_block" if "k_cluster_block" in name else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prof-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("cluster_bench needs a CUDA device")
    from sniffles_b200 import abi, binding, config as sconfig
    out = {"card": card(), "config": a.config, "scale": a.scale}
    spec = bench.workload_spec(a)
    cfg = sconfig.default_config(*spec["cli"])
    blk, _ = bench.workload(a, None, os.cpu_count() or 1)
    blk.pack16()
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    ctx.load(blk)

    def step():
        return ctx.run(want_leads=False, want_cands=True, want_seqs=True, copy=False)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    cl, dev = [], []
    for _ in range(a.steps):
        res = step()
        t = {}
        for n, ms, _b in ctx.timings():
            t[n] = t.get(n, 0.0) + ms
        cl.append(t["cluster_call"])
        dev.append(t["total"])
    torch.cuda.synchronize()
    out["candidates"] = int(len(res.cand))
    out["cluster_call_ms"] = {"mean": statistics.mean(cl), "median": statistics.median(cl), "min": min(cl), "max": max(cl)}
    out["device_ms_per_step"] = statistics.mean(dev)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.prof_steps):
            step()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        lab = kernel_label(ev.key)
        if lab is not None:
            d = per.setdefault(lab, {"ms": 0.0, "launches": 0})
            d["ms"] += ev.device_time_total / 1e3
            d["launches"] += ev.count
    out["kernels_ms_per_step"] = {k: {"ms": v["ms"] / a.prof_steps, "launches": v["launches"] / a.prof_steps} for k, v in sorted(per.items())}
    ctx.close()
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
