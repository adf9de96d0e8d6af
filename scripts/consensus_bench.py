"""Stage C (the INS consensus) on a bench.py workload (config 2, full size, by default).  Prints one JSON line: the card, its power limit
and top SM clock; the stage-C interval of ctx.timings() (`consensus` + `consensus_align` + `consensus_vote`: mean, median, min and max over
--steps timed steps after --warmup, inputs resident as bench.py loads them) with the step's device time; from a separate torch.profiler
run of --prof-steps steps, the device time per step of k_prep, k_align and k_vote; and the shape of the work: the heavy and light
(candidate, supporting read) items and a histogram of the consensus length L, counted from the step's candidates as k_plan counts them.

    python scripts/consensus_bench.py [--config 2] [--scale 1.0] [--steps 30] [--warmup 5] [--prof-steps 3] [--out FILE]
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

STAGE_C = ("consensus", "consensus_align", "consensus_vote")
HEAVY_L = 3000                    # consensus.cuh: items of longer insertions are taken by a whole block
HAS_SEQ = 1 << 10                 # SNFB_LF_HAS_SEQ
L_EDGES = [0, 100, 300, 1000, 3000, 10000, 1 << 31]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, power, sm = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "clocks_max_sm": sm}


def kernel_label(name):
    """stable label of a stage-C kernel from its demangled name, None for every other kernel"""
    m = re.search(r"consensus::(k_prep|k_align|k_vote)\b", name)
    return m.group(1) if m else None


def work_shape(res, cfg):
    """k_plan's items: per INS candidate with an ALT, nm seq-bearing leads, L = the best read's length; with a consensus
    (nm - 1 >= consensus_min_reads) one item per other read, heavy when L > HEAVY_L"""
    c = res.cand
    ins = np.flatnonzero((c["svtype"] == 0) & (c["alt_off"] >= 0) & (c["alt_len"] > 0))
    has = np.concatenate([[0], np.cumsum((res.cand_leads["flags"] & HAS_SEQ) != 0)])
    lo, n = c["lead_off"][ins].astype(np.int64), c["lead_n"][ins].astype(np.int64)
    nm = has[lo + n] - has[lo]
    L = c["alt_len"][ins].astype(np.int64)
    cons = (nm - 1 >= cfg.consensus_min_reads) & (not cfg.no_consensus)
    items = np.where(cons, nm - 1, 0)
    heavy = L > HEAVY_L
    hist = np.histogram(L[cons], bins=L_EDGES)[0]
    return {"candidates_with_consensus": int(cons.sum()), "items_heavy": int(items[heavy].sum()), "items_light": int(items[~heavy].sum()),
            "L_histogram": {f"{a}-{b - 1}" if b < (1 << 31) else f">={a}": int(h) for a, b, h in zip(L_EDGES, L_EDGES[1:], hist)},
            "L_items_histogram": {f"{a}-{b - 1}" if b < (1 << 31) else f">={a}": int(items[cons & (L >= a) & (L < b)].sum()) for a, b in zip(L_EDGES, L_EDGES[1:])}}


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
        raise SystemExit("consensus_bench needs a CUDA device")
    from sniffles_b200 import abi, binding, config as sconfig
    out = {"card": card(), "config": a.config, "scale": a.scale}
    spec = bench.workload_spec(a)
    cfg = sconfig.default_config(*spec["cli"])
    acfg = abi.Config.from_sniffles(cfg)
    blk, _ = bench.workload(a, None, os.cpu_count() or 1)
    blk.pack16()
    ctx = binding.Context(0)
    ctx.set_config(acfg)
    ctx.load(blk)

    def step(leads=False):
        return ctx.run(want_leads=leads, want_cands=True, want_seqs=True, copy=False)

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    sc, dev = [], []
    for _ in range(a.steps):
        step()
        t = {}
        for n, ms, _b in ctx.timings():
            t[n] = t.get(n, 0.0) + ms
        sc.append(sum(t.get(k, 0.0) for k in STAGE_C))
        dev.append(t["total"])
    torch.cuda.synchronize()
    out["stage_c_ms"] = {"mean": statistics.mean(sc), "median": statistics.median(sc), "min": min(sc), "max": max(sc)}
    out["device_ms_per_step"] = statistics.mean(dev)
    out["work"] = work_shape(step(), acfg)

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
