"""Where the step's wall time goes after its last kernel: the device-to-host copies at the end of snfb_run.  Prints one JSON line with
the card and its power limit; over --steps steps after --warmup (the workload of bench.py, inputs resident, the same ctx.run call) the
median wall time, the median `total` device time of the marks and the gap between them; the bytes of every device-to-host copy of
the step; and, from a separate torch.profiler run with CUDA activities (traces written under --out-dir), the start, end and duration
of every `Memcpy DtoH` of a step relative to the end of the step's last kernel.

    python scripts/copy_tail_bench.py [--config 2] [--scale 1.0] [--steps 30] [--warmup 5] [--profile-steps 3] [--slices K] [--out-dir DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power}


def copy_bytes(res, n_task):
    """the device-to-host copies of one snfb_run with candidates and ALT bytes (api.cu run_pipeline / enqueue_cand_copies)"""
    from sniffles_b200 import abi
    counters = 2 * 8 * 30         # DevCounters, once when stage B ends and once at the end (the consensus work table goes with each)
    return {"cand": len(res.cand) * abi.CAND_DTYPE.itemsize, "rn_off": 4 * len(res.cand), "cand_leads": len(res.cand_leads) * abi.LEAD_DTYPE.itemsize,
            "rnames": 8 * len(res.rnames), "task_cov": 8 * n_task, "alt": len(res.alt), "counters": counters}


def trace_tail(path):
    """every DtoH copy of the traced step, relative to the end of its last kernel (ms)"""
    with open(path) as f:
        ev = json.load(f)["traceEvents"]
    kern = [e for e in ev if e.get("ph") == "X" and e.get("cat") == "kernel"]
    cps = [e for e in ev if e.get("ph") == "X" and e.get("cat") == "gpu_memcpy" and "DtoH" in e.get("name", "")]
    k_end = max(e["ts"] + e["dur"] for e in kern)
    k_start = min(e["ts"] for e in kern)
    out = []
    for e in sorted(cps, key=lambda e: e["ts"]):
        if e["ts"] + e["dur"] < k_start:
            continue
        a = e.get("args", {})
        out.append({"bytes": a.get("bytes"), "stream": a.get("stream"), "start_ms": (e["ts"] - k_end) / 1e3, "end_ms": (e["ts"] + e["dur"] - k_end) / 1e3,
                    "dur_ms": e["dur"] / 1e3, "GBps": (a.get("bytes") or 0) / (e["dur"] * 1e3) if e["dur"] else None})
    return {"kernels_span_ms": (k_end - k_start) / 1e3, "last_copy_end_ms": max([c["end_ms"] for c in out] or [0.0]), "copies": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--slices", type=int, default=None, help="snfb_set_consensus_slices (default: the library's)")
    ap.add_argument("--out-dir", default=None, help="where the traces and the JSON line go (default: a new temporary directory)")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("copy_tail_bench needs a CUDA device")
    from sniffles_b200 import abi, binding, synth, config as sconfig
    a.out_dir = a.out_dir or tempfile.mkdtemp(prefix="snfb_copy_tail_")
    os.makedirs(a.out_dir, exist_ok=True)
    out = {"card": card(), "config": a.config, "scale": a.scale}
    cfg = sconfig.default_config(*(["--mosaic"] if a.config == 3 else []))
    blk = synth.config_block(a.config, a.scale, threads=os.cpu_count() or 1)
    blk.pack16()
    L = binding.lib()
    for arr in (blk.rec16, blk.cigar16, blk.var, blk.seq):
        if arr.nbytes:
            L.snfb_pin_host(C.c_void_p(arr.ctypes.data), arr.nbytes)
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    if a.slices:
        ctx.set_consensus_slices(a.slices)
        out["slices"] = a.slices
    ctx.load(blk)
    for _ in range(a.warmup):
        res = ctx.run(want_leads=False, want_cands=True, want_seqs=True, copy=False)
    torch.cuda.synchronize()
    wall, dev = [], []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        res = ctx.run(want_leads=False, want_cands=True, want_seqs=True, copy=False)
        wall.append((time.perf_counter() - t0) * 1e3)
        dev.append(next(ms for n, ms, _ in ctx.timings() if n == "total"))
    gaps = [w - d for w, d in zip(wall, dev)]
    out["steps"] = a.steps
    out["wall_ms_median"], out["device_ms_median"], out["gap_ms_median"] = statistics.median(wall), statistics.median(dev), statistics.median(gaps)
    out["gap_ms_min"], out["gap_ms_max"] = min(gaps), max(gaps)
    out["reruns"] = ctx.rerun_count()
    out["d2h_bytes"] = copy_bytes(res, len(blk.task))
    stage = {}
    for n, ms, _ in ctx.timings():
        stage[n] = stage.get(n, 0.0) + ms
    out["stage_ms_last_step"] = stage
    from torch.profiler import profile, ProfilerActivity
    traces = []
    for k in range(a.profile_steps):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            ctx.run(want_leads=False, want_cands=True, want_seqs=True, copy=False)
            torch.cuda.synchronize()
        path = os.path.join(a.out_dir, f"step{k}_slices{a.slices or 0}.pt.trace.json")
        prof.export_chrome_trace(path)
        traces.append(trace_tail(path))
    out["profiled"] = traces
    ctx.close()
    line = json.dumps(out)
    with open(os.path.join(a.out_dir, f"copy_tail{a.slices or ''}.json"), "w") as f:
        f.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
