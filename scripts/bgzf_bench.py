"""BGZF compression of a large VCF: the device encoder (snfb_deflate_bgzf) against zlib on the CPU.

    python scripts/bgzf_bench.py [--mb 200] [--calls 10] [--warmup 2] [--seed 1]

Builds a seeded text of fixture VCF lines tiled with shifted POS (tests/bgzf_host.tiled_vcf_text), checks that the device output
inflates back with zlib, then times:
  * the CPU arms first, in worker processes forked before this process touches CUDA: zlib level 6 on one core (what
    pysam.tabix_index does for the reference's `--vcf out.vcf.gz`), and levels 1 and 6 over all cores, one 0xff00 block per task;
  * the device: the whole call host bytes -> host bytes (warm-up calls, then --calls timed calls) and the kernel time of its
    "deflate" mark (snfb_last_timings).
Prints one JSON line with the times, the size ratios against zlib levels 1 and 6, and the card's name and power limit read with
nvidia-smi in the same run.
"""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bgzf_host  # noqa: E402

BLOCK = 0xff00
_DATA = None


def _member_size(args):
    k, level = args
    c = zlib.compressobj(level, zlib.DEFLATED, -15)
    return len(c.compress(_DATA[k:k + BLOCK]) + c.flush()) + 26


def cpu_arm(data, level, procs):
    """seconds and total BGZF bytes of zlib at `level` over `procs` forked workers (1 = this process)"""
    global _DATA
    _DATA = data
    ks = [(k, level) for k in range(0, len(data), BLOCK)]
    t0 = time.perf_counter()
    if procs == 1:
        sizes = [_member_size(a) for a in ks]
    else:
        with mp.get_context("fork").Pool(procs) as pool:
            sizes = pool.map(_member_size, ks, chunksize=16)
    return time.perf_counter() - t0, sum(sizes)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=200)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    data = bgzf_host.tiled_vcf_text(a.mb << 20, a.seed)
    ncpu = os.cpu_count() or 1
    # CPU arms before CUDA is initialised in this process: forking after it is not safe
    t_z6_1, n_z6 = cpu_arm(data, 6, 1)
    t_z1_all, n_z1 = cpu_arm(data, 1, ncpu)
    t_z6_all, _ = cpu_arm(data, 6, ncpu)

    from sniffles_b200 import binding
    ctx = binding.Context(0)
    z, co = ctx.deflate_bgzf(data)
    import gzip
    assert gzip.decompress(z) == data, "round trip through zlib failed"
    for _ in range(a.warmup):
        ctx.deflate_bgzf(data)
    call_s, kern_ms = [], []
    for _ in range(a.calls):
        t0 = time.perf_counter()
        z2, _ = ctx.deflate_bgzf(data)
        call_s.append(time.perf_counter() - t0)
        kern_ms.append(next(ms for n, ms, _ in ctx.timings() if n == "deflate"))
        assert z2 == z
    ctx.close()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    med = lambda xs: sorted(xs)[len(xs) // 2]
    mb = len(data) / 1e6
    print(json.dumps({
        "metric": "bgzf_compress", "input_mb": round(mb, 1), "blocks": len(co), "gpu": q[0] if q else "unknown",
        "device_kernel_ms_median": round(med(kern_ms), 3), "device_kernel_ms_min": round(min(kern_ms), 3),
        "device_call_ms_median": round(1e3 * med(call_s), 3), "device_call_ms_min": round(1e3 * min(call_s), 3),
        "kernel_gb_per_s": round(mb / med(kern_ms), 2), "call_gb_per_s": round(mb / 1e3 / med(call_s), 2),
        "zlib6_1core_ms": round(1e3 * t_z6_1, 1), "zlib1_allcores_ms": round(1e3 * t_z1_all, 1), "zlib6_allcores_ms": round(1e3 * t_z6_all, 1), "cpu_cores": ncpu,
        "size_vs_zlib1": round(len(z) / n_z1, 4), "size_vs_zlib6": round(len(z) / n_z6, 4), "device_bytes": len(z)}))


if __name__ == "__main__":
    main()
