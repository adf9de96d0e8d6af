"""Index build time on the GPU (bamio.build_index -> snfb_index_bam), printed as one JSON line.

Input: the config-6 BAM of scripts/call_sample_bench.py (bench.py --config 6's generator: four 1.5 Mb contigs, 30x, 15 kb reads; DEFLATE
level 1, noisy base qualities), written to a temporary directory.  Arms:
  * "one_window": BAI with the default window (sized from the free device memory: the whole file is one window);
  * "windows":    BAI with --window-mb windows, so the file is several times larger than a window and records cross window edges;
  * "csi":        CSI with the default window;
  * "cpu":        the host restatement (tests/bam_index_host.py, one record at a time through bamio.BgzfReader) over the first
                  --cpu-records records, as a records-per-second rate.
Each GPU arm: wall seconds of build_index (file reading, the device work, serialization; a CSI's compression), the device milliseconds
snfb_index_bam reports (CUDA events around its phases), windows used and the device bytes held at the widest point; the best of --repeat
runs after one warm-up build.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--window-mb", type=float, default=64.0)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--cpu-records", type=int, default=2000)
    a = ap.parse_args()
    import bam_index_host as H
    from call_sample_bench import make_input
    from sniffles_b200 import bamio, binding
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        path, n_rec, _ = make_input("c6", 1.0, tmp)
        write_s = time.perf_counter() - t0
        bam_bytes = os.path.getsize(path)
        inflated = sum(isize for _, _, _, isize in bamio.bgzf_members(open(path, "rb").read()))
        res = dict(metric="bam_index", gpu=gpu_info(), records=n_rec, bam_bytes=bam_bytes, inflated_bytes=inflated, write_s=round(write_s, 2))
        ref = None
        for arm, fmt, window in (("one_window", "bai", None), ("windows", "bai", int(a.window_mb * (1 << 20))), ("csi", "csi", None)):
            ctx = binding.Context(0)                  # a fresh context per arm: its buffers only grow, and device_bytes reports them
            bamio.build_index(path, fmt, window_bytes=window, ctx=ctx)                  # warm-up
            best = None
            for _ in range(a.repeat):
                st = {}
                t = time.perf_counter()
                data = bamio.build_index(path, fmt, window_bytes=window, ctx=ctx, stats=st)
                wall = time.perf_counter() - t
                if best is None or wall < best[0]:
                    best = (wall, st)
            if fmt == "bai":
                ref = data if ref is None else ref
                assert data == ref, "the windowed build differs from the one-window build"
            wall, st = best
            res[arm] = dict(wall_s=round(wall, 4), device_ms=round(st["device_ms"], 3), windows=st["n_windows"], device_bytes=st["device_bytes"],
                            records=st["n_records"], inflated_gb_per_s_wall=round(inflated / wall / 1e9, 3))
            ctx.close()
        t = time.perf_counter()
        contigs, recs = H.rows(path, a.cpu_records)
        H.tables(contigs, recs)
        cpu_s = time.perf_counter() - t
        res["cpu"] = dict(records=len(recs), seconds=round(cpu_s, 3), records_per_s=round(len(recs) / cpu_s, 1),
                          extrapolated_s=round(n_rec * cpu_s / max(len(recs), 1), 1))
        res["gpu_records_per_s_wall"] = round(n_rec / res["one_window"]["wall_s"], 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
