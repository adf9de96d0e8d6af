"""Coordinate sort on the GPU (bamio.sort_bam -> snfb_sort_bam), printed as one JSON line.

Input: the config-6 BAM of scripts/call_sample_bench.py (bench.py --config 6's generator: four 1.5 Mb contigs, 30x, 15 kb reads, noisy
base qualities), rewritten by tests/bam_sort_host.shuffled_bam in a seeded random record order (zlib level 6, htslib's member cuts), in a
temporary directory.  Arms:
  * "default":      budgets sized from the free device memory (the whole file is one window and one bucket);
  * "quarter":      bucket_bytes = 1/4 of the inflated size, so every bucket pass re-reads the windows holding its records;
  * "sorted_input": the default arm's output sorted again with --window-mb windows and quarter buckets: each window's records fall in
                    one or two buckets, so a bucket pass skips the other windows;
  * "cpu":          the host restatement (tests/bam_sort_host.py: records through bamio.BgzfReader, a stable Python sort, zlib members)
                    over the first --cpu-records records of the shuffled file, as a records-per-second rate.  It is not samtools.
Each GPU arm: wall seconds of sort_bam (file reading and writing, the device work), the device milliseconds per phase snfb_sort_bam
reports (CUDA events), the host's member-cut loop, windows, buckets, window reads of the input, output bytes against the input's zlib-6
bytes, and the device bytes held at the widest point; the best of --repeat runs after one warm-up.  Every arm's output is checked to
inflate to the default arm's stream.  The card's name and power limit are read in the same run."""
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
    ap.add_argument("--window-mb", type=float, default=16.0)
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--cpu-records", type=int, default=2000)
    a = ap.parse_args()
    import bam_sort_host as H
    from call_sample_bench import make_input
    from sniffles_b200 import bamio, binding
    with tempfile.TemporaryDirectory() as tmp:
        path, n_rec, _ = make_input("c6", 1.0, tmp)
        shuf = H.shuffled_bam(path, os.path.join(tmp, "shuf.bam"), seed=6)
        os.remove(path)
        inflated = sum(isize for _, _, _, isize in bamio.bgzf_members(open(shuf, "rb").read()))
        in_bytes = os.path.getsize(shuf)
        res = dict(metric="bam_sort", gpu=gpu_info(), records=n_rec, input_zlib6_bytes=in_bytes, inflated_bytes=inflated)
        stream = None
        out0 = os.path.join(tmp, "sorted.bam")
        arms = (("default", shuf, out0, {}), ("quarter", shuf, os.path.join(tmp, "q.bam"), dict(bucket_bytes=inflated // 4)),
                ("sorted_input", out0, os.path.join(tmp, "s2.bam"), dict(window_bytes=int(a.window_mb * (1 << 20)), bucket_bytes=inflated // 4)))
        for arm, src, out, budgets in arms:
            ctx = binding.Context(0)                  # a fresh context per arm: its buffers only grow, and device_bytes reports them
            bamio.sort_bam(src, out, ctx=ctx, **budgets)                                # warm-up
            best = None
            for _ in range(a.repeat):
                st = {}
                t = time.perf_counter()
                bamio.sort_bam(src, out, ctx=ctx, stats=st, **budgets)
                wall = time.perf_counter() - t
                if best is None or wall < best[0]:
                    best = (wall, st)
            ctx.close()
            data = b"".join(d for _, d in H.members(out))
            stream = data if stream is None else stream
            assert data == stream, f"arm {arm}: the output differs from the default arm's"
            wall, st = best
            res[arm] = dict(wall_s=round(wall, 4), device_ms={k[3:]: round(st[k], 3) for k in ("ms_keys", "ms_sort", "ms_layout", "ms_scatter", "ms_deflate")},
                            layout_host_ms=round(st["ms_layout_host"], 3), windows=st["n_windows"], buckets=st["n_buckets"], input_reads=st["n_input_reads"],
                            bytes_in=st["bytes_in"], bytes_out=st["bytes_out"], out_over_zlib6=round(st["bytes_out"] / in_bytes, 4),
                            device_bytes=st["device_bytes"], records=st["n_records"], inflated_gb_per_s_wall=round(inflated / wall / 1e9, 3))
        t = time.perf_counter()
        header, recs = H.records(shuf)
        recs = recs[:a.cpu_records]
        header = H.rewrite_header(header)
        recs = H.sort_records(header, recs)
        data = header + b"".join(recs)
        u = 0
        for s in H.member_sizes(len(header), [len(r) for r in recs]):
            bamio._bgzf_block(data[u:u + s])
            u += s
        cpu_s = time.perf_counter() - t
        res["cpu_restatement_prefix"] = dict(records=len(recs), seconds=round(cpu_s, 3), records_per_s=round(len(recs) / cpu_s, 1))
        res["gpu_records_per_s_wall"] = round(n_rec / res["default"]["wall_s"], 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
