"""Measures the --reference path on one GPU and prints one JSON line.

A seeded genome of config 2's 24 GRCh38-length contigs (times --scale) with a GRCh38-like gap layout (telomere and centromere 'N'
blocks, scattered gaps, single bases) and soft-masked stretches is written as plain FASTA (60 columns) and as BGZF (compressed with
snfb_deflate_bgzf), with their .fai, into a temporary directory.  Device arm: snfb_load_reference wall time and its timing marks for both
files, then snfb_fetch_reference for 50,000 seeded DEL intervals plus their anchor bases.  CPU arm: a numpy N scan of the plain text and
a zlib inflate of the BGZF members on all cores.  Also the card's name and power limit, and device memory in use with the genome
resident (cudaMemGetInfo through torch).

    python scripts/reference_bench.py [--scale 1.0] [--seed 7]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from sniffles_b200 import abi, bamio, binding, fasta, synth  # noqa: E402


def contig(rng, L):
    s = np.frombuffer(b"ACGT", "u1")[rng.integers(0, 4, L, dtype=np.uint8)]
    for a in rng.integers(0, L, max(1, L // 20_000)):                   # soft-masked repeats: about half the bases
        s[a:a + int(rng.integers(1_000, 20_000))] |= 0x20
    gaps = [(0, 10_000), (L - 10_000, L), (L // 2 - L // 60, L // 2 + L // 60)]
    gaps += [(int(a), int(a) + int(rng.integers(100, 100_000))) for a in rng.integers(0, L, 12)]
    gaps += [(int(a), int(a) + 1) for a in rng.integers(0, L, 20)]
    for a, b in gaps:
        s[max(0, a):min(L, b)] = ord("N")
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    rng = np.random.default_rng(a.seed)
    lengths = [max(200_000, int(x * a.scale)) for x in synth.GRCH38]
    names = [f"chr{k + 1}" for k in range(len(lengths))]
    tmp = tempfile.mkdtemp(prefix="refbench_")
    plain, gz = os.path.join(tmp, "g.fa"), os.path.join(tmp, "g.fa.gz")
    fai, off = [], 0
    with open(plain, "wb") as f:
        for n, L in zip(names, lengths):
            head = f">{n}\n".encode()
            f.write(head)
            off += len(head)
            s = contig(rng, L)
            full = L // 60
            body = np.full((full, 61), 10, np.uint8)
            body[:, :60] = s[:full * 60].reshape(full, 60)
            f.write(body.tobytes())
            if L % 60:
                f.write(s[full * 60:].tobytes() + b"\n")
            fai.append(f"{n}\t{L}\t{off}\t60\t61")
            off += L + (L + 59) // 60
    with open(plain + ".fai", "w") as f:
        f.write("\n".join(fai) + "\n")
    text = np.fromfile(plain, dtype="u1")
    ctx = binding.Context(0)
    members = []
    step = 0xff00 * 60000
    for k in range(0, len(text), step):
        z, _ = ctx.deflate_bgzf(text[k:k + step].tobytes())
        members.append(z)
    zdata = b"".join(members)
    with open(gz, "wb") as f:
        f.write(zdata + bamio._BGZF_EOF)
    with open(gz + ".fai", "w") as f:
        f.write("\n".join(fai) + "\n")
    out = dict(workload="reference_load", scale=a.scale, genome_bp=int(sum(lengths)), plain_bytes=int(len(text)), bgzf_bytes=len(zdata))
    try:
        import torch
        out["gpu"] = torch.cuda.get_device_name(0)
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        out["power_limit"] = q.stdout.strip()
    except Exception as e:       # the numbers are still printed; the card is then unnamed
        out["gpu_query_error"] = str(e)
    _, rows = fasta.parse_fai(open(plain + ".fai").read())
    table = np.zeros(len(rows), abi.REF_CONTIG_DTYPE)
    table["length"], table["linebases"], table["linewidth"] = rows["length"], rows["linebases"], rows["linewidth"]
    for arm, data, is_bgzf in (("plain", text, False), ("bgzf", np.frombuffer(zdata, "u1"), True)):
        table["offset"] = rows["offset"]
        ctx.load_reference(data, table, is_bgzf=is_bgzf)          # warm-up (allocations)
        t0 = time.perf_counter()
        runs, coff = ctx.load_reference(data, table, is_bgzf=is_bgzf)
        out[f"{arm}_load_s"] = time.perf_counter() - t0
        out[f"{arm}_marks_ms"] = {n: round(ms, 3) for n, ms, _ in ctx.timings()}
    out["n_runs"] = int(len(runs))
    qr = np.random.default_rng(a.seed + 1)
    n = 50_000
    q = np.zeros(2 * n, abi.REF_QUERY_DTYPE)
    c = qr.integers(0, len(lengths), n)
    dl = np.minimum(np.exp(qr.normal(5.5, 1.2, n)).astype(np.int64) + 50, 50_000)
    st = (qr.random(n) * (np.array(lengths)[c] - dl - 1)).astype(np.int64)
    q["contig"][:n], q["start"][:n], q["length"][:n] = c, st, dl + 1
    q["contig"][n:], q["start"][n:], q["length"][n:] = c, st, 1
    q["out_off"] = np.concatenate(([0], np.cumsum(q["length"][:-1])))
    ctx.fetch_reference(q)
    t0 = time.perf_counter()
    ctx.fetch_reference(q)
    out["fetch_100k_queries_s"] = time.perf_counter() - t0
    out["fetch_marks_ms"] = {n: round(ms, 3) for n, ms, _ in ctx.timings()}
    try:
        import torch
        free, total = torch.cuda.mem_get_info(0)
        out["device_mem_used_gb_with_genome"] = round((total - free) / 1e9, 2)
    except Exception:
        pass
    t0 = time.perf_counter()
    m = text == 78
    d = np.diff(np.concatenate(([0], m.view(np.int8), [0])))
    int(np.count_nonzero(d == 1))
    out["cpu_numpy_nscan_s"] = time.perf_counter() - t0
    blocks = [(po, pl) for _, po, pl, _ in bamio.bgzf_members(zdata)]
    t0 = time.perf_counter()
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        sum(len(x) for x in ex.map(lambda b: zlib.decompress(zdata[b[0]:b[0] + b[1]], -15), blocks, chunksize=256))
    out["cpu_zlib_inflate_s"] = time.perf_counter() - t0
    out["cpu_threads"] = os.cpu_count()
    ctx.close()
    for p in (plain, plain + ".fai", gz, gz + ".fai"):
        os.remove(p)
    os.rmdir(tmp)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
