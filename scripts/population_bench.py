"""Population annotation benchmark (--combine-population): one JSON line.

A seeded synthetic population SNF (about 250k variants over config 2's 24 contigs, INS ALTs of realistic lengths) is written to a
temporary directory, decoded by the host (combine_run.Population) and loaded to the device; about 200k calls drawn near its variants are
matched.  Reported: the host decode; CUDA-event medians of population_load and population_match over repeated calls after two warm-up
calls; the device memory the table holds (cudaMemGetInfo around the first load); oracle/population.py on a bounded sample of the calls,
per call on that sample (not extrapolated); the GPU's name and power limit, read in the same run.
    python scripts/population_bench.py [--variants N] [--queries N] [--reps K] [--cpu-sample N]"""
import argparse
import gzip
import json
import os
import pickle
import random
import statistics
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import population as opop                   # noqa: E402
from sniffles_b200 import combine_run, snf, synth, tasks  # noqa: E402

CONTIGS = [(f"chr{c}", n) for c, n in zip([*range(1, 23), "X", "Y"], synth.GRCH38)]
BS = 100_000


def write_population(path, n_var, rng):
    """mostly 50-400 bp INS, some mobile-element and 6-kb ones; DEL / DUP / INV of 50 bp - 5 kb; BND"""
    V = snf.population_class()
    total = sum(n for _, n in CONTIGS)
    index, parts, offset = {}, [], 0
    for name, length in CONTIGS:
        blocks = {}
        for i in range(max(1, round(n_var * length / total))):
            pos, st = rng.randrange(length), rng.choice(["INS", "INS", "DEL", "DEL", "DUP", "INV", "BND"])
            r = rng.random()
            svlen = ((rng.randrange(50, 400) if r < 0.8 else rng.randrange(280, 340) if r < 0.9 else rng.randrange(5900, 6100)) if st == "INS"
                     else 0 if st == "BND" else rng.randrange(50, 5000) * (-1 if st == "DEL" else 1))
            alt = "".join(rng.choice("ACGT") for _ in range(svlen)) if st == "INS" else f"<{st}>"
            v = V(name, pos, f"{st}.{i}", alt, st, svlen, pos + abs(svlen), rng.random(), rng.randrange(40, 51), rng.randrange(1, 40))
            blocks.setdefault(pos // BS * BS, {t: [] for t in snf.TYPES} | {"_COVERAGE": {}})[st].append(v)
        index[name] = {}
        for b in sorted(blocks):
            parts.append(gzip.compress(pickle.dumps(blocks[b])))
            index[name][str(b)] = [(offset, len(parts[-1]))]
            offset += len(parts[-1])
    header = {"config": {"snf_block_size": BS, "contig_lengths": CONTIGS}, "index": index, "population": {"version": 1, "name": "Population",
              "description": "synthetic", "size": 50}}
    with open(path, "wb") as f:
        f.write((json.dumps(header) + "\n").encode() + b"".join(parts))


def queries(pop, n_q, rng):
    q = {k: [] for k in ("contig", "svtype", "pos", "svlen", "alt")}
    for _ in range(n_q):
        i = rng.randrange(len(pop.variants))
        st, a = int(pop.cols["svtype"][i]), bytearray(pop.alts[i])
        for _ in range(rng.randrange(0, 1 + len(a) // 20) if st == 0 else 0):
            a[rng.randrange(len(a))] = rng.choice(b"ACGT")
        q["contig"].append(int(pop.cols["contig"][i]))
        q["svtype"].append(st)
        q["pos"].append(max(0, int(pop.cols["pos"][i]) + rng.randrange(-200, 200)))
        q["svlen"].append(0 if st == 4 else int(pop.cols["svlen"][i]) + rng.randrange(-30, 30))
        q["alt"].append(bytes(a))
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", type=int, default=250_000)
    ap.add_argument("--queries", type=int, default=200_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-sample", type=int, default=2000)
    a = ap.parse_args()
    import torch
    rng = random.Random(2026)
    prm = (250, 1000, 0.7)                           # combine_match, combine_match_max, combine_pctseq
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "population.snf")
        write_population(path, a.variants, rng)
        t0 = time.perf_counter()
        pop = combine_run.Population(path, [name for name, _ in CONTIGS])
        decode_s = time.perf_counter() - t0
    q = queries(pop, a.queries, rng)
    ctx = tasks.device_context(0)
    free0, _ = torch.cuda.mem_get_info()
    pop.load(ctx)
    free1, _ = torch.cuda.mem_get_info()
    ms = {"population_load": [], "population_match": []}
    for k in range(a.reps + 2):                      # two warm-up rounds of each step
        for step in (lambda: pop.load(ctx), lambda: ctx.population_match(*q.values(), *prm, BS)):
            step()
            for name, t, _ in ctx.timings():
                if name in ms and k >= 2:
                    ms[name].append(t)
    best = ctx.population_match(*q.values(), *prm, BS)
    n_cpu = min(a.cpu_sample, a.queries)
    table = dict(pop.cols, alt=pop.alts)
    t0 = time.perf_counter()
    want = opop.match(table, {k: v[:n_cpu] for k, v in q.items()}, *prm, BS)
    cpu_s = time.perf_counter() - t0
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"bench": "population", "gpu": gpu, "variants": len(pop.variants), "queries": a.queries, "matched": int((best >= 0).sum()),
                      "decode_s": round(decode_s, 3), "population_load_ms": round(statistics.median(ms["population_load"]), 3),
                      "population_match_ms": round(statistics.median(ms["population_match"]), 3), "reps": a.reps, "table_bytes": int(free0 - free1),
                      "cpu_oracle_sample": n_cpu, "cpu_oracle_us_per_query": round(1e6 * cpu_s / n_cpu, 1), "cpu_sample_agrees": best[:n_cpu].tolist() == want}))


if __name__ == "__main__":
    main()
