"""Force-calling benchmark: snfb_genotype_targets on BASELINE config 2 at full size (resident block), 1,000,000 targets = the run's
candidates jittered plus seeded decoys.  Prints one JSON line: card and power limit, the "genotype" device time (median of 10 calls
after 2 warm-ups), the host time to parse and to write 1M records, the match count, and the CPU arm: oracle/genotype.py's matching on one
core, same targets.  The CPU arm leaves out the coverage restatement: its per-base vectors of a 3 Gbp genome do not fit in host memory next
to the resident block (tests/test_gpu_genotype.py checks it at 1/100 scale).

    python scripts/genotype_bench.py [--scale 1.0] [--targets 1000000] [--no-cpu]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]

from sniffles_b200 import abi, binding, genotype, synth  # noqa: E402
from sniffles_b200 import config as sconfig  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = [x.strip() for x in q.splitlines()[0].split(",")]
        return name, power
    except Exception as e:       # the numbers are still printed, without the card
        return f"unknown ({e})", "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--targets", type=int, default=1_000_000)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    blk = synth.config_block(2, a.scale)
    cfg = sconfig.default_config()
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    ctx.load(blk)
    res = ctx.run()
    cols = synth.genotype_targets(res.cand, len(blk.task), blk.task["contig_len"], np.random.default_rng(11), a.targets)
    ms = []
    for i in range(12):
        match = ctx.genotype_targets(*cols, cfg.combine_match, cfg.combine_match_max)[0]
        if i >= 2:
            ms.append(next(t for n, t, _ in ctx.timings() if n == "genotype"))
    n_match = int((match >= 0).sum())
    # host: a VCF of the same targets, parsed and rewritten
    names = blk.contig_names
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "t.vcf")
        with open(path, "w") as f:
            f.write("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS\n")
            for t, st, pos, svlen, first, mate in zip(*(c.tolist() for c in cols)):
                sv = abi.SVTYPE_NAMES[st] if st >= 0 else "CNV"
                alt = (f"N[{names[mate] if mate >= 0 else 'chrUn'}:100[" if first else f"]{names[mate] if mate >= 0 else 'chrUn'}:100]N") if sv == "BND" else f"<{sv}>"
                f.write(f"{names[t]}\t{pos + 1}\t.\tN\t{alt}\t.\tPASS\tSVTYPE={sv};SVLEN={svlen}\tGT\t0/1\n")
        t0 = time.perf_counter()
        header, targets = genotype.read_targets(path)
        parse_ms = (time.perf_counter() - t0) * 1e3
    for t in targets:
        t.coverage_start, t.coverage_center, t.coverage_end = 3, 4, 5
    t0 = time.perf_counter()
    text = genotype.rewrite_header(header, cfg) + "".join(genotype.rewrite_line(t, cfg) + "\n" for t in targets)
    write_ms = (time.perf_counter() - t0) * 1e3
    out = {"card": card()[0], "power_limit": card()[1], "n_cand": int(len(res.cand)), "n_targets": int(a.targets), "n_match": n_match,
           "genotype_device_ms": float(np.median(ms)), "genotype_device_ms_all": [round(x, 4) for x in ms],
           "host_parse_ms": round(parse_ms, 1), "host_write_ms": round(write_ms, 1), "out_bytes": len(text)}
    if not a.no_cpu:
        from oracle import genotype as ogt
        task = cols[0]
        ranges = np.searchsorted(res.cand["task"], np.arange(len(blk.task) + 1))
        cpu_s, agree = 0.0, True
        for t in np.unique(task):
            idx = np.nonzero(task == t)[0]
            lo, hi = int(ranges[t]), int(ranges[t + 1])
            cands = ogt.cand_svs(res.cand[lo:hi], names)
            tl = [ogt.Sv(abi.SVTYPE_NAMES[st] if st >= 0 else "CNV", pos, svlen, first, names[mate] if mate >= 0 else "unknown")
                  for st, pos, svlen, first, mate in zip(*(cols[k][idx].tolist() for k in (1, 2, 3, 4, 5)))]
            t0 = time.perf_counter()
            m = ogt.match(cands, tl, cfg.combine_match, cfg.combine_match_max, cfg.cluster_merge_bnd)
            cpu_s += time.perf_counter() - t0
            agree = agree and np.array_equal(match[idx], np.array([lo + x if x >= 0 else -1 for x in m], dtype=np.int64))
        out["cpu_oracle_match_ms"] = round(cpu_s * 1e3, 1)
        out["cpu_matches_agree"] = bool(agree)
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
