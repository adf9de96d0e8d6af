"""Calling inside regions, measured: the config-2 generator at 1/100 written as a BAM, called three ways -- the whole genome, 20,000
sorted disjoint regions, and the same regions with 20 % of them overlapping or moved out of order.  Prints one JSON line: the card's
name and power limit (read in the same call), and per way the wall time, the index and read time, per pass the load / run time, the
coverage-order sort's device time (timing mark `cov_order` of the last pass), the launches and the inflated bytes loaded.  Numbers this
script does not take are written as "not measured".  Inputs and outputs go to a temporary directory.

    python scripts/regions_bench.py [--scale 0.01] [--regions 20000]"""
import argparse
import json
import os
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from call_sample_bench import card  # noqa: E402


def write_bed(path, bam, n, shuffle_frac, seed):
    """n regions spread over the contigs in proportion to their length, sorted and disjoint; with shuffle_frac, that share of them is
    widened over its neighbour (overlap) or moved to a random place in the list (out of order)"""
    import numpy as np
    rng = np.random.default_rng(seed)
    total = sum(L for _, L in bam.contigs)
    rows = []
    for name, L in bam.contigs:
        k = max(1, round(n * L / total))
        step = L // k
        for i in range(k):
            a = i * step + int(rng.integers(0, step // 4 + 1))
            rows.append([name, a, min(L, a + step // 2)])
    m = int(len(rows) * shuffle_frac)
    for j in rng.choice(len(rows), m, replace=False):
        if rng.random() < 0.5:
            rows[j][2] = min(rows[j][2] + (rows[j][2] - rows[j][1]), dict(bam.contigs)[rows[j][0]])
        else:
            r = rows.pop(int(j))
            rows.insert(int(rng.integers(0, len(rows))), r)
    with open(path, "w") as f:
        f.writelines(f"{c}\t{a}\t{b}\n" for c, a, b in rows)
    return len(rows)


def run(path, tmp, tag, extra):
    from sniffles_b200 import call, tasks
    from sniffles_b200 import config as sconfig
    cfg = sconfig.default_config("--input", path, "--vcf", os.path.join(tmp, tag + ".vcf"), "--allow-overwrite", *extra)
    cfg.input = path
    ctx = tasks.device_context(0)
    l0 = ctx.launch_count()
    stats = {}
    call.call_sample(cfg, stats=stats)
    t = {name: ms for name, ms, _ in ctx.timings()}
    return {"wall_s": stats["wall_s"], "index_s": stats["index_s"], "read_s": stats["read_s"], "passes": stats["passes"],
            "load_bam_s": stats["load_bam_s"], "run_s": stats["run_s"], "inflated_bytes": stats["pass_inflated_bytes"],
            "launches": ctx.launch_count() - l0, "cov_order_ms_last_pass": t.get("cov_order", "not measured")}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.01)
    ap.add_argument("--regions", type=int, default=20000)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("regions_bench needs a CUDA device")
    from sniffles_b200 import bamio, synth
    tmp = tempfile.mkdtemp(prefix="snfb_regions_")
    blk = synth.config_block(2, a.scale)
    path = os.path.join(tmp, "c2.bam")
    bamio.write_bam(path, blk, level=1, qual_seed=7)
    bam = bamio.BamFile(path)
    beds = {}
    for tag, frac in (("sorted", 0.0), ("overlap_unsorted", 0.2)):
        beds[tag] = os.path.join(tmp, tag + ".bed")
        write_bed(beds[tag], bam, a.regions, frac, 11)
    bam.close()
    out = {"card": card(), "scale": a.scale, "records": len(blk.rec), "n_regions": a.regions, "ways": {}}
    run(path, tmp, "warm", ["--all-contigs"])
    out["ways"]["whole_genome"] = run(path, tmp, "whole", ["--all-contigs"])
    for tag, bed in beds.items():
        out["ways"][tag] = run(path, tmp, tag, ["--regions", bed])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
