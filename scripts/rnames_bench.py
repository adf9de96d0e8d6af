"""The cost of --output-rnames on whole-sample calling.  Prints one JSON line: the card and its power limit; per input the wall time of
call.call_sample without and with --output-rnames (plain VCF + SNF) and the growth of both files; and, on one pass over the whole BAM,
the device time of snfb_read_names (CUDA events of its two marks, median of --reps calls after --warmup), the names and text bytes, the
host decode of every candidate's names (median), and the device memory the first call adds (free memory before and after it).

    python scripts/rnames_bench.py [--inputs c6,c2] [--c2-scale 0.01] [--reps 20] [--warmup 3] [--out FILE]

"c6" / "c2" are the inputs of scripts/call_sample_bench.py (bench.py --config 6's generator; the config-2 generator at --c2-scale)."""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

import call_sample_bench as csb  # noqa: E402


def run_call(path, tmp, tag, rnames):
    from sniffles_b200 import call
    from sniffles_b200 import config as sconfig
    vcf_path, snf_path = os.path.join(tmp, tag + ".vcf"), os.path.join(tmp, tag + ".snf")
    cfg = sconfig.default_config("--input", path, "--vcf", vcf_path, "--snf", snf_path, "--all-contigs", "--allow-overwrite",
                                 *(["--output-rnames"] if rnames else []))
    cfg.input = path
    stats = {}
    call.call_sample(cfg, stats=stats)
    return {"wall_s": stats["wall_s"], "passes": stats["passes"], "run_s": sum(stats["run_s"]), "rnames_s": sum(stats["rnames_s"]),
            "finalize_s": stats["finalize_s"], "vcf_write_s": stats["vcf_write_s"], "snf_write_s": stats["snf_write_s"],
            "vcf_bytes": os.path.getsize(vcf_path), "snf_bytes": os.path.getsize(snf_path)}


def names_step(path, reps, warmup):
    """one load_bam + run over the whole BAM, then snfb_read_names: device ms, sizes, host decode, device memory of the first call"""
    import torch
    from sniffles_b200 import abi, bamio, binding, call, tasks
    from sniffles_b200 import config as sconfig
    cfg = sconfig.default_config("--all-contigs")
    bam = bamio.BamFile(path)
    items = list(call.task_inputs(bam, tasks.plan(bam.contigs, cfg)[1]))
    z, spans = call.join_inputs([(it.bgzf, it.spans) for it in items])
    block = bamio.pack_records(bam.contigs, [], [(bam.name_to_id[it.contig], it.start, it.end, it.id) for it in items])
    bam.close()
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    ctx.load_bam(z, spans, block)
    res = ctx.run()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    names = ctx.read_names()
    free1 = torch.cuda.mem_get_info(0)[0]
    dev_ms, decode_s = [], []
    for k in range(warmup + reps):
        names = ctx.read_names()
        t = {n: ms for n, ms, _ in ctx.timings()}
        t0 = time.perf_counter()
        fresh = binding.ReadNames(names.text, names.off)
        fresh.per_candidate(res.rn_off, 0, len(res.cand))
        t1 = time.perf_counter()
        if k >= warmup:
            dev_ms.append(t["rnames_resolve"] + t["rnames_copy"])
            decode_s.append(t1 - t0)
    ctx.close()
    n = len(res.rnames)
    return {"candidates": len(res.cand), "names": n, "text_bytes": int(len(names.text)), "collisions": names.collisions,
            "device_ms_median": statistics.median(dev_ms), "device_ms_min": min(dev_ms), "device_ms_max": max(dev_ms),
            "host_decode_ms_median": 1e3 * statistics.median(decode_s),
            "device_bytes_added": int(free0 - free1), "device_bytes_per_name": (free0 - free1) / n if n else None,
            "inflated_bytes": sum(it.inflated for it in items)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", default="c6,c2")
    ap.add_argument("--c2-scale", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("rnames_bench needs a CUDA device")
    out = {"card": csb.card(), "inputs": {}}
    tmp = tempfile.mkdtemp(prefix="snfb_rnames_")
    for kind in a.inputs.split(","):
        path, n_rec, _ = csb.make_input(kind, a.c2_scale, tmp)
        r = {"records": n_rec}
        run_call(path, tmp, kind + "_warm", True)
        runs = {"without": [], "with": []}
        for k in range(2):                                          # alternated, twice
            runs["without"].append(run_call(path, tmp, f"{kind}_off{k}", False))
            runs["with"].append(run_call(path, tmp, f"{kind}_on{k}", True))
        r["without"], r["with"] = runs["without"], runs["with"]
        r["vcf_growth"] = runs["with"][0]["vcf_bytes"] / runs["without"][0]["vcf_bytes"]
        r["snf_growth"] = runs["with"][0]["snf_bytes"] / runs["without"][0]["snf_bytes"]
        r["names_step"] = names_step(path, a.reps, a.warmup)
        out["inputs"][kind] = r
        print(f"[rnames_bench] {kind}: {json.dumps(r)}", file=sys.stderr, flush=True)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
