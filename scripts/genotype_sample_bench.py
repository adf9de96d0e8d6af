"""Force calling a whole sample (genotype.genotype_vcf) on synthetic BAMs in device passes, and the device memory of one pass with its
targets.  Prints one JSON line: the card and its power limit; per input the wall time of genotype_vcf and its split (target parse, index
and BGZF read, snfb_load_bam, snfb_run and snfb_genotype_targets per pass, rewrite and output), the passes and their inflated bytes, at
the default budget, at ¼ of it and at about ¼ of the BAM's inflated bytes; whether the three outputs are byte-equal; and the peak device
memory of one load_bam + run + genotype_targets over the whole BAM and every target on a fresh context (free memory polled every
millisecond), per inflated byte.

    python scripts/genotype_sample_bench.py [--inputs c6,c2] [--c2-scale 0.01] [--targets 500000] [--out FILE]

The inputs are those of scripts/call_sample_bench.py.  The targets are synth.genotype_targets over the candidates of one device run of the
BAM: half of them jittered copies of the candidates, half seeded decoys and edge cases, written sorted by contig and position (a catalog's
order, which the .vcf.gz output's index needs); targets outside their contig's task and BND targets before the first other target of
their contig are left out."""
import argparse
import json
import logging
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts")]

import call_sample_bench as csb  # noqa: E402


def _device_pass(path, cfg, cols=None):
    """one snfb_load_bam + snfb_run over every contig of the BAM on a fresh context, then (cols given) one snfb_genotype_targets over
    them: (inflated bytes, candidates, task contig names, peak device bytes of load + run, peak of the whole)"""
    from sniffles_b200 import abi, bamio, binding, call, tasks
    bam = bamio.BamFile(path)
    items = list(call.task_inputs(bam, tasks.plan(bam.contigs, cfg)[1]))
    z, spans = call.join_inputs([(it.bgzf, it.spans) for it in items])
    block = bamio.pack_records(bam.contigs, [], [(bam.name_to_id[it.contig], it.start, it.end, it.id) for it in items])
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    with csb.MemPoll() as m:
        ctx.load_bam(z, spans, block)
        res = ctx.run()
        run_low = m.low = min(m.low, m.free())
        if cols is not None:
            ctx.genotype_targets(*cols, cfg.combine_match, cfg.combine_match_max)
    ctx.close()
    bam.close()
    return sum(it.inflated for it in items), res.cand.copy(), [it.contig for it in items], m.start - run_low, m.start - m.low


def write_targets(cand, names, lengths, n, path):
    """n seeded targets over the run's candidates as a VCF; returns the number written"""
    from sniffles_b200 import abi, synth
    cols = synth.genotype_targets(cand, len(names), np.array(lengths), np.random.default_rng(11), n)
    rows = sorted(zip(*(c.tolist() for c in cols)), key=lambda r: (r[0], r[2]))
    lines, anchored = [], set()
    for t, st, pos, svlen, first, mate in rows:
        sv = abi.SVTYPE_NAMES[st] if st >= 0 else "CNV"
        if not 0 <= pos < lengths[t] - 1 or (sv == "BND" and t not in anchored):         # outside every task, or its task would fail
            continue
        anchored.add(t)
        mate_name = names[mate] if 0 <= mate < len(names) else "chrUn"
        alt = (f"N[{mate_name}:100[" if first else f"]{mate_name}:100]N") if sv == "BND" else f"<{sv}>"
        lines.append(f"{names[t]}\t{pos + 1}\t.\tN\t{alt}\t.\tPASS\tSVTYPE={sv};SVLEN={svlen}\tGT\t0/1\n")
    with open(path, "w") as f:
        f.write("##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS\n")
        f.writelines(lines)
    return len(lines)


def target_cols(path, bam_path, cfg):
    """the snfb_gt_in columns genotype_vcf makes from the target VCF, for one pass over every planned task (task index = plan order)"""
    from sniffles_b200 import bamio, genotype
    bam = bamio.BamFile(bam_path)
    _, targets = genotype.read_targets(path)
    parts = [genotype.encode(p[4], k, bam.name_to_id) for k, p in enumerate(genotype.plan(bam.contigs, targets, cfg)) if p[4]]
    bam.close()
    keys = ("task", "svtype", "pos", "svlen", "bnd_is_first", "mate_contig")
    return [np.concatenate([p[k] for p in parts]) for k in keys]


def run_genotype(path, targets, tmp, budget, tag):
    from sniffles_b200 import genotype
    from sniffles_b200 import config as sconfig
    out = os.path.join(tmp, tag + ".vcf.gz")
    cfg = sconfig.default_config("--input", path, "--genotype-vcf", targets, "--vcf", out, "--all-contigs")
    cfg.input = path
    stats = {}
    with csb.MemPoll() as m:
        n = genotype.genotype_vcf(cfg, budget=budget, stats=stats)
    stats["peak_device_bytes_added"] = int(m.start - m.low)          # over the free memory before the call; contexts of earlier calls stay
    stats["records_written"] = n
    stats["budget"] = budget
    with open(out, "rb") as f, open(out + ".tbi", "rb") as g:
        return stats, f.read() + g.read()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", default="c6,c2")
    ap.add_argument("--c2-scale", type=float, default=0.01)
    ap.add_argument("--targets", type=int, default=500_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("genotype_sample_bench needs a CUDA device")
    logging.getLogger("sniffles_b200").setLevel(logging.ERROR)      # one "Unsupported SVTYPE" warning per decoy of an unknown type
    from sniffles_b200 import call, bamio
    from sniffles_b200 import config as sconfig
    out = {"card": csb.card(), "device": torch.cuda.get_device_name(0), "inputs": {}}
    tmp = tempfile.mkdtemp(prefix="snfb_genotype_sample_")
    cfg = sconfig.default_config("--all-contigs")
    for kind in a.inputs.split(","):
        t0 = time.perf_counter()
        path, n_rec, bp = csb.make_input(kind, a.c2_scale, tmp)
        r = {"records": n_rec, "aligned_bp": bp, "bam_bytes": os.path.getsize(path), "bam_write_s": time.perf_counter() - t0}
        infl, cand, names, _, _ = _device_pass(path, cfg)
        bam = bamio.BamFile(path)
        lengths = [bam.get_reference_length(n) for n in names]
        bam.close()
        targets = os.path.join(tmp, kind + ".targets.vcf")
        r["candidates"], r["targets"] = int(len(cand)), write_targets(cand, names, lengths, a.targets, targets)
        r["warmup"] = run_genotype(path, targets, tmp, None, kind + "_warm")[0]["wall_s"]
        infl, _, _, run_peak, peak = _device_pass(path, cfg, target_cols(targets, path, cfg))
        r["one_pass_inflated_bytes"], r["one_pass_peak_device_bytes_run"], r["one_pass_peak_device_bytes_with_targets"] = infl, run_peak, peak
        r["device_bytes_per_inflated_byte_with_targets"] = peak / infl
        budget = call.device_budget(0)
        runs = {"default_budget": None, "quarter_budget": max(1, budget // 4), "split": max(1, infl // 4)}
        files = {}
        for name, b in runs.items():
            r[name], files[name] = run_genotype(path, targets, tmp, b, f"{kind}_{name}")
        r["outputs_byte_equal"] = len(set(files.values())) == 1
        r["budget_model"] = {"fixed_bytes": call.DEVICE_BYTES_FIXED, "bytes_per_inflated_byte": call.DEVICE_BYTES_PER_INFLATED_BYTE}
        out["inputs"][kind] = r
        print(f"[genotype_sample_bench] {kind}: {json.dumps(r)}", file=sys.stderr, flush=True)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
