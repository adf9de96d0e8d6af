"""Combine mode with and without `--reference` on one GPU; prints one JSON line.

The cohort is scripts/combine_sample_bench.py's (bench.combine_workload: 50 samples on 24 GRCh38-length contigs, times --scale), written
as SNF files into a temporary directory, with a seeded genome over its contigs (tests/ref_fasta.genome: N runs, soft-masked stretches,
IUPAC codes) written there as plain FASTA with its .fai.  combine_run.combine_snfs runs over it once without and once with --reference,
on one context created before either run.  Reported: the card and its power limit; the wall time of both runs and their split from
`stats`; the FASTA load (tasks.reference_for: read, snfb_load_reference); per pass the prefetch time and the bases gathered
(snfb_fetch_reference); the host time write_call's allele branch adds, taken as the difference of the two runs' VCF write times (it is
not timed on its own); and the device memory of the run with the genome resident (free memory polled every millisecond, as
call_sample_bench polls it): the lowest free memory seen against the free memory after the run without it, and the card's memory in use
at that low point; for the run without it, the lowest free memory against the free memory after the context was created.

    python scripts/combine_reference_bench.py [--scale 0.1] [--seed 7]"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    import ref_fasta
    from call_sample_bench import MemPoll, card
    from combine_sample_bench import write_cohort
    from sniffles_b200 import combine_run, tasks
    from sniffles_b200 import config as sconfig
    if not torch.cuda.is_available():
        raise SystemExit("combine_reference_bench needs a CUDA device")
    out = {"workload": f"config-4 shape: 50 samples, scale {args.scale}, seeded genome over its contigs", **card()}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        paths = write_cohort(tmp, args.scale)
        contigs = [(str(n), int(L)) for n, L in combine_run.read_header(paths[0])["config"]["contig_lengths"]]
        seqs = ref_fasta.genome(args.seed, contigs)
        fa = os.path.join(tmp, "genome.fa")
        with open(fa, "wb") as f:
            f.write(ref_fasta.fasta_text(seqs))
        with open(fa + ".fai", "wb") as f:
            f.write(ref_fasta.fai_text(seqs))
        del seqs
        out["inputs_write_s"] = round(time.perf_counter() - t0, 3)
        out["genome_bp"] = sum(L for _, L in contigs)
        tasks.device_context(0)                                      # context creation outside the timed runs
        runs = {}
        for arm, extra in (("without", []), ("with", ["--reference", fa])):
            cfg = sconfig.SnifflesConfig("-i", *paths, "-v", os.path.join(tmp, f"{arm}.vcf"), *extra)
            st = {}
            with MemPoll() as m:
                n = combine_run.combine_snfs(cfg, stats=st)
            runs[arm] = (n, st, m)
        n0, st0, m0 = runs["without"]
        n1, st1, m1 = runs["with"]
        total = torch.cuda.mem_get_info(0)[1]
    out.update(records_without=n0, records_with=n1, passes=st1["passes"], candidates=sum(st1["pass_candidates"]),
               wall_s_without=round(st0["wall_s"], 3), wall_s_with=round(st1["wall_s"], 3), fasta_load_s=round(st1["reference_s"], 3),
               prefetch_s=[round(x, 4) for x in st1["prefetch_s"]], prefetch_bases=st1["prefetch_bytes"],
               write_s_without=round(st0["write_s"], 3), write_s_with=round(st1["write_s"], 3),
               allele_branch_s_difference=round(st1["write_s"] - st0["write_s"], 3),
               split_with={k: round(st1[k], 3) for k in ("header_s", "decode_s", "device_s", "call_group_s", "write_s")},
               peak_device_bytes_added_without=int(m0.start - m0.low), peak_device_bytes_added=int(m1.start - m1.low),
               device_bytes_in_use_at_peak=int(total - m1.low))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
