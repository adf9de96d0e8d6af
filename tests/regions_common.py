"""Inputs of tests/golden/make_regions_golden.py (the unmodified reference's whole-sample run with --regions / --region) and of the tests
that compare call.call_sample with it (tests/golden/regions/expected.json).  A case is (input, BED lines or None, extra arguments); the
BED lines and `--region` strings are functions of the BAM header's contigs [(name, length)], so the same case fits any input."""
import os

HERE = os.path.dirname(os.path.abspath(__file__))
EXPECTED = os.path.join(HERE, "golden", "regions", "expected.json")


def _sorted(ctg):
    (a, L), rest = ctg[0], ctg[1:]
    lines = [f"{a}\t{L // 10}\t{L // 4}", f"{a}\t{L // 3}\t{L // 2}", f"{a}\t{L // 2}\t{(3 * L) // 4}"]       # the last two adjacent
    lines += [f"{b}\t0\t{M // 2}" for b, M in rest[:2]]
    return lines


def _overlap_unsorted(ctg):
    (a, L) = ctg[0]
    return [f"{a}\t{L // 2}\t{(9 * L) // 10}", f"{a}\t{L // 5}\t{(3 * L) // 5}", f"{a}\t{L // 4}\t{L // 3}", f"{a}\t0\t{L // 6}"]


def _edges(ctg):
    (a, L) = ctg[0]
    return ["# a comment line", "", f"{a}\t{L - 40000}\t{L}", f"{a}\t{L // 3}\t{L // 3}", f"{a}\tnot_a_number\t5",
            f"{a}\t{L // 2}\t{L + 50000}", "no_such_contig\t0\t1000", f"{a}\t{L + 10}\t{L + 20}"]


def _bad(ctg):
    (a, L) = ctg[0]
    lines = [f"{a}\t{L // 2}\t{L // 4}"]
    lines += [f"{b}\t{M // 4}\t{M // 2}" for b, M in ctg[1:2]]
    return lines


def _genotype(ctg):
    """targets inside, outside and across the regions of the first contig (overlapping, unsorted), one region on the second"""
    lines = _overlap_unsorted(ctg)
    lines += [f"{b}\t{M // 3}\t{(2 * M) // 3}" for b, M in ctg[1:2]]
    return lines


def _fasta_short(ctg):
    """regions of the first contig, one of them reaching past the end of that contig in the FASTA, which is cut short
    (SHORT_FASTA_CUT bases): that region's fetch does not fit its slice, and the task goes unmasked"""
    (a, L) = ctg[0]
    lines = [f"{a}\t{L // 5}\t{L // 2}", f"{a}\t{L - 3 * SHORT_FASTA_CUT}\t{L - 1}"]
    lines += [f"{b}\t0\t{M // 2}" for b, M in ctg[1:2]]
    return lines


SHORT_FASTA_CUT = 10_000


def _strings(ctg):
    (a, L) = ctg[0]
    return ["--region", f"{a}:{L // 5}-{L // 2}", "--region", "missing_colon", "--region", f"{a}:{L // 10}-{L // 4}"]


CASES = {
    "c1_sorted": ("c1_ont_1mb", _sorted, []),
    "c1_overlap_unsorted": ("c1_ont_1mb", _overlap_unsorted, []),
    "c1_edges": ("c1_ont_1mb", _edges, []),
    "c1_strings": ("c1_ont_1mb", None, _strings),
    "c1_sorted_snf": ("c1_ont_1mb", _sorted, ["--snf", "{snf}"]),
    "c1_overlap_snf": ("c1_ont_1mb", _overlap_unsorted, ["--snf", "{snf}"]),
    "phased_sorted": ("phased_phase", _sorted, ["--phase"]),
    "phased_bad": ("phased_phase", _bad, ["--phase"]),
    "phased_overlap_reference": ("phased_phase", _overlap_unsorted, ["--phase", "--reference", "{fasta}", "--snf", "{snf}"]),
    "c1_overlap_tandem_repeats": ("c1_ont_1mb", _overlap_unsorted, ["--tandem-repeats", "{tr}"]),
    "hg002_overlap": ("hg002", _overlap_unsorted, ["--snf", "{snf}"]),
    "phased_fasta_short": ("phased_phase", _fasta_short, ["--phase", "--reference", "{fasta_short}", "--snf", "{snf}"]),
}
# --genotype-vcf with --regions: (input, BED, extra arguments, targets VCF under tests/golden/genotype)
GENOTYPE_CASES = {
    "phased_genotype": ("phased_phase", _genotype, ["--phase"], "phased_phase.targets.vcf"),
    "c1_genotype": ("c1_ont_1mb", _genotype, [], "c1_ont_1mb.targets.vcf"),
}


def write_short_fasta(paths, tmp):
    """the input's FASTA with its first contig cut short by SHORT_FASTA_CUT bases, + .fai: paths["fasta_short"]"""
    import ref_fasta
    name = os.path.splitext(os.path.basename(paths["fasta"]))[0]
    _, seqs = ref_fasta.golden_fasta(name)
    seqs = [(seqs[0][0], seqs[0][1][:-SHORT_FASTA_CUT])] + list(seqs[1:])
    out = os.path.join(tmp, name + ".short.fa")
    with open(out, "wb") as f:
        f.write(ref_fasta.fasta_text(seqs))
    with open(out + ".fai", "wb") as f:
        f.write(ref_fasta.fai_text(seqs))
    paths["fasta_short"] = out
    return paths


def contigs_with_reads(bam):
    """the header's contigs that hold mapped reads, in header order: the regions are placed on them"""
    return [(n, L) for n, L in bam.contigs if (bam.count_mapped(n) or 0) > 0]


def case_args(case, paths, bam, tmp, vcf_path, snf_path, cases=None):
    """the command line of a case: its BED written under `tmp`, its placeholders filled"""
    _, bed, extra = (cases or CASES)[case][:3]
    ctg = contigs_with_reads(bam)
    args = ["--input", paths["bam"], "--vcf", vcf_path]
    if bed is not None:
        path = os.path.join(tmp, case + ".bed")
        with open(path, "w") as f:
            f.write("".join(line + "\n" for line in bed(ctg)))
        args += ["--regions", path]
    if "{fasta_short}" in (extra if not callable(extra) else []):
        write_short_fasta(paths, tmp)
    fill = {"{tr}": paths.get("tr"), "{fasta}": paths.get("fasta"), "{fasta_short}": paths.get("fasta_short"), "{snf}": snf_path}
    return args + [fill.get(a, a) for a in (extra(ctg) if callable(extra) else extra)]
