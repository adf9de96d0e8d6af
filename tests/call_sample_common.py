"""Inputs and digests shared by tests/golden/make_call_sample_golden.py (the unmodified reference's whole-sample run) and the tests that
compare call.call_sample with it (tests/golden/call_sample/expected.json).

Inputs: BAMs written by bamio.write_bam from four fixture blocks (one contig per task, every contig of the block's header kept, so hg008
carries 218 contigs of which three have reads) and the reference's own htslib-written hg002.bam.  A case is (input, argument list); the
argument list may name `{tr}` (a BED of the block's tandem repeats) and `{fasta}` (the seeded FASTA of tests/ref_fasta.py)."""
import hashlib
import json
import os
import shutil
import sys

import ref_fasta

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "oracle", "pyref"))     # harness.combine_call_dict
GOLDEN = os.path.join(HERE, "golden")
EXPECTED = os.path.join(GOLDEN, "call_sample", "expected.json")
HG002 = os.path.join(GOLDEN, "bams", "hg002.bam")
STAMP = {"command": "sniffles --input sample.bam --vcf out.vcf", "start_date": "2026/10/16 00:00:00", "version": "Sniffles2", "build": "2.6.3"}

CASES = {
    "c1_default": ("c1_ont_1mb", []),
    "c1_snf": ("c1_ont_1mb", ["--snf", "{snf}"]),
    "c1_no_qc": ("c1_ont_1mb", ["--no-qc"]),
    "c1_tandem_repeats": ("c1_ont_1mb", ["--tandem-repeats", "{tr}", "--snf", "{snf}"]),
    "phased_all_contigs": ("phased_phase", ["--phase", "--all-contigs", "--snf", "{snf}"]),
    "phased_contig": ("phased_phase", ["--phase", "--contig", "ctg2"]),
    "phased_reference": ("phased_phase", ["--phase", "--all-contigs", "--reference", "{fasta}", "--snf", "{snf}"]),
    "c3_mosaic": ("c3_hifi_mosaic", ["--mosaic", "--all-contigs", "--snf", "{snf}"]),
    "hg008_default": ("hg008", []),
    "hg008_all_contigs": ("hg008", ["--all-contigs", "--snf", "{snf}", "--sample-id", "HG008"]),
    "hg002_default": ("hg002", []),
    "hg002_all_contigs": ("hg002", ["--all-contigs", "--snf", "{snf}"]),
}
COMBINE_CASES = ["phased_all_contigs", "phased_reference"]     # two samples' SNFs of the same contigs, combined
SNF_FIELDS = ["svtype", "pos", "end", "svlen", "support", "qual", "filter", "qc", "precise", "alt", "ref", "id", "fwd", "rev", "coverage_upstream",
              "coverage_start", "coverage_center", "coverage_end", "coverage_downstream", "genotypes", "rnames", "nm"]


def load_block(name):
    import test_oracle_golden as tog
    return tog._bam_block("hg008") if name == "hg008" else tog.load_fixture(name)[1]


def write_inputs(name, tmp):
    """the BAM of an input (+ its BED of tandem repeats and FASTA where it has them) under `tmp`: {"bam", "tr", "fasta"}"""
    from sniffles_b200 import bamio
    from sniffles_b200 import config as sconfig
    os.makedirs(tmp, exist_ok=True)
    out = {}
    if name == "hg002":
        out["bam"] = os.path.join(tmp, "hg002.bam")
        shutil.copyfile(HG002, out["bam"])
        shutil.copyfile(HG002 + ".csi", out["bam"] + ".csi")
        return out
    blk = load_block(name)
    out["bam"], _ = bamio.write_bam(os.path.join(tmp, name + ".bam"), blk)
    if len(blk.tr):                 # the block's repeats are padded intervals: a BED that load_tandem_repeats pads back to them
        pad = sconfig.default_config().tandem_repeat_region_pad
        out["tr"] = os.path.join(tmp, name + ".tr.bed")
        with open(out["tr"], "w") as f:
            for t in range(len(blk.task)):
                o, n = int(blk.task[t]["tr_off"]), int(blk.task[t]["tr_n"])
                for k in range(n):
                    a, b = int(blk.tr[2 * (o + k)]), int(blk.tr[2 * (o + k) + 1])
                    f.write(f"{blk.contig_names[int(blk.task[t]['contig'])]}\t{a + pad if a > 0 else pad}\t{b - pad}\n")
    if name in ref_fasta.GOLDEN_FASTA:
        out["fasta"] = os.path.join(tmp, name + ".fa")
        text, seqs = ref_fasta.golden_fasta(name)
        with open(out["fasta"], "wb") as f:
            f.write(text)
        with open(out["fasta"] + ".fai", "wb") as f:
            f.write(ref_fasta.fai_text(seqs))
    return out


def case_args(case, paths, vcf_path, snf_path):
    """the command-line arguments of a case, its placeholders filled"""
    _, args = CASES[case]
    fill = {"{tr}": paths.get("tr"), "{fasta}": paths.get("fasta"), "{snf}": snf_path}
    return ["--input", paths["bam"], "--vcf", vcf_path] + [fill.get(a, a) for a in args]


def digest(obj):
    """the sha256 prefix of an object's canonical JSON: numpy scalars as Python numbers, tuples as lists, keys sorted.  Values that
    compare equal hash equal: a bool and an integral float are written as ints (the reference stores nm -1 where this package has -1.0,
    STDEV_POS 0.0 where it has 0; the pickled candidates compare equal field by field, as tests/test_snf.py compares them)"""
    def plain(v):
        if isinstance(v, dict):
            return {str(k): plain(x) for k, x in v.items()}
        if isinstance(v, (list, tuple)):
            return [plain(x) for x in v]
        v = v.item() if hasattr(v, "item") else v
        if isinstance(v, bool) or (isinstance(v, float) and v.is_integer()):
            return int(v)
        return v
    return hashlib.sha256(json.dumps(plain(obj), sort_keys=True).encode()).hexdigest()[:16]


def vcf_digest(text):
    """a VCF file as the golden data stores it: the header's hash and contig count, each record in ref_fasta.vcf_digest's short form with
    the hash of the full line"""
    lines = text.splitlines()
    head = [l for l in lines if l.startswith("#")]
    return {"header": [digest(head), sum(l.startswith("##contig=") for l in head)],
            "records": [ref_fasta.vcf_digest(l) for l in lines if not l.startswith("#")]}


def snf_digest(path):
    """an SNF file's content as the golden data stores it: the index as {contig: {block: number of parts}}, the candidate count and the
    contig coverages of the header, and per block part the hash of its `_COVERAGE` and, per SV type, the number of candidates and the hash
    of their fields (SNF_FIELDS and the INFO entries that are set)"""
    from sniffles_b200 import snf
    rd = snf.SNFReader(path)
    out = {"index": {c: {b: len(v) for b, v in d.items()} for c, d in rd.index.items()}, "snf_candidate_count": rd.header["snf_candidate_count"],
           "contig_coverages": rd.header["config"]["contig_coverages"], "blocks": {}}
    for contig in rd.index:
        for block in sorted(rd.index[contig], key=int):
            for k, b in enumerate(rd.read_blocks(contig, block)):
                cands = {t: [[getattr(c, f) for f in SNF_FIELDS] + [{i: v for i, v in c.info.items() if v is not None}] for c in b[t]] for t in snf.TYPES}
                out["blocks"][f"{contig}:{block}:{k}"] = {"_COVERAGE": digest(sorted(b["_COVERAGE"].items())),
                                                          **{t: [len(v), digest(v)] for t, v in cands.items() if v}}
    rd.close()
    return json.loads(json.dumps(out))


def combine_digest(calls):
    """combined calls as the golden data stores them: [svtype, pos, svlen, filter, hash of harness.combine_call_dict] per call"""
    import harness
    return [[c.svtype, c.pos, c.svlen, c.filter, digest(harness.combine_call_dict(c))] for c in calls]
