"""Cases and stored forms shared by tests/golden/make_rnames_golden.py (the unmodified reference's whole-sample runs and combine with
--output-rnames) and the tests that compare this package with them (tests/golden/rnames/expected.json).

The reference lists a call's read names as list(set(...)) of strings (sv.py:520, 555), an order that depends on PYTHONHASHSEED; this
package lists them by ascending 64-bit name hash.  So a called record is stored as its line with the RNAMES entry cut out plus its names
sorted, and an SNF candidate as the hash of its other fields plus its names sorted.  Combine mode concatenates the pickled lists in group
order (sv.py:349-354), which is deterministic for given SNF files: its RNAMES are stored in order."""
import os

import call_sample_common as csc

GOLDEN = os.path.join(csc.GOLDEN, "rnames")
EXPECTED = os.path.join(GOLDEN, "expected.json")

# case -> (input, argument list), the placeholders of call_sample_common.case_args
CASES = {
    "rn_c1_snf": ("c1_ont_1mb", ["--snf", "{snf}", "--output-rnames"]),
    "rn_phased_all_contigs": ("phased_phase", ["--phase", "--all-contigs", "--snf", "{snf}", "--output-rnames"]),
    "rn_phased_reference": ("phased_phase", ["--phase", "--all-contigs", "--reference", "{fasta}", "--snf", "{snf}", "--output-rnames"]),
    # --long-ins-length 500: an insertion of 609 bp takes a name that only its leads_long carry (sv.py:520-525)
    "rn_c3_mosaic": ("c3_hifi_mosaic", ["--mosaic", "--all-contigs", "--snf", "{snf}", "--output-rnames", "--long-ins-length", "500"]),
    # the real BAM yields SVs only with the filters relaxed: its few calls carry real ONT read names
    "rn_hg002_all_contigs": ("hg002", ["--all-contigs", "--snf", "{snf}", "--output-rnames", "--minsupport", "1", "--mapq", "0", "--minsvlen", "20",
                                       "--no-qc"]),
}
# the two cases whose reference-written SNFs are stored under tests/golden/rnames/ (<case>.snf) and combined
COMBINE_CASES = ["rn_phased_all_contigs", "rn_phased_reference"]
SNF_FIELDS = [f for f in csc.SNF_FIELDS if f != "rnames"]


def register():
    """makes the cases known to call_sample_common.case_args in this process (the golden generator runs them through its harness)"""
    csc.CASES.update(CASES)


def case_args(case, paths, vcf_path, snf_path):
    """the command-line arguments of a case, its placeholders filled as call_sample_common.case_args fills them"""
    _, args = CASES[case]
    fill = {"{tr}": paths.get("tr"), "{fasta}": paths.get("fasta"), "{snf}": snf_path}
    return ["--input", paths["bam"], "--vcf", vcf_path] + [fill.get(a, a) for a in args]


def split_rnames(line):
    """a VCF record -> (the line with its RNAMES entry removed, the names in their listed order; None when the record has none)"""
    cols = line.split("\t")
    info, names = [], None
    for kv in cols[7].split(";"):
        if kv.startswith("RNAMES="):
            names = kv[len("RNAMES="):].split(",")
        else:
            info.append(kv)
    cols[7] = ";".join(info)
    return "\t".join(cols), names


def vcf_form(text):
    """a called VCF as the golden data stores it: the header's hash, then per record [CHROM, POS, ID, hash of the line without RNAMES,
    sorted names (None without RNAMES)]"""
    lines = text.splitlines()
    recs = []
    for l in lines:
        if not l.startswith("#"):
            rest, names = split_rnames(l)
            c = l.split("\t")
            recs.append([c[0], int(c[1]), c[2], csc.digest(rest), None if names is None else sorted(names)])
    return {"header": csc.digest([l for l in lines if l.startswith("#")]), "records": recs}


def snf_form(path):
    """an SNF file as the golden data stores it: per block part and SV type, per candidate [hash of SNF_FIELDS and the set INFO entries,
    sorted rnames (None when the candidate has none)]"""
    from sniffles_b200 import snf
    rd = snf.SNFReader(path)
    out = {"snf_candidate_count": rd.header["snf_candidate_count"], "blocks": {}}
    for contig in rd.index:
        for block in sorted(rd.index[contig], key=int):
            for k, b in enumerate(rd.read_blocks(contig, block)):
                out["blocks"][f"{contig}:{block}:{k}"] = {
                    t: [[csc.digest([getattr(c, f) for f in SNF_FIELDS] + [{i: v for i, v in c.info.items() if v is not None}]),
                         None if c.rnames is None else sorted(c.rnames)] for c in b[t]] for t in snf.TYPES if b[t]}
    rd.close()
    return out


def combine_form(lines):
    """combined VCF records as the golden data stores them: per record [CHROM, POS, ID, hash of the line without RNAMES, names in order]"""
    out = []
    for l in lines:
        rest, names = split_rnames(l)
        c = l.split("\t")
        out.append([c[0], int(c[1]), c[2], csc.digest(rest), names])
    return out
