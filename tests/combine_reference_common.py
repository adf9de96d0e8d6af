"""Inputs and golden format of the combine-mode `--reference` tests (tests/golden/make_combine_reference_golden.py writes the golden data,
tests/test_gpu_combine_reference.py reads it).

The SNF inputs are combine_cli_common's.  The FASTA is a seeded genome over their contigs (tests/ref_fasta.genome: N runs, soft-masked
stretches, IUPAC codes) with sequence planted at the SNFs' own candidate sites, so that the combined calls meet every allele rule:
  * a DEL span made wholly of N (dropped at the default --max-unknown-pct 0.5);
  * a DEL span whose first 30 % is N (kept at 0.5, dropped at 0.1);
  * IUPAC codes around a DEL's anchor base (written as they are: the clean-up only runs on the branch where REF is still N);
  * IUPAC codes or N around the anchor base of an INS, BND, DUP or INV (an INS or BND ALT takes the anchor base; IUPAC codes in REF and
    ALT become N, the letters of a symbolic ALT included, as in the reference);
  * and sites of each kind left alone.
A site covers the anchor bases of every sample's candidate of one SV, since a combined call's position is its group's, not one
candidate's.  The FASTA is written with its .fai, 60 columns per line."""
import json
import os

import combine_cli_common as ccc
import population_common as pc
import ref_fasta

HERE = os.path.dirname(os.path.abspath(__file__))
EXPECTED = os.path.join(HERE, "golden", "combine_reference", "expected.json")
SEED = 20261018
S4 = ["s1.snf", "s2.snf", "s3.snf", "s4.snf"]

# (label, inputs, extra arguments, FASTA: "full" or "no_ctg2", population SNF name or None)
CASES = [
    ("in_memory", S4, [], "full", None),
    ("two", ["s1.snf", "s2.snf"], [], "full", None),
    ("tmpfile", S4, ["--combine-max-inmemory-results", "1"], "full", None),
    ("symbolic", S4, ["--symbolic"], "full", None),
    ("max_unknown", S4, ["--max-unknown-pct", "0.1"], "full", None),
    ("contig_absent", S4, [], "no_ctg2", None),
    ("population", S4, [], "full", "P_edit"),
    ("population_tmpfile", S4, ["--combine-max-inmemory-results", "1"], "full", "P_edit"),
    ("contig", ["s1.snf", "s2.snf", "s3.snf"], ["--contig", "ctg2"], "full", None),
    ("regions", ["s1.snf", "s2.snf", "s3.snf"], ["--regions", "regions.bed"], "full", None),
]
IUPAC = b"RYSWKMBDHV"


def candidate_sites():
    """[(contig, pos, svtype, svlen)] of every candidate of the committed combine SNFs, sorted and distinct"""
    from sniffles_b200 import snf
    out = set()
    for k in range(1, 5):
        r = snf.SNFReader(os.path.join(ccc.SRC, f"sample{k}.snf"))
        try:
            for contig, length in ccc.CONTIGS:
                for b in range(0, length + r.header["config"]["snf_block_size"], r.header["config"]["snf_block_size"]):
                    for part in r.read_blocks(contig, b) or []:
                        for t in snf.TYPES:
                            out.update((c.contig, int(c.pos), t, int(c.svlen)) for c in part[t])
        finally:
            r.close()
    return sorted(out)


def site_groups():
    """[(contig, svtype, first pos, last pos, longest |svlen|)]: the candidate sites of one svtype closer than 500 bp to the previous one,
    taken as one site (the samples' candidates of one SV)"""
    out = []
    for contig, pos, t, svlen in sorted(candidate_sites(), key=lambda x: (x[0], x[2], x[1])):
        g = out[-1] if out else None
        if g is not None and g[0] == contig and g[1] == t and pos - g[3] < 500:
            out[-1] = (contig, t, g[2], pos, max(g[4], abs(svlen)))
        else:
            out.append((contig, t, pos, pos, abs(svlen)))
    return out


def genome():
    """[(name, bases)] over combine_cli_common.CONTIGS with the planted sites: DEL sites in turn wholly N, 30 % N, IUPAC at the anchor
    or left alone; other sites in turn IUPAC at the anchor, N at the anchor, left alone twice"""
    seqs = dict((n, bytearray(s)) for n, s in ref_fasta.genome(SEED, [tuple(c) for c in ccc.CONTIGS]))
    k_del = k_other = 0
    for contig, t, lo, hi, span in site_groups():
        s = seqs[contig]
        a, b = max(0, lo - 4), min(len(s), hi + 3)                     # the anchor bases of every candidate of the site
        if t == "DEL":
            kind, k_del = k_del % 4, k_del + 1
            if kind == 0:
                b = min(len(s), hi + span + 4)
                s[a:b] = b"N" * (b - a)
            elif kind == 1:
                b = min(len(s), hi - 1 + max(2, int(span * 0.3)))
                s[a:b] = b"N" * (b - a)
            elif kind == 2:
                s[a:b] = bytes(IUPAC[j % len(IUPAC)] for j in range(a, b))
        else:
            kind, k_other = k_other % 4, k_other + 1
            if kind == 0:
                s[a:b] = bytes(IUPAC[j % len(IUPAC)] for j in range(a, b))
            elif kind == 1:
                s[a:b] = b"N" * (b - a)
    return [(n, bytes(s)) for n, s in seqs.items()]


def fasta_files(kind, directory):
    """writes the FASTA of `kind` ("full", or "no_ctg2": ctg2 left out) and its .fai into `directory`; returns (path, sha256 of the text)"""
    seqs = genome()
    if kind == "no_ctg2":
        seqs = [(n, s) for n, s in seqs if n != "ctg2"]
    text = ref_fasta.fasta_text(seqs)
    path = os.path.join(directory, f"{kind}.fa")
    with open(path, "wb") as f:
        f.write(text)
    with open(path + ".fai", "wb") as f:
        f.write(ref_fasta.fai_text(seqs))
    return path, ref_fasta.sha256(text)


def case_args(inputs, extra, population, out, fasta):
    args = ["-i", *inputs, "-v", out, *extra, "--reference", fasta]
    if population:
        args += ["--combine-population", pc.snf_path(population)]
    return args


def load_expected():
    """(FASTA sha256 per kind, {label: case with "vcf" as combine_cli_common.load_expected gives it})"""
    with open(EXPECTED) as f:
        g = json.load(f)
    out = {}
    for label, case in g["cases"].items():
        c = dict(case)
        c["vcf"] = [g["headers"][i] for i in case["headers"]] + [g["records"][i] for i in case["records"]]
        out[label] = c
    return g["fasta_sha256"], out


def allele_counts(text):
    """per VCF text, the records by how their alleles were resolved: a DEL with its REF bases, an INS or BND with an anchor base, and
    symbolic or N anchored ones"""
    out = {"del_sequence": 0, "anchored": 0, "n_ref": 0}
    for line in text.splitlines():
        if line.startswith("#"):
            continue
        f = line.split("\t")
        ref, svtype = f[3], f[7].split("SVTYPE=")[1].split(";")[0]
        if ref == "N":
            out["n_ref"] += 1
        elif svtype == "DEL" and len(ref) > 1:
            out["del_sequence"] += 1
        else:
            out["anchored"] += 1
    return out


vcf_lines = ccc.vcf_lines
