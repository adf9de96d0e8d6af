"""Inputs and golden format of the combine-mode command-line tests (tests/golden/make_combine_cli_golden.py writes the golden data,
tests/test_combine_cli.py and tests/test_gpu_combine_cli.py read it).

The SNF inputs are derived, at test time, from the committed tests/golden/combine/sample*.snf: `contig_lengths` is added to the JSON header
line (block offsets are relative to the end of that line, so rewriting it is safe), one copy drops `build` (re-QC'd under --re-qc auto),
and two copies make ctg1 520 Mb long, so that `scatter` splits it at --threads 4.

The golden VCFs are stored compactly: every distinct header line once, every distinct record once as [CHROM, POS, ID, sha256 of the
whole line], and per case the indices of its lines.  A record matches only when its whole text does."""
import hashlib
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "golden", "combine")
EXPECTED = os.path.join(HERE, "golden", "combine_cli", "expected.json")
CONTIGS = [["ctg1", 350_000], ["ctg2", 260_000]]
LONG = [["ctg1", 520_000_000], ["ctg2", 260_000]]
STAMPS = ("##source=", "##command=", "##fileDate=")

# (label, inputs, extra arguments); inputs are names relative to the directory write_inputs filled, which is the working directory
CASES = [
    ("two", ["s1.snf", "s2.snf"], []),
    ("three", ["s1.snf", "s2.snf", "s3.snf"], []),
    ("tsv", ["samples.tsv"], []),
    ("reqc_auto_nobuild", ["s1.snf", "s3_nobuild.snf"], []),
    ("reqc0", ["s1.snf", "s2.snf", "s3.snf"], ["--re-qc", "0"]),
    ("reqc1", ["s1.snf", "s2.snf", "s3.snf"], ["--re-qc", "1"]),
    ("contig", ["s1.snf", "s2.snf", "s3.snf"], ["--contig", "ctg2"]),
    ("regions", ["s1.snf", "s2.snf", "s3.snf"], ["--regions", "regions.bed"]),
    ("scatter", ["long1.snf", "long2.snf"], ["--threads", "4"]),
    ("tmpfile", ["s1.snf", "s2.snf", "s3.snf", "s4.snf"], ["--combine-max-inmemory-results", "1"]),
    ("default4", ["s1.snf", "s2.snf", "s3.snf", "s4.snf"], []),
    ("no_alignment4", ["s1.snf", "s2.snf", "s3.snf", "s4.snf"], ["--combine-pctseq", "0"]),
    ("strict_alignment4", ["s1.snf", "s2.snf", "s3.snf", "s4.snf"], ["--combine-pctseq", "0.985", "--combine-separate-intra"]),
    ("loose4", ["s1.snf", "s2.snf", "s3.snf", "s4.snf"], ["--combine-match", "100", "--combine-low-confidence", "0.6", "--combine-output-filtered"]),
]


def _rewrite(src, dst, contig_lengths, drop_build=False):
    with open(src, "rb") as f:
        header = json.loads(f.readline())
        rest = f.read()
    header["config"]["contig_lengths"] = contig_lengths
    if drop_build:
        del header["config"]["build"]
    with open(dst, "wb") as f:
        f.write((json.dumps(header) + "\n").encode())
        f.write(rest)


def write_inputs(directory):
    """the SNFs, the sample list and the BED of the cases, under `directory`"""
    os.makedirs(directory, exist_ok=True)
    for k in range(1, 5):
        _rewrite(os.path.join(SRC, f"sample{k}.snf"), os.path.join(directory, f"s{k}.snf"), CONTIGS)
    _rewrite(os.path.join(SRC, "sample3.snf"), os.path.join(directory, "s3_nobuild.snf"), CONTIGS, drop_build=True)
    for k in (1, 2):
        _rewrite(os.path.join(SRC, f"sample{k}.snf"), os.path.join(directory, f"long{k}.snf"), LONG)
    with open(os.path.join(directory, "samples.tsv"), "w") as f:
        f.write("# sample list\n\ns1.snf\ns2.snf\tOVERRIDE\n")
    with open(os.path.join(directory, "regions.bed"), "w") as f:
        f.write("ctg1\t120000\t180000\nctg2\t5000\t90000\n")
    return directory


def record_key(line):
    f = line.split("\t", 3)
    return [f[0], int(f[1]), f[2], hashlib.sha256(line.encode()).hexdigest()[:24]]


def vcf_lines(text):
    """a VCF's lines without the run-stamp lines, records as record_key"""
    return [line if line.startswith("#") else record_key(line) for line in text.splitlines() if not line.startswith(STAMPS)]


def load_expected():
    """{label: {"inputs", "args", "dropped", "tasks", "vcf": the lines as vcf_lines gives them}}"""
    with open(EXPECTED) as f:
        g = json.load(f)
    out = {}
    for label, case in g["cases"].items():
        c = dict(case)
        c["vcf"] = [g["headers"][i] for i in case["headers"]] + [g["records"][i] for i in case["records"]]
        out[label] = c
    return out
