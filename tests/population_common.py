"""Golden data of the population annotation (tests/golden/make_population_golden.py writes it; tests/test_population.py and
tests/test_gpu_population.py read it): the population SNFs, the reference's VCFs in combine_cli_common's compact form, and the
reference's picks for seeded queries against P_edit, which seeded_queries draws again from P_edit's variants."""
import json
import os
import random

import combine_cli_common as ccc

HERE = os.path.dirname(os.path.abspath(__file__))
DIR = os.path.join(HERE, "golden", "population")
TYPES = ["INS", "DEL", "DUP", "INV", "BND"]


def snf_path(name):
    return os.path.join(DIR, name + ".snf")


def load_expected():
    """(populations, {label: case with "vcf" as combine_cli_common.load_expected gives it})"""
    with open(os.path.join(DIR, "expected.json")) as f:
        g = json.load(f)
    out = {}
    for label, case in g["cases"].items():
        c = dict(case)
        c["vcf"] = [g["headers"][i] for i in case["headers"]] + [g["records"][i] for i in case["records"]]
        out[label] = c
    return g["populations"], out


def seeded_queries(contig, svtype, pos, svlen, alts, n, seed):
    """n calls drawn near the given variants (file-order columns, contig names, ALT bytes), and a zero-length INS at ctg2:259990:
    positions within 300 bp (a fifth anywhere on a 350-kb contig), lengths within 60, up to 24 substitutions in an INS ALT, and 3 %
    on a contig the population lacks"""
    rng = random.Random(seed)
    q = {k: [] for k in ("contig", "svtype", "pos", "svlen", "alt")}
    for _ in range(n):
        i = rng.randrange(len(pos))
        p = max(0, pos[i] + rng.randrange(-300, 300)) if rng.random() < 0.8 else rng.randrange(0, 350_000)
        a = bytearray(alts[i])
        if svtype[i] == "INS" and a and a[:1] != b"<":
            for _ in range(rng.randrange(0, min(24, max(1, len(a) // 4)))):
                a[rng.randrange(len(a))] = ord(rng.choice("ACGTN"))
        for k, v in zip(q, (contig[i] if rng.random() < 0.97 else "ctg9", svtype[i], p, svlen[i] + rng.randrange(-60, 60) if svtype[i] != "BND" else 0, bytes(a))):
            q[k].append(v)
    for k, v in zip(q, ("ctg2", "INS", 259_990, 0, b"")):
        q[k].append(v)
    return q


def load_vectors():
    """(table columns in file order over the vectors' contigs, query columns as snfb_population_match takes them, parameter sets)"""
    from sniffles_b200 import combine_run          # not at import: the golden generator runs the reference's own `sniffles` package
    with open(os.path.join(DIR, "match_vectors.json")) as f:
        vec = json.load(f)
    pop = combine_run.Population(snf_path("P_edit"), vec["contigs"])
    table = dict(pop.cols)
    table["alt"] = pop.alts
    names = {i: name for name, i in pop.contig_ids.items()}
    q = seeded_queries([names[c] for c in pop.cols["contig"].tolist()], [v.svtype for v in pop.variants], pop.cols["pos"].tolist(),
                       pop.cols["svlen"].tolist(), pop.alts, vec["n"], vec["seed"])
    q["contig"] = [pop.contig_ids.get(c, -1) for c in q["contig"]]
    q["svtype"] = [TYPES.index(t) for t in q["svtype"]]
    return table, q, vec["sets"]


def case_args(case, workdir, out):
    return ["-i", *case["inputs"], "-v", out, *case["args"], "--combine-population", snf_path(case["population"])]


vcf_lines = ccc.vcf_lines
