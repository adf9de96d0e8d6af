"""Force calling (--genotype-vcf) on the host: the target parser and the rewrite against the reference's own output
(tests/golden/genotype, written by make_genotype_golden.py), the .vcf.gz reader, the genotype rule for unmatched targets, the
task planning, and the plain-Python matching restatement that the device kernel is checked against."""
import json
import os
from types import SimpleNamespace as NS

import pytest

from oracle import genotype as ogt
from sniffles_b200 import bamio, genotype
from sniffles_b200 import config as sconfig

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "genotype")
EXPECTED = json.load(open(os.path.join(G, "expected.json")))


def _config():
    c = sconfig.default_config()
    for k, v in EXPECTED["config"].items():
        setattr(c, k, v)
    return c


def _bgzip(src, dst):
    data = open(src, "rb").read()
    with open(dst, "wb") as f:
        for o in range(0, len(data), 0xff00):
            f.write(bamio._bgzf_block(data[o:o + 0xff00], 6))
        f.write(bamio._BGZF_EOF)


@pytest.mark.parametrize("name", sorted(EXPECTED["files"]))
@pytest.mark.parametrize("gz", [False, True])
def test_parser_and_rewrite_match_reference(name, gz, tmp_path):
    want = EXPECTED["files"][name]
    path = os.path.join(G, name + ".vcf")
    if gz:
        path = str(tmp_path / (name + ".vcf.gz"))
        _bgzip(os.path.join(G, name + ".vcf"), path)
    if "error" in want:
        with pytest.raises(genotype.TargetVcfError) as e:
            genotype.read_targets(path)
        assert str(e.value) == want["error"]
        return
    header, targets = genotype.read_targets(path)
    got = [[t.contig, t.pos, t.svtype, t.svlen, t.end, t.bnd_info.mate_contig if t.bnd_info else None,
            bool(t.bnd_info.is_first) if t.bnd_info else None, t.raw_vcf_line_index] for t in targets]
    assert got == want["targets"]
    config = _config()
    gts = [tuple(g[:5]) + (tuple(g[5]),) for g in EXPECTED["genotypes"]]
    out = [genotype.rewrite_header(header, config)]
    for i, t in enumerate(targets):
        t.genotype_match_sv = NS(genotypes={0: gts[i % len(gts)]})
        out.append(genotype.rewrite_line(t, config) + "\n")
    assert "".join(out) == want["output"]


def test_defaults_agree_with_reference():
    c = _config()
    want = EXPECTED["reference_defaults"]
    assert (c.genotype_format, bool(c.phase), list(c.genotype_none[:5])) == (want["genotype_format"], want["phase"], want["genotype_none"])


def test_other_extensions_are_refused(tmp_path):
    p = tmp_path / "t.bcf"
    p.write_text("")
    with pytest.raises(genotype.TargetVcfError, match="Expected a .vcf or .vcf.gz"):
        genotype.read_targets(str(p))


def test_unmatched_genotype_from_coverage():
    config = _config()
    def gt(s, c, e, match=None):
        return genotype.genotype_of(NS(genotype_match_sv=match, coverage_start=s, coverage_center=c, coverage_end=e), config)
    assert gt(0, 0, 1) == config.genotype_none                  # round(1 / 3) = 0
    assert gt(2, 2, 1) == (0, 0, 0, 2, 0, (None, None))          # round(5 / 3) = 2
    assert gt(0, 1, 2) == (0, 0, 0, 1, 0, (None, None))
    assert gt(0, 0, 0, NS(genotypes={})) == config.genotype_none  # a match without a genotype falls back to the target's own
    assert gt(9, 9, 9, NS(genotypes={0: (0, 1, 5, 3, 4, (None, None))})) == (0, 1, 5, 3, 4, (None, None))


def test_plan_keeps_processed_contigs_and_targets_inside_tasks():
    config = sconfig.default_config("--genotype-vcf", "t.vcf")
    assert config.mode == "genotype_vcf"
    T = lambda contig, pos: NS(contig=contig, pos=pos)
    targets = [T("a", 5), T("b", 0), T("a", -1), T("a", 1_999_998), T("a", 1_999_999), T("short", 10), T("a", 7)]
    plan = genotype.plan([("a", 2_000_000), ("short", 5000), ("b", 1_000_000)], targets, config)
    assert [(tid, name, s, e) for tid, name, s, e, _ in plan] == [(0, "a", 0, 1_999_999), (1, "b", 0, 999_999)]
    assert [t.pos for t in plan[0][4]] == [5, 1_999_998, 7] and [t.pos for t in plan[1][4]] == [0]
    config = sconfig.default_config("--genotype-vcf", "t.vcf", "--contig", "short")
    assert [p[1] for p in genotype.plan([("a", 2_000_000), ("short", 5000)], targets, config)] == ["short"]


def test_snf_output_is_refused_in_genotype_mode():
    with pytest.raises(SystemExit):
        sconfig.default_config("--genotype-vcf", "t.vcf", "--snf", "x.snf")


def _sv(svtype, pos, svlen=0, mate=None, first=False):
    return NS(svtype=svtype, pos=pos, svlen=svlen, bnd_info=NS(mate_contig=mate, is_first=first) if svtype == "BND" else None)


def test_oracle_matching_rules():
    cands = [_sv("DEL", 10_000, -500), _sv("DEL", 10_010, -500), _sv("SINGLE_LEFT", 10_000), _sv("DEL", 4_990, -500),
             _sv("BND", 20_000, 0, "chr2"), _sv("BND", 20_100, 0, "chr3"), _sv("INS", 0, 300)]
    targets = [_sv("DEL", 10_005, -500),       # equal distance to cands 0 and 1: the earlier wins
               _sv("DEL", 5_010, -500),        # pos % 5000 < 500: also looks in the previous bin (cand 3)
               _sv("DEL", 10_000, 0),          # minlen 0 never matches
               _sv("BND", 20_050, 0, "chr3"),  # mate contig decides
               _sv("BND", 20_050, 0, None),
               _sv("INS", -1, 300),            # POS 0: bin 0, and pos % 5000 = 4999 adds bin 5000
               _sv("CNV", 10_000, -500)]
    assert ogt.match(cands, targets, 250, 1000, 1000) == [0, 3, -1, 5, -1, 6, -1]
    assert ogt.match(cands, [_sv("DEL", 10_000, -9000)], 250, 1000, 1000) == [-1]


def test_oracle_coverage_leaks_end_and_wraps():
    import numpy as np
    cv = np.arange(1000, dtype=np.uint16)
    t = [_sv("DEL", 100, -200), _sv("BND", 500, 0, "x", True), _sv("INS", 990, 10), _sv("BND", 10, 0, "x")]
    assert ogt.coverage(t, cv, 100) == [(100, 200, 200), (399, 499, 400), (890, 990, 0), (910, 10, 0)]
    with pytest.raises(UnboundLocalError):
        ogt.coverage([_sv("BND", 10, 0, "x")], cv, 100)
