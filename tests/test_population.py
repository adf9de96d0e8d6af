"""Population annotation of combine mode (--combine-population) without a GPU: the population SNF reader against the reference's files
(tests/golden/population, made by tests/golden/make_population_golden.py), the refusals, the header lines, the host INFO step, and the
oracle against the reference's picks."""
import gzip
import json
import logging
import pickle
import types

import pytest

import combine_cli_common as ccc
import population_common as pc
from oracle import population as opop
from sniffles_b200 import __main__ as cli
from sniffles_b200 import combine_run, snf, vcf
from sniffles_b200 import config as sconfig

POPS, GOLD = pc.load_expected()


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return ccc.write_inputs(str(tmp_path_factory.mktemp("population_inputs")))


def test_reader_against_the_reference_files():
    for name, meta in POPS.items():
        r = snf.PopulationReader(pc.snf_path(name))
        try:
            assert r.population == {"version": 1, "name": "Population", "description": "A sample population", "size": 4}
            seen = []
            for contig in ("ctg1", "ctg2"):
                for block, blk in r.blocks(contig):
                    assert blk["_COVERAGE"] == {}
                    for t in pc.TYPES:
                        for v in blk[t]:
                            assert (type(v).__module__, type(v).__name__) == ("sniffles.snfp", "PopulationVariant")
                            assert v.contig == contig and v.svtype == t and isinstance(v.af, float) and v.rnames is None
                            assert all(hasattr(v, f) for f in ("pos", "id", "alt", "svlen", "end", "genotyped_sample_count", "variant_sample_count"))
                            seen.append(v.id)
            # the [0] rule: only P_edit lists a block in two parts, and no variant of its second part is read
            two = [(c, b) for c, blocks in r.index.items() for b, parts in blocks.items() if len(parts) > 1]
            assert len(two) == (name == "P_edit")
            assert not any(x.endswith("_part2") for x in seen)
            if name == "P_edit":
                contig, block = two[0]
                start, length = r.index[contig][block][1]
                r.f.seek(r.header_length + start)
                blk = pickle.loads(gzip.decompress(r.f.read(length)))
                second = [v.id for t in pc.TYPES for v in blk[t]]
                assert second and all(x.endswith("_part2") for x in second) and len(seen) + len(second) == meta["variants"]
            else:
                assert len(seen) == meta["variants"]
        finally:
            r.close()


def test_population_table_flattening():
    pop = combine_run.Population(pc.snf_path("P_edit"), ["ctg2"])
    assert set(pop.cols["contig"].tolist()) == {0} and len(pop.variants) == len(pop.alts)
    assert [v.svtype for v in pop.variants] == [pc.TYPES[t] for t in pop.cols["svtype"].tolist()]
    assert "zero_len_ins" in [v.id for v in pop.variants]


def _refused(args, out, caplog, msg):
    caplog.clear()
    assert cli.main(args) == 1, args
    assert msg in caplog.text and "--combine-population" in caplog.text and "(Fatal error, exiting.)" in caplog.text, caplog.text
    assert not out.exists()


def test_refusals(inputs, tmp_path, caplog, monkeypatch):
    monkeypatch.chdir(inputs)
    out = tmp_path / "o.vcf"
    base = ["-i", "s1.snf", "s2.snf", "-v", str(out)]
    _refused(base + ["--combine-population", str(tmp_path / "missing.snf")], out, caplog, "missing.snf")
    _refused(base + ["--combine-population", "s3.snf"], out, caplog, "no population record")
    _refused(base + ["--dev-population-snf", str(tmp_path / "p.snf")], out, caplog, "writing a population SNF is not supported")
    # a population header over blocks of sample candidates
    with open("s3.snf", "rb") as f:
        header, rest = json.loads(f.readline()), f.read()
    header["population"] = {"version": 1, "name": "Population", "description": "x", "size": 1}
    bad = tmp_path / "fake_pop.snf"
    bad.write_bytes((json.dumps(header) + "\n").encode() + rest)
    _refused(base + ["--combine-population", str(bad)], out, caplog, "does not hold PopulationVariant lists")
    not_snf = tmp_path / "text.snf"
    not_snf.write_text("not json\n")
    _refused(base + ["--combine-population", str(not_snf)], out, caplog, "Unable to read")


def _header(cfg):
    import io
    buf = io.StringIO()
    vcf.VCFWriter(cfg, buf).write_header([("ctg1", 10)])
    return [line for line in buf.getvalue().splitlines() if "POPULATION" in line]


def test_header_lines(caplog):
    want = ['##INFO=<ID=POPULATION_AF,Number=1,Type=Float,Description="Population Allele Frequency">',
            '##INFO=<ID=POPULATION_SIZE,Number=1,Type=Integer,Description="Size of genotyped population for this variant">']
    cfg = sconfig.SnifflesConfig("-i", "a.snf", "b.snf", "-v", "o.vcf", "--combine-population", "p.snf", "--phase")
    cfg.mode = "combine"
    caplog.set_level(logging.WARNING)
    assert _header(cfg) == want and "does not provide population phasing" in caplog.text
    cfg = sconfig.SnifflesConfig("-i", "a.snf", "b.snf", "-v", "o.vcf")
    cfg.mode = "combine"
    assert _header(cfg) == []
    # the golden headers: the two lines right after LASM
    for case in GOLD.values():
        heads = [x for x in case["vcf"] if isinstance(x, str)]
        k = next(i for i, x in enumerate(heads) if "ID=LASM" in x)
        assert heads[k + 1:k + 3] == want


def test_host_info_step():
    V = snf.population_class()
    v = V("ctg1", 10, "x", "A", "INS", 5, 10, 2 / 3, 7, 3)
    call = types.SimpleNamespace(info={"STDEV_POS": 1.0})
    call.set_info = lambda k, val: call.info.__setitem__(k, val)
    combine_run.set_population_info(call, v)
    assert call.info["POPULATION_AF"] == 0.66667 and call.info["POPULATION_SIZE"] == 7
    assert vcf._fmt_info("POPULATION_AF", call.info["POPULATION_AF"]) == "POPULATION_AF=0.667"
    combine_run.set_population_info(call, None)
    af, sz = call.info["POPULATION_AF"], call.info["POPULATION_SIZE"]
    assert (af, sz) == (0, 0) and type(af) is int and type(sz) is int
    assert vcf._fmt_info("POPULATION_AF", af) == "POPULATION_AF=0"
    assert sorted(call.info) == ["POPULATION_AF", "POPULATION_SIZE", "STDEV_POS"]
    # n_samples == 1: the call's info is its first candidate's own dict, which receives the two values
    cand_info = {"VAF": 0.5}
    one = types.SimpleNamespace(info=cand_info)
    one.set_info = lambda k, val: one.info.__setitem__(k, val)
    combine_run.set_population_info(one, v)
    assert cand_info == {"VAF": 0.5, "POPULATION_AF": 0.66667, "POPULATION_SIZE": 7}


def test_oracle_against_the_reference_picks():
    table, q, sets = pc.load_vectors()
    for s in sets:
        got = opop.match(table, q, s["combine_match"], s["combine_match_max"], s["combine_pctseq"], 100_000)
        assert got == s["best"], s["combine_pctseq"]


def test_golden_cases_cover_every_class():
    total = {}
    for case in GOLD.values():
        for k, n in case["classes"].items():
            total[k] = total.get(k, 0) + n
    for k in ("ins_aligned_match", "ins_alignment_rejected", "non_ins_match", "unmatched", "contig_absent"):
        assert total[k] > 0, k
    assert GOLD["contig_absent"]["classes"]["contig_absent"] == len([x for x in GOLD["contig_absent"]["vcf"] if not isinstance(x, str)])
