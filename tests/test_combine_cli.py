"""Combine mode's host side without a GPU: the sample list, header checks, the re-QC rule, the task plan with scatter against the
reference's (tests/golden/combine_cli, over the inputs of combine_cli_common), CombineResultTmpFile's ordering, and the command line's
refusals."""
import json
import types

import pytest

import combine_cli_common as ccc
from sniffles_b200 import __main__ as cli
from sniffles_b200 import abi, binding, combine_run
from sniffles_b200 import config as sconfig

GOLD = ccc.load_expected()


def _snf(path, **cfg):
    """an SNF with a header only"""
    header = {"config": dict({"snf_block_size": 100000, "snf_format_version": "S2_rc4", "sample_id": None, "build": "2.8.1",
                              "contig_lengths": [["c1", 1000]]}, **cfg), "index": {}, "snf_candidate_count": 0}
    with open(path, "w") as f:
        f.write(json.dumps(header) + "\n")
    return str(path)


def _config(*args):
    cfg = sconfig.SnifflesConfig(*args)
    cfg.mode = "combine"
    return cfg


def test_struct_sizes():
    L = binding.lib()
    import ctypes as C
    assert [L.snfb_sizeof(i) for i in (14, 15)] == [C.sizeof(abi.CombinePlanIn), C.sizeof(abi.CombinePlanOut)]


def test_tsv_sample_list(tmp_path):
    tsv = tmp_path / "s.tsv"
    tsv.write_text("# header\n\n  \na.snf\nb.snf\tB\n")
    assert combine_run.sample_list([str(tsv)]) == [("a.snf", None), ("b.snf", "B")]
    tsv.write_text("a.snf\n# x\nb.snf\tB\textra\n")
    with pytest.raises(combine_run.CombineError, match=r"Line 3 - expected either one or two columns"):
        combine_run.sample_list([str(tsv)])


def test_sample_id_precedence(tmp_path):
    a = _snf(tmp_path / "a.snf", sample_id="HEADER")
    b = _snf(tmp_path / "b.snf")
    tsv = tmp_path / "s.tsv"
    tsv.write_text(f"{a}\tTSV\n{a}\n{b}\n")
    cfg = _config("-i", str(tsv), "-v", str(tmp_path / "o.vcf"))
    combine_run.read_inputs(cfg)
    assert [s["sample_id"] for s in cfg.snf_input_info] == ["TSV", "HEADER", "b"]
    assert cfg.sample_ids_vcf == [(0, "TSV"), (1, "HEADER"), (2, "b")]


def test_header_validation(tmp_path):
    a = _snf(tmp_path / "a.snf")
    bad_bs = _snf(tmp_path / "bs.snf", snf_block_size=50000)
    bad_v = _snf(tmp_path / "v.snf", snf_format_version="S2_rc3")
    for path, msg in ((bad_bs, "SNF block size differs"), (bad_v, "SNF format version")):
        with pytest.raises(combine_run.CombineError, match=msg):
            combine_run.read_inputs(_config("-i", a, path, "-v", "o.vcf"))
        combine_run.read_inputs(_config("-i", a, path, "-v", "o.vcf", "--dev-skip-snf-validation"))
    # the SNF writer of this package leaves no snf_format_version: taken as the current one
    plain = _snf(tmp_path / "p.snf")
    h = json.loads(open(plain).readline())
    del h["config"]["snf_format_version"]
    open(plain, "w").write(json.dumps(h) + "\n")
    combine_run.read_inputs(_config("-i", a, plain, "-v", "o.vcf"))
    for path, cl in (("none.snf", None), ("odd.snf", "c1")):
        p = _snf(tmp_path / path, contig_lengths=cl)
        with pytest.raises(combine_run.CombineError, match=f"{path} has no contig_lengths"):
            combine_run.read_inputs(_config("-i", a, p, "-v", "o.vcf"))


@pytest.mark.parametrize("build,want", [(None, True), ("2.5.2", True), ("2.5.3", False), ("2.10.0", True), ("2.8.1-dev", False)])
def test_reqc_rule(build, want):
    cfg = {} if build is None else {"build": build}
    assert combine_run.needs_reqc({"config": cfg}, "auto") is want
    assert combine_run.needs_reqc({"config": cfg}, combine_run.parse_reqc("0")) is False
    assert combine_run.needs_reqc({"config": cfg}, combine_run.parse_reqc("1")) is True
    with pytest.raises(combine_run.CombineError, match="allowed values are: auto, 0, 1"):
        combine_run.parse_reqc("yes")


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return ccc.write_inputs(str(tmp_path_factory.mktemp("combine_cli_inputs")))


@pytest.mark.parametrize("label", sorted(GOLD))
def test_task_plan_matches_the_reference(label, inputs, monkeypatch):
    case = GOLD[label]
    monkeypatch.chdir(inputs)
    cfg = _config("-i", *case["inputs"], "-v", "o.vcf", *case["args"])
    contig_lengths, _ = combine_run.read_inputs(cfg)
    got = [[t.id, t.contig, t.block_indices[0], t.block_indices[-1], len(t.block_indices)] for t in combine_run.plan_tasks(cfg, contig_lengths)]
    want = case["tasks"]
    if isinstance(want, dict):
        assert [len(got), got[:3], got[-3:]] == [want["n"], want["first"], want["last"]]
    else:
        assert got == want


def test_scatter_ids_follow_the_clones():
    cfg = _config("-i", "a.snf", "-v", "o.vcf", "--threads", "4")
    cfg.sample_ids_vcf = [(k, str(k)) for k in range(3)]
    planned = combine_run.plan_tasks(cfg, [("a", 350_000_000), ("b", 1000)])
    # 3501 blocks x 3 samples = 10503 > 10000: clones of one block, ids 1 .. 3501, the next contig 3502
    assert [t.id for t in planned[:2]] == [1, 2] and planned[-2].id == 3501 and planned[-1].id == 3502 and planned[-1].contig == "b"
    cfg.threads = 1
    assert [t.id for t in combine_run.plan_tasks(cfg, [("a", 350_000_000), ("b", 1000)])] == [0, 1]


def test_tmpfile_result_on_hand_built_batches():
    c = lambda pos: types.SimpleNamespace(pos=pos)
    pairs = [(0, c(50)), (0, c(10)), (2, c(40)), (2, c(60)), (2, c(5)), (3, c(60)), (3, c(70))]
    calls, dropped = combine_run.stored_calls(pairs, True, True)
    assert [x.pos for x in calls] == [10, 50, 60, 60, 70] and dropped == 2         # 5 and 40 fall below 50, the first batch's highest
    calls, dropped = combine_run.stored_calls(pairs, True, False)
    assert [x.pos for x in calls] == [50, 10, 40, 60, 5, 60, 70] and dropped == 0
    calls, dropped = combine_run.stored_calls(pairs, False, True)
    assert [x.pos for x in calls] == [5, 10, 40, 50, 60, 60, 70] and dropped == 0


def test_command_line_refusals(tmp_path, caplog, monkeypatch):
    a = _snf(tmp_path / "a.snf")
    out = tmp_path / "o.vcf"
    cases = [
        (["-i", a, str(tmp_path / "x.tsv"), "-v", str(out)], "Please specify either"),
        (["-i", a, str(tmp_path / "missing.snf"), "-v", str(out)], "missing.snf"),
        (["-i", a, "-v", str(out), "--snf", str(tmp_path / "o.snf")], "--snf cannot be used with run mode combine"),
        (["-i", a], "Please specify at least one of"),
        (["-i", a, "-v", str(tmp_path / "no" / "o.vcf")], "does not exists"),
        (["-i", a, _snf(tmp_path / "b.snf", snf_block_size=1), "-v", str(out)], "SNF block size differs"),
        (["-i", a, "-v", str(out), "--re-qc", "2"], "allowed values are: auto, 0, 1"),
        (["-i", a, "-v", str(out), "--combine-consensus"], "--combine-consensus"),
        (["-i", a, "-v", str(out), "--combine-population", "p.snf"], "--combine-population"),
        (["-i", a, "-v", str(out), "--dev-population-snf", "p.snf"], "--combine-population"),
    ]
    for args, msg in cases:
        caplog.clear()
        assert cli.main(args) == 1, args
        assert msg in caplog.text and "(Fatal error, exiting.)" in caplog.text, (args, caplog.text)
        assert not out.exists()
    monkeypatch.setenv("WORLD_SIZE", "2")
    caplog.clear()
    assert cli.main(["-i", a, "-v", str(out)]) == 1
    assert "combine mode (.snf / .tsv input) runs on one GPU" in caplog.text and not out.exists()
    out.write_text("keep")
    monkeypatch.setenv("WORLD_SIZE", "1")
    assert cli.main(["-i", a, "-v", str(out)]) == 1 and "already exists" in caplog.text and out.read_text() == "keep"
