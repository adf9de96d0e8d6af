"""call.call_sample on the device against the unmodified reference's whole-sample run (tests/golden/call_sample/expected.json, written by
tests/golden/make_call_sample_golden.py): every VCF byte, the SNF content field by field, the same output at any pass budget, a
.vcf.gz that decompresses to the same text with its .tbi, the command line, and combine mode over two samples' SNFs."""
import gzip
import json
import os

import pytest

import call_sample_common as csc
from sniffles_b200 import __main__ as cli
from sniffles_b200 import call
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

with open(csc.EXPECTED) as _f:
    GOLD = json.load(_f)


def _config(case, paths, out_dir, vcf_name="out.vcf"):
    vcf_path, snf_path = os.path.join(out_dir, vcf_name), os.path.join(out_dir, "out.snf")
    args = csc.case_args(case, paths, vcf_path, snf_path)
    cfg = sconfig.default_config(*args)
    for k, v in GOLD["stamp"].items():
        setattr(cfg, k, v)
    cfg.input = paths["bam"]
    return cfg


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("call_sample_inputs")
    return {name: csc.write_inputs(name, str(d / name)) for name in {n for n, _ in csc.CASES.values()}}


@pytest.mark.parametrize("case", sorted(csc.CASES))
def test_call_sample_matches_reference(case, inputs, tmp_path):
    gold = GOLD["cases"][case]
    cfg = _config(case, inputs[gold["input"]], str(tmp_path))
    n = call.call_sample(cfg)
    text = (tmp_path / "out.vcf").read_text()
    assert n == gold["n_written"]
    assert cfg.task_read_id_offset_mult == gold["task_read_id_offset_mult"]
    assert csc.vcf_digest(text) == gold["vcf"]
    if "snf" in gold:
        assert csc.snf_digest(str(tmp_path / "out.snf")) == gold["snf"]
    else:
        assert not (tmp_path / "out.snf").exists()


@pytest.mark.parametrize("case", ["c3_mosaic", "phased_reference", "hg008_all_contigs"])
def test_any_budget_gives_the_same_files(case, inputs, tmp_path):
    """one task per pass (a budget of 1 byte: tasks without reads still share a pass) and a two-pass split give the bytes of one pass"""
    from sniffles_b200 import bamio, tasks
    gold = GOLD["cases"][case]
    cfg = _config(case, inputs[gold["input"]], str(tmp_path))
    bam = bamio.BamFile(cfg.input)
    sizes = [it.inflated for it in call.task_inputs(bam, tasks.plan(bam.contigs, cfg)[1])]
    bam.close()
    outs = []
    for k, budget in enumerate((1 << 40, 1, max(sum(sizes) - 1, max(sizes)))):
        d = tmp_path / str(k)
        d.mkdir()
        stats = {}
        call.call_sample(_config(case, inputs[gold["input"]], str(d)), budget=budget, stats=stats)
        assert stats["passes"] == len(list(call.group_passes(sizes, budget, size=lambda n: n)))
        assert stats["passes"] == 1 if k == 0 else stats["passes"] >= 2
        assert all(b <= budget for b in stats["pass_inflated_bytes"]) or k == 1
        outs.append(((d / "out.vcf").read_bytes(), csc.snf_digest(str(d / "out.snf"))))
    assert outs[0] == outs[1] == outs[2]
    assert csc.vcf_digest(outs[0][0].decode()) == gold["vcf"] and outs[0][1] == gold["snf"]


def test_vcf_gz_and_snf_only(inputs, tmp_path):
    case = "c1_snf"
    gold = GOLD["cases"][case]
    cfg = _config(case, inputs["c1_ont_1mb"], str(tmp_path), vcf_name="out.vcf.gz")
    assert call.call_sample(cfg) == gold["n_written"]
    with gzip.open(tmp_path / "out.vcf.gz", "rt") as f:
        assert csc.vcf_digest(f.read()) == gold["vcf"]
    assert (tmp_path / "out.vcf.gz.tbi").stat().st_size > 0
    d = tmp_path / "snf_only"
    d.mkdir()
    cfg = _config(case, inputs["c1_ont_1mb"], str(d))
    cfg.vcf = None
    assert call.call_sample(cfg) == 0
    assert sorted(os.listdir(d)) == ["out.snf"] and csc.snf_digest(str(d / "out.snf")) == gold["snf"]
    with pytest.raises(call.CallSampleError, match="already exists"):
        call.call_sample(cfg)
    cfg.allow_overwrite = True
    call.call_sample(cfg)
    assert csc.snf_digest(str(d / "out.snf")) == gold["snf"]


def test_command_line_gives_the_same_files(inputs, tmp_path):
    case = "phased_reference"
    gold = GOLD["cases"][case]
    cfg = _config(case, inputs["phased_phase"], str(tmp_path))
    call.call_sample(cfg)
    d = tmp_path / "cli"
    d.mkdir()
    args = csc.case_args(case, inputs["phased_phase"], str(d / "out.vcf"), str(d / "out.snf"))
    assert cli.main(args) == 0
    strip = lambda t: [l for l in t.splitlines() if not l.startswith(("##source=", "##command=", "##fileDate="))]     # the run's own stamp
    assert strip((d / "out.vcf").read_text()) == strip((tmp_path / "out.vcf").read_text())
    assert csc.snf_digest(str(d / "out.snf")) == csc.snf_digest(str(tmp_path / "out.snf")) == gold["snf"]


def test_combine_over_call_sample_snfs(inputs, tmp_path):
    """combine.CombineTask over two samples' SNFs written by call_sample gives the calls of the reference's CombineTask over the
    reference's own SNFs of the same two runs (stored by the generator under "combine")"""
    from sniffles_b200 import combine, tasks
    snfs = []
    for case in csc.COMBINE_CASES:
        d = tmp_path / case
        d.mkdir()
        call.call_sample(_config(case, inputs["phased_phase"], str(d)))
        snfs.append(str(d / "out.snf"))
    cfg = sconfig.default_config()
    cfg.mode, cfg.input = "combine", snfs
    cfg.snf_input_info, cfg.sample_ids_vcf = [], []
    for k, path in enumerate(snfs):
        cfg.snf_input_info.append({"internal_id": k, "sample_id": f"s{k}", "filename": path})
        cfg.sample_ids_vcf.append((k, f"s{k}"))
    ctx = tasks.device_context(0)
    blk = csc.load_block("phased_phase")
    for tid, (name, c) in enumerate(zip(blk.contig_names, blk.contig)):
        got = combine.CombineTask(tid, name, 0, int(c["length"]) - 1, cfg).execute(ctx=ctx)
        assert json.loads(json.dumps(csc.combine_digest(got))) == GOLD["combine"][name], name
