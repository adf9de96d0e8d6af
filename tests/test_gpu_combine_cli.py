"""Combine mode on the device: snfb_combine_plan's chunk plan against the host restatement (CombineTask.plan + plan_arrays), and the
command line against the reference's combine mode (tests/golden/combine_cli, made by tests/golden/make_combine_cli_golden.py over the
inputs of combine_cli_common)."""
import gzip
import json
import os
import random

import numpy as np
import pytest

import call_sample_common as csc
import combine_cli_common as ccc
from sniffles_b200 import __main__ as cli, combine, combine_run, snf, tasks
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = ccc.load_expected()


def _config(n_samples, *extra):
    cfg = sconfig.default_config(*extra)
    cfg.mode = "combine"
    cfg.snf_input_info = [{"internal_id": k, "sample_id": f"s{k}", "filename": ""} for k in range(n_samples)]
    cfg.sample_ids_vcf = [(k, f"s{k}") for k in range(n_samples)]
    return cfg


def _device_vs_host(ctx, cfg, planned, readers):
    """one snfb_combine_plan over `planned` equals CombineTask.plan + plan_arrays (+ snfb_combine_groups on that plan)"""
    fp = combine_run.join([_decode(cfg, t, readers) for t in planned])
    flat = fp.arrays()
    res = ctx.combine_plan(flat, cfg)
    got, out = fp.plan(res, flat)
    want = combine.Plan()
    for k, t in enumerate(planned):
        t.plan(readers, want, k)
    a = combine.plan_arrays(want, cfg)
    key = lambda c: (c.svtype, c.id, c.pos, c.svlen, c.support, c._sample_index)      # an SNFReader unpickles new objects per read
    assert [key(c) for c in got.cands] == [key(c) for c in want.cands]
    assert got.chains == want.chains and got.chunks == want.chunks
    np.testing.assert_array_equal(res["chains"], a["chains"])
    np.testing.assert_array_equal(res["chunks"], a["chunks"])
    for k in ("pos", "svlen", "sample", "mate_pos", "alt_len"):
        np.testing.assert_array_equal(flat[k][res["perm"]], a[k])
    names = {i: n for n, i in fp.contig_ids.items()}
    names_h = {i: n for n, i in want.contig_ids.items()}
    bnd = a["mate_contig"] != 0
    assert [names[i] for i in flat["mate_contig"][res["perm"]][bnd]] == [names_h[i] for i in a["mate_contig"][bnd]]
    host = ctx.combine_groups(want, cfg)
    n = len(want.cands)
    np.testing.assert_array_equal(out[0], host[0][:n])
    np.testing.assert_array_equal(out[1], host[1][:n])
    used = out[1] >= 0                                   # emit_ord and cov_non of an unused group slot are not written
    np.testing.assert_array_equal(out[2][used], host[2][:n][used])
    np.testing.assert_array_equal(out[3][used], host[3][:n][used])
    return len(want.cands)


def _decode(cfg, task, readers):
    fp = combine_run.FlatPass(cfg)
    fp.add_task(task, readers)
    return fp


def test_device_plan_on_committed_snfs():
    paths = [os.path.join(HERE, "golden", "combine", f"sample{k}.snf") for k in range(1, 5)]
    ctx = tasks.device_context(0)
    for extra in ((), ("--combine-pctseq", "0")):
        cfg = _config(4, *extra)
        readers = {k: snf.SNFReader(p) for k, p in enumerate(paths)}
        planned = [combine.CombineTask(0, "ctg1", 0, 349_999, cfg), combine.CombineTask(1, "ctg2", 0, 259_999, cfg)]
        assert _device_vs_host(ctx, cfg, planned, readers) > 0
        for r in readers.values():
            r.close()


class _Reader:
    """an SNFReader look-alike over blocks held in memory: {(contig, block): [parts]}"""

    def __init__(self, blocks):
        self.blocks = blocks

    def read_blocks(self, contig, block):
        return self.blocks.get((contig, block))


def _seeded(seed, n_samples, n_blocks, bs=100_000):
    SVCall, BND, _ = snf.compat_classes()
    rnd = random.Random(seed)
    readers = {}
    for s in range(n_samples):
        blocks = {}
        for b in range(n_blocks):
            if rnd.random() < 0.25:                                    # the sample has no such block
                continue
            parts = []
            for _ in range(rnd.choice([1, 1, 2])):
                part = {t: [] for t in snf.TYPES}
                part["_COVERAGE"] = {b * bs + i * 500: rnd.randrange(0, 40) for i in range(0, 200, rnd.choice([1, 3]))}
                for t in snf.TYPES:
                    for _ in range(rnd.choice([0, 3, 12, 40])):
                        # a few sites per block, so that bins fill and chunks close exactly at bin_max; pos < 0 in block 0 (truncation)
                        site = rnd.choice([-250, -99, 0, 99, 100, 4_950, 5_000, 37_777, 99_999]) if b == 0 else rnd.choice([100, 199, 200, 4_999, 60_000])
                        pos = b * bs + site + rnd.randrange(-3, 4)
                        svlen = rnd.choice([-1, 1]) * rnd.randrange(50, 900) if t != "BND" else 0
                        c = SVCall(contig="c1", pos=pos, id=f"{t}.{rnd.randrange(1 << 20):X}", ref="N", alt="ACGT" * rnd.randrange(1, 30), qual=rnd.randrange(0, 60),
                                   filter="PASS", info={}, svtype=t, svlen=svlen, end=pos + abs(svlen), genotypes={0: (0, 1, 20, 5, 5, (None, None))}, precise=True,
                                   support=rnd.choice([1, 2, 3, 3, 3, 5, 5, 8]), rnames=None, qc=True, nm=-1, postprocess=None, fwd=1, rev=1)
                        if t == "BND":
                            c.bnd_info = BND(rnd.choice(["c1", "c2", "c3"]), rnd.randrange(0, 10_000), True, False)
                        part[t].append(c)
                parts.append(part)
            blocks[("c1", b * bs)] = parts
        readers[s] = _Reader(blocks)
    return readers


@pytest.mark.parametrize("seed,n_samples", [(1, 2), (2, 5), (3, 30), (4, 60)])
def test_device_plan_on_seeded_shapes(seed, n_samples):
    """support ties, bins that close a chunk exactly at bin_max, empty and missing blocks, absent samples, BND mates, pos < 0; several
    tasks in one call, one of them with no blocks at all"""
    ctx = tasks.device_context(0)
    cfg = _config(n_samples)
    readers = _seeded(seed, n_samples, 6)
    bs = cfg.snf_block_size
    planned = [combine.CombineTask(0, "c1", 0, 2 * bs - 1, cfg), combine.CombineTask(1, "c1", 0, 0, cfg, block_indices=[7 * bs]),
               combine.CombineTask(2, "c1", 2 * bs, 6 * bs - 1, cfg)]
    assert _device_vs_host(ctx, cfg, planned, readers) > 0


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return ccc.write_inputs(str(tmp_path_factory.mktemp("combine_cli_inputs")))


def _args(case, out):
    return ["-i"] + case["inputs"] + ["-v", out] + case["args"]


def _lines(path):
    data = open(path, "rb").read()
    return ccc.vcf_lines((gzip.decompress(data) if path.endswith(".gz") else data).decode())


@pytest.mark.parametrize("label", sorted(GOLD))
def test_command_line_matches_the_reference(label, inputs, tmp_path, monkeypatch):
    case = GOLD[label]
    monkeypatch.chdir(inputs)                      # a .tsv names its SNFs relative to the working directory, as the reference reads it
    out = str(tmp_path / "out.vcf")
    assert cli.main(_args(case, out)) == 0
    assert _lines(out) == case["vcf"]
    if label in ("two", "tmpfile", "regions"):
        gz = str(tmp_path / "out.vcf.gz")
        assert cli.main(_args(case, gz)) == 0
        if label == "tmpfile":
            # above --combine-max-inmemory-results a .vcf.gz becomes the plain file, unsorted: nothing is dropped
            got = _lines(str(tmp_path / "out.vcf"))
            assert not os.path.exists(gz) and [x for x in got if isinstance(x, str)] == [x for x in case["vcf"] if isinstance(x, str)]
            keys = {tuple(x) for x in got if not isinstance(x, str)}
            assert {tuple(x) for x in case["vcf"] if not isinstance(x, str)} <= keys and len(got) == len(case["vcf"]) + case["dropped"]
        else:
            assert _lines(gz) == case["vcf"] and os.path.getsize(gz + ".tbi") > 0


@pytest.mark.parametrize("label", ["default4", "tmpfile", "regions", "scatter"])
def test_pass_budgets_give_the_same_file(label, inputs, tmp_path, monkeypatch):
    case = GOLD[label]
    monkeypatch.chdir(inputs)
    texts = []
    for budget in (1, 10 ** 9):
        cfg = sconfig.SnifflesConfig(*_args(case, str(tmp_path / f"b{budget}.vcf")))
        st = {}
        combine_run.combine_snfs(cfg, budget=budget, stats=st)
        assert st["dropped"] == case["dropped"]
        texts.append(_lines(str(tmp_path / f"b{budget}.vcf")))
        if budget == 1:
            assert st["passes"] >= 2 or label == "scatter"
    assert texts[0] == texts[1] == case["vcf"]


@pytest.fixture(scope="module")
def bam_inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("combine_cli_inputs")
    return csc.write_inputs("phased_phase", str(d / "phased_phase"))


def test_command_line_over_call_sample_snfs(bam_inputs, tmp_path):
    """SNFs written by call_sample on the device, combined through the command line with --re-qc 0, give the calls of the reference's
    CombineTask over the reference's own SNFs of the same runs (tests/golden/call_sample, "combine")"""
    from sniffles_b200 import call
    gold = json.load(open(csc.EXPECTED))
    snfs = []
    for case in csc.COMBINE_CASES:
        d = tmp_path / case
        d.mkdir()
        cfg = sconfig.default_config(*csc.case_args(case, bam_inputs, str(d / "out.vcf"), str(d / "out.snf")))
        for k, v in gold["stamp"].items():
            setattr(cfg, k, v)
        cfg.input = bam_inputs["bam"]
        call.call_sample(cfg)
        snfs.append(str(d / "out.snf"))
    out = str(tmp_path / "combined.vcf")
    assert cli.main(["-i", *snfs, "-v", out, "--re-qc", "0"]) == 0
    records = [line.split("\t") for line in open(out) if not line.startswith("#")]
    # the same run's calls, taken before the VCF writer: one device pass over every task, as the command line made it
    cfg = sconfig.SnifflesConfig("-i", *snfs, "-v", str(tmp_path / "unused.vcf"), "--re-qc", "0")
    cfg.mode = "combine"
    contig_lengths, reqc = combine_run.read_inputs(cfg)
    assert not any(reqc.values())
    readers = {s["internal_id"]: snf.SNFReader(s["filename"]) for s in cfg.snf_input_info}
    fp = combine_run.join([_decode(cfg, t, readers) for t in combine_run.plan_tasks(cfg, contig_lengths)])
    flat = fp.arrays()
    plan, res = fp.plan(tasks.device_context(0).combine_plan(flat, cfg), flat)
    calls = combine.CombineTask.emit(fp.tasks, plan, res)
    for k, t in enumerate(fp.tasks):
        assert json.loads(json.dumps(csc.combine_digest(calls[k]))) == gold["combine"][t.contig], t.contig
    ids = {f"Sniffles2.{c.id}" for k in calls for c in calls[k]}
    assert records and all(r[2] in ids for r in records)
