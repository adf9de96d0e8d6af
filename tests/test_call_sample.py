"""call_sample's host side without a GPU: the task plan against the reference's rule (sniffles:311-358 over util.should_process_contig),
the grouping of tasks into device passes, the offset rule of sniffles:304-309, the
refusal of existing outputs and of what the mode does not run, and the command line's dispatch."""
import math
import os

import numpy as np
import pytest

import call_sample_common as csc
from sniffles_b200 import bamio, call, genotype, tasks
from sniffles_b200 import __main__ as cli
from sniffles_b200 import config as sconfig

HEADER = [("chr1", 248_956_422), ("short_a", 999_999), ("chr2", 1_000_000), ("one", 1), ("two", 2), ("short_b", 5000), ("chr3", 3_000_000)]


def _ref_plan(contigs, config):
    """sniffles:311-358 with task_count 1, written out as the reference loops (the contig kept in the header even when no task fits)"""
    names, planned = [], []
    for name, L in contigs:
        if config.contig and name not in config.contig:
            continue
        if not config.all_contigs and L < 1_000_000 and not (config.contig and name in config.contig):
            continue
        names.append((name, L))
        start = 0
        while start < L - 1:
            planned.append((len(planned), name, start, min(L - 1, start + L)))
            start += L
    return names, planned


@pytest.mark.parametrize("args", [[], ["--all-contigs"], ["--contig", "short_b", "--contig", "chr3"], ["--contig", "one", "--contig", "two"],
                                  ["--contig", "nope"], ["--all-contigs", "--contig", "chr2"]])
def test_plan_follows_the_reference_rule(args):
    cfg = sconfig.default_config(*args)
    assert tasks.plan(HEADER, cfg) == _ref_plan(HEADER, cfg)


def test_genotype_plan_is_the_shared_plan():
    cfg = sconfig.default_config("--all-contigs")
    T = genotype.Target
    targets = [T("chr2", 5, 1, "N", "<DEL>", None, "PASS", {}), T("two", 0, 2, "N", "<DEL>", None, "PASS", {}),
               T("chr2", 999_999, 3, "N", "<DEL>", None, "PASS", {})]
    got = genotype.plan(HEADER, targets, cfg)
    assert [p[:4] for p in got] == tasks.plan(HEADER, cfg)[1]
    assert {p[1]: [t.id for t in p[4]] for p in got}["chr2"] == [1] and {p[1]: [t.id for t in p[4]] for p in got}["two"] == [2]


@pytest.mark.parametrize("n", [0, 1, 2, 9, 10, 11, 339, 1225, 6_270_000, 10 ** 8])
def test_offset_rule(n):
    want = 10 ** 9 if n == 0 else 10 ** math.ceil(math.log(n) + 1)
    assert call.read_id_offset_mult(n) == want
    assert n == 0 or call.read_id_offset_mult(n) > n          # read ids of one task never reach the next task's


@pytest.mark.parametrize("seed", range(6))
def test_passes_keep_order_and_budget(seed):
    rng = np.random.default_rng(seed)
    sizes = [int(x) for x in rng.integers(0, 1000, int(rng.integers(1, 60)))]
    budget = int(rng.integers(1, 2500))
    items = [(k, s) for k, s in enumerate(sizes)]
    groups = list(call.group_passes(iter(items), budget))
    assert [it for g in groups for it in g] == items                               # every task once, in task order
    for k, g in enumerate(groups):
        total = sum(s for _, s in g)
        assert total <= budget or len(g) == 1                                      # over budget only alone
        if k + 1 < len(groups):
            assert total + groups[k + 1][0][1] > budget                            # greedy: the next task did not fit


def test_oversized_task_runs_alone():
    items = [("a", 10), ("big", 500), ("b", 10), ("c", 10), ("huge", 10 ** 9), ("d", 0)]
    assert [[n for n, _ in g] for g in call.group_passes(items, 100)] == [["a"], ["big"], ["b", "c"], ["huge"], ["d"]]
    assert [[n for n, _ in g] for g in call.group_passes(items, 1)] == [["a"], ["big"], ["b"], ["c"], ["huge"], ["d"]]
    assert [[n for n, _ in g] for g in call.group_passes(items, 10 ** 10)] == [[n for n, _ in items]]
    assert list(call.group_passes([], 5)) == []


def test_passes_are_lazy():
    taken = []

    def gen():
        for k in range(5):
            taken.append(k)
            yield (k, 10)
    g = call.group_passes(gen(), 20)
    assert next(g) == [(0, 10), (1, 10)] and taken == [0, 1, 2]       # the third task is read only to close the first pass


def test_join_inputs_shifts_spans(tmp_path):
    blk = csc.load_block("c3_hifi_mosaic")
    path, _ = bamio.write_bam(str(tmp_path / "s.bam"), blk, block_bytes=4000)
    bam = bamio.BamFile(path)
    regions = [(n, 0, L - 1) for n, L in bam.contigs]
    parts = [bam.device_input([r]) for r in regions]
    z, spans = call.join_inputs(parts)
    assert len(z) == sum(len(p[0]) for p in parts) and len(spans) == sum(len(p[1]) for p in parts)
    assert np.array_equal(spans["task"], np.repeat(np.arange(len(parts)), [len(p[1]) for p in parts]))
    o = 0
    for k, (zk, sk) in enumerate(parts):
        sel = spans[spans["task"] == k]
        assert np.array_equal(sel["cbeg"], sk["cbeg"] + o) and np.array_equal(sel["cend"], sk["cend"] + o)
        assert np.array_equal(sel["ubeg"], sk["ubeg"]) and np.array_equal(sel["uend"], sk["uend"])
        assert bytes(z[o:o + len(zk)]) == bytes(zk)
        o += len(zk)
    assert call.inflated_bytes(parts[0][0]) == sum(m[3] for m in bamio.bgzf_members(bytes(parts[0][0])))
    bam.close()


def test_existing_outputs_are_refused(tmp_path):
    vcf_path, snf_path = tmp_path / "o.vcf", tmp_path / "o.snf"
    for existing in (vcf_path, snf_path):
        existing.write_text("keep")
        cfg = sconfig.default_config("--vcf", str(vcf_path), "--snf", str(snf_path))
        with pytest.raises(call.CallSampleError, match=f"Output file '{existing}' already exists! Use --allow-overwrite"):
            call.call_sample(cfg)
        assert existing.read_text() == "keep"
        existing.unlink()
    cfg = sconfig.default_config("--vcf", str(tmp_path / "missing_dir" / "o.vcf"))
    with pytest.raises(call.CallSampleError, match="does not exists"):
        call.call_sample(cfg)
    cfg = sconfig.default_config()
    cfg.vcf = None
    with pytest.raises(call.CallSampleError, match="at least one of: --vcf or --snf"):
        call.call_sample(cfg)
    with pytest.raises(call.CallSampleError, match="--gpus"):
        call.call_sample(sconfig.default_config("--vcf", str(tmp_path / "x.vcf"), "--gpus", "2"))


def test_command_line_refuses_what_it_does_not_run(tmp_path, caplog):
    assert cli.main(["--input", "a.snf", "b.snf", "--vcf", str(tmp_path / "o.vcf")]) == 1
    assert cli.main(["--input", "a.cram", "--vcf", str(tmp_path / "o.vcf")]) == 1
    assert "single .bam" in caplog.text
    (tmp_path / "o.vcf").write_text("keep")
    assert cli.main(["--input", "a.bam", "--vcf", str(tmp_path / "o.vcf")]) == 1
    assert "already exists" in caplog.text and (tmp_path / "o.vcf").read_text() == "keep"
