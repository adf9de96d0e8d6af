"""call_sample on several ranks, without a GPU: the task weights read from the BAM index and their assignment to ranks, rank 0's merge of
the ranks' payloads into the output files, and the refusals of a world size of 2 on gloo with two spawned CPU processes."""
import io
import os

import pytest

import call_sample_common as csc
import ranks_common
from sniffles_b200 import bamio, call, dist, snf, tasks
from sniffles_b200 import config as sconfig


@pytest.fixture(scope="module")
def bams(tmp_path_factory):
    """hg002.bam (htslib-written, one contig with reads among many) and phased_phase written by bamio.write_bam in small BGZF blocks"""
    d = tmp_path_factory.mktemp("ranks_bams")
    path, _ = bamio.write_bam(str(d / "phased.bam"), csc.load_block("phased_phase"), block_bytes=4000)
    return {"hg002": csc.HG002, "phased": path}


@pytest.mark.parametrize("which", ["hg002", "phased"])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_weights_and_assignment(bams, which, world):
    cfg = sconfig.default_config("--all-contigs")
    runs = []
    for _ in range(2):                                   # two fresh opens of the BAM: the same weights and owners
        bam = bamio.BamFile(bams[which])
        planned = tasks.plan(bam.contigs, cfg)[1]
        w = dist.task_weights(bam, planned)
        runs.append((w, dist.lpt_assign(w, world)))
        with_reads = [(bam.count_mapped(name) or 0) > 0 for _, name, _, _ in planned]
        bam.close()
    assert runs[0] == runs[1]
    w, owner = runs[0]
    assert len(owner) == len(planned) and set(owner) <= set(range(world))      # every planned task on exactly one rank
    assert [x > 0 for x in w] == with_reads and any(with_reads)
    size = os.path.getsize(bams[which])                  # the compressed bytes of the records: most of the file, never more
    assert 0.9 * size <= sum(w) <= size


def test_regions_weigh_only_their_windows(bams):
    bam = bamio.BamFile(bams["phased"])
    (a, La), (b, Lb) = bam.contigs[:2]
    whole = dist.task_weights(bam, tasks.plan(bam.contigs, sconfig.default_config("--all-contigs"))[1])
    windows = [(La // 4, La // 3), (La // 2, La // 2 + 5000)]
    cfg = sconfig.default_config("--all-contigs", *[x for s, e in windows for x in ("--region", f"{a}:{s}-{e}")],
                                 "--region", f"{b}:{Lb // 2}-{Lb // 4}")
    planned = tasks.plan(bam.contigs, cfg)[1]
    assert [p[1] for p in planned] == [a, b]
    w = dist.task_weights(bam, planned, cfg.regions_by_contig)
    assert w[0] == sum(dist.task_weights(bam, [(0, a, s, e)])[0] for s, e in windows)
    assert 0 < w[0] < whole[0]
    assert w[1] == 0                                     # start > end: the task fails on whichever rank runs it
    bam.close()


def test_three_ranks_on_two_tasks_leave_one_empty(bams):
    bam = bamio.BamFile(bams["phased"])
    planned = tasks.plan(bam.contigs, sconfig.default_config("--all-contigs"))[1]
    assert len(planned) == 2
    owner = dist.lpt_assign(dist.task_weights(bam, planned), 3)
    assert len(set(owner)) == 2                          # both tasks weigh: two ranks get one each, the third none
    bam.close()


def _part(tid, contig, blocks):
    """a hand-made SNF part: blocks {block: bytes}"""
    index, data = {}, b""
    for blk, raw in blocks.items():
        index[blk] = (len(data), len(raw))
        data += raw
    return (tid, contig, index, data, len(blocks), float(tid))


def _payload(rank, items, nm=None, error=None):
    return {"rank": rank, "tasks": items, "failed": [], "nm": nm, "stats": {}, "error": error}


def _merge_config(tmp_path):
    cfg = sconfig.default_config("--vcf", str(tmp_path / "o.vcf"), "--snf", str(tmp_path / "o.snf"))
    for k, v in csc.STAMP.items():
        setattr(cfg, k, v)
    cfg.sample_ids_vcf = [(0, "SAMPLE")]
    return cfg


CONTIGS = [("ctg1", 300_000), ("ctg2", 200_000), ("ctg3", 100_000)]


def test_merge_writes_tasks_in_task_order(tmp_path):
    cfg = _merge_config(tmp_path)
    p2 = _part(2, "ctg3", {0: b"c" * 7})
    p0 = _part(0, "ctg1", {0: b"a" * 5, 100000: b"b" * 3})
    payloads = [_payload(0, [(2, "ctg3\t5\tr2\n", 1, p2)], nm=(2, 0.5, 0.5)),
                _payload(1, []),                                                     # an empty rank
                _payload(2, [(0, "ctg1\t1\tr0a\nctg1\t9\tr0b\n", 2, p0), (1, "", 0, None)], nm=(1, 0.25, 0.25))]
    written, _, _ = call.write_rank_outputs(cfg, CONTIGS, payloads)
    assert written == 3
    head = io.StringIO()
    from sniffles_b200 import vcf
    vcf.VCFWriter(cfg, head).write_header(CONTIGS)
    assert (tmp_path / "o.vcf").read_text() == head.getvalue() + "ctg1\t1\tr0a\nctg1\t9\tr0b\nctg3\t5\tr2\n"
    assert (cfg.average_regional_nm, cfg.qc_nm_threshold) == (0.5, 0.5)             # the last task's, as a one-GPU run leaves them
    want = io.BytesIO()
    snf.write_results(want, cfg, [p0, p2], [n for n, _ in CONTIGS])
    assert (tmp_path / "o.snf").read_bytes() == want.getvalue()


def test_merge_refuses_a_failed_rank_and_writes_nothing(tmp_path):
    cfg = _merge_config(tmp_path)
    payloads = [_payload(0, [(0, "ctg1\t1\tr0\n", 1, _part(0, "ctg1", {0: b"a"}))]), _payload(1, [], error="the pass over ctg2 failed")]
    with pytest.raises(call.CallSampleError, match="rank 1: the pass over ctg2 failed"):
        call.write_rank_outputs(cfg, CONTIGS, payloads)
    assert os.listdir(tmp_path) == []


def _existing_output(rank, world, vcf_path):
    """--gpus 2 with an existing --vcf: rank 0 alone checks it (check_outputs is not called on rank 1)"""
    seen = []
    if rank == 1:
        call.check_outputs = lambda config: seen.append(config)
    cfg = sconfig.default_config("--vcf", vcf_path, "--gpus", "2")
    try:
        call.call_sample(cfg)
    except call.CallSampleError as e:
        return str(e), len(seen)
    return None, len(seen)


def test_existing_output_is_refused_on_every_rank(tmp_path):
    path = tmp_path / "o.vcf"
    path.write_text("keep")
    got = ranks_common.run_ranks(_existing_output, 2, str(path), timeout=240)
    assert all(ok for ok, _ in got), got
    (m0, _), (m1, seen1) = got[0][1], got[1][1]
    assert m0 == m1 == f"Output file '{path}' already exists! Use --allow-overwrite to ignore this check and overwrite."
    assert seen1 == 0 and path.read_text() == "keep"


def _cli(rank, world, args):
    """the command line of one rank of a torchrun launch: its exit code and what it logged"""
    import logging
    from sniffles_b200 import __main__ as cli
    buf = io.StringIO()
    handler = logging.StreamHandler(buf)
    logging.getLogger().addHandler(handler)
    try:
        code = cli.main(args)
    finally:
        logging.getLogger().removeHandler(handler)
    return code, buf.getvalue()


@pytest.mark.parametrize("extra, message", [(["--genotype-vcf", "targets.vcf", "--gpus", "2"], "--genotype-vcf runs on one GPU"),
                                            (["--gpus", "3"], "--gpus 3 does not match the 2 processes")])
def test_command_line_refuses_under_two_ranks(tmp_path, extra, message):
    args = ["--input", str(tmp_path / "s.bam"), "--vcf", str(tmp_path / "o.vcf")] + extra
    got = ranks_common.run_ranks(_cli, 2, args, init=False, timeout=240)
    assert all(ok for ok, _ in got), got
    assert [code for _, (code, _) in got] == [1, 1]
    assert all(message in text for _, (_, text) in got)
    assert os.listdir(tmp_path) == []
