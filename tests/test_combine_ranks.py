"""Combine mode on several ranks, without a GPU: the combine task weights read from the SNF headers and their assignment to ranks, rank
0's merge of the ranks' payloads into the output file, and the refusals of a world size of 2 on gloo with two spawned CPU processes."""
import io
import json
import logging
import os

import pytest

import combine_cli_common as ccc
import ranks_common
from sniffles_b200 import combine_run, dist, snf, vcf
from sniffles_b200 import config as sconfig

CLI_GOLD = ccc.load_expected()


def n_tasks(case):
    """the planned task count of a golden case: its task list, or the count a long one is stored with"""
    return case["tasks"]["n"] if isinstance(case["tasks"], dict) else len(case["tasks"])


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return ccc.write_inputs(str(tmp_path_factory.mktemp("combine_ranks_inputs")))


def _plan(label, workdir):
    """(readers, planned tasks) of a combine_cli_common case as a run plans them"""
    case = CLI_GOLD[label]
    cwd = os.getcwd()
    os.chdir(workdir)
    try:
        cfg = sconfig.SnifflesConfig("-i", *case["inputs"], "-v", "unused.vcf", *case["args"])
        cfg.mode = "combine"
        contig_lengths, _ = combine_run.read_inputs(cfg)
        planned = combine_run.plan_tasks(cfg, contig_lengths)
        readers = {s["internal_id"]: snf.SNFReader(os.path.join(workdir, s["filename"])) for s in cfg.snf_input_info}
    finally:
        os.chdir(cwd)
    return cfg, readers, planned


def _hand_weights(cfg, workdir, planned):
    """the part lengths of every sample's index entries for each task's blocks, read from the JSON header line itself"""
    indexes = []
    for s in cfg.snf_input_info:
        with open(os.path.join(workdir, s["filename"]), "rb") as f:
            indexes.append(json.loads(f.readline())["index"])
    out = []
    for t in planned:
        w = 0
        for index in indexes:
            for b in t.block_indices:
                for _, length in index.get(t.contig, {}).get(str(b), []):
                    w += length
        out.append(w)
    return out


@pytest.mark.parametrize("label", ["two", "three", "tsv", "default4", "tmpfile", "scatter", "regions", "contig"])
def test_weights_are_the_index_lengths(inputs, label):
    cfg, readers, planned = _plan(label, inputs)
    try:
        w = dist.combine_task_weights(readers, planned)
    finally:
        for r in readers.values():
            r.close()
    assert len(planned) == n_tasks(CLI_GOLD[label])
    assert w == _hand_weights(cfg, inputs, planned)
    assert sum(w) > 0
    if label == "scatter":                               # clones of one long contig: most of its blocks are in no sample
        assert len(planned) > 1000 and 0 < sum(x > 0 for x in w) < len(planned)
    if label == "contig":
        assert {t.contig for t in planned} == {"ctg2"}
    if label == "regions":                               # only the blocks the regions touch
        whole = _plan("three", inputs)
        assert 0 < sum(w) < sum(dist.combine_task_weights(whole[1], whole[2]))


def _assignment(rank, world, workdir, label, worlds):
    cfg, readers, planned = _plan(label, workdir)
    w = dist.combine_task_weights(readers, planned)
    for r in readers.values():
        r.close()
    return w, [dist.lpt_assign(w, n) for n in worlds]


def test_assignment_is_the_same_on_every_rank(inputs):
    worlds = [1, 2, 3, 4, 8]
    got = ranks_common.run_ranks(_assignment, 2, inputs, "scatter", worlds, init=False, timeout=240)
    assert all(ok for ok, _ in got), got
    assert got[0][1] == got[1][1] == _assignment(0, 1, inputs, "scatter", worlds)
    w, owners = got[0][1]
    for n, owner in zip(worlds, owners):
        assert len(owner) == len(w) and set(owner) <= set(range(n))


@pytest.mark.parametrize("label", ["two", "default4"])
def test_three_ranks_on_two_tasks_leave_one_empty(inputs, label):
    _, readers, planned = _plan(label, inputs)
    w = dist.combine_task_weights(readers, planned)
    for r in readers.values():
        r.close()
    assert len(planned) == 2 and all(x > 0 for x in w)
    assert len(set(dist.lpt_assign(w, 3))) == 2


CONTIGS = [("ctg1", 350_000), ("ctg2", 260_000)]


def _merge_config(tmp_path, name="o.vcf"):
    cfg = sconfig.default_config("--vcf", str(tmp_path / name))
    cfg.mode = "combine"
    cfg.command, cfg.start_date = "sniffles merge-test", "2026/01/01 00:00:00"
    cfg.sample_ids_vcf = [(0, "A"), (1, "B")]
    return cfg


def _payload(rank, items, dropped=0, error=None):
    return {"rank": rank, "tasks": items, "dropped": dropped, "stats": {}, "error": error}


def test_merge_writes_tasks_in_task_order(tmp_path, caplog):
    cfg = _merge_config(tmp_path)
    payloads = [_payload(0, [(3, "ctg2\t7\tr3\n", 1), (1, "ctg1\t5\tr1a\nctg1\t6\tr1b\n", 2)], dropped=2),
                _payload(1, []),                                                     # an empty rank
                _payload(2, [(2, "", 0), (0, "ctg1\t1\tr0\n", 1)], dropped=1)]
    caplog.set_level(logging.INFO)
    assert combine_run.write_rank_outputs(cfg, CONTIGS, payloads) == (4, 3)
    head = io.StringIO()
    vcf.VCFWriter(cfg, head).write_header(CONTIGS)
    assert (tmp_path / "o.vcf").read_text() == head.getvalue() + "ctg1\t1\tr0\nctg1\t5\tr1a\nctg1\t6\tr1b\nctg2\t7\tr3\n"
    assert caplog.text.count("3 calls came out of position order") == 1 and caplog.text.count("Wrote 4 called SVs") == 1


def test_merge_refuses_a_failed_rank_and_writes_nothing(tmp_path):
    cfg = _merge_config(tmp_path)
    payloads = [_payload(0, [(0, "ctg1\t1\tr0\n", 1)]), _payload(1, [], error="the device pass over 1 task(s) failed"),
                _payload(2, [], error="a later failure")]
    with pytest.raises(combine_run.CombineError, match="^rank 1: the device pass over 1 task\\(s\\) failed$"):
        combine_run.write_rank_outputs(cfg, CONTIGS, payloads)
    assert os.listdir(tmp_path) == []


def _existing_output(rank, world, workdir, vcf_path):
    """--gpus 2 with an existing --vcf: rank 0 alone checks it (check_outputs is not called on rank 1)"""
    seen = []
    if rank == 1:
        combine_run.check_outputs = lambda config: seen.append(config)
    os.chdir(workdir)
    cfg = sconfig.SnifflesConfig("-i", "s1.snf", "s2.snf", "-v", vcf_path, "--gpus", "2")
    try:
        combine_run.combine_snfs(cfg)
    except combine_run.CombineError as e:
        return str(e), len(seen)
    return None, len(seen)


def test_existing_output_is_refused_on_every_rank(inputs, tmp_path):
    path = tmp_path / "o.vcf"
    path.write_text("keep")
    got = ranks_common.run_ranks(_existing_output, 2, inputs, str(path), timeout=240)
    assert all(ok for ok, _ in got), got
    (m0, _), (m1, seen1) = got[0][1], got[1][1]
    assert m0 == m1 == f"Output file '{path}' already exists! Use --allow-overwrite to ignore this check and overwrite."
    assert seen1 == 0 and path.read_text() == "keep"


def _cli(rank, world, workdir, args):
    """the command line of one rank of a torchrun launch: its exit code and what it logged"""
    from sniffles_b200 import __main__ as cli
    os.chdir(workdir)
    buf = io.StringIO()
    handler = logging.StreamHandler(buf)
    logging.getLogger().addHandler(handler)
    try:
        code = cli.main(args)
    finally:
        logging.getLogger().removeHandler(handler)
    return code, buf.getvalue()


@pytest.mark.parametrize("extra, message", [(["--gpus", "3"], "--gpus 3 does not match the 2 processes torchrun started"),
                                            (["--gpus", "2", "--combine-consensus"], "--combine-consensus is not supported"),
                                            (["--gpus", "2", "--dev-population-snf", "p.snf"], "--dev-population-snf: writing a population SNF"),
                                            ([], "combine mode (.snf / .tsv input) runs on one GPU")])
def test_command_line_refuses_under_two_ranks(inputs, tmp_path, extra, message):
    args = ["-i", "s1.snf", "s2.snf", "-v", str(tmp_path / "o.vcf")] + extra
    got = ranks_common.run_ranks(_cli, 2, inputs, args, init=False, timeout=240)
    assert all(ok for ok, _ in got), got
    assert [code for _, (code, _) in got] == [1, 1]
    assert all(message in text and "(Fatal error, exiting.)" in text for _, (_, text) in got), got
    assert os.listdir(tmp_path) == []


def test_several_gpus_without_torchrun_warn_and_run_on_one(inputs, tmp_path, monkeypatch, caplog):
    """--gpus 2 without a process group is combine mode on one GPU, with one warning naming the torchrun command line (here the
    existing output stops the run before any device work)"""
    from sniffles_b200 import __main__ as cli
    monkeypatch.chdir(inputs)
    monkeypatch.delenv("WORLD_SIZE", raising=False)
    out = tmp_path / "o.vcf"
    out.write_text("keep")
    assert cli.main(["-i", "s1.snf", "s2.snf", "-v", str(out), "--gpus", "2"]) == 1
    assert caplog.text.count("torchrun --standalone --nproc-per-node 2 -m sniffles_b200 ... --gpus 2") == 1
    assert "already exists" in caplog.text and out.read_text() == "keep"


def _missing_inputs(rank, world, vcf_path):
    cfg = sconfig.SnifflesConfig("-i", "nope1.snf", "nope2.snf", "-v", vcf_path, "--gpus", "2")
    try:
        combine_run.combine_snfs(cfg)
    except combine_run.CombineError as e:
        return str(e)
    return None


def test_a_failed_header_pass_names_the_rank_on_every_rank(tmp_path):
    """the header pass fails on every rank before rank 0 has its contig lengths: the error names rank 0 and its message"""
    got = ranks_common.run_ranks(_missing_inputs, 2, str(tmp_path / "o.vcf"), timeout=240)
    assert all(ok for ok, _ in got), got
    m0, m1 = got[0][1], got[1][1]
    assert m0 == m1 and m0.startswith("rank 0: Unable to read the SNF file nope1.snf: "), got
    assert os.listdir(tmp_path) == []


def _reference_verdict(rank, world, workdir, vcf_path, unreadable_rank):
    """a two-rank run with --reference whose device inputs and passes are stand-ins: the FASTA object each rank loads ("FASTA", or None
    on `unreadable_rank`, as tasks.reference_for returns when it cannot read the contigs), and the one each pass is given"""
    from sniffles_b200 import tasks
    os.chdir(workdir)
    seen = []

    def device_inputs(config, device, contigs, st, load=True):
        return None, None, (None if rank == unreadable_rank else "FASTA") if load else None

    def run_pass(ctx, fp, config, reqc, write, tmpfile, st, pop=None, reference=None):
        seen.append(reference)
        return 0
    combine_run._device_inputs, combine_run._run_pass = device_inputs, run_pass
    tasks.device_context = lambda device=0: None
    cfg = sconfig.SnifflesConfig("-i", "s1.snf", "s2.snf", "-v", vcf_path, "--reference", "genome.fa", "--gpus", "2")
    combine_run.combine_snfs(cfg)
    return seen


@pytest.mark.parametrize("unreadable_rank", [None, 0, 1])
def test_every_rank_drops_the_fasta_when_one_cannot_read_it(inputs, tmp_path, unreadable_rank):
    """one GPU runs without a FASTA any of whose planned contigs it cannot read; on two ranks, each loading its own contigs, so does
    every rank when one of them cannot"""
    got = ranks_common.run_ranks(_reference_verdict, 2, inputs, str(tmp_path / "o.vcf"), unreadable_rank, timeout=240)
    assert all(ok for ok, _ in got), got
    seen = [v for _, v in got]
    assert all(len(s) == 1 for s in seen), seen                    # "two" plans two tasks: one on each rank
    want = "FASTA" if unreadable_rank is None else None
    assert seen == [[want], [want]]
