"""Combine mode on several ranks of a gloo group, spawned as processes on device 0 with a small candidate budget: every rank's combine
tasks on the device, rank 0 writing the file.  The files equal the reference's (tests/golden/combine_cli, combine_reference, population)
and a one-rank run's byte for byte, the .tbi of a .vcf.gz included.  Also: a seeded cohort above --combine-max-inmemory-results at 1, 2
and 4 ranks, a rank that fails, and the torchrun command line where two devices are visible."""
import gzip
import json
import os
import subprocess
import sys

import pytest
import torch

import combine_cli_common as ccc
import combine_reference_common as crc
import population_common as pc
import ranks_common
from sniffles_b200 import combine_run
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUDGET = 200                                      # candidates per pass: several passes on every case
STAMP = {"command": "sniffles combine-ranks-test", "start_date": "2026/01/01 00:00:00"}
CLI_GOLD = ccc.load_expected()
REF_SHA, REF_GOLD = crc.load_expected()
_, POP_GOLD = pc.load_expected()


def n_tasks(case):
    """the planned task count of a golden case: its task list, or the count a long one is stored with"""
    return case["tasks"]["n"] if isinstance(case["tasks"], dict) else len(case["tasks"])


def _config(args, world):
    cfg = sconfig.SnifflesConfig(*args, "--gpus", str(world))
    for k, v in STAMP.items():
        setattr(cfg, k, v)
    return cfg


def _run_cases(rank, world, workdir, runs, budget, fail_rank=None):
    """combine_snfs over every (tag, arguments) of `runs` on this rank, from `workdir`: per tag the records written, the dropped calls and
    rank 0's per-rank stats, or the error.  fail_rank: that rank's device passes raise CombineError (a host-side stand-in for a failing
    pass)."""
    os.chdir(workdir)
    if rank == fail_rank:
        def failing_pass(*args, **kwargs):
            raise combine_run.CombineError(f"injected failure of a device pass on rank {rank}")
        combine_run._run_pass = failing_pass
    out = {}
    for tag, args in runs:
        stats = {}
        try:
            n = combine_run.combine_snfs(_config(args, world), device=0, budget=budget, stats=stats)
            out[tag] = {"n": n, "dropped": stats.get("dropped"), "ranks": stats.get("ranks")}
        except combine_run.CombineError as e:
            out[tag] = {"error": str(e)}
    return out


def _spawn(world, workdir, runs, budget=BUDGET, fail_rank=None):
    """rank 0's results; asserts that every rank returned the same count or raised the same error"""
    got = ranks_common.run_ranks(_run_cases, world, workdir, runs, budget, fail_rank)
    assert all(ok for ok, _ in got), got
    per_rank = [v for _, v in got]
    for tag, _ in runs:
        assert len({json.dumps([r[tag].get("n"), r[tag].get("error")]) for r in per_rank}) == 1, (tag, [r[tag] for r in per_rank])
    return per_rank[0]


def _one(workdir, args, budget=BUDGET):
    """the same run on one GPU in this process: (records, dropped)"""
    cwd = os.getcwd()
    os.chdir(workdir)
    try:
        st = {}
        n = combine_run.combine_snfs(_config(args, 1), device=0, budget=budget, stats=st)
    finally:
        os.chdir(cwd)
    return n, st["dropped"]


def _lines(path):
    data = open(path, "rb").read()
    return ccc.vcf_lines((gzip.decompress(data) if path.endswith(".gz") else data).decode())


def _same_files(a, b):
    """the VCF at `a` and `b` byte for byte, and their .tbi when they are .vcf.gz"""
    assert open(a, "rb").read() == open(b, "rb").read(), (a, b)
    if a.endswith(".gz"):
        assert open(a + ".tbi", "rb").read() == open(b + ".tbi", "rb").read(), (a, b)


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """(SNF input directory, {FASTA kind: path}) of combine_cli_common and combine_reference_common"""
    d = tmp_path_factory.mktemp("combine_ranks")
    fastas = {}
    for kind in ("full", "no_ctg2"):
        fastas[kind], sha = crc.fasta_files(kind, str(d))
        assert sha == REF_SHA[kind], kind
    return ccc.write_inputs(str(d / "in")), fastas


def _cli_args(label, out):
    case = CLI_GOLD[label]
    return ["-i"] + case["inputs"] + ["-v", out] + case["args"]


def _ref_args(label, fastas, out):
    _, files, extra, kind, population = next(c for c in crc.CASES if c[0] == label)
    return crc.case_args(files, extra, population, out, fastas[kind])


def _written(path):
    """the file a run wrote: above --combine-max-inmemory-results a sorted .vcf.gz becomes the plain file"""
    return path if os.path.exists(path) else path.removesuffix(".gz")


def _check(workdir, runs, res):
    """per (tag, arguments, golden lines or None): rank 0's count and dropped calls equal a one-GPU run's, the file equals the golden
    lines and the one-GPU file byte for byte"""
    for tag, args, gold in runs:
        many = args[args.index("-v") + 1]
        one = many.replace(os.sep + "many" + os.sep, os.sep + "one" + os.sep)
        os.makedirs(os.path.dirname(one))
        n, dropped = _one(workdir, [one if a == many else a for a in args])
        assert res[tag].get("n") == n and res[tag]["dropped"] == dropped, (tag, res[tag], n, dropped)
        _same_files(_written(one), _written(many))
        if gold is not None:
            assert _lines(_written(many)) == gold, tag


def _make_dirs(runs):
    for _, args, _ in runs:
        os.makedirs(os.path.dirname(args[args.index("-v") + 1]))
    return [(tag, args) for tag, args, _ in runs]


@pytest.mark.parametrize("world", [2, 3])
def test_cli_cases_match_reference_and_one_rank(world, inputs, tmp_path):
    workdir, _ = inputs
    many = tmp_path / "many"
    runs = [(label, _cli_args(label, str(many / label / "out.vcf")), CLI_GOLD[label]["vcf"]) for label in sorted(CLI_GOLD)]
    runs += [(label + "_gz", _cli_args(label, str(many / (label + "_gz") / "out.vcf.gz")), None) for label in ("default4", "tmpfile")]
    res = _spawn(world, workdir, _make_dirs(runs))
    _check(workdir, runs, res)
    assert os.path.getsize(many / "default4_gz" / "out.vcf.gz.tbi") > 0
    for label, case in CLI_GOLD.items():
        assert res[label]["dropped"] == case["dropped"], label
        ranks = res[label]["ranks"]
        assert len(ranks) == world and sum(r["tasks"] for r in ranks) == n_tasks(case), label


def test_reference_and_population_cases_at_two_ranks(inputs, tmp_path):
    workdir, fastas = inputs
    many = tmp_path / "many"
    runs = [("ref_" + label, _ref_args(label, fastas, str(many / ("ref_" + label) / "out.vcf")), REF_GOLD[label]["vcf"]) for label in sorted(REF_GOLD)]
    runs += [("pop_" + label, pc.case_args(case, workdir, str(many / ("pop_" + label) / "out.vcf")), case["vcf"]) for label, case in sorted(POP_GOLD.items())]
    runs += [("ref_population_gz", _ref_args("population", fastas, str(many / "ref_population_gz" / "out.vcf.gz")), REF_GOLD["population"]["vcf"])]
    res = _spawn(2, workdir, _make_dirs(runs))
    _check(workdir, runs, res)
    assert os.path.getsize(many / "ref_population_gz" / "out.vcf.gz.tbi") > 0


def test_seeded_cohort_at_one_two_and_four_ranks(tmp_path):
    scripts = os.path.join(ROOT, "scripts")
    sys.path.insert(0, scripts)
    try:
        import combine_sample_bench
    finally:
        sys.path.remove(scripts)
    cohort = tmp_path / "cohort"
    cohort.mkdir()
    paths = combine_sample_bench.write_cohort(str(cohort), 0.01)
    cfg = sconfig.SnifflesConfig("-i", *paths, "-v", "x.vcf")
    assert len(paths) > cfg.combine_max_inmemory_results         # results kept as CombineResultTmpFile keeps them
    budget = 3000
    (tmp_path / "w1").mkdir()
    n1, dropped1 = _one(str(cohort), ["-i", *paths, "-v", str(tmp_path / "w1" / "out.vcf")], budget)
    assert n1 > 0
    for world in (2, 4):
        (tmp_path / f"w{world}").mkdir()
        res = _spawn(world, str(cohort), [("cohort", ["-i", *paths, "-v", str(tmp_path / f"w{world}" / "out.vcf")])], budget)
        assert res["cohort"]["n"] == n1 and res["cohort"]["dropped"] == dropped1, res["cohort"]
        assert sum(r["tasks"] > 0 for r in res["cohort"]["ranks"]) == world
        _same_files(str(tmp_path / "w1" / "out.vcf"), str(tmp_path / f"w{world}" / "out.vcf"))


def test_a_failing_rank_fails_every_rank_and_writes_nothing(inputs, tmp_path):
    workdir, _ = inputs
    out = tmp_path / "out"
    out.mkdir()
    for name in ("out.vcf", "out.vcf.gz"):
        res = _spawn(2, workdir, [("default4", _cli_args("default4", str(out / name)))], fail_rank=1)
        assert res["default4"] == {"error": "rank 1: injected failure of a device pass on rank 1"}
    assert os.listdir(out) == []


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="the torchrun command line runs one process per GPU: it needs two visible devices")
def test_torchrun_command_line_gives_the_same_file(inputs, tmp_path):
    from sniffles_b200 import __main__ as cli
    workdir, fastas = inputs
    one, two = str(tmp_path / "one.vcf.gz"), str(tmp_path / "two.vcf.gz")
    args = lambda out: [os.path.join(workdir, a) if a.endswith(".snf") else a for a in _ref_args("population", fastas, out)]
    assert cli.main(args(one)) == 0
    proc = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2", "-m", "sniffles_b200"]
                          + args(two) + ["--gpus", "2"], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    assert _lines(two) == _lines(one) == REF_GOLD["population"]["vcf"]
    assert os.path.getsize(two + ".tbi") > 0
