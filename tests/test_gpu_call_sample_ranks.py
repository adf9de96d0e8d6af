"""call_sample on several ranks of a gloo group, spawned as processes on device 0 with a small pass budget: every rank's tasks on the
device, rank 0 writing the files.  The files equal the reference's (tests/golden/call_sample, tests/golden/regions) and a one-rank run's:
the VCF and the .tbi byte for byte, the SNF byte for byte apart from each gzip member's write time and the header's record of --gpus and
the output paths.  Also: a rank that fails, and the torchrun command line where two devices are visible."""
import gzip
import json
import os
import subprocess
import sys

import pytest
import torch

import call_sample_common as csc
import ranks_common
import regions_common as rc
from sniffles_b200 import bamio, call, tasks
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUDGET = 1 << 22                                  # inflated BAM bytes per pass: several passes on the larger inputs
with open(csc.EXPECTED) as _f:
    GOLD = json.load(_f)
with open(rc.EXPECTED) as _f:
    REGIONS = json.load(_f)


def _config(args, world):
    cfg = sconfig.SnifflesConfig(*args, "--gpus", str(world))
    for k, v in csc.STAMP.items():
        setattr(cfg, k, v)
    return cfg


def _run_cases(rank, world, runs, budget, fail_rank=None):
    """call_sample over every (tag, arguments) of `runs` on this rank: per tag the records written or the error, and rank 0's stats.
    fail_rank: that rank's device passes raise CallSampleError (a host-side stand-in for a failing pass)."""
    if rank == fail_rank:
        def failing_pass(*args, **kwargs):
            raise call.CallSampleError(f"injected failure of a device pass on rank {rank}")
        call.load_pass = failing_pass
    out = {}
    for tag, args in runs:
        stats = {}
        try:
            n = call.call_sample(_config(args, world), device=0, budget=budget, stats=stats)
            out[tag] = {"n": n, "ranks": stats.get("ranks")}
        except call.CallSampleError as e:
            out[tag] = {"error": str(e)}
    return out


def _spawn(world, runs, budget=BUDGET, fail_rank=None):
    """rank 0's results; asserts that every rank returned the same count or raised the same error"""
    got = ranks_common.run_ranks(_run_cases, world, runs, budget, fail_rank)
    assert all(ok for ok, _ in got), got
    per_rank = [v for _, v in got]
    for tag, _ in runs:
        assert len({json.dumps([r[tag].get("n"), r[tag].get("error")]) for r in per_rank}) == 1, (tag, [r[tag] for r in per_rank])
    return per_rank[0]


def _n_planned(bam_path, args):
    bam = bamio.BamFile(bam_path)
    n = len(tasks.plan(bam.contigs, _config(args, 1))[1])
    bam.close()
    return n


def snf_content(path):
    """an SNF file without what a run stamps on it: the header without `gpus`, `vcf` and `snf`, the body with the MTIME of every gzip
    member zeroed"""
    with open(path, "rb") as f:
        header = json.loads(f.readline())
        body = bytearray(f.read())
    for k in ("gpus", "vcf", "snf"):
        header["config"].pop(k)
    for blocks in header["index"].values():
        for parts in blocks.values():
            for off, _ in parts:
                assert body[off:off + 2] == b"\x1f\x8b"
                body[off + 4:off + 8] = b"\0\0\0\0"
    return header, bytes(body)


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("ranks_inputs")
    return {name: csc.write_inputs(name, str(d / name)) for name in {n for n, _ in csc.CASES.values()}}


@pytest.fixture(scope="module")
def two_ranks(inputs, tmp_path_factory):
    """every case of call_sample_common.CASES at two ranks"""
    d = tmp_path_factory.mktemp("two_ranks")
    runs = []
    for case in sorted(csc.CASES):
        os.makedirs(d / case)
        runs.append((case, csc.case_args(case, inputs[GOLD["cases"][case]["input"]], str(d / case / "out.vcf"), str(d / case / "out.snf"))))
    return d, dict(runs), _spawn(2, runs)


@pytest.mark.parametrize("case", sorted(csc.CASES))
def test_two_ranks_match_reference(case, two_ranks, inputs):
    d, args, res = two_ranks
    gold = GOLD["cases"][case]
    assert res[case].get("n") == gold["n_written"], res[case]
    assert csc.vcf_digest((d / case / "out.vcf").read_text()) == gold["vcf"]
    if "snf" in gold:
        assert csc.snf_digest(str(d / case / "out.snf")) == gold["snf"]
    else:
        assert not (d / case / "out.snf").exists()
    ranks = res[case]["ranks"]
    assert len(ranks) == 2 and sum(r["tasks"] for r in ranks) == _n_planned(inputs[gold["input"]]["bam"], args[case])


def test_three_ranks_give_the_files_of_one(inputs, tmp_path):
    """three ranks (one of them without tasks on the two-contig inputs, two of them on the one-contig c1) against one rank in this
    process: the same VCF bytes, the same SNF, and for a .vcf.gz the same decompressed text and .tbi bytes"""
    runs = [(c, c, "out.vcf") for c in ("phased_all_contigs", "phased_reference", "hg008_all_contigs", "c1_snf")]
    runs += [("phased_reference_gz", "phased_reference", "out.vcf.gz"), ("c1_snf_gz", "c1_snf", "out.vcf.gz")]
    many, want = [], {}
    for tag, case, vcf_name in runs:
        paths = inputs[GOLD["cases"][case]["input"]]
        for sub in ("one", "many"):
            os.makedirs(tmp_path / sub / tag)
        one = csc.case_args(case, paths, str(tmp_path / "one" / tag / vcf_name), str(tmp_path / "one" / tag / "out.snf"))
        want[tag] = call.call_sample(_config(one, 1), device=0)
        many.append((tag, csc.case_args(case, paths, str(tmp_path / "many" / tag / vcf_name), str(tmp_path / "many" / tag / "out.snf"))))
    res = _spawn(3, many)
    for tag, case, vcf_name in runs:
        a, b = tmp_path / "one" / tag, tmp_path / "many" / tag
        assert res[tag].get("n") == want[tag] == GOLD["cases"][case]["n_written"], (tag, res[tag])
        if vcf_name.endswith(".gz"):
            assert gzip.decompress((a / vcf_name).read_bytes()) == gzip.decompress((b / vcf_name).read_bytes())
            assert (a / (vcf_name + ".tbi")).read_bytes() == (b / (vcf_name + ".tbi")).read_bytes()
        else:
            assert (a / vcf_name).read_bytes() == (b / vcf_name).read_bytes()
        assert csc.vcf_digest(gzip.decompress((b / vcf_name).read_bytes()).decode() if vcf_name.endswith(".gz") else (b / vcf_name).read_text()) \
            == GOLD["cases"][case]["vcf"]
        assert snf_content(str(a / "out.snf")) == snf_content(str(b / "out.snf"))
        assert sorted(r["tasks"] for r in res[tag]["ranks"])[0] == 0 or case == "hg008_all_contigs"


def test_regions_at_two_ranks_match_reference(tmp_path):
    """every --regions / --region case at two ranks, the tasks that fail included"""
    runs, names = [], {}
    for case in sorted(rc.CASES):
        name = rc.CASES[case][0]
        if name not in names:
            names[name] = csc.write_inputs(name, str(tmp_path / name))
        paths = dict(names[name])
        bam = bamio.BamFile(paths["bam"])
        runs.append((case, rc.case_args(case, paths, bam, str(tmp_path), str(tmp_path / (case + ".vcf")), str(tmp_path / (case + ".snf")))))
        bam.close()
    res = _spawn(2, runs)
    for case, _ in runs:
        want = REGIONS["cases"][case]
        assert res[case].get("n") == want["n_written"], (case, res[case])
        with open(tmp_path / (case + ".vcf")) as f:
            assert csc.vcf_digest(f.read())["records"] == want["vcf"]["records"], case
        if "snf" in want:
            assert csc.snf_digest(str(tmp_path / (case + ".snf"))) == want["snf"], case
        failed = sorted(list(t) for r in res[case]["ranks"] for t in r["failed"])
        assert failed == want["failed_tasks"], case


def test_a_failing_rank_fails_every_rank_and_writes_nothing(inputs, tmp_path):
    case = "phased_all_contigs"
    args = csc.case_args(case, inputs["phased_phase"], str(tmp_path / "out.vcf"), str(tmp_path / "out.snf"))
    res = _spawn(2, [(case, args)], fail_rank=1)
    assert res[case] == {"error": "rank 1: injected failure of a device pass on rank 1"}
    assert os.listdir(tmp_path) == []


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="the torchrun command line runs one process per GPU: it needs two visible devices")
def test_torchrun_command_line_gives_the_same_files(inputs, tmp_path):
    from sniffles_b200 import __main__ as cli
    case = "phased_reference"
    paths = inputs["phased_phase"]
    for sub in ("one", "two"):
        os.makedirs(tmp_path / sub)
    assert cli.main(csc.case_args(case, paths, str(tmp_path / "one" / "out.vcf"), str(tmp_path / "one" / "out.snf"))) == 0
    args = csc.case_args(case, paths, str(tmp_path / "two" / "out.vcf"), str(tmp_path / "two" / "out.snf")) + ["--gpus", "2"]
    proc = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", "--nproc-per-node", "2", "-m", "sniffles_b200"] + args,
                          cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    strip = lambda t: [l for l in t.splitlines() if not l.startswith(("##source=", "##command=", "##fileDate="))]     # the run's own stamp
    assert strip((tmp_path / "two" / "out.vcf").read_text()) == strip((tmp_path / "one" / "out.vcf").read_text())
    assert csc.snf_digest(str(tmp_path / "two" / "out.snf")) == csc.snf_digest(str(tmp_path / "one" / "out.snf")) == GOLD["cases"][case]["snf"]
