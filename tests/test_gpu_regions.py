"""`--regions` / `--region` on the device against the unmodified reference (tests/golden/regions/expected.json, made by
tests/golden/make_regions_golden.py): every case through call.call_sample, VCF records and SNF contents compared byte for byte."""
import gzip
import json

import numpy as np
import pytest

import call_sample_common as csc
import regions_common as rc
from sniffles_b200 import bamio, call
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

with open(rc.EXPECTED) as _f:
    EXPECTED = json.load(_f)


def _run(case, tmp_path, budget=None):
    name = rc.CASES[case][0]
    paths = csc.write_inputs(name, str(tmp_path / name))
    bam = bamio.BamFile(paths["bam"])
    vcf_path, snf_path = str(tmp_path / (case + ".vcf")), str(tmp_path / (case + ".snf"))
    cfg = sconfig.SnifflesConfig(*rc.case_args(case, paths, bam, str(tmp_path), vcf_path, snf_path))
    bam.close()
    for k, v in csc.STAMP.items():
        setattr(cfg, k, v)
    n = call.call_sample(cfg, budget=budget)
    with open(vcf_path) as f:
        got = {"n_written": n, "vcf": csc.vcf_digest(f.read())}
    if cfg.snf is not None:
        got["snf"] = csc.snf_digest(snf_path)
    return got


@pytest.mark.parametrize("case", sorted(rc.CASES))
def test_regions_case_matches_reference(case, tmp_path):
    want = EXPECTED["cases"][case]
    got = _run(case, tmp_path)
    assert got["n_written"] == want["n_written"]
    assert got["vcf"]["records"] == want["vcf"]["records"]
    if "snf" in want:
        assert got["snf"] == want["snf"]


def test_regions_one_task_per_pass_same_bytes(tmp_path):
    """two tasks with regions in one pass, and one task per pass, give the same records"""
    a = _run("phased_sorted", tmp_path / "a")
    b = _run("phased_sorted", tmp_path / "b", budget=1)
    assert a == b
    assert a["vcf"]["records"] == EXPECTED["cases"]["phased_sorted"]["vcf"]["records"]


def test_whole_contig_region_is_the_default_task(tmp_path):
    """one region [0, L - 1] per contig reads what the default task reads: the same records as a run without regions"""
    paths = csc.write_inputs("phased_phase", str(tmp_path / "in"))
    bam = bamio.BamFile(paths["bam"])
    ctg = rc.contigs_with_reads(bam)
    bam.close()
    out = {}
    for tag, extra in (("plain", ["--all-contigs"]), ("regions", [x for n, L in ctg for x in ("--region", f"{n}:0-{L - 1}")])):
        vcf_path = str(tmp_path / (tag + ".vcf"))
        cfg = sconfig.SnifflesConfig("--input", paths["bam"], "--vcf", vcf_path, "--phase", *extra)
        for k, v in csc.STAMP.items():
            setattr(cfg, k, v)
        if tag == "plain":
            cfg.all_contigs = False
            cfg.contig = [n for n, _ in ctg]
        call.call_sample(cfg)
        with open(vcf_path) as f:
            out[tag] = [l for l in f.read().splitlines() if not l.startswith("#")]
    assert out["regions"] == out["plain"] and out["plain"]


def test_host_reader_matches_device_ingest_with_overlapping_regions(tmp_path):
    """Task.build_leadtab on the host reader and on the device ingest, overlapping and unsorted regions: same candidates and coverage"""
    from sniffles_b200 import tasks
    paths = csc.write_inputs("c1_ont_1mb", str(tmp_path / "in"))
    bam = bamio.BamFile(paths["bam"])
    (name, L), = rc.contigs_with_reads(bam)[:1]
    regions = [(name, *map(int, line.split("\t")[1:3])) for line in rc._overlap_unsorted([(name, L)])]
    res = {}
    for dev in (True, False):
        cfg = sconfig.default_config("--snf", str(tmp_path / "x.snf"))
        t = tasks.CallTask(id=0, sv_id=0, contig=name, start=0, end=L - 1, config=cfg, bam=bam, regions=regions, device_ingest=dev)
        calls, n_reads = t.execute()
        res[dev] = ([(c.svtype, c.pos, c.svlen, c.support, c.coverage_start, c.coverage_center, c.coverage_end, c.alt) for c in calls],
                    n_reads, t.coverage_average_total, gzip.decompress(t.snf_part[3]))      # the gzip headers carry the write time
    assert res[True] == res[False]
    assert res[True][1] > 0


@pytest.mark.parametrize("case", sorted(rc.GENOTYPE_CASES))
def test_genotype_vcf_with_regions_matches_reference(case, tmp_path):
    """--genotype-vcf with --regions: target matches and start / center / end coverage from the regions' reads only"""
    import os
    from sniffles_b200 import genotype
    want = EXPECTED["genotype"][case]
    name, _, _, targets = rc.GENOTYPE_CASES[case]
    paths = csc.write_inputs(name, str(tmp_path / name))
    bam = bamio.BamFile(paths["bam"])
    vcf_path = str(tmp_path / (case + ".vcf"))
    args = rc.case_args(case, paths, bam, str(tmp_path), vcf_path, None, rc.GENOTYPE_CASES)
    bam.close()
    cfg = sconfig.SnifflesConfig(*args, "--genotype-vcf", os.path.join(rc.HERE, "golden", "genotype", targets))
    for k, v in csc.STAMP.items():
        setattr(cfg, k, v)
    assert genotype.genotype_vcf(cfg) == want["n_written"]
    with open(vcf_path) as f:
        assert f.read() == want["output"]


def _task_results(bam, cfg, name, L, regions, dev, ctx_device=0):
    from sniffles_b200 import tasks
    tr = None
    if cfg.tandem_repeats:
        tr = tasks.load_tandem_repeats(cfg.tandem_repeats, cfg.tandem_repeat_region_pad).get(name)
    t = tasks.CallTask(id=0, sv_id=0, contig=name, start=0, end=L - 1, config=cfg, bam=bam, regions=regions, device_ingest=dev,
                       tandem_repeats=tr, device=ctx_device)
    calls, n_reads = t.execute()
    return ([(c.svtype, c.pos, c.svlen, c.support, c.qc, c.coverage_upstream, c.coverage_start, c.coverage_center, c.coverage_end,
              c.coverage_downstream, c.alt, c.nm) for c in calls], n_reads, t.coverage_average_total,
            gzip.decompress(t.snf_part[3]) if t.snf_part else None)      # the gzip headers carry the write time


@pytest.mark.parametrize("case", sorted(rc.CASES))
def test_host_reader_matches_device_ingest(case, tmp_path):
    """every task of every case on the host reader (device_ingest=False) and on the device ingest: the same calls, coverage and SNF part.
    The device ingest reproduces the reference (test_regions_case_matches_reference), so the host reader does too."""
    name = rc.CASES[case][0]
    paths = csc.write_inputs(name, str(tmp_path / name))
    bam = bamio.BamFile(paths["bam"])
    cfg = sconfig.SnifflesConfig(*rc.case_args(case, paths, bam, str(tmp_path), str(tmp_path / "x.vcf"), str(tmp_path / "x.snf")))
    for cname, L in bam.contigs:
        rg = cfg.regions_by_contig.get(cname)
        if not rg or any(s < 0 or s > e for _, s, e in rg):
            continue
        got = [_task_results(bam, cfg, cname, L, rg, dev) for dev in (True, False)]
        assert got[0] == got[1], cname
    bam.close()


def test_run_without_regions_after_regions_on_the_same_context(tmp_path):
    """the region table applies to one load only: a task without regions after a task with regions, on the same device context, gives
    the bytes and the launch count of the same task run first"""
    from sniffles_b200 import tasks
    paths = csc.write_inputs("c1_ont_1mb", str(tmp_path / "in"))
    bam = bamio.BamFile(paths["bam"])
    (name, L), = rc.contigs_with_reads(bam)[:1]
    cfg = sconfig.default_config("--snf", str(tmp_path / "x.snf"))
    ctx = tasks.device_context(0)
    regions = [(name, *map(int, line.split("\t")[1:3])) for line in rc._overlap_unsorted([(name, L)])]
    out = []
    for rg in (None, regions, None):
        for dev in (True, False):
            l0 = ctx.launch_count()
            out.append((rg is None, dev, _task_results(bam, cfg, name, L, rg, dev), ctx.launch_count() - l0))
    bam.close()
    assert out[4] == out[0] and out[5] == out[1]
    assert out[2][2] != out[0][2]


def _alen(cigar):
    ops = cigar & 0xf
    lens = cigar >> 4
    return int(lens[np.isin(ops, (0, 1, 7, 8))].sum())


def test_thousands_of_random_regions(tmp_path):
    """2,400 random regions on one contig (overlapping, unsorted, empty and past-the-end ones): both readers agree, and the read count and
    coverage_average_total equal a restatement of the reference's per-region loop (leadprov.py:475-510): every read that passes the
    filters and starts inside a region counts once per such region, its bases [start, end) clipped to the contig"""
    paths = csc.write_inputs("c1_ont_1mb", str(tmp_path / "in"))
    bam = bamio.BamFile(paths["bam"])
    (name, L), = rc.contigs_with_reads(bam)[:1]
    rng = np.random.default_rng(2024)
    starts = rng.integers(0, L, 2400)
    widths = rng.choice([0, 50, 2_000, 20_000, 150_000], 2400)
    regions = [(name, int(s), int(s + w)) for s, w in zip(starts, widths)]
    cfg = sconfig.default_config("--snf", str(tmp_path / "x.snf"))
    got = [_task_results(bam, cfg, name, L, regions, dev) for dev in (True, False)]
    assert got[0] == got[1]
    recs = list(bam.fetch(name, 0, L))
    n_reads, bases = 0, 0
    for _, s, e in regions:
        for r in recs:
            alen = _alen(np.asarray(r["cigar"], dtype=np.int64))
            if r["mapq"] < cfg.mapq or r["flag"] & 256 or alen < cfg.min_alignment_length or not s <= r["pos"] < e:
                continue
            n_reads += 1
            bases += min(r["pos"] + bamio.ref_span(r["cigar"]), L) - r["pos"]
    assert got[0][1] == n_reads > 0
    assert got[0][2] == bases / L
    bam.close()
