"""GPU parity: the CUDA path through the C ABI vs the CPU oracle on the same seeded inputs."""
import pytest

from sniffles_b200 import abi, binding, synth
from sniffles_b200 import config as sconfig
import devcheck

pytestmark = pytest.mark.gpu


def _run(blk, *args, cigar16=True):
    import oracle.oracle as orc
    cfg = abi.Config.from_sniffles(sconfig.default_config(*args))
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk, cigar16=cigar16)
        got = ctx.run()
    finally:
        ctx.close()
    want = orc.run(blk, cfg, 3, 4)
    devcheck.assert_same(want, got)
    return got


def test_config1_shape():
    got = _run(synth.config_block(1))
    assert len(got.cand) > 20


# --minsvlen 8 screens for events below the E threshold the block was packed with: the library re-flags the arena (k_reflag)
@pytest.mark.parametrize("args", [(), ("--mosaic",), ("--no-qc",), ("--repeat",), ("--minsvlen", "30"), ("--minsvlen", "8")])
def test_config2_scaled(args):
    _run(synth.config_block(2, 0.004), *args)


def test_bam_words_converted_by_the_library():
    """SNFB_CIGAR_BAM32 host arenas: snfb_load_records converts them itself."""
    _run(synth.config_block(2, 0.003), cigar16=False)


def test_wrong_chain_cut_is_detected_and_recovered():
    """Stage B cuts chains of bins where the gap exceeds max(cluster_merge_bnd, cluster_repeat_h_max) and verifies the stdev criterion afterwards
    (k_verify_cuts).  With an absurd --cluster-r the criterion does fire across such gaps: the library must notice (unverified_breaks), run again
    without cuts, and still return the reference's clusters (here 11 candidates instead of 456)."""
    import oracle.oracle as orc
    blk = synth.generate(77, [600000], 20.0, len_model=0, len_mean=20000.0, len_sd=2000.0, len_min=5000, len_max=60000, tech="ont", sv_spacing=1300.0,
                         ins_only=True, tr_frac=0.0, clip_prob=0.0, sv_min=50, sv_max=400, threads=4)
    cfg = abi.Config.from_sniffles(sconfig.default_config("--cluster-r", "2000"))
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk)
        got = ctx.run()
        reruns = ctx.rerun_count()
        again = ctx.run()                          # the decision is remembered for this block: no further re-run
        assert ctx.rerun_count() == reruns
    finally:
        ctx.close()
    want = orc.run(blk, cfg, 3, 4)
    devcheck.assert_same(want, got)
    devcheck.assert_same(want, again)
    assert reruns >= 1 and len(got.cand) < 50


def test_config3_hifi_mosaic():
    _run(synth.config_block(3, 0.003), "--mosaic")


def test_config5_ins_heavy():
    got = _run(synth.config_block(5, 0.05))
    assert (got.cand["svtype"] == 0).sum() > 100


@pytest.mark.parametrize("seed", range(8))
def test_random_shapes(seed):
    import random
    rnd = random.Random(seed)
    lens = [rnd.randrange(150000, 600000) for _ in range(rnd.choice([1, 2, 3]))]
    blk = synth.generate(1000 + seed, lens, coverage=rnd.choice([8, 15, 30, 60]), len_mean=rnd.choice([3000.0, 8000.0, 20000.0]),
                         len_sd=rnd.choice([300.0, 2000.0]), tech=rnd.choice(["ont", "hifi"]), sv_spacing=rnd.choice([800.0, 3000.0, 20000.0]),
                         phased_frac=rnd.choice([0.0, 0.5, 1.0]), tr_frac=rnd.choice([0.0, 0.15, 0.6]), ins_only=rnd.random() < 0.2,
                         clip_prob=rnd.choice([0.0, 0.1, 0.5]), lowmapq_prob=rnd.choice([0.05, 0.3]))
    _run(blk, *rnd.choice([(), ("--mosaic",), ("--no-qc",), ("--qc-nm",), ("--cluster-merge-pos", "50")]))


@pytest.mark.parametrize("name", ["c1_ont_1mb", "c2_ont_wgs_small", "c3_hifi_mosaic", "c5_ins_heavy", "tr_repeat_noqc", "auto_support_qcnm", "phased_phase",
                                  "filters_binsize", "long_ins_minsv", "hifi_strict"])
def test_device_against_reference_golden(name):
    """CUDA path -> host epilogue vs what the unmodified reference produced (tests/golden/*.json):
    lead table, candidates, FILTER / GT / ALT of the finalized calls."""
    from test_oracle_golden import load_fixture, check_against_golden
    from test_host_epilogue import check_final
    from sniffles_b200 import tasks
    fx, blk = load_fixture(name)
    cfg = sconfig.default_config(*fx["args"])
    br = tasks.run_block(blk, cfg, 0)
    check_against_golden(fx, blk, br.result)
    check_final(fx, blk, br.result, br.rec_nm, cfg)


def test_calltask_surface():
    """The Task mirror keeps the reference's call sequence (parallel.py:256-271)."""
    from sniffles_b200 import tasks
    blk = synth.config_block(1)
    cfg = sconfig.default_config()
    br = tasks.run_block(blk, cfg, 0)
    t = tasks.CallTask(id=0, sv_id=0, contig=blk.contig_names[0], start=0, end=int(blk.task[0]["end"]), config=cfg, block_run=br, task_index=0)
    calls, read_count = t.execute()
    assert read_count == int(br.result.task_read_count[0]) and len(calls) > 10
    assert all(c.qc for c in calls) and calls == sorted(calls, key=lambda c: c.pos)
    assert {c.svtype for c in calls} >= {"INS", "DEL"}


def test_seq_on_demand_gives_identical_alts():
    """e2e mode: the seq arena stays on the host, only the requested slices cross PCIe; results must not change."""
    import oracle.oracle as orc
    blk = synth.config_block(5, 0.05)
    cfg = abi.Config.from_sniffles(sconfig.default_config())
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk, seq_on_demand=True)
        got = ctx.run()
    finally:
        ctx.close()
    devcheck.assert_same(orc.run(blk, cfg, 3, 4), got)
    assert len(got.alt) > 10000


@pytest.mark.parametrize("prefix", ["hg008", "hg002"])
def test_reference_bnd_vectors_on_device(prefix):
    """The reference's own vectors (src/tests/test_bnd_leads.py: 8 tuples + 9 "no lead" on hg008.bam / hg002.bam) through the CUDA path."""
    import json
    import os
    from test_oracle_golden import GOLDEN, _bam_block, bnd_leads_by_record
    with open(os.path.join(GOLDEN, "hg008_bnd.json")) as f:
        exp = [e for e in json.load(f)["records"] if e["file"].startswith(prefix)]
    blk = _bam_block(prefix)
    cfg = abi.Config.from_sniffles(sconfig.default_config("--dev-no-qc"))
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk, cigar16=False)
        res = ctx.extract_leads()
    finally:
        ctx.close()
    got = bnd_leads_by_record(blk, res.leads)
    assert len(exp) == len(blk.rec)
    for i, e in enumerate(exp):
        assert got.get(i) == e["lead"], (i, e, got.get(i))
    if prefix == "hg008":
        assert sum(e["lead"] is not None for e in exp) == 8


def test_coverage_bins_match_numpy():
    """snfb_coverage_bins = the reshape-mean of the per-base coverage vector the SNF writer stores (snf.py:248-267)."""
    import numpy as np
    from test_gpu_full_size import numpy_filter
    blk = synth.config_block(2, 0.003)
    cfg_ns = sconfig.default_config()
    ok, _ = numpy_filter(blk, cfg_ns)
    ops = blk.cigar & 15
    adv = np.isin(ops, [0, 2, 3, 7, 8])
    span = np.add.reduceat(np.where(adv, blk.cigar >> 4, 0).astype(np.int64), blk.rec["cigar_off"].astype(np.int64))
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(cfg_ns))
        ctx.load(blk)
        ctx.extract_leads()
        for t in (0, 5, len(blk.task) - 1):
            L = int(blk.task[t]["contig_len"])
            cov = np.zeros(L + 1, np.int64)
            sel = ok & (blk.rec["task"] == t)
            s = blk.rec["pos"][sel].astype(np.int64)
            e = np.minimum(s + span[sel], L)
            np.add.at(cov, s, 1)
            np.add.at(cov, e, -1)
            cov = np.cumsum(cov)[:L]
            pad = -L % 500
            want = np.pad(cov, (0, pad)).reshape(-1, 500).mean(axis=1)
            got = ctx.coverage_bins(t, 500)
            assert len(got) == len(want) and np.array_equal(got, want), t
    finally:
        ctx.close()


def test_calltask_from_bam_region(tmp_path):
    """A CallTask built the reference's way (id, contig, region, config, bam path, tandem repeats — sniffles:313-358) executes through
    BAM region fetch -> packer -> snfb_load_records -> the three per-stage exports, bound to device worker.id % n_gpus, and gives the
    calls of the block-level run."""
    from sniffles_b200 import bamio, tasks
    blk = synth.generate(91, [260_000, 150_000], 20.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=6000.0, tr_frac=0.2)
    path = str(tmp_path / "x.bam")
    bamio.write_bam(path, blk)
    cfg = sconfig.default_config()
    br = tasks.run_block(blk, cfg, 0)

    class Worker:
        id = 5

    for t, name in enumerate(blk.contig_names):
        tk = blk.task[t]
        o, n = int(tk["tr_off"]), int(tk["tr_n"])
        tr = [(int(blk.tr[2 * (o + k)]), int(blk.tr[2 * (o + k) + 1])) for k in range(n)]
        want = tasks.CallTask(id=t, sv_id=0, contig=name, start=0, end=int(tk["end"]), config=sconfig.default_config(), block_run=br, task_index=t)
        w_calls, w_reads = want.execute()
        for device_ingest in (True, False):            # compressed bytes decoded on the GPU (snfb_load_bam) / host reader + snfb_load_records
            got = tasks.CallTask(id=t, sv_id=0, contig=name, start=0, end=int(tk["end"]), config=sconfig.default_config(), bam=path, tandem_repeats=tr, device_ingest=device_ingest)
            g_calls, g_reads = got.execute(Worker())
            assert got.device == 5 % tasks.gpu_count()
            assert g_reads == w_reads and len(g_calls) == len(w_calls) > 5
            for a, b in zip(g_calls, w_calls):
                assert (a.svtype, a.pos, a.end, a.svlen, a.support, a.filter, a.alt, a.id) == (b.svtype, b.pos, b.end, b.svlen, b.support, b.filter, b.alt, b.id)
                assert a.genotypes == b.genotypes and a.info == b.info
