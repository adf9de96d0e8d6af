"""N-masked coverage on the device (--reference) against independent answers, with runs placed where the probes read them.

Candidate positions do not depend on the mask, so every block runs once unmasked; the probe positions of postprocessing.coverage
(postprocessing.py:69-130, restated here) then place runs on, just before, just after and around each probe, and the masked run is
compared field by field with the C oracle (oracle/snf_oracle.c: coverage zeroed inside [max(a, start), min(b, end)) clipped to [0, L)).
Around those runs: runs at base 0 and at the contig end (where upstream probes that wrap to a negative index land), runs past the
contig end, runs across region edges, adjacent and single-base runs, a run over a whole read, a run over a whole task, one task with
tens of thousands of runs, and tasks with none between tasks with some.  Region tasks (start > 0, and two tasks of one contig with a
run list each) and a task whose header length is shorter than its reads reach put the clipping of every path to work.

snfb_coverage_bins (the SNF `_COVERAGE` means) is checked against the numpy restatement of the masked vector at several bin sizes and
against what the reference itself stored (tests/golden/reference/snf_coverage.json); snfb_genotype_targets' probes against
oracle/genotype.py on a masked block; and snfb_load_records refuses runs that are not sorted and disjoint."""
import dataclasses
import json
import os

import numpy as np
import pytest

from oracle import genotype as ogt
from sniffles_b200 import abi, binding, snf, synth
from sniffles_b200 import config as sconfig
import devcheck
import ref_fasta
from test_gpu_full_size import numpy_filter

pytestmark = pytest.mark.gpu

WALK_WIDE_MIN = 32 * 132 * 4 * 8          # blocks this large are walked in 32-record tiles (test_gpu_cigar_walk_passes.py)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference")


def probe_positions(cand, bs, ud):
    """{task: [positions]} every candidate's coverage probes read, in emission order: a BND takes the `end` of the last non-BND call
    of its task before it, and has no end probes when there is none (the reference's UnboundLocalError)"""
    out, last_end = {}, {}
    for c in cand:
        t, ty, pos, svlen = int(c["task"]), int(c["svtype"]), int(c["pos"]), int(c["svlen"])
        start, end = pos, None
        if ty == abi.INS:
            end = start + 1
        elif ty == abi.BND:
            start -= int(c["bnd_is_first"])
            end = last_end.get(t)
        else:
            end = pos + abs(svlen)
        if ty != abi.BND:
            last_end[t] = end
        if ty in (abi.INS, abi.BND):
            ps = [start - bs, start] + ([end + bs] if end is not None else [])
        else:
            ps = [start, int((start + end) / 2), end - bs]
        ps += [start - ud] + ([end + ud] if end is not None else [])
        out.setdefault(t, []).extend(ps)
    return out


def disjoint(iv):
    """sorted, pairwise disjoint runs (adjacent allowed): the first of any overlapping pair is kept"""
    out = []
    for a, b in sorted((max(0, int(a)), int(b)) for a, b in iv):
        if a <= b and (not out or a >= out[-1][1]):
            out.append((a, b))
    return out


def place_runs(blk, probes, rng, deep=None, whole=None, skip=3):
    """{task: runs}: per probe one of [p, p+1), [p-k, p), [p+1, p+k), [p-k, p+k) in turn (a negative probe wrapped as numpy
    indexes), plus the edge cases of the module doc; every `skip`-th task gets none, `deep` ten thousands, `whole` one over its region"""
    spans = ogt.record_spans(blk)
    runs = {}
    for t, tk in enumerate(blk.task):
        L, start, end = int(tk["contig_len"]), int(tk["start"]), int(tk["end"])
        if t % skip == skip - 1:
            continue
        if t == deep:
            x = np.arange(0, L + 200, 17)
            runs[t] = disjoint(zip(x, x + rng.integers(0, 17, len(x))))        # empty, single-base and adjacent runs, some past L
            continue
        if t == whole:
            runs[t] = [(start, end), (L, L + 10)]
            continue
        iv = []
        for j, p in enumerate(sorted(set(probes.get(t, [])))):
            if p < 0:
                p += L
            k = int(rng.integers(2, 300))
            iv.append([(p, p + 1), (p - k, p), (p + 1, p + k), (p - k, p + k)][j % 4])
        iv += [(0, int(rng.integers(1, 400))), (L - int(rng.integers(1, 400)), L), (L, L + 3), (L + 50, L + 5000)]
        iv += [(start - 40, start + 40), (end - 40, end + 40), (start, start + 1), (end - 1, end)]
        for x in rng.integers(0, max(L, 1), 6):
            iv += [(int(x), int(x) + 10), (int(x) + 10, int(x) + 11)]                  # adjacent, single base
        mine = np.nonzero(blk.rec["task"] == t)[0]
        if len(mine):
            r = int(mine[len(mine) // 2])
            iv.append((int(blk.rec["pos"][r]), int(blk.rec["pos"][r]) + int(spans[r])))   # a whole read
        runs[t] = disjoint(iv)
    return runs


def with_regions(blk):
    """task 1 narrowed to a region with start > 0, and task 0's contig split into two tasks [0, m) and [m, L) with the records
    of the contig in both (appended as the last task, so records stay ordered by task)"""
    task = blk.task.copy()
    if len(task) > 1:
        L1 = int(task[1]["contig_len"])
        task[1]["start"], task[1]["end"] = L1 // 5, (3 * L1) // 4
    L0 = int(task[0]["contig_len"])
    m = L0 // 2 + 777
    extra = task[0:1].copy()
    extra["start"], extra["task_id"] = m, int(task["task_id"].max()) + 1
    task[0]["end"] = m
    dup = blk.rec[blk.rec["task"] == 0].copy()
    dup["task"] = len(task)
    return dataclasses.replace(blk, rec=np.concatenate([blk.rec, dup]), task=np.concatenate([task, extra]), rec16=None, cigar16=None,
                               mask=None, mask_task_off=None)


def with_short_header(blk, t=0, cut=3000):
    """task t's contig length (and region end) cut short of where its reads reach: read ends clip to L, runs past L clip away"""
    task = blk.task.copy()
    task[t]["contig_len"] -= cut
    task[t]["end"] = min(int(task[t]["end"]), int(task[t]["contig_len"]))
    return dataclasses.replace(blk, task=task, rec16=None, cigar16=None, mask=None, mask_task_off=None)


def numpy_bins_check(ctx, blk, cfg_ns, runs, binsizes=None):
    """snfb_coverage_bins = the padded reshape-means of the per-base vector with the runs zeroed, every task, every bin size"""
    ok, span = numpy_filter(blk, cfg_ns)[0], ogt.record_spans(blk)
    for t in range(len(blk.task)):
        L = int(blk.task[t]["contig_len"])
        cv = ogt.coverage_vector(blk, ok, span, t, runs.get(t))
        for b in binsizes or (1, 7, 100, 500, L, L + 1):
            got, want = ctx.coverage_bins(t, b), ref_fasta.coverage_bins(cv, b)
            assert len(got) == len(want), (t, b)
            i = np.nonzero(got != want)[0]
            assert len(i) == 0, f"task {t} binsize {b}: bin {i[0]} device {got[i[0]]} != masked numpy {want[i[0]]}"


def run_masked(blk, args, seed, deep=None, whole=None, bins=True):
    import oracle.oracle as orc
    cfg_ns = sconfig.default_config(*args)
    cfg = abi.Config.from_sniffles(cfg_ns)
    rng = np.random.default_rng(seed)
    blk.mask = blk.mask_task_off = None
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk)
        plain = ctx.run()
        runs = place_runs(blk, probe_positions(plain.cand, cfg_ns.coverage_binsize, cfg_ns.coverage_binsize * cfg_ns.coverage_updown_bins),
                          rng, deep, whole)
        blk.set_n_mask(runs)
        ctx.load(blk)
        got = ctx.run()
        devcheck.assert_same(orc.run(blk, cfg, 3, 8), got)
        if bins:
            numpy_bins_check(ctx, blk, cfg_ns, runs)
        # the same context reloaded without a mask: a fresh unmasked run, nothing of the mask left over
        blk.mask = blk.mask_task_off = None
        ctx.load(blk)
        again = ctx.run()
        assert again.cand.tobytes() == plain.cand.tobytes() and again.alt.tobytes() == plain.alt.tobytes()
        assert (again.task_cov_mean == plain.task_cov_mean).all()
        if bins:
            numpy_bins_check(ctx, blk, cfg_ns, {}, (500,))
    finally:
        ctx.close()
    assert sum(len(r) for r in runs.values()) > 50 and (got.task_cov_mean < plain.task_cov_mean).any()
    return runs, got


def test_config1_masked():
    run_masked(synth.config_block(1), (), 1)


@pytest.mark.parametrize("args", [(), ("--mosaic",), ("--qc-nm",), ("--minsupport", "auto")])
def test_config2_masked(args):
    runs, _ = run_masked(synth.config_block(2, 0.004), args, 2, deep=0, whole=4)
    assert len(runs[0]) > 20_000


def test_config2_regions_masked():
    """region tasks: start > 0, and two tasks of one contig, each with its own runs; records outside a region are filtered"""
    blk = with_regions(synth.config_block(2, 0.004))
    runs, got = run_masked(blk, (), 3)
    n = len(blk.task) - 1
    assert runs.get(0) and runs.get(n) and runs[0] != runs[n] and int(blk.task[1]["start"]) > 0


def test_short_contig_header_masked():
    """reads that run past the task's contig length: their ends clip to L in every coverage path"""
    blk = with_short_header(synth.config_block(2, 0.004), t=0)
    spans = ogt.record_spans(blk)
    sel = blk.rec["task"] == 0
    assert (blk.rec["pos"][sel] + spans[sel] > int(blk.task[0]["contig_len"])).any()
    run_masked(blk, (), 4)


def test_config3_masked():
    run_masked(synth.config_block(3, 0.003), ("--mosaic",), 5, whole=1)


def test_config5_masked():
    run_masked(synth.config_block(5, 0.05), (), 6)


@pytest.mark.parametrize("seed", range(4))
def test_random_shapes_masked(seed):
    """BND-heavy and long-read shapes"""
    shapes = [dict(len_mean=30000.0, len_sd=5000.0, sv_spacing=1500.0, clip_prob=0.5, tr_frac=0.1),
              dict(len_mean=60000.0, len_sd=20000.0, len_max=200000, sv_spacing=5000.0, clip_prob=0.3, tr_frac=0.0),
              dict(len_mean=8000.0, len_sd=2000.0, sv_spacing=800.0, clip_prob=0.5, tr_frac=0.3, tech="hifi"),
              dict(len_mean=20000.0, len_sd=300.0, sv_spacing=3000.0, clip_prob=0.4, phased_frac=1.0)][seed]
    blk = synth.generate(3100 + seed, [450_000, 180_000, 260_000][:2 + seed % 2], 25.0, **shapes)
    run_masked(blk, (), 10 + seed)


def test_wide_walk_block_masked():
    blk = synth.config_block(3, 0.015)
    assert len(blk.rec) >= WALK_WIDE_MIN
    run_masked(blk, ("--mosaic",), 7, deep=2, bins=False)


# ------------------------------------------------------------------------------------------------ force calling probes under a mask
def edge_targets(t, runs, bs, rng, n=60):
    """targets of task t whose start / center / end probes fall on the first base of a run, the base before it, its last base and the
    base after it, and BND targets whose end probe is the leaked `end` of the DEL before them landing there"""
    rows = []
    for a, b in [runs[i] for i in rng.integers(0, len(runs), n)]:
        for p in (a - 1, a, b - 1, b):
            rows += [(t, abi.INS, p, 100, 0, 0), (t, abi.INS, p + bs, 100, 0, 0), (t, abi.DEL, p - 300, 600, 0, 0),
                     (t, abi.DEL, p + bs - 400, 400, 0, 0), (t, abi.BND, p + 1, 0, 1, 0),
                     (t, abi.DEL, p - bs - 500, 500, 0, 0), (t, abi.BND, p + 5000, 0, 0, 0)]
    return rows


def test_genotype_probes_under_a_mask():
    """on region tasks too: past a region's end the passing reads still cover the probes, and a run there is not masked"""
    blk = with_regions(synth.config_block(2, 0.01))
    cfg_ns = sconfig.default_config()
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(cfg_ns))
        ctx.load(blk)
        plain = ctx.run()
        rng = np.random.default_rng(11)
        runs = place_runs(blk, probe_positions(plain.cand, cfg_ns.coverage_binsize, cfg_ns.coverage_binsize * cfg_ns.coverage_updown_bins),
                          rng, deep=1)
        blk.set_n_mask(runs)
        ctx.load(blk)
        res = ctx.run()
        cols = synth.genotype_targets(res.cand, len(blk.task), blk.task["contig_len"], rng, 100_000)
        rows = list(zip(*(np.asarray(c).tolist() for c in cols)))
        for t, r in runs.items():
            if r:
                rows += edge_targets(t, r, cfg_ns.coverage_binsize, rng)
        rows.sort(key=lambda x: x[0])                                  # stable: input order kept inside a task
        cols = [np.array(c, np.int32) for c in zip(*rows)]
        match, cs, cc, ce, flag = ctx.genotype_targets(*cols, cfg_ns.combine_match, cfg_ns.combine_match_max)
    finally:
        ctx.close()
    task = cols[0]
    ranges = np.searchsorted(res.cand["task"], np.arange(len(blk.task) + 1))
    ok, span = numpy_filter(blk, cfg_ns)[0], ogt.record_spans(blk)
    masked = 0
    for t in np.unique(task):
        idx = np.nonzero(task == t)[0]
        lo, hi = int(ranges[t]), int(ranges[t + 1])
        cands = ogt.cand_svs(res.cand[lo:hi], blk.contig_names)
        targets = [ogt.Sv(abi.SVTYPE_NAMES[int(cols[1][i])] if int(cols[1][i]) >= 0 else "CNV", int(cols[2][i]), int(cols[3][i]), int(cols[4][i]),
                          blk.contig_names[int(cols[5][i])] if int(cols[5][i]) >= 0 else "unknown") for i in idx]
        want = np.array([lo + m if m >= 0 else -1 for m in ogt.match(cands, targets, cfg_ns.combine_match, cfg_ns.combine_match_max, cfg_ns.cluster_merge_bnd)])
        assert np.array_equal(match[idx], want), int(t)
        try:
            cov = np.array(ogt.coverage(targets, ogt.coverage_vector(blk, ok, span, int(t), runs.get(int(t))), cfg_ns.coverage_binsize))
            plain_cov = np.array(ogt.coverage(targets, ogt.coverage_vector(blk, ok, span, int(t)), cfg_ns.coverage_binsize))
        except UnboundLocalError:
            assert flag[idx].any(), int(t)
            continue
        assert not flag[idx].any(), int(t)
        got = np.stack([cs[idx], cc[idx], ce[idx]], 1)
        bad = np.nonzero((got != cov).any(axis=1))[0]
        assert len(bad) == 0, f"task {t} target {idx[bad[0]]} {rows[idx[bad[0]]]}: device {got[bad[0]]} != masked restatement {cov[bad[0]]}"
        masked += int((cov != plain_cov).sum())
    assert masked > 1000


# ------------------------------------------------------------------------------------------------ SNF bins against the reference
@pytest.mark.parametrize("name", sorted(ref_fasta.GOLDEN_FASTA))
def test_device_bins_to_snf_coverage_match_the_reference(name):
    """device bins -> SNFWriter.annotate_block_coverages = the `_COVERAGE` the reference stored with --snf --reference"""
    from test_oracle_golden import load_fixture
    with open(os.path.join(GOLDEN, "snf_coverage.json")) as f:
        gold = json.load(f)["blocks"][name]
    _, blk = load_fixture(name)
    text, seqs = ref_fasta.golden_fasta(name)
    assert ref_fasta.sha256(text) == gold["fasta_sha256"]
    blk.set_n_mask(ref_fasta.task_runs(blk, seqs))
    cfg = sconfig.default_config("--snf", "x.snf", *gold["args"])
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(cfg))
        ctx.load(blk)
        ctx.extract_leads()
        n = 0
        for t in range(len(blk.task)):
            contig = blk.contig_names[int(blk.task[t]["contig"])]
            want = {int(b): {int(p): v for p, v in e.items()} for b, e in gold["coverage"].get(contig, {}).items()}
            w = snf.SNFWriter(cfg, None)
            w.blocks = {b: {"_COVERAGE": {}} for b in want}
            w.annotate_block_coverages(ctx.coverage_bins(t, cfg.coverage_binsize_combine))
            assert {b: w.blocks[b]["_COVERAGE"] for b in want} == want, (name, contig)
            n += len(want)
    finally:
        ctx.close()
    assert n == sum(len(v) for v in gold["coverage"].values()) > 0


# ------------------------------------------------------------------------------------------------ masks that break the contract
@pytest.mark.parametrize("runs, message", [
    ({1: [(100, 200), (50, 60)]}, "N mask of task 1: run 1 starts before run 0 ends"),
    ({1: [(100, 200), (150, 300)]}, "N mask of task 1: run 1 starts before run 0 ends"),
    ({0: [(10, 20)], 1: [(5, 9), (300, 200)]}, "N mask of task 1: run 1 has start > end"),
])
def test_unsorted_overlapping_or_reversed_runs_are_refused(runs, message):
    blk = synth.generate(4243, [200_000, 150_000], 15.0, len_mean=9000.0, len_sd=2000.0, sv_spacing=8000.0)
    off, flat = [0], []
    for t in range(len(blk.task)):
        flat += [x for ab in runs.get(t, []) for x in ab]                  # as given: set_n_mask would sort them
        off.append(len(flat) // 2)
    blk.mask, blk.mask_task_off = np.array(flat, "<i4"), np.array(off, "<u4")
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(sconfig.default_config()))
        with pytest.raises(binding.SnfbError, match=message):
            ctx.load(blk)
        blk.set_n_mask({t: sorted(set(r)) for t, r in runs.items() if t == 0})
        ctx.load(blk)                                                   # the context stays usable
        assert len(ctx.run().cand) > 5
    finally:
        ctx.close()
