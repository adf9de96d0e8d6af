"""Stage C in slices (snfb_set_consensus_slices): the candidates, ALT bytes and read names are byte-identical for every slice count and
equal to the oracle's, on blocks where the slices are uneven or empty: no candidate at all, candidates without ALT bytes, one consensus
candidate, one candidate holding almost all the work, and a run redone after the consensus kernels were already queued."""
import numpy as np
import pytest

from sniffles_b200 import abi, binding, synth
from sniffles_b200 import config as sconfig
import devcheck

pytestmark = pytest.mark.gpu

SLICES = (1, 2, 4, 7)


def _runs(blk, *args, slices=SLICES, seq_on_demand=False):
    """{k: Result} over `slices` on one context, and the oracle's result"""
    import oracle.oracle as orc
    cfg = abi.Config.from_sniffles(sconfig.default_config(*args))
    ctx = binding.Context(0)
    got = {}
    try:
        ctx.set_config(cfg)
        ctx.load(blk, seq_on_demand=seq_on_demand)
        for k in slices:
            ctx.set_consensus_slices(k)
            got[k] = ctx.run(want_leads=False)
    finally:
        ctx.close()
    return got, orc.run(blk, cfg, 3, 4)


def _check(blk, *args, slices=SLICES, seq_on_demand=False):
    got, want = _runs(blk, *args, slices=slices, seq_on_demand=seq_on_demand)
    one = got[slices[0]]
    for k, res in got.items():
        for name in ("cand", "cand_leads", "rnames", "rn_off", "alt"):
            a, b = getattr(one, name), getattr(res, name)
            assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), f"{name} with {k} slices differs from {slices[0]}"
        devcheck.assert_same(want, res, check_leads=False)
    return one


def _ins_work(res):
    ins = res.cand[(res.cand["svtype"] == 0) & (res.cand["alt_len"] > 0)]
    return ins["alt_len"].astype(np.float64) * ins["lead_n"]


@pytest.mark.parametrize("name", ["c5_ins_heavy", "long_ins_minsv", "c1_ont_1mb"])
def test_golden_fixtures(name):
    from test_oracle_golden import load_fixture
    fx, blk = load_fixture(name)
    res = _check(blk, *fx["args"])
    assert len(_ins_work(res)) > 0


def test_no_candidate():
    res = _check(synth.generate(11, [300000], 20.0, sv_spacing=1e9, tr_frac=0.0, threads=4))
    assert len(res.cand) == 0 and len(res.alt) == 0


def test_candidates_without_alt_bytes():
    res = _check(synth.config_block(2, 0.002), "--symbolic")
    assert len(res.cand) > 0 and len(res.alt) == 0


def test_single_consensus_candidate():
    res = _check(synth.generate(12, [200000], 20.0, sv_spacing=150000.0, ins_only=True, tr_frac=0.0, sv_min=1500, sv_max=1500, ins_noise=0.0, clip_prob=0.0, threads=4))
    assert len(_ins_work(res)) == 1


def test_one_candidate_holds_most_of_the_work():
    """a 3,057-bp insertion (heavy items) carries 92 % of the rows x length: most slices are cut inside or around it"""
    res = _check(synth.generate(44, [400000], 20.0, sv_spacing=90000.0, ins_only=True, tr_frac=0.0, sv_min=50, sv_max=5000, threads=4))
    w = _ins_work(res)
    assert len(w) >= 3 and w.max() / w.sum() > 0.9


def test_rerun_after_stage_c_was_queued():
    """a chain cut found wrong at the counters read mid-run: the run is redone while the first attempt's consensus kernels are in flight"""
    blk = synth.generate(77, [600000], 20.0, len_model=0, len_mean=20000.0, len_sd=2000.0, len_min=5000, len_max=60000, tech="ont", sv_spacing=1300.0,
                         ins_only=True, tr_frac=0.0, clip_prob=0.0, sv_min=50, sv_max=400, threads=4)
    _check(blk, "--cluster-r", "2000")


def test_slice_count_is_checked():
    ctx = binding.Context(0)
    try:
        for k in (0, 9):
            with pytest.raises(binding.SnfbError):
                ctx.set_consensus_slices(k)
    finally:
        ctx.close()
