"""snfb_allgather_candidates on one rank without a communicator.  Rebasing is the identity at one rank, so the gathered arrays equal the
run's own.  A second block several times larger makes the agreed slot size and the pinned result grow between calls on the same context."""
import ctypes as C

import numpy as np
import pytest

from sniffles_b200 import abi, binding, synth
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    c.set_config(abi.Config.from_sniffles(sconfig.default_config()))
    yield c
    c.close()


def _same_records(got, want):
    assert len(got) == len(want)
    for f in want.dtype.names:
        np.testing.assert_array_equal(got[f], want[f], err_msg=f)


def _gather_and_compare(ctx, contig_len):
    """load a synthetic block, run it, and check every form of the gather against the run; returns the largest slot size used"""
    ctx.load(synth.generate(4242, [contig_len], 20.0, len_mean=12000.0, len_sd=3000.0, sv_spacing=8000.0, tr_frac=0.2))
    r = ctx.run()
    assert len(r.cand) > 0
    slot = 0
    for with_leads in (False, True):
        g = ctx.allgather_candidates(with_leads=with_leads)
        assert (g.n_cand, g.n_alt_bytes, g.n_rnames) == (len(r.cand), len(r.alt), len(r.rnames))
        assert g.n_cand_leads == (len(r.cand_leads) if with_leads else 0)
        _same_records(g.cand, r.cand)
        np.testing.assert_array_equal(g.alt, r.alt)
        np.testing.assert_array_equal(g.rnames, r.rnames)
        np.testing.assert_array_equal(g.rn_off, r.rn_off)
        _same_records(g.cand_leads, r.cand_leads if with_leads else np.zeros(0, abi.LEAD_DTYPE))
        slot = max(slot, g.dev_bytes_per_rank)
    g = ctx.allgather_candidates(device_only=True)
    assert (g.n_cand, g.n_alt_bytes, g.n_rnames, g.n_cand_leads) == (len(r.cand), len(r.alt), len(r.rnames), 0)
    assert g.dev_bytes_per_rank > 0
    # the per-rank candidate counts the binding does not expose
    gv = abi.GatherView()
    assert ctx._lib.snfb_allgather_candidates(ctx._h, abi.GATHER_DEVICE_ONLY, C.byref(gv)) == 0
    assert list(abi.view(gv.rank_n_cand, "<u8", 1)) == [len(r.cand)]
    return max(slot, g.dev_bytes_per_rank)


def test_gather_equals_run_and_grows(ctx):
    small = _gather_and_compare(ctx, 400_000)
    large = _gather_and_compare(ctx, 2_400_000)
    assert large > small, "the larger block should have needed a larger slot"
