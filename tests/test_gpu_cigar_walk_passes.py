"""GPU parity of k_cigar_walk's decode of flagged groups on blocks walked in 32-record tiles (at least WALK_WIDE_MIN = 135,168
records; smaller blocks are walked one record per warp).  The flagged chunks of a round are decoded together, one group per lane,
in passes of 32 groups: these shapes put many passes into one round, several E words into one group, and E words next to
extension words."""
import pytest

from sniffles_b200 import synth
from test_gpu_parity import _run

pytestmark = pytest.mark.gpu

WALK_WIDE_MIN = 32 * 132 * 4 * 8


@pytest.mark.parametrize("args", [(), ("--qc-nm",)])
def test_dense_svs_in_long_ont_reads(args):
    """An SV every 2 kb, from just below the 45-base screen threshold: most chunks are flagged, a round holds several passes of 32
    flagged groups, and some groups hold more than one E word.  With --qc-nm the big-indel sums of the decoded groups feed the NM
    correction."""
    blk = synth.generate(2025, [7_500_000] * 4, 20.0, len_mean=4000.0, len_sd=1000.0, len_min=2000, len_max=12000, tech="ont",
                         sv_spacing=2000.0, sv_min=40, sv_max=150, tr_frac=0.05, threads=8)
    assert len(blk.rec) >= WALK_WIDE_MIN
    got = _run(blk, *args)
    assert len(got.cand) > 1000


def test_hifi_extension_words_next_to_e_words():
    """HiFi: long matches put extension words into most chunks, so most flagged groups are decoded op by op."""
    blk = synth.config_block(3, 0.015)
    assert len(blk.rec) >= WALK_WIDE_MIN
    got = _run(blk, "--mosaic")
    assert len(got.cand) > 20
