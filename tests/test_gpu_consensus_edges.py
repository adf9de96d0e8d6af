"""Stage C on the device at its dispatch, vote and alphabet edges: every case block of tests/consensus_common.py gives the oracle's
result field by field and the reference's calls and ALTs (tests/golden/consensus/expected.json), with the consensus in 1 and 7 slices,
from the full sequence arena and with the sequences fetched on demand."""
import pytest

import consensus_common as cc
from test_consensus_edges import calls, golden
from test_gpu_consensus_slices import _check

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    return golden()


@pytest.mark.parametrize("seq_on_demand", [False, True], ids=["arena", "on_demand"])
@pytest.mark.parametrize("name", sorted(cc.CASES))
def test_consensus_edges_match_oracle_and_reference(name, seq_on_demand, gold):
    blk, _, args = cc.build(name)
    assert cc.digest(blk) == gold[name]["digest"]
    res = _check(blk, *args, slices=(1, 7), seq_on_demand=seq_on_demand)
    got = calls(res)
    assert len(got) == len(gold[name]["calls"])
    for i, (a, b) in enumerate(zip(got, gold[name]["calls"])):
        assert a == b, f"call {i}: device {a} != reference {b}"
