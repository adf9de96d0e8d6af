"""GPU tests of k_rec_index: the clips at the two ends of a record, found from its first and last 16-byte CIGAR16 groups (word by word
when the clip ops at an end leave those groups), and the record checks that make a malformed block fail the run."""
import numpy as np
import pytest

from sniffles_b200 import abi, binding, synth
from sniffles_b200 import config as sconfig
from test_gpu_parity import _run

pytestmark = pytest.mark.gpu

MALFORMED = "the record block is malformed: a record points outside its task table or arenas"
M, D, S = 0, 2, 4                         # BAM CIGAR op codes


def _cigar(n_ops, l_seq, tail_clip):
    """BAM words of a CIGAR of n_ops one-word CIGAR16 ops (so n_ops words, no pad words): a 5-base soft clip first when needed for the
    count, M and 1-base D ops alternating, ending with M, then a 7-base soft clip when tail_clip; the M ops share the other query bases."""
    tail = [(7, S)] if tail_clip else []
    mid = n_ops - len(tail)
    head = [(5, S)] if mid % 2 == 0 else []
    n_m = (mid - len(head) + 1) // 2
    base, extra = divmod(l_seq - sum(ln for ln, _ in head + tail), n_m)
    ops = list(head)
    for i in range(n_m):
        ops.append((base + (1 if i < extra else 0), M))
        if i + 1 < n_m:
            ops.append((1, D))
    ops += tail
    assert len(ops) == n_ops and all(0 < ln < 2048 for ln, _ in ops)
    return np.array([(ln << 4) | op for ln, op in ops], dtype="<u4")


# (CIGAR16 words, a soft clip at the end): 1 = a single M op (with its extension word), whose first op is its last; 129 and 257 words
# end with a clip that is alone in the last group, so the walk from the end continues into the group before it
SHAPES = [(1, False), (128, False), (129, True), (136, False), (256, False), (257, True)]


def test_records_of_chosen_group_counts():
    """Every third passing record is rewritten to one of SHAPES: records of 1, 16, 17, 32 and 33 groups, clips found inside the end groups
    and clips that take the word-by-word walk."""
    blk = synth.config_block(2, 0.004)
    rec = blk.rec
    pick = np.flatnonzero((rec["mapq"] >= 20) & (rec["l_seq"] >= 2000) & (rec["l_seq"] <= 60000) & ((rec["flag"] & 256) == 0))[::3]
    words, off = [blk.cigar], len(blk.cigar)
    for i, r in enumerate(pick):
        n_ops, tail_clip = SHAPES[i % len(SHAPES)]
        l_seq = int(rec["l_seq"][r])
        cg = np.array([(l_seq << 4) | M], dtype="<u4") if n_ops == 1 else _cigar(n_ops, l_seq, tail_clip)
        rec["cigar_off"][r], rec["n_cigar"][r] = off, len(cg)
        words.append(cg)
        off += len(cg)
    blk.cigar = np.concatenate(words)
    groups = (blk.pack16().rec16["n_cigar"][pick].astype(np.int64) + 7) // 8
    assert set(groups.tolist()) == {1, 16, 17, 32, 33}
    _run(blk, "--qc-nm")


def _corrupt(field):
    blk = synth.config_block(2, 0.004).pack16()
    r16 = blk.rec16
    i = len(r16) // 2
    if field == "task":
        r16["task"][i] = len(blk.task)
    elif field == "cigar_align":
        r16["cigar_off"][i] += 1
    elif field == "cigar_range":
        r16["cigar_off"][i] = len(blk.cigar16) - 8
        assert r16["n_cigar"][i] > 8
    return blk


@pytest.mark.parametrize("field", ["task", "cigar_align", "cigar_range"])
def test_malformed_record_fails_the_run(field):
    """One record with its task out of range, its CIGAR16 offset not a multiple of 8, or its CIGAR running past the arena: the run fails
    with the malformed-block message (k_rec_index counts the record and reads nothing through the bad field)."""
    blk = _corrupt(field)
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(sconfig.default_config()))
        ctx.load(blk)
        with pytest.raises(binding.SnfbError, match=MALFORMED):
            ctx.run()
    finally:
        ctx.close()
