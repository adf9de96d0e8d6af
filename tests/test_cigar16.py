"""CIGAR16 (include/snfb.h): snfb_pack_cigar16 is host code, so the format is checked without a GPU:
every op survives the round trip, groups never straddle a 16-byte boundary, records start on one.
`check_record` decodes with this file's own reading of the format, independent of sniffles_b200/csrc/cigar16.h; the ingest tests
check the device encoder's words with it as well."""
import numpy as np
import pytest

from sniffles_b200 import abi, binding, synth

CLASS = [3, 1, 2, 6, 5, 4, 0, 3, 3]          # M I D N S H P = X


def decode(words):
    """CIGAR16 words -> [(length, class, E)]; pad words are skipped.  An op's extension words follow it directly, level 1 then 2."""
    ops, level = [], 0          # the level the next extension word must have (0: none may come)
    for k, w in enumerate(int(x) for x in words):
        if w & 0x8000:
            assert k % 8 != 0, "an extension word starts a 16-byte group"
            assert level and (w >> 12) & 7 == level, "extension word without its base word or out of order"
            ln, c, e = ops[-1]
            ops[-1] = (ln + ((w & 0xfff) << (11 + 12 * (level - 1))), c, e)
            level = 2 if level == 1 else 0
        elif w != 0:
            ops.append((w & 0x7ff, (w >> 11) & 7, bool(w & 0x4000)))
            level = 1
        else:
            level = 0
    return ops


def n_words(cigar32):
    """words of one record: 1, 2 or 3 per op (length below 2^11, 2^23, or more), and pad words only where a group would straddle 16 bytes"""
    k = 0
    for w in cigar32:
        ln = int(w) >> 4
        g = 1 if ln < 1 << 11 else 2 if ln < 1 << 23 else 3
        if k % 8 + g > 8:
            k = (k + 7) // 8 * 8
        k += g
    return k


def check_record(words, cigar32, evt_min=11):
    """one record's CIGAR16 words (from its first word to its last op's last word) against its BAM CIGAR words"""
    assert len(words) == n_words(cigar32)
    got = decode(words)
    want = [(int(w) >> 4, CLASS[int(w) & 15]) for w in cigar32]
    want = [(ln, c) for ln, c in want if not (ln == 0 and c == 0)]        # a zero-length P is a pad word
    assert [(ln, c) for ln, c, _ in got] == want
    for ln, c, e in got:          # E bit: an I / D / S of at least evt_min bases
        assert e == (c in (1, 2, 5) and ln >= evt_min), (ln, c, e)


def block_of(cigars):
    rec = np.zeros(len(cigars), abi.REC_DTYPE)
    flat, off = [], 0
    for i, cg in enumerate(cigars):
        rec[i]["cigar_off"], rec[i]["n_cigar"] = off, len(cg)
        flat.extend((ln << 4) | op for ln, op in cg)
        off += len(cg)
    return rec, np.asarray(flat, dtype="<u4")


def check(rec, cigar32):
    rec16, c16 = binding.pack_cigar16(rec, cigar32)
    assert len(c16) % 8 == 0
    for r, r16 in zip(rec, rec16):
        assert int(r16["cigar_off"]) % 8 == 0
        o, n = int(r16["cigar_off"]), int(r16["n_cigar"])
        check_record(c16[o:o + n], cigar32[int(r["cigar_off"]):int(r["cigar_off"]) + int(r["n_cigar"])])
        for f in ("task", "pos", "flag", "mapq", "l_seq", "seq_off", "var_off", "nm"):
            assert r[f] == r16[f]
    return rec16, c16


def test_round_trip_random_ops():
    rnd = np.random.default_rng(7)
    cigars = []
    for _ in range(300):
        n = int(rnd.integers(1, 60))
        lens = np.where(rnd.random(n) < 0.15, rnd.integers(2048, 1 << 23, n), rnd.integers(0, 300, n))
        lens = np.where(rnd.random(n) < 0.03, rnd.integers(1 << 23, 1 << 28, n), lens)
        cigars.append([(int(l), int(o)) for l, o in zip(lens, rnd.integers(0, 9, n))])
    check(*block_of(cigars))


def test_length_boundaries():
    cigars = [[(2047, 0), (2048, 1), (2049, 2), ((1 << 23) - 1, 3), (1 << 23, 4), ((1 << 28) - 1, 2), (0, 0), (1, 8), (10, 1), (11, 2)],
              [(5000, 4)] * 9, [((1 << 24) + 5, 2)] * 7, [(10, 0)]]
    rec16, c16 = check(*block_of(cigars))
    # [(5000, S)] x 9: two-word groups, four per 16 bytes -> 8, 8, 2 words
    assert int(rec16[1]["n_cigar"]) == 18
    # three-word groups: two per 16 bytes, two pad words each time
    assert int(rec16[2]["n_cigar"]) == 8 * 3 + 3


def test_unknown_op_is_rejected():
    rec, cg = block_of([[(10, 0), (3, 9)]])
    with pytest.raises(binding.SnfbError):
        binding.pack_cigar16(rec, cg)


def test_synthetic_block():
    blk = synth.config_block(2, 0.002)
    check(blk.rec[::53].copy(), blk.cigar)
    blk.pack16()
    assert blk.cigar16.nbytes < 0.52 * blk.cigar.nbytes
