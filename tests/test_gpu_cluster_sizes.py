"""Stage B's per-cluster kernels at their size boundaries: hand-built blocks that put a chosen number of leads into one cluster (1 to 1025
leads: both sides of 32 and 48 — the dense warp kernel's rank sort in registers and its capacity —, 64, 128 — the mid-sized warp kernel — and 1024
— a block staging the leads in shared memory or working in global memory), for every SV type, and the tie rules of the per-cluster code:
the modal mate contig of a BND with tied counts, the names of long insertions read twice, phase sets that tie in count and differ in
decimal order, a cluster that resplit splits, and --qc-nm.  Each block runs on the device and in the oracle and must give the same result."""
import numpy as np
import pytest

import devcheck
import oracle.oracle as orc
from sniffles_b200 import abi, bamio
from sniffles_b200 import config as sconfig

SIZES = [1, 2, 31, 32, 33, 47, 48, 49, 63, 64, 65, 128, 129, 1024, 1025]
ARGS = ("--minsvlen", "35", "--minsupport", "2", "--mapq", "0")
SPACING = 60_000              # between the clusters of one block: far beyond every merge distance
FLANK = 2000


def _seq(rnd, l_seq):
    return rnd.integers(0, 256, (l_seq + 1) // 2, dtype=np.uint8) & 0x99 | 0x11


def _rec(rnd, pos, cigar, l_seq, qname, flag=0, aux=None):
    return dict(pos=pos, flag=flag, mapq=60, l_seq=l_seq, qname=qname, cigar=np.array(cigar, "<u4"), seq=_seq(rnd, l_seq), aux=aux or {"NM": 10})


def _indel(rnd, pos, k, op, length, qname, aux=None):
    """<FLANK>M <length>{I,D} <FLANK>M at about pos"""
    j = k % 3
    return _rec(rnd, pos - FLANK + j, [((FLANK - j) << 4) | 0, (length << 4) | op, ((FLANK + j) << 4) | 0],
                2 * FLANK + (length if op == 1 else 0), qname, flag=0 if k % 2 else 16, aux=aux)


def _split(rnd, pos, k, sa, qname, rev=False):
    """<FLANK>M <FLANK>S at about pos, the clipped half aligned where the SA entry says"""
    j = k % 3
    return _rec(rnd, pos - FLANK + j, [(FLANK << 4) | 0, (FLANK << 4) | 4], 2 * FLANK, qname, flag=16 if rev else 0,
                aux={"NM": 5, "SA": sa})


def _block(contigs, recs):
    """recs: (contig index, record) in any order; one task per contig"""
    by = sorted(recs, key=lambda cr: (cr[0], cr[1]["pos"]))
    return bamio.pack_records(contigs, [(c, r) for c, r in by], [(c, 0, ln, c) for c, (_, ln) in enumerate(contigs)])


def _sized(kind, sizes=SIZES):
    """one cluster of n leads per size, SPACING apart on ctgA; BND mates on ctgB"""
    rnd = np.random.default_rng(sum(sizes) * 31 + len(kind))
    contigs = [("ctgA", SPACING * (len(sizes) + 2)), ("ctgB", SPACING * (len(sizes) + 2))]
    recs = []
    for s, n in enumerate(sizes):
        pos = SPACING * (s + 1)
        for k in range(n):
            name = b"%s_%d_%04d" % (kind.encode(), n, k)
            if kind == "INS":
                recs.append((0, _indel(rnd, pos, k, 1, 200 + (k % 7), name)))
            elif kind == "DEL":
                recs.append((0, _indel(rnd, pos, k, 2, 300 + (k % 5), name)))
            elif kind == "DUP":            # the clipped half maps back upstream, same strand
                recs.append((0, _split(rnd, pos, k, b"ctgA,%d,+,%dS%dM,60,3;" % (pos - 3000 + 1 + (k % 4), FLANK, FLANK), name)))
            elif kind == "INV":            # the clipped half maps downstream on the other strand
                recs.append((0, _split(rnd, pos, k, b"ctgA,%d,-,%dM%dS,60,3;" % (pos + 4000 + 1 + (k % 4), FLANK, FLANK), name)))
            elif kind == "BND":            # the clipped half maps to the other contig
                recs.append((0, _split(rnd, pos, k, b"ctgB,%d,-,%dM%dS,60,3;" % (pos + 1 + (k % 4), FLANK, FLANK), name)))
    return _block(contigs, recs)


def _bnd_tied():
    """BND clusters whose leads split evenly between two mate contigs: the tie goes to the smaller name (beta), which has the larger index"""
    rnd = np.random.default_rng(7)
    sizes = [2, 16, 24, 32, 40, 300]
    contigs = [("ctgA", SPACING * (len(sizes) + 2)), ("zeta", 10_000_000), ("beta", 10_000_000)]
    recs = []
    for s, half in enumerate(sizes):
        pos = SPACING * (s + 1)
        for k in range(2 * half):
            mate = b"zeta" if k % 2 == 0 else b"beta"
            recs.append((0, _split(rnd, pos, k, b"%s,%d,-,%dM%dS,60,2;" % (mate, 100_000 + 1 + (k % 4), FLANK, FLANK), b"t_%d_%04d" % (half, k))))
    return _block(contigs, recs)


def _long_ins():
    """long insertions (svlen >= long_ins_length) whose clusters also hold clipped reads (leads_long), each clipped read's name twice"""
    rnd = np.random.default_rng(11)
    sizes = [(3, 4), (20, 12), (40, 30), (60, 50), (130, 40)]
    contigs = [("ctgA", SPACING * (len(sizes) + 2))]
    recs = []
    for s, (n_ins, n_clip) in enumerate(sizes):
        pos = SPACING * (s + 1)
        for k in range(n_ins):
            recs.append((0, _indel(rnd, pos, k, 1, 3000 + (k % 5), b"li_%d_%04d" % (s, k))))
        for k in range(n_clip):
            j = k % 3
            recs.append((0, _rec(rnd, pos - FLANK + j, [((FLANK - j) << 4) | 0, (3000 << 4) | 4], FLANK - j + 3000, b"lc_%d_%04d" % (s, k // 2))))
    return _block(contigs, recs)


def _phased():
    """INS clusters of phased reads: PS 9 and PS 10 tie in count at most sizes (str order: "10" < "9"), with unphased reads and a third,
    rarer PS"""
    rnd = np.random.default_rng(13)
    sizes = [4, 12, 30, 48, 64, 100, 200]
    contigs = [("ctgA", SPACING * (len(sizes) + 2))]
    recs = []
    for s, n in enumerate(sizes):
        pos = SPACING * (s + 1)
        for k in range(n):
            m = k % 5
            aux = {"NM": 10, "HP": 1 + (m % 2), "PS": (9, 10, 9, 10)[m]} if m < 4 else {"NM": 10}
            if k % 20 == 4:
                aux = {"NM": 10, "HP": 1, "PS": 123}
            recs.append((0, _indel(rnd, pos, k, 1, 150 + (k % 3), b"ph_%d_%04d" % (n, k), aux=aux)))
    return _block(contigs, recs)


def _resplit():
    """INS clusters with two length groups far apart (resplit makes two sub-clusters), at sizes around the warp kernels' limits"""
    rnd = np.random.default_rng(17)
    sizes = [4, 32, 48, 64, 128, 400]
    contigs = [("ctgA", SPACING * (len(sizes) + 2))]
    recs = []
    for s, n in enumerate(sizes):
        pos = SPACING * (s + 1)
        for k in range(n):
            recs.append((0, _indel(rnd, pos, k, 1, (100 if k % 3 else 600) + (k % 4), b"rs_%d_%04d" % (n, k))))
    return _block(contigs, recs)


BLOCKS = {"ins": lambda: _sized("INS"), "del": lambda: _sized("DEL"), "dup": lambda: _sized("DUP"), "inv": lambda: _sized("INV"),
          "bnd": lambda: _sized("BND"), "bnd_tied_mates": _bnd_tied, "long_ins_dup_names": _long_ins, "phase_set_ties": _phased,
          "resplit": _resplit}


def _run_both(blk, *extra):
    from sniffles_b200 import binding
    cfg = abi.Config.from_sniffles(sconfig.default_config(*ARGS, *extra))
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk)
        got = ctx.run()
    finally:
        ctx.close()
    want = orc.run(blk, cfg, 3, 1)
    return want, got


@pytest.mark.parametrize("name", sorted(BLOCKS))
def test_blocks_make_the_clusters_they_are_built_for(name):
    """CPU: the oracle calls something on every block, so the device comparison below compares candidates"""
    blk = BLOCKS[name]()
    res = orc.run(blk, abi.Config.from_sniffles(sconfig.default_config(*ARGS)), 2, 1)
    assert len(res.cand) > 0, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BLOCKS))
def test_cluster_sizes_match_the_oracle(name):
    want, got = _run_both(BLOCKS[name]())
    devcheck.assert_same(want, got)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ins", "del", "bnd", "long_ins_dup_names"])
def test_cluster_sizes_match_the_oracle_qc_nm(name):
    want, got = _run_both(BLOCKS[name](), "--qc-nm")
    devcheck.assert_same(want, got)


@pytest.mark.gpu
def test_tied_mate_contigs_in_one_sub_cluster_match_the_oracle():
    """without resplit a BND sub-cluster holds both mate contigs, so resolve_bnd's tie rule decides which leads stay"""
    want, got = _run_both(_bnd_tied(), "--dev-no-resplit")
    devcheck.assert_same(want, got)
