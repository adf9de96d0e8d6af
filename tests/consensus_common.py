"""Hand-built record blocks for stage C (the INS consensus) at its dispatch, vote and alphabet edges.

Every case is one block of INS clusters, SPACING apart on one contig.  A cluster is a truth insertion T and the reads that carry it as one
CIGAR I op between two FLANK-long M ops, all at one reference position unless the case says otherwise.  The best read is chosen by
construction (the first read of the lowest-difference group, see `_place`), the other reads carry planted edits so the column vote
decides something: substitutions give rows whose acceptance is known, and the edits of the threshold cases are placed relative to the
strided anchor k-mers, so a segment's or a run's identity or a row's span lands exactly on its threshold.  `hits` restates which anchors a
read finds; the builder asserts with it that every planted edit does what its case says.

Blocks are rebuilt from seeds here and on the GPU machine; tests/golden/make_consensus_golden.py runs the reference on them."""
import hashlib

import numpy as np

from test_gpu_cluster_sizes import _block, _rec

FLANK = 1000
SPACING = 20_000
K = 6
A, C, G, T = 1, 2, 4, 8
ACGT = np.array([A, C, G, T], np.uint8)
CODE = "=ACMGRSVTWYHKDBN"
NOQC = ("--no-qc",)


def skip_of(L):
    """consensus_kmer_skip_base + int(L * consensus_kmer_skip_seqlen_mult) at the default settings"""
    return 3 + int(L * (1.0 / 500.0))


def text(codes):
    return "".join(CODE[c] for c in codes)


def anchors(best, skip):
    """{k-mer: i} of the best read's strided k-mers, repeated ones left out (taboo)"""
    out, taboo = {}, set()
    for i in range(0, len(best) - K, skip):
        km = bytes(best[i:i + K])
        if km in taboo:
            continue
        if km in out:
            del out[km]
            taboo.add(km)
            continue
        out[km] = i
    return out, taboo


def hits(best, read, skip):
    """the anchors (i, j) a read accepts, in j order"""
    an, _ = anchors(best, skip)
    got, last = [], None
    for j in range(0, len(read) - K, skip):
        i = an.get(bytes(read[j:j + K]))
        if i is None or abs(i - j) > K or (last is not None and i <= last):
            continue
        got.append((i, j))
        last = i
    return got


def _other(rnd, c):
    return int(rnd.choice([x for x in ACGT if x != c]))


def _subst(rnd, seq, cols):
    s = seq.copy()
    for p in cols:
        s[p] = _other(rnd, s[p])
    return s


def _sparse(rnd, seq, n, lo=8, hi=None):
    hi = len(seq) - 8 if hi is None else hi
    return _subst(rnd, seq, rnd.choice(np.arange(lo, hi), n, replace=False))


def _pack(codes):
    c = np.asarray(codes, np.uint8)
    if len(c) & 1:
        c = np.append(c, 0)
    return (c[0::2] << 4) | c[1::2]


def _read(rnd, lead_pos, ins, name, pieces=None, clip=0):
    """one record: [<clip>S] <FLANK>M <ins>I <FLANK>M with the insertion at reference position lead_pos; pieces = (a, g) splits the
    insertion into a bases, g M, the rest (two I ops merge_inner joins again); clip shifts the query offsets"""
    ins = np.asarray(ins, np.uint8)
    left, right = rnd.choice(ACGT, clip + FLANK), rnd.choice(ACGT, FLANK)
    cig = [(clip << 4) | 4] if clip else []
    if pieces is None:
        cig += [(FLANK << 4) | 0, (len(ins) << 4) | 1, (FLANK << 4) | 0]
        q = np.concatenate([left, ins, right])
    else:
        a, g = pieces
        cig += [(FLANK << 4) | 0, (a << 4) | 1, (g << 4) | 0, ((len(ins) - a) << 4) | 1, ((FLANK - g) << 4) | 0]
        q = np.concatenate([left, ins[:a], rnd.choice(ACGT, g), ins[a:], right[g:]])
    r = _rec(rnd, lead_pos - FLANK, cig, len(q), name)
    r["seq"] = _pack(q)
    return r


def _place(pos, n):
    """lead positions of n reads of one cluster: all at pos"""
    return [pos] * n


def _cluster(rnd, k, pos, best, others, positions=None, pieces=None, clips=None, need=()):
    """records of cluster k: the best read first, then the others; returns (records, meta).  need: anchor positions the case is built
    around (a random repeat of their k-mer elsewhere in the best read would make them taboo)"""
    seqs = [best] + list(others)
    positions = positions or _place(pos, len(seqs))
    recs = []
    for r, s in enumerate(seqs):
        pc = pieces[r] if pieces else None
        recs.append((0, _read(rnd, positions[r], s, b"c%02d_r%03d" % (k, r), pc, clips[r] if clips else 0)))
    sk = skip_of(len(best))
    clean = all(i == j for o in others for i, j in hits(best, o, sk))      # no k-mer planted by an edit anchors a read elsewhere
    have = set(anchors(best, sk)[0].values())
    clean = clean and all(p in have for p in need)
    return recs, dict(L=len(best), n_other=len(others), best=text(best), best_name="c%02d_r%03d" % (k, 0), clean=clean)


def _truth(rnd, L):
    return rnd.choice(ACGT, L).astype(np.uint8)


# ---------------------------------------------------------------- cluster kinds

def _unique(rnd, t, skip):
    """t with its strided k-mers made distinct (a base of each repeat redrawn), so every one of them is an anchor"""
    for _ in range(200):
        seen, dup = set(), []
        for i in range(0, len(t) - K, skip):
            km = bytes(t[i:i + K])
            (dup.append(i) if km in seen else seen.add(km))
        if not dup:
            return t
        for i in dup:
            t[i + 2] = _other(rnd, t[i + 2])
    raise AssertionError("no repeat-free insertion")


def _std(rnd, k, pos, L, n_other=6, copy_best=False):
    """T (all strided k-mers distinct) with errors in the best read, three of them in the last 60 bases, where a read's last hits
    land, and sparse errors in the others: the vote corrects the best read's errors.  With skip >= 7 the best read's errors sit between
    the strided k-mers, so it keeps every anchor.  copy_best: one other read equals the best read (it finds every anchor:
    (L - 6 + skip - 1) // skip hits)"""
    sk = skip_of(L)
    t = _unique(rnd, _truth(rnd, L), sk)
    cols = np.arange(8, L - 60)
    if sk >= 7:
        cols = cols[cols % sk >= K]
    tail = [p for p in range(L - 60, L - 20) if sk < 7 or p % sk >= K][-3:]
    best = _subst(rnd, _subst(rnd, t, rnd.choice(cols, max(4, L // 150), replace=False)), tail)
    others = [_sparse(rnd, t, max(1, L // 600)) for _ in range(n_other)]
    if copy_best:
        others[0] = best.copy()
    return _cluster(rnd, k, pos, best, others)


def _rows(rnd, k, pos, n_other, L=600):
    """n_other + 1 reads, at most 10 per 10-bp bin (--cluster-binsize 10 keeps every read's sequence), four of them at pos, so pos is the
    only mode of the positions and the first of those four is the best read.  The best read is T; at the ladder columns the last m other
    reads (in cluster order) carry X and the first z a third base, so X leads T by d = 2m + z - n_other - 1 for d = 1..4"""
    n = n_other + 1
    mid = n // 20
    positions = []
    for r in range(n):
        b, o = r // 10, r % 10
        positions.append(pos + 10 * (b - mid) + (0 if b == mid and o < 4 else o))
    order = sorted(range(n), key=lambda r: (positions[r], r))
    best_r = order.index(10 * mid)           # the first read at pos in record order
    t = _truth(rnd, L)
    seqs = [t.copy() for _ in range(n)]
    oth = [r for r in order if r != order[best_r]]
    cols = []
    for d, col in zip((1, 2, 3, 4, 3, 2), range(120, 480, 60)):
        z = (n_other + 1 + d) & 1
        m = (n_other + 1 + d - z) // 2
        x = _other(rnd, t[col])
        y = int(rnd.choice([c for c in ACGT if c not in (x, t[col])]))
        for r in oth[len(oth) - m:]:
            seqs[r][col] = x
        for r in oth[:z]:
            seqs[r][col] = y
        cols.append(dict(col=col, d=d, m=m, z=z))
    recs = []
    bi = order[best_r]
    for r in range(n):
        recs.append((0, _read(rnd, positions[r], seqs[r], b"c%02d_r%03d" % (k, r))))
    return recs, dict(L=L, n_other=n_other, best=text(seqs[bi]), best_name="c%02d_r%03d" % (k, bi), ladder=cols, clean=True)


def _tie(rnd, k, pos, L=800):
    """a 2-tie: r1 and r2 at pos, the others 2 bp away (pos stays the median of the position modes); r1 is chosen.  r1 and r2 differ
    where the others split three ways, so whichever is chosen shows in the ALT"""
    t = _truth(rnd, L)
    r1 = _sparse(rnd, t, 4)
    r2 = r1.copy()
    others = [_sparse(rnd, t, 2) for _ in range(3)]
    for col in (200, 333, 500, 650):
        a, b, c = rnd.permutation(ACGT)[:3]
        r1[col], r2[col] = a, b
        others[0][col], others[1][col], others[2][col] = a, b, c
    seqs = [r1, r2] + others
    positions = [pos, pos, pos - 2, pos + 2, pos + 2]
    return _cluster(rnd, k, pos, seqs[0], seqs[1:], positions=positions)


def _alphabet(rnd, k, pos, where, L=700):
    """'=', N and IUPAC codes in the best read, in the others, or in both"""
    t = _truth(rnd, L)
    best = _sparse(rnd, t, 5)
    others = [_sparse(rnd, t, 1) for _ in range(4 if where == "both" else 5)]
    cols = list(range(100, 620, 40))
    odd = [0, 15, 5, 10, 3, 12, 6, 9, 7, 11, 13, 14, 15]
    for col, code in zip(cols, odd):
        if where in ("best", "both"):
            best[col] = code
        if where in ("others", "both"):
            for o in others:                         # the other reads agree on the code: it wins over a one-hot best base
                o[col] = code
    if where == "both":
        # the best read holds R (A|G): three others say A, one C.  Counted as a code, R keeps the column (A 3, R 1, C 1); counted by
        # its bits it would tip it to A (A 4, G 1, C 1)
        for col in (140 + 2, 300 + 2, 460 + 2):
            best[col] = 5
            for o in others[:3]:
                o[col] = A
            others[3][col] = C
    return _cluster(rnd, k, pos, best, others)


def _repeat(rnd, k, pos, mode, L=600):
    """low complexity: 'part' a 100-bp stretch of a period-4 repeat (its strided k-mers are one taboo k-mer), 'all' the whole insertion
    one repeat (no anchor at all), 'period3' a period-3 repeat (three taboo k-mers, no anchor)"""
    t = _truth(rnd, L)
    if mode == "part":
        t[200:300] = np.tile([A, C, G, T], 25)
    elif mode == "all":
        t = np.tile([A, C, G, T], L // 4).astype(np.uint8)
    else:
        t = np.tile([A, G, T], L // 3).astype(np.uint8)
    best = _sparse(rnd, t, 4) if mode == "part" else t.copy()
    others = [_sparse(rnd, t, 1) for _ in range(5)]
    return _cluster(rnd, k, pos, best, others)


def _merged(rnd, k, pos, best_merged, L=301):
    """reads whose insertion is two I ops a few M apart (merge_inner joins them), with odd and even query offsets and odd l_seq"""
    t = _truth(rnd, L)
    best = _sparse(rnd, t, 3)
    others = [_sparse(rnd, t, 1) for _ in range(5)]          # three merged reads and three single: 9 leads in the bin, all keep their sequence
    seqs = [best] + others
    pieces, clips = [], []
    for r in range(len(seqs)):
        merged = (r % 2 == 0) == best_merged
        pieces.append((120 + r, 3 + (r % 4)) if merged else None)
        clips.append(r % 3)
    return _cluster(rnd, k, pos, best, others, pieces=pieces, clips=clips)


def _votes(rnd, k, pos, L=600):
    """top-two differences 2, 3 and 4 among seven others (m carry X, z a third base: X m, the best read's base 8 - m - z, the third z), and
    columns with one and two aligned rows (a read whose first anchors are spoiled has dashes before its first anchor): columns 0..3 have
    one row and are not voted, columns 4..11 have two and are voted (2 / maxal 8 is exactly a quarter).  The nal 1 / 2 edge cannot change
    a column: with the best read's base and at most two rows the top two counts differ by at most 2"""
    t = _truth(rnd, L)
    others = [t.copy() for _ in range(7)]
    for col, m, z in ((150, 5, 1), (250, 5, 0), (350, 6, 0), (450, 5, 1), (153, 5, 0), (253, 6, 0)):
        x = _other(rnd, t[col])
        y = int(rnd.choice([c for c in ACGT if c not in (x, t[col])]))
        for o in others[:m]:
            o[col] = x
        for o in others[m:m + z]:
            o[col] = y
    # others[0] keeps its start, others[1] loses the anchor at 0 (first anchor at 4), the rest lose 0, 4 and 8 (first anchor at 12):
    # the columns before 12 have 2 aligned rows (4..11) or 1 (0..3)
    others[1][1] = _other(rnd, t[1])
    for o in others[2:]:
        o[2], o[9] = _other(rnd, t[2]), _other(rnd, t[9])
    return _cluster(rnd, k, pos, t.copy(), others)


def _lead_in(rnd, k, pos):
    """a plain cluster first on the contig: the bin merge never re-tests the first cluster after its first merge, so a many-bin cluster
    must not come first"""
    return _std(rnd, k, pos, 300, n_other=4)


def _bad(rnd, read, t, a, d):
    """spoil the segment between the anchors at a and a + d: every base of a + 6 .. a + d - 1 differs from T"""
    for p in range(a + 6, a + d):
        read[p] = _other(rnd, t[p])


def _quarter(rnd, k, pos, L=600):
    """15 accepted rows (maxal 16); at column c only four rows are aligned (the other eleven have a dashed segment over it) and all four
    carry X: nal / maxal is exactly 0.25, so the column is voted and X (4 against 1) wins"""
    t = _truth(rnd, L)
    c = 300
    others = [t.copy() for _ in range(15)]
    x = _other(rnd, t[c])
    for o in others[:4]:
        o[c] = x
    for o in others[4:]:
        _bad(rnd, o, t, 288, 24)
    # ten reads at pos and six in the next 100-bp bin (at most ten reads of a bin keep their sequence); pos is the only position mode
    return _cluster(rnd, k, pos, t.copy(), others, positions=[pos] * 10 + [pos + 100] * 6, need=range(280, 320, 4))


def _seg_half(rnd, k, pos, L=600):
    """skip 4: between the anchors at a and a + 24 the other reads match the best read at exactly 12 of the 24 compared positions
    (a + 1 .. a + 24), so the segment's identity is exactly 0.5 and it is copied; the run around it is long and passes"""
    t = _truth(rnd, L)
    a = 300
    mis = [a + 6, a + 7, a + 9, a + 12, a + 13, a + 16, a + 17, a + 18, a + 20, a + 21, a + 22, a + 23]
    assert len(mis) == 12
    x = t.copy()
    for p in mis:
        x[p] = _other(rnd, t[p])
    others = [x.copy() for _ in range(4)]
    return _cluster(rnd, k, pos, t.copy(), others, need=range(a - 20, a + 48, 4)), dict(a=a, d=24, matches=12)


def _run_half(rnd, k, pos, L=600):
    """skip 4: a run of one segment (a .. a + 15) between two dashed segments, matching the best read at exactly 8 of its 16 columns
    (identity 0.5, not above it; its segment identity is 0.5 too, so it is copied and then dropped by the run test)"""
    t = _truth(rnd, L)
    a = 300
    x = t.copy()
    _bad(rnd, x, t, a - 16, 16)
    for p in (a + 6, a + 7, a + 8, a + 9, a + 12, a + 13, a + 14, a + 15):
        x[p] = _other(rnd, t[p])
    _bad(rnd, x, t, a + 16, 16)
    others = [x.copy() for _ in range(4)]
    return _cluster(rnd, k, pos, t.copy(), others, need=range(a - 32, a + 48, 4)), dict(a=a, d=16, matches=8)


def _run_abs(rnd, k, pos, ident, L=1200):
    """skip 5: a run of one segment between two dashed segments.  ident 6: the four other reads' run a .. a + 9 matches at its first six
    columns and carries X at the last four (identity 0.6, 6 matches: kept, X wins).  ident 5: two reads have a run a .. a + 4 that matches
    at all five columns (identity 1, 5 matches: dropped), four more carry X at a + 1 and a + 3 (X 4 against 1; with the two runs kept
    it would be 4 against 3)"""
    t = _truth(rnd, L)
    a = 600
    if ident == 6:
        x = t.copy()
        _bad(rnd, x, t, a - 15, 15)
        for p in range(a + 6, a + 10):
            x[p] = _other(rnd, t[p])
        _bad(rnd, x, t, a + 10, 15)
        others = [x.copy() for _ in range(4)]
        return _cluster(rnd, k, pos, t.copy(), others, need=range(a - 30, a + 45, 5)), dict(a=a, d=10, matches=6)
    y = t.copy()
    _bad(rnd, y, t, a - 15, 15)
    _bad(rnd, y, t, a + 5, 15)
    x = t.copy()
    for p in (a + 1, a + 3):
        x[p] = _other(rnd, t[p])
    others = [x.copy() for _ in range(4)] + [y.copy(), y.copy()]
    return _cluster(rnd, k, pos, t.copy(), others, need=range(a - 30, a + 45, 5)), dict(a=a, d=5, matches=5)


def _span(rnd, k, pos, last, L=500):
    """skip 4: four other reads follow T up to their anchor at `last` and are unrelated after it, so the row's span is `last` (100:
    span / L exactly 0.2, not above it: rejected; 104: accepted).  They carry X at columns 50 and 70, which wins only when they count"""
    t = _truth(rnd, L)
    x = t.copy()
    for p in range(last + 6, L):
        x[p] = _other(rnd, t[p])
    for p in (50, 70):
        x[p] = _other(rnd, t[p])
    others = [x.copy() for _ in range(4)]
    return _cluster(rnd, k, pos, t.copy(), others, need=range(0, last + 1, 4)), dict(span=last)


# ---------------------------------------------------------------- cases

def _sized(lengths, **kw):
    return [lambda rnd, k, pos, L=L: _std(rnd, k, pos, L, **kw) for L in lengths]


def _with(fn, *a):
    """a kind whose builder returns ((records, meta), extra): the extra facts go into meta"""
    def f(rnd, k, pos):
        (recs, meta), extra = fn(rnd, k, pos, *a)
        meta.update(extra)
        return recs, meta
    return f


CASES = {
    # name: (seed, cluster builders, extra CLI args, family)
    "heavy_l": (101, [lambda rnd, k, pos, L=L: _std(rnd, k, pos, L, copy_best=True) for L in (2999, 3000, 3001)], (), "HEAVY_L"),
    "vote_tiles": (102, _sized((4095, 4096, 4097, 8193), n_other=4), (), "vote tiles"),
    "segments_g": (103, _sized((4999, 5000), n_other=4), (), "segments_pass<1> / <8>"),
    "skip_500": (104, _sized((499, 500, 501)), (), "skip"),
    "min_reads": (105, [lambda rnd, k, pos, n=n: _std(rnd, k, pos, 900, n_other=n) for n in (3, 4)], (), "consensus_min_reads"),
    "rows_247_249": (106, [_lead_in] + [lambda rnd, k, pos, n=n: _rows(rnd, k, pos, n) for n in (247, 248, 249)], ("--cluster-binsize", "10"), "rows"),
    "rows_256_257": (107, [_lead_in] + [lambda rnd, k, pos, n=n: _rows(rnd, k, pos, n) for n in (256, 257)], ("--cluster-binsize", "10"), "rows"),
    "best_tie": (108, [_tie], (), "best-read tie"),
    "alphabet": (109, [lambda rnd, k, pos, w=w: _alphabet(rnd, k, pos, w) for w in ("best", "others", "both")], (), "alphabet"),
    "low_complexity": (110, [lambda rnd, k, pos, m=m: _repeat(rnd, k, pos, m) for m in ("part", "all", "period3")], (), "taboo anchors"),
    "merged_leads": (111, [lambda rnd, k, pos, b=b: _merged(rnd, k, pos, b) for b in (True, False)], (), "merged leads"),
    "vote_thresholds": (112, [_votes, _quarter], (), "vote thresholds"),
    "identity": (113, [_with(_seg_half), _with(_run_half), _with(_run_abs, 5), _with(_run_abs, 6)], (), "identity thresholds"),
    "span": (114, [_with(_span, 100), _with(_span, 104)], (), "span"),
}


def clusters(name):
    """[(records, meta)] of case `name`, one per cluster"""
    seed, kinds, _, _ = CASES[name]
    rnd = np.random.default_rng(seed)
    out = []
    for k, fn in enumerate(kinds):
        for _ in range(50):                # redrawn until no planted edit makes an anchor of its own
            r, m = fn(rnd, k, SPACING * (k + 1))
            if m.pop("clean"):
                break
        else:
            raise AssertionError(f"{name}: cluster {k} keeps a stray anchor")
        out.append((r, m))
    return out


def build(name):
    """(block, [cluster meta], CLI args) of case `name`"""
    cl = clusters(name)
    contigs = [("ctgA", SPACING * (len(cl) + 2))]
    return _block(contigs, [x for r, _ in cl for x in r]), [m for _, m in cl], NOQC + tuple(CASES[name][2])


def insertion(rec, L):
    """the insertion of a record built here, as codes (the pieces of a split insertion joined)"""
    s = rec["seq"]
    q = np.empty(2 * len(s), np.uint8)
    q[0::2], q[1::2] = s >> 4, s & 15
    cig = [(int(x) & 15, int(x) >> 4) for x in rec["cigar"]]
    out, o = [], 0
    for op, n in cig:
        if op == 1:
            out.append(q[o:o + n])
        o += n
    return np.concatenate(out)[:L]


def digest(blk):
    h = hashlib.sha256()
    for a in (blk.rec, blk.cigar, blk.var, blk.seq, blk.task, blk.tr):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def alt_digest(s):
    return hashlib.sha256(s.encode()).hexdigest()[:24]
