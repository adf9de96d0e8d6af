"""Plain-Python restatement of force calling's matching and target coverage (parallel.py:300-347, postprocessing.py:69-130), the
checker of snfb_genotype_targets.  The matching is the reference's loop as written: bins of targets, then the candidates visited in
emission order.  Coverage reads a per-base numpy vector with the reference's indexing, IndexError and leaked `end` included.

Calls and targets are any objects with svtype, pos, svlen and, for a BND, bnd_info.mate_contig / bnd_info.is_first."""
import math

BINSIZE = 5000
BINEDGE = int(BINSIZE / 10)
TYPES = ["INS", "DEL", "DUP", "INV", "BND"]


def match(cands, targets, combine_match, combine_match_max, cluster_merge_bnd):
    """per target: the index into `cands` (emission order of the task) of its match, or -1"""
    best = [(math.inf, -1)] * len(targets)
    bins = {svtype: {} for svtype in TYPES}
    for i, t in enumerate(targets):
        if t.svtype not in bins:
            continue
        bs = [int(t.pos / BINSIZE) * BINSIZE]
        if t.pos % BINSIZE < BINEDGE:
            bs.append((int(t.pos / BINSIZE) - 1) * BINSIZE)
        if t.pos % BINSIZE > BINSIZE - BINEDGE:
            bs.append((int(t.pos / BINSIZE) + 1) * BINSIZE)
        for b in bs:
            bins[t.svtype].setdefault(b, []).append(i)
    for ci, cand in enumerate(cands):
        if cand.svtype.startswith("SINGLE"):
            continue
        b = int(cand.pos / BINSIZE) * BINSIZE
        if b not in bins[cand.svtype]:
            continue
        for i in bins[cand.svtype][b]:
            t = targets[i]
            if cand.svtype == "BND":
                dist = abs(t.pos - cand.pos)
                if dist < best[i][0] and dist <= cluster_merge_bnd and cand.bnd_info.mate_contig == t.bnd_info.mate_contig:
                    best[i] = (dist, ci)
            else:
                dist = abs(t.pos - cand.pos) + abs(abs(t.svlen) - abs(cand.svlen))
                minlen = float(min(abs(t.svlen), abs(cand.svlen)))
                if minlen > 0 and dist < best[i][0] and dist <= combine_match * math.sqrt(minlen) and dist <= combine_match_max:
                    best[i] = (dist, ci)
    return [ci for _, ci in best]


def coverage(targets, cv, coverage_binsize):
    """per target (start, center, end) probes of postprocessing.coverage over the per-base vector cv; raises UnboundLocalError for a
    BND with no earlier non-BND target, as the reference does"""
    out = []
    for t in targets:
        start = t.pos
        if t.svtype == "INS":
            end = start + 1
        elif t.svtype == "BND":
            if t.bnd_info.is_first:
                start -= 1
        else:
            end = t.pos + abs(t.svlen)
        if t.svtype in ("INS", "BND"):
            idx = (start - coverage_binsize, start, end + coverage_binsize)
        else:
            idx = (start, int((start + end) / 2), end - coverage_binsize)
        v = []
        for x in idx:
            try:
                v.append(int(cv[x]))
            except IndexError:
                v.append(0)
        out.append(tuple(v))
    return out


def record_spans(blk):
    """reference span of every record of a packed block (BAM CIGAR words: M, D, N, =, X advance the reference)"""
    import numpy as np
    adv = np.isin(blk.cigar & 15, [0, 2, 3, 7, 8])
    cs = np.concatenate(([0], np.cumsum(np.where(adv, blk.cigar >> 4, 0), dtype=np.int64)))     # records may share or reorder CIGARs
    off = blk.rec["cigar_off"].astype(np.int64)
    return cs[off + blk.rec["n_cigar"].astype(np.int64)] - cs[off]


def coverage_vector(blk, ok, span, t, runs=None):
    """LeadProvider.coverage of task t as a per-base uint16 vector: reads passing the filters (`ok`) over [pos, pos + span).  `runs`:
    reference 'N' runs [(a, b)] of the task; _mask_N_coverage zeroes them inside the task region only (the mask is fetched per region,
    leadprov.py:436-439), and the slice clips to the vector"""
    import numpy as np
    L = int(blk.task[t]["contig_len"])
    sel = ok & (blk.rec["task"] == t)
    s = blk.rec["pos"][sel].astype(np.int64)
    cov = np.zeros(L + 1, np.int64)
    np.add.at(cov, s, 1)
    np.add.at(cov, np.minimum(s + span[sel], L), -1)
    cov = np.cumsum(cov)[:L].astype(np.uint16)
    start, end = int(blk.task[t]["start"]), int(blk.task[t]["end"])
    for a, b in runs or ():
        a, b = max(int(a), start, 0), min(int(b), end, L)
        if a < b:
            cov[a:b] = 0
    return cov


class Sv:
    """a call or target as match() and coverage() read it"""
    def __init__(self, svtype, pos, svlen, is_first=False, mate=None):
        self.svtype, self.pos, self.svlen = svtype, pos, svlen
        self.bnd_info = type("Bnd", (), dict(is_first=bool(is_first), mate_contig=mate))() if svtype == "BND" else None


def cand_svs(cand, contig_names):
    """snfb_cand rows -> Sv (mate contig by name, as the reference compares it)"""
    names = ["INS", "DEL", "DUP", "INV", "BND", "SINGLE_LEFT", "SINGLE_RIGHT"]
    return [Sv(names[int(c["svtype"])], int(c["pos"]), int(c["svlen"]), int(c["bnd_is_first"]),
               contig_names[int(c["bnd_mate_contig"])] if int(c["bnd_mate_contig"]) >= 0 else "?") for c in cand]


def task_results(cand, lo, targets, cv, combine_match, combine_match_max, cluster_merge_bnd, coverage_binsize):
    """what snfb_genotype_targets returns for one task's targets: (match as emission index, cov_start, cov_center, cov_end, bnd_no_prev)"""
    import numpy as np
    n = len(targets)
    m = match(cand, targets, combine_match, combine_match_max, cluster_merge_bnd)
    out = [np.array([lo + x if x >= 0 else -1 for x in m], dtype=np.int64)] + [np.zeros(n, np.int32) for _ in range(4)]
    try:
        cov = coverage(targets, cv, coverage_binsize)
    except UnboundLocalError:
        out[4][:] = 1
        return tuple(out)
    for k in range(3):
        out[1 + k][:] = [c[k] for c in cov]
    return tuple(out)
