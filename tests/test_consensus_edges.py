"""Stage C's edges on the CPU: the case blocks of tests/consensus_common.py rebuild the blocks the reference ran on
(tests/golden/consensus/expected.json, made by tests/golden/make_consensus_golden.py), the oracle's calls and ALTs equal the reference's,
and what the reference logged while building each consensus shows that the case reaches the edge it is built for."""
import json
import os

import numpy as np
import pytest

import consensus_common as cc
import oracle.oracle as orc
from sniffles_b200 import abi
from sniffles_b200 import config as sconfig

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "consensus", "expected.json")
SVTYPE = {0: "INS", 1: "DEL", 2: "DUP", 3: "INV", 4: "BND"}


def golden():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def calls(res):
    """[svtype, pos, svlen, ALT length, ALT digest] per candidate, as the golden data stores the reference's"""
    out = []
    for i, c in enumerate(res.cand):
        alt = res.alt_of(i) if int(c["alt_len"]) > 0 else ""
        out.append([SVTYPE[int(c["svtype"])], int(c["pos"]), int(c["svlen"]), len(alt), cc.alt_digest(alt)])
    return out


def votes(entry):
    """[(nal, t0, t1, changed)] of one consensus"""
    return [tuple(int(x) for x in k.split(",")) for k in entry["votes"]]


def oracle_alts(name):
    blk, metas, args = cc.build(name)
    res = orc.run(blk, abi.Config.from_sniffles(sconfig.default_config(*args)), 3, 1)
    return [res.alt_of(i) for i in range(len(res.cand))], metas


@pytest.fixture(scope="module")
def gold():
    return golden()


@pytest.mark.parametrize("name", sorted(cc.CASES))
def test_oracle_matches_reference(name, gold):
    g = gold[name]
    blk, _, args = cc.build(name)
    assert cc.digest(blk) == g["digest"], "tests/consensus_common.py no longer builds the block the golden data was made from"
    assert list(args) == g["args"]
    res = orc.run(blk, abi.Config.from_sniffles(sconfig.default_config(*args)), 3, 1)
    got = calls(res)
    assert len(got) == len(g["calls"])
    for i, (a, b) in enumerate(zip(got, g["calls"])):
        assert a == b, f"call {i}: oracle {a} != reference {b}"


def _by_best(entries, metas):
    """the reference's consensus log entry of each cluster (None: the cluster's ALT is its best read)"""
    by = {e["best"]: e for e in entries}
    return [by.get(m["best_name"]) for m in metas]


def _changed(e, diff=None, nal=None):
    return any(c and (diff is None or t0 - t1 == diff) and (nal is None or n == nal) for n, t0, t1, c in votes(e))


def _kept(e, diff):
    return any(not c and t0 - t1 == diff for n, t0, t1, c in votes(e))


def test_evidence_sizes(gold):
    """HEAVY_L, the vote tiles, segments_pass<1> / <8> and the skip steps: L and skip as logged, and the vote corrected every cluster"""
    for name, want in (("heavy_l", [(2999, 8), (3000, 9), (3001, 9)]), ("vote_tiles", [(4095, 11), (4096, 11), (4097, 11), (8193, 19)]),
                       ("segments_g", [(4999, 12), (5000, 13)]), ("skip_500", [(499, 3), (500, 4), (501, 4)])):
        log = gold[name]["consensus"]
        assert [(e["L"], e["skip"]) for e in log] == want, name
        assert all(_changed(e) for e in log), name
    # 2999: the other read equal to the best read finds 375 strided k-mers less the few taboo ones: more than 368 hits of the 384 a warp holds
    for recs, m in cc.clusters("heavy_l"):
        best = np.array([cc.CODE.index(ch) for ch in m["best"]], np.uint8)
        n = len(cc.hits(best, cc.insertion(recs[1][1], m["L"]), cc.skip_of(m["L"])))
        assert n <= 384 and (m["L"] != 2999 or n > 368), (m["L"], n)
    # the vote corrects the best read in the last columns of the first tile (the last 96 it has) and, for 8193, in the last tile (columns
    # 8192..: its only one is past the last anchor, so the corrections lie in the second tile's tail).  The partial tile of 4097 holds
    # column 4096 only, which lies past every row's last anchor: no row reaches it, its ALT byte is the best read's, written by that tile
    # alone (the device's ALT is compared with the golden one byte for byte)
    alts, metas = oracle_alts("vote_tiles")
    for alt, m in zip(alts, metas):
        end = min(m["L"], 4096)
        assert alt[end - 96:end] != m["best"][end - 96:end], m["L"]
        if m["L"] == 4097:
            assert alt[4096] == m["best"][4096]
        if m["L"] == 8193:
            assert alt[8192 - 96:] != m["best"][8192 - 96:]


def test_evidence_min_reads(gold):
    """3 other reads: no consensus, the ALT is the best read; 4: a consensus that changes columns"""
    log = gold["min_reads"]["consensus"]
    alts, metas = oracle_alts("min_reads")
    ent = _by_best(log, metas)
    assert ent[0] is None and alts[0] == metas[0]["best"] and metas[0]["n_other"] == 3
    assert ent[1]["n_other"] == 4 and _changed(ent[1]) and alts[1] != metas[1]["best"]


@pytest.mark.parametrize("name,counts", [("rows_247_249", (247, 248, 249)), ("rows_256_257", (256, 257))])
def test_evidence_rows(name, counts, gold):
    """247 / 248 / 249 / 256 / 257 accepted rows: every other read's row is aligned at the ladder columns (the largest nal is the number
    of other reads, so every row was accepted), and the ladder's columns lead by 2 (kept) and 3 (changed)"""
    log = gold[name]["consensus"]
    _, metas = oracle_alts(name)
    ent = _by_best(log, metas)[1:]
    for e, n in zip(ent, counts):
        assert e["n_other"] == n
        assert max(v[0] for v in votes(e)) == n
        assert _changed(e, 3, n) and _changed(e, 4, n) and _kept(e, 2) and _kept(e, 1)


def test_evidence_tie(gold):
    """two reads tie for the smallest |len - svlen| + 1.5 |start - pos|; the first one is the best read"""
    (e,) = gold["best_tie"]["consensus"]
    call = gold["best_tie"]["calls"][0]
    d = {q: 2 * abs(n - call[2]) + 3 * abs(p - call[1]) for q, n, p in e["leads"]}
    assert e["best"] == "c00_r000" and d["c00_r000"] == d["c00_r001"] == min(d.values())
    assert sorted(d.values())[2] > d["c00_r000"]


def test_evidence_alphabet(gold):
    alts, metas = oracle_alts("alphabet")
    log = _by_best(gold["alphabet"]["consensus"], metas)
    odd = set("=MRSVWYHKDBN")
    assert odd & set(metas[0]["best"]) and odd & set(metas[2]["best"])
    assert not odd & set(alts[0]) and _changed(log[0])                       # the best read's codes voted out by four one-hot reads
    assert odd & set(alts[1]) and not odd & set(metas[1]["best"])          # four reads' codes voted in
    assert all(alts[2][c] == "R" for c in (142, 302, 462)) and _kept(log[2], 2)


def test_evidence_low_complexity(gold):
    alts, metas = oracle_alts("low_complexity")
    log = _by_best(gold["low_complexity"]["consensus"], metas)
    for m, e, alt in zip(metas, log, alts):
        best = np.array([cc.CODE.index(ch) for ch in m["best"]], np.uint8)
        an, taboo = cc.anchors(best, cc.skip_of(m["L"]))
        assert taboo
        if m is metas[0]:
            assert an and _changed(e)
        else:
            assert not an and not votes(e) and alt == m["best"]                # no anchor at all: nothing aligns, the best read stays


def test_evidence_merged_leads(gold):
    """each cluster's best read and other reads come from two I ops joined by merge_inner, at odd and even query offsets"""
    cl = cc.clusters("merged_leads")
    log = _by_best(gold["merged_leads"]["consensus"], [m for _, m in cl])
    def ins_offsets(r):
        out, q = [], 0
        for x in r["cigar"]:
            op, n = int(x) & 15, int(x) >> 4
            if op == 1:
                out.append(q)
            if op in (0, 1, 4):
                q += n
        return out
    for (recs, m), e in zip(cl, log):
        two = [r for _, r in recs if len(ins_offsets(r)) == 2]
        assert len(two) == 3 and all(n == 301 for _, n, _ in e["leads"]) and e["n_other"] == 5
        offs = [o for r in two for o in ins_offsets(r)]
        assert {o & 1 for o in offs[0::2]} == {0, 1} and {o & 1 for o in offs[1::2]} == {0, 1}
        assert any(r["l_seq"] & 1 for r in two) and _changed(e)
    assert len(ins_offsets(cl[0][0][0][1])) == 2 and len(ins_offsets(cl[1][0][0][1])) == 1     # the best read merged, then single


def test_evidence_vote_thresholds(gold):
    log = gold["vote_thresholds"]["consensus"]
    a, b = log
    assert _changed(a, 3) and _kept(a, 2) and _changed(a, 4)
    # columns 4..11: two rows aligned, voted (changes nothing, the rows agree with the best read); columns 0..3 (one row) are not voted
    assert a["votes"].get("2,3,0,0") == 8 and not [v for v in votes(a) if v[0] < 2]
    assert b["n_other"] == 15 and max(v[0] for v in votes(b)) == 15             # 15 accepted rows: maxal 16
    assert (4, 4, 1, 1) in votes(b)                                           # nal 4 = 0.25 maxal: voted, and X wins


def _matches(t, x, lo, hi):
    return int((t[lo:hi] == x[lo:hi]).sum())


def test_evidence_identity(gold):
    """by construction, checked on the reads: the segment at a with identity exactly 12 / 24; the run with 8 / 16; the runs with 5 and 6
    matches.  In the log: X wins where the segment is copied and where the 6-match run stays, and not where the runs are dropped"""
    cl = cc.clusters("identity")
    alts, metas = oracle_alts("identity")
    for (recs, m), alt in zip(cl, alts):
        t = np.array([cc.CODE.index(ch) for ch in m["best"]], np.uint8)
        a, d, sk = m["a"], m["d"], cc.skip_of(m["L"])
        reads = [cc.insertion(r, m["L"]) for _, r in recs[1:]]
        x = reads[-1]
        h = [j for i, j in cc.hits(t, x, sk)]
        assert a in h and a + d in h and not [j for j in h if a < j < a + d]          # one segment between the anchors at a and a + d
        assert _matches(t, x, a + 1, a + d + 1) == m["matches"]                       # the segment's compared positions
        assert _matches(t, x, a, a + d) == m["matches"]                               # the run's columns
        if d != 24:                                                                   # the run is bounded by dashed segments
            before, after = max(j for j in h if j < a), min(j for j in h if j > a + d - 1 and j != a + d)
            assert _matches(t, x, before + 1, a + 1) / (a - before) < 0.5
            assert _matches(t, x, a + d + 1, after + 1) / (after - a - d) < 0.5
    seg, run, five, six = alts
    assert seg != metas[0]["best"] and run == metas[1]["best"] and five != metas[2]["best"] and six != metas[3]["best"]


def test_evidence_span(gold):
    """the four other reads' anchors run from 0 to 100 (span / L exactly 0.2: rejected) and to 104 (accepted)"""
    cl = cc.clusters("span")
    alts, metas = oracle_alts("span")
    log = _by_best(gold["span"]["consensus"], metas)
    for (recs, m), alt, e in zip(cl, alts, log):
        t = np.array([cc.CODE.index(ch) for ch in m["best"]], np.uint8)
        h = cc.hits(t, cc.insertion(recs[1][1], m["L"]), 4)
        assert h[0] == (0, 0) and h[-1] == (m["span"], m["span"])
    assert metas[0]["span"] / metas[0]["L"] == 0.2 and alts[0] == metas[0]["best"] and not votes(log[0])
    assert alts[1] != metas[1]["best"] and _changed(log[1], 3, 4)


def test_every_case_has_evidence():
    """each case above is checked by one of the evidence tests"""
    covered = {"heavy_l", "vote_tiles", "segments_g", "skip_500", "min_reads", "rows_247_249", "rows_256_257", "best_tie", "alphabet",
               "low_complexity", "merged_leads", "vote_thresholds", "identity", "span"}
    assert covered == set(cc.CASES)
