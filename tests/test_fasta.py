"""The host side of --reference (sniffles_b200/fasta.py, vcf.reference_intervals) without a GPU: the .fai parser and in-memory builder,
the BGZF member-to-contig plan, pysam's fetch rules, and the intervals a call set needs.  The device is stood in for by `HostCtx`, a
numpy restatement of snfb_load_reference / snfb_fetch_reference."""
import copy
import io
import json
import os
import zlib

import numpy as np
import pytest

from sniffles_b200 import abi, bamio, fasta, vcf
from sniffles_b200 import config as sconfig
import ref_fasta

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "golden.json")


def unwrap(raw, row):
    """newline-free bases of one contig by its .fai geometry (the kernel's formula)"""
    L, lb, lw = int(row["length"]), int(row["linebases"]), int(row["linewidth"])
    p = np.arange(L, dtype=np.int64)
    return np.asarray(raw, "u1")[int(row["offset"]) + (p // max(lb, 1)) * lw + p % max(lb, 1)].tobytes() if L else b""


class HostCtx:
    """numpy stand-in for binding.Context's reference calls"""

    def load_reference(self, data, table, is_bgzf=False):
        raw = np.frombuffer(bytes(data), "u1")
        if is_bgzf:
            raw = np.frombuffer(b"".join(zlib.decompress(bytes(data[po:po + pl]), -15) for _, po, pl, _ in bamio.bgzf_members(bytes(data))), "u1")
        self.seqs = [unwrap(raw, r) for r in table]
        runs = [ref_fasta.n_runs(s) for s in self.seqs]
        off = np.concatenate(([0], np.cumsum([len(r) for r in runs]))).astype("<u8")
        return (np.concatenate(runs) if runs else np.zeros((0, 2), "<i4")), off

    def fetch_reference(self, q):
        out = np.zeros(int((q["out_off"] + q["length"]).max()) if len(q) else 0, "u1")
        for r in q:
            s = self.seqs[int(r["contig"])][int(r["start"]):int(r["start"]) + int(r["length"])]
            assert len(s) == int(r["length"])
            out[int(r["out_off"]):int(r["out_off"]) + len(s)] = np.frombuffer(s, "u1")
        return out


def seqs_for(seed, lengths):
    return ref_fasta.genome(seed, [(f"s{k}", L) for k, L in enumerate(lengths)])


# ---------------------------------------------------------------------------------------------------------------- .fai
@pytest.mark.parametrize("crlf", [False, True])
def test_fai_build_matches_htslib_layout_every_width(crlf):
    for width in range(1, 131):
        lengths = [3 * width, 3 * width + 1, width - 1 if width > 1 else 1, 0, 2 * width + width // 2, 1]     # last line full, short, one line, empty
        seqs = seqs_for(width, lengths)
        text = ref_fasta.fasta_text(seqs, width=width, crlf=crlf)
        names, rows = fasta.build_fai(text)
        want_names, want = fasta.parse_fai(ref_fasta.fai_text(seqs, width=width, crlf=crlf).decode())
        assert names == want_names == [n for n, _ in seqs]
        for a, b in zip(rows, want):
            if int(b["length"]) == 0:
                assert int(a["length"]) == 0
                continue
            assert tuple(a) == tuple(b), (width, crlf, a, b)
        for (n, s), r in zip(seqs, rows):
            assert unwrap(np.frombuffer(text, "u1"), r) == s


def test_fai_build_without_final_newline_and_with_trailing_blank_line():
    seqs = seqs_for(5, [125, 60])
    text = ref_fasta.fasta_text(seqs, last_newline=False)
    names, rows = fasta.build_fai(text)
    assert [int(x) for x in rows["length"]] == [125, 60]
    assert unwrap(np.frombuffer(text, "u1"), rows[1]) == seqs[1][1]
    text2 = ref_fasta.fasta_text(seqs[:1]).replace(b"\n>", b"\n\n>") + b"\n"
    names, rows = fasta.build_fai(text2)
    assert int(rows["length"][0]) == 125


def test_fai_errors():
    with pytest.raises(fasta.ReferenceError, match="different line length in sequence 'b'"):
        fasta.build_fai(b">a\nACGT\nAC\n>b\nACGT\nACG\nACGT\n")
    with pytest.raises(fasta.ReferenceError, match="different line length in sequence 'a'"):
        fasta.build_fai(b">a x\nACG\nACGT\n")
    with pytest.raises(fasta.ReferenceError, match="duplicate sequence name 'a'"):
        fasta.build_fai(b">a\nACGT\n>a second\nAC\n")
    with pytest.raises(fasta.ReferenceError, match="before the first"):
        fasta.build_fai(b"ACGT\n>a\nAC\n")
    with pytest.raises(fasta.ReferenceError, match="malformed"):
        fasta.parse_fai("a\t10\t3\n")
    with pytest.raises(fasta.ReferenceError, match="duplicate"):
        fasta.parse_fai("a\t1\t3\t1\t2\na\t1\t8\t1\t2\n")
    names, rows = fasta.build_fai(b">chr1 description here\tx\nAC\n")
    assert names == ["chr1"] and tuple(rows[0]) == (2, 25, 2, 3)


def test_refuses_plain_gzip_and_bgzf_without_fai(tmp_path):
    seqs = seqs_for(3, [500])
    text = ref_fasta.fasta_text(seqs)
    p = tmp_path / "x.fa.gz"
    import gzip
    p.write_bytes(gzip.compress(text))
    with pytest.raises(fasta.ReferenceError, match="gzip, not BGZF"):
        fasta.Reference(str(p), HostCtx())
    q = tmp_path / "y.fa.gz"
    q.write_bytes(bamio._bgzf_block(text) + bamio._BGZF_EOF)
    with pytest.raises(fasta.ReferenceError, match=r"y\.fa\.gz\.fai is missing"):
        fasta.Reference(str(q), HostCtx())


# ---------------------------------------------------------------------------------------------------------------- BGZF plan
@pytest.mark.parametrize("block", [777, 4096, 0xff00])
def test_bgzf_members_map_to_contigs(block):
    seqs = seqs_for(11, [70_000, 0, 1, 3_000, 140_000])
    text = ref_fasta.fasta_text(seqs)
    names, rows = fasta.parse_fai(ref_fasta.fai_text(seqs).decode())
    z = b"".join(bamio._bgzf_block(text[k:k + block]) for k in range(0, len(text), block)) + bamio._BGZF_EOF
    for pick in ([0, 1, 2, 3, 4], [3], [4, 0], [1], [2, 4]):
        spans = [(int(rows[k]["offset"]), fasta._raw_end(rows[k])) for k in pick]
        shipped, offs = fasta.bgzf_plan(z, spans)
        raw = b"".join(zlib.decompress(shipped[po:po + pl], -15) for _, po, pl, _ in bamio.bgzf_members(shipped))
        nmem = sum(1 for _ in bamio.bgzf_members(shipped))
        need = sum(1 for _, _, _, isz in bamio.bgzf_members(z) if isz) if pick == [0, 1, 2, 3, 4] else None
        if need is not None:
            assert nmem == need
        for k, o in zip(pick, offs):
            r = rows[k].copy()
            r["offset"] = o
            assert unwrap(np.frombuffer(raw, "u1"), r) == seqs[k][1]
        if pick == [3]:
            assert nmem < sum(1 for _ in bamio.bgzf_members(z)) - 1          # only the members of the picked contig travel


# ---------------------------------------------------------------------------------------------------------------- fetch rules
def test_fetch_resolution_against_slicing(tmp_path):
    seqs = seqs_for(21, [5_000, 1, 0, 61, 120, 9_999])
    path = tmp_path / "r.fa"
    path.write_bytes(ref_fasta.fasta_text(seqs, width=61))          # no .fai: indexed in memory
    ref = fasta.Reference(str(path), HostCtx())
    assert ref.references == tuple(n for n, _ in seqs) and ref.lengths == tuple(len(s) for _, s in seqs)
    assert not os.path.exists(str(path) + ".fai")
    d = dict(seqs)
    rng = np.random.default_rng(5)
    edge = [(None, None), (0, 0), (3, 3), (0, 1), (-1, 5), (5, 4), (0, 10 ** 9), (10 ** 9, 10 ** 9 + 5), (10 ** 9, 10), (59, 62), (60, 61)]
    cases = []
    for _ in range(10_000):
        name = seqs[int(rng.integers(0, len(seqs)))][0]
        L = len(d[name])
        if rng.random() < 0.1:
            s, e = edge[int(rng.integers(0, len(edge)))]
        else:
            s = int(rng.integers(-2, L + 3)); e = s + int(rng.integers(-2, 200))
        cases.append((name, s, e))
    cases += [("missing", 0, 1)]
    half = cases[::2]
    ref.prefetch(half + [("missing", 0, 1), ("s0", -1, 3)])
    for name, s, e in cases:
        if name not in d:
            with pytest.raises(KeyError):
                ref.fetch(name, s, e)
            continue
        seq = d[name].decode()
        if s is not None and (s < 0 or (e is not None and s > e)):
            with pytest.raises(ValueError):
                ref.fetch(name, s, e)
            continue
        assert ref.fetch(name, s, e) == seq[(s or 0):(len(seq) if e is None else e)], (name, s, e)
    assert ref.fetch("s0") == d["s0"].decode()


def test_task_runs_follow_the_references_mask_rules(tmp_path, caplog):
    seqs = seqs_for(8, [50_000, 30_000])
    path = tmp_path / "r.fa"
    path.write_bytes(ref_fasta.fasta_text(seqs))
    ref = fasta.Reference(str(path), HostCtx())
    assert np.array_equal(ref.task_runs("s0", 0, 49_999), ref_fasta.n_runs(seqs[0][1]))
    assert np.array_equal(ref.task_runs("s1", 0, 30_000), ref_fasta.n_runs(seqs[1][1]))     # FASTA at least as long as the region: masked
    with caplog.at_level("WARNING"):
        assert ref.task_runs("s1", 0, 30_001) is None                                    # shorter than the region: unmasked
        assert ref.task_runs("chrZ", 0, 10) is None                                      # missing: unmasked
    assert sum("Unable to mask N regions in coverage vector" in r.message for r in caplog.records) == 2


# ---------------------------------------------------------------------------------------------------------------- call sets
class Recorder:
    def __init__(self):
        self.asked = []

    def fetch(self, contig, start=None, end=None):
        self.asked.append((contig, start, end))
        if start is None or end is None or start < 0 or end < start:
            raise ValueError("bad interval")
        return ("ACGTN" * (1 + (end - start) // 5))[:end - start]


@pytest.mark.parametrize("name", sorted(ref_fasta.GOLDEN_FASTA))
def test_reference_intervals_cover_every_fetch(name):
    import oracle.oracle as orc
    from test_oracle_golden import load_fixture
    from test_vcf import final_calls
    with open(GOLDEN) as f:
        gold = json.load(f)["blocks"][name]
    fx, blk = load_fixture(name)
    n = 0
    for key, entry in gold["args"].items():
        cfg = sconfig.default_config(*entry["argv"])
        res = orc.run(blk, abi.Config.from_sniffles(cfg), 3, 2, keep_rec_nm=True)
        for t in range(len(blk.task)):
            calls = final_calls(fx, blk, res, cfg, t)
            want = set(vcf.reference_intervals(calls, cfg))
            rec = Recorder()
            w = vcf.VCFWriter(cfg, io.StringIO(), reference=rec)
            for c in calls:
                w.write_call(copy.deepcopy(c))
            assert set(rec.asked) <= want, set(rec.asked) - want
            n += len(rec.asked)
    assert n > 50


@pytest.mark.parametrize("name", sorted(ref_fasta.GOLDEN_FASTA))
def test_golden_fasta_and_n_run_restatement(name):
    with open(GOLDEN) as f:
        gold = json.load(f)["blocks"][name]
    text, seqs = ref_fasta.golden_fasta(name)
    assert ref_fasta.sha256(text) == gold["fasta_sha256"], "tests/ref_fasta.py no longer writes the FASTA the golden data was made with"
    for cname, s in seqs:
        runs = ref_fasta.n_runs(s)
        mask = np.frombuffer(s, "u1") == 78                       # the reference's `mask == 78`
        got = np.zeros(len(s), bool)
        for a, b in runs:
            got[a:b] = True
        assert np.array_equal(got, mask) and np.all(runs[1:, 0] > runs[:-1, 1])
    lengths = dict((n, len(s)) for n, s in seqs)
    assert 0 in [int(a) for a, _ in ref_fasta.n_runs(seqs[0][1])] and lengths[seqs[0][0]] in [int(b) for _, b in ref_fasta.n_runs(seqs[0][1])]
