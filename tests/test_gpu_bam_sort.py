"""bamio.sort_bam on the device (snfb_sort_bam) against the host restatement (tests/bam_sort_host.py): shuffled inputs give the restatement's
inflated stream and member sizes, every member checks with zlib, the bytes do not depend on the window and bucket budgets, the sorted file
indexes and calls as the original does, and bad input is refused naming the block or the record."""
import logging
import os
import struct

import numpy as np
import pytest

import bam_index_host as IH
import bam_sort_host as H
import call_sample_common as csc
from sniffles_b200 import bamio, binding, call, synth
from sniffles_b200 import config as sconfig
from sniffles_b200 import index as index_cli
from sniffles_b200 import sort as sort_cli

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    yield c
    c.close()


def _check(ctx, src, out, **budgets):
    """sort_bam(src) -> out equals the restatement's stream and member sizes; every member checks; the EOF marker ends the file"""
    stats = {}
    bamio.sort_bam(src, out, ctx=ctx, stats=stats, **budgets)
    want, sizes = H.sorted_stream(src)
    got = H.members(out)
    assert got[-1][0] == 0 and open(out, "rb").read().endswith(bamio._BGZF_EOF)
    assert b"".join(d for _, d in got) == want
    assert [i for i, _ in got[:-1]] == sizes
    assert stats["n_members"] == len(sizes) and stats["bytes_out"] == os.path.getsize(out)
    return stats


def _record(tid, pos, flag, l_seq, name, rng):
    """one BAM record with its block_size prefix: a match CIGAR of l_seq (none when unmapped), random bases, 0xff qualities"""
    cig = b"" if flag & 4 else struct.pack("<I", (l_seq << 4) | 0)
    q = name.encode() + b"\0"
    end = pos + (l_seq if not flag & 4 else 1)
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(q), 60, bamio.reg2bin(max(pos, 0), max(end, 1)), len(cig) // 4, flag, l_seq, -1, -1, 0) + q + cig \
        + rng.integers(0, 256, (l_seq + 1) // 2, dtype=np.uint8).tobytes() + b"\xff" * l_seq
    return struct.pack("<i", len(body)) + body


def _write(path, text, contigs, recs):
    head = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(contigs)) \
        + b"".join(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln) for n, ln in contigs)
    data = head + b"".join(recs)
    with open(path, "wb") as f:
        u = 0
        for s in H.member_sizes(len(head), [len(r) for r in recs]):
            f.write(bamio._bgzf_block(data[u:u + s]))
            u += s
        f.write(bamio._BGZF_EOF)
    return path


def _synthetic(path, seed=5, n=3000, big=True):
    """ties on (tid, pos) on both strands, placed unmapped reads, unplaced reads with and without a pos, records larger than a member,
    in random order under an unsorted header"""
    rng = np.random.default_rng(seed)
    contigs = [(f"c{k}", 5_000_000) for k in range(5)]
    recs = []
    for j in range(n):
        kind = int(rng.integers(0, 20))
        tid, pos = int(rng.integers(0, 5)), int(rng.integers(0, 200)) * 97       # few positions: many ties
        flag = int(rng.choice([0, 16]))
        l_seq = int(rng.integers(20, 3000))
        if kind == 0:
            flag |= 4                                                           # placed unmapped
        elif kind == 1:
            tid, pos, flag = -1, -1, 4                                          # unplaced, no pos
        elif kind == 2:
            tid, flag = -1, 4                                                   # unplaced with a pos
        elif kind == 3 and big:
            l_seq = int(rng.integers(70_000, 200_000))                          # spans several members
        recs.append(_record(tid, pos, flag, l_seq, f"r{j}", rng))
    rng.shuffle(recs)
    return _write(path, b"@HD\tVN:1.6\tSO:unsorted\n" + b"".join(f"@SQ\tSN:{c}\tLN:{ln}\n".encode() for c, ln in contigs), contigs, recs)


def test_hg008_comes_back_with_htslib_layout(ctx, tmp_path):
    src = IH.hg008_bam(str(tmp_path / "hg008.bam"))
    shuf = H.shuffled_bam(src, str(tmp_path / "shuf.bam"), seed=2, sort_order=b"unsorted")
    out = str(tmp_path / "s.bam")
    _check(ctx, shuf, out)
    got = H.members(out)
    want = H.members(src)
    assert [d for _, d in got] == [d for _, d in want]


@pytest.mark.parametrize("case", ["synthetic", "no_contigs", "header_only", "sorted"])
def test_inputs_match_the_restatement(ctx, tmp_path, case):
    src = str(tmp_path / "in.bam")
    rng = np.random.default_rng(1)
    if case == "synthetic":
        _synthetic(src)
    elif case == "no_contigs":
        recs = [_record(-1, int(rng.integers(-1, 3)), 4, int(rng.integers(10, 400)), f"u{j}", rng) for j in range(200)]
        _write(src, b"", [], recs)
    elif case == "header_only":
        _write(src, b"@HD\tVN:1.6\tSO:queryname\n@SQ\tSN:c0\tLN:100\n", [("c0", 100)], [])
    else:
        _synthetic(str(tmp_path / "raw.bam"), big=False)
        H.write_sorted(str(tmp_path / "raw.bam"), src)
    st = _check(ctx, src, str(tmp_path / "s.bam"))
    if case == "sorted":
        assert [d for _, d in H.members(src)] == [d for _, d in H.members(str(tmp_path / "s.bam"))]
    if case == "header_only":
        assert st["n_records"] == 0 and st["n_buckets"] == 1


def test_budgets_do_not_change_the_bytes(ctx, tmp_path):
    """default budgets, windows of one member (records carried across windows) and >= 8 buckets write the same file"""
    src = _synthetic(str(tmp_path / "in.bam"), seed=8)
    outs = []
    raw = sum(i for i, _ in H.members(src))
    for k, budgets in enumerate(({}, dict(window_bytes=1), dict(bucket_bytes=raw // 12))):
        out = str(tmp_path / f"s{k}.bam")
        st = _check(ctx, src, out, **budgets)
        if "window_bytes" in budgets:
            assert st["n_windows"] == len(H.members(src))
        if "bucket_bytes" in budgets:
            assert st["n_buckets"] >= 8 and st["n_input_reads"] > st["n_windows"] + 1
        outs.append(open(out, "rb").read())
    assert outs[0] == outs[1] == outs[2]


def test_write_index_matches_the_index_tool_and_the_host(tmp_path, caplog):
    src = _synthetic(str(tmp_path / "in.bam"), seed=4)
    out = str(tmp_path / "s.bam")
    assert sort_cli.main([src, "-o", out, "--write-index"]) == 0
    assert sorted(os.listdir(tmp_path)) == ["in.bam", "s.bam", "s.bam.csi"]
    with open(out + ".csi", "rb") as f:
        mine = IH.parse_index(f.read())
    assert index_cli.main([out, "-c", "-o", str(tmp_path / "tool.csi")]) == 0
    with open(str(tmp_path / "tool.csi"), "rb") as f:
        assert IH.parse_index(f.read()) == mine
    assert IH.parse_index(IH.host_index(out, "csi")[0]) == mine


def test_shuffled_golden_bam_calls_as_the_original(tmp_path):
    """a call_sample golden BAM, put in the sort's order by the restatement, indexed and called; then shuffled, sorted on the device with
    --write-index and called: the VCFs are byte-equal"""
    case = "c1_default"
    name = csc.CASES[case][0]
    paths = csc.write_inputs(name, str(tmp_path / "gold"))
    orig = str(tmp_path / "orig.bam")
    H.write_sorted(paths["bam"], orig)
    with open(orig + ".csi", "wb") as f:
        f.write(bamio.build_index(orig, "csi"))
    shuf = H.shuffled_bam(orig, str(tmp_path / "shuf.bam"), seed=9)
    out = str(tmp_path / "sorted.bam")
    assert sort_cli.main([shuf, "-o", out, "--write-index"]) == 0
    assert [d for _, d in H.members(out)] == [d for _, d in H.members(orig)]
    vcfs = []
    for bam in (orig, out):
        vcf = str(tmp_path / (os.path.basename(bam) + ".vcf"))
        cfg = sconfig.default_config(*csc.case_args(case, dict(paths, bam=bam), vcf, str(tmp_path / "x.snf")))
        cfg.input = bam
        call.call_sample(cfg)
        vcfs.append(open(vcf).read())
    assert csc.vcf_digest(vcfs[0]) == csc.vcf_digest(vcfs[1])
    body = [[x for x in v.splitlines() if not x.startswith("##")] for v in vcfs]
    assert body[0] == body[1] and len(body[0]) > 1


def _refusal(path, out, caplog):
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="sniffles_b200.sort"):
        code = sort_cli.main([path, "-o", out, "--write-index"])
    errs = [r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR]
    assert code == 1 and len(errs) == 1 and errs[0].endswith("(Fatal error, exiting.)")
    assert not any(os.path.exists(out + x) for x in ("", ".tmp", ".csi", ".csi.tmp"))
    return errs[0]


def test_bad_input_is_refused(tmp_path, caplog):
    src = _synthetic(str(tmp_path / "src.bam"), seed=6)
    out = str(tmp_path / "s.bam")
    z = open(src, "rb").read()
    starts = [o for o, *_ in bamio.bgzf_members(z)]
    k = len(starts) // 2
    bsize = starts[k + 1] - starts[k]
    bad = bytearray(z)
    bad[starts[k] + bsize - 8] ^= 0x5a                  # the member's CRC-32
    p = str(tmp_path / "crc.bam")
    open(p, "wb").write(bytes(bad))
    assert f"BGZF block at file offset {starts[k]}: CRC32 mismatch" in _refusal(p, out, caplog)
    p = str(tmp_path / "cut.bam")
    open(p, "wb").write(z[:starts[k] + bsize // 2])
    assert f"truncated BGZF block at file offset {starts[k]}" in _refusal(p, out, caplog)
    p = str(tmp_path / "text.bam")
    open(p, "wb").write(b"not a bam\n" * 10)
    assert f"Unable to sort '{p}'" in _refusal(p, out, caplog)
    # a record whose tid is past the header's references: the strict record test refuses it, naming the record before it
    rng = np.random.default_rng(0)
    contigs = [("c0", 1000)]
    recs = [_record(0, 10, 0, 50, "good", rng), _record(3, 10, 0, 50, "bad_tid", rng), _record(0, 5, 0, 50, "after", rng)]
    p = _write(str(tmp_path / "tid.bam"), b"", contigs, recs)
    msg = _refusal(p, out, caplog)
    assert "the record chain breaks after record 'good'" in msg, msg


def test_synth_long_reads(ctx, tmp_path):
    """reads of ~150 kb from the synthetic generator, shuffled: most records span members; many buckets and small windows"""
    blk = synth.generate(11, [3_000_000, 1_200_000], 6.0, len_mean=150_000.0, len_sd=20_000.0, len_min=60_000, len_max=300_000)
    src, _ = bamio.write_bam(str(tmp_path / "long.bam"), blk, qual_seed=11)
    shuf = H.shuffled_bam(src, str(tmp_path / "shuf.bam"), seed=1)
    raw = sum(i for i, _ in H.members(shuf))
    a = _check(ctx, shuf, str(tmp_path / "a.bam"), window_bytes=300_000, bucket_bytes=raw // 10)
    assert a["n_buckets"] >= 8
    _check(ctx, shuf, str(tmp_path / "b.bam"))
    assert open(str(tmp_path / "a.bam"), "rb").read() == open(str(tmp_path / "b.bam"), "rb").read()
