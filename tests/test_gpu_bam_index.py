"""bamio.build_index on the device (snfb_index_bam), BAI and CSI: the two htslib-written CSI fixtures, synthetic BAMs byte for byte against
the host restatement (tests/bam_index_host.py) at the record-boundary, CIGAR, placement and window edges, the built index answering
queries as the original does, every call_sample golden case through a built index, and the refusals of unsorted, truncated and corrupted
input, naming the record or the block."""
import json
import logging
import os
import shutil
import zlib

import numpy as np
import pytest

import bam_index_host as H
import call_sample_common as csc
from sniffles_b200 import bamio, binding, call, synth
from sniffles_b200 import config as sconfig
from sniffles_b200 import index as index_cli

pytestmark = pytest.mark.gpu

BAMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bams")


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    yield c
    c.close()


def _plain(data):
    """an index file with a CSI's BGZF compression undone"""
    if data[:2] != b"\x1f\x8b":
        return data
    out, o = b"", 0
    while o < len(data):
        d = zlib.decompressobj(31)
        out += d.decompress(data[o:])
        o = len(data) - len(d.unused_data)
    return out


def _check_host(ctx, path, fmt, min_shift=14, window=None):
    """the device's index equals the host restatement's byte for byte (the CSI after its compression is undone); returns build stats"""
    stats = {}
    got = bamio.build_index(path, fmt, min_shift, window_bytes=window, ctx=ctx, stats=stats)
    want, tab = H.host_index(path, fmt, min_shift)
    assert _plain(got) == want
    assert stats["n_records"] == tab["n_records"]
    if fmt == "csi":
        assert got.endswith(bamio._BGZF_EOF)
    return stats


@pytest.mark.parametrize("fmt", ["bai", "csi"])
@pytest.mark.parametrize("name", ["hg002", "hg008"])
def test_fixtures_match_htslib(ctx, name, fmt, tmp_path):
    path = H.fixture_bam(name, tmp_path)
    with open(os.path.join(BAMS, name + ".bam.csi"), "rb") as f:
        want = H.parse_index(f.read())
    got = H.parse_index(_plain(bamio.build_index(path, fmt, ctx=ctx)))
    if fmt == "csi":
        assert got["refs"] == want["refs"]
    else:                                   # the same bins and chunks; BAI has no loffsets
        assert [{b: c for b, (_, c) in r.items()} for r in got["refs"]] == [{b: c for b, (_, c) in r.items()} for r in want["refs"]]
    assert got["n_no_coor"] == want["n_no_coor"]
    _check_host(ctx, path, fmt)


def _record(pos, flag, ops, l_seq, name, rng):
    cig = np.array([(n << 4) | o for n, o in ops], "<u4")
    return dict(pos=pos, mapq=60, flag=flag, l_seq=l_seq, qname=name.encode(), cigar=cig,
                seq=rng.integers(0, 256, (l_seq + 1) // 2, dtype=np.uint8), aux={})


def _edge_bam(path, seed=7, n_contig=300):
    """many contigs (every 7th empty), placed unmapped reads, zero-span CIGARs, a CG-escaped CIGAR of 70,000 operations, reads longer than
    a BGZF member, and 30 unplaced reads (reference -1) at the end"""
    rng = np.random.default_rng(seed)
    contigs = [(f"chr{k}", int(rng.integers(60_000, 3_000_000))) for k in range(n_contig)]
    tasks, recs = [], []
    for c, (_, ln) in enumerate(contigs):
        if c % 7 == 3:
            continue
        t = len(tasks)
        tasks.append((c, 0, ln, t))
        for j, pos in enumerate(sorted(int(x) for x in rng.integers(0, ln - 50_000, int(rng.integers(1, 8))))):
            kind = int(rng.integers(0, 10))
            name = f"r{c}_{j}"
            if j == 0 and c % 50 == 1:
                ops = [(1, 0), (1, 1)] * 35_000
                recs.append((t, _record(pos, 0, ops, 70_000, name, rng)))
            elif kind == 0:
                recs.append((t, _record(pos, 4, [], int(rng.integers(50, 3000)), name, rng)))
            elif kind == 1:
                l_seq = int(rng.integers(10, 500))
                recs.append((t, _record(pos, 0, [(l_seq, 4)], l_seq, name, rng)))
            else:
                m = int(rng.integers(500, 20_000))
                clip = int(rng.integers(0, 90_000)) if kind == 3 else 0
                ops = ([(clip, 4)] if clip else []) + [(m // 2, 0), (int(rng.integers(1, 300)), 2), (m - m // 2, 0)]
                recs.append((t, _record(pos, 16 if kind == 4 else 0, ops, clip + m, name, rng)))
    t = len(tasks)
    tasks.append((-1, 0, 1, t))
    for j in range(30):
        recs.append((t, _record(-1, 4, [], 200, f"unplaced{j}", rng)))
    blk = bamio.pack_records(contigs, recs, tasks)
    bamio.write_bam(path, blk, qual_seed=seed)
    return path


@pytest.mark.parametrize("fmt", ["bai", "csi"])
def test_edge_bam_matches_host(ctx, tmp_path, fmt):
    path = _edge_bam(str(tmp_path / "edge.bam"))
    st = _check_host(ctx, path, fmt)
    assert st["n_windows"] >= 1


def _long_read_bam(path, seed=11):
    """reads of ~150 kb with noisy qualities: most records span several BGZF members, and runs of members hold no record start"""
    blk = synth.generate(seed, [3_000_000, 1_200_000], 6.0, len_mean=150_000.0, len_sd=20_000.0, len_min=60_000, len_max=300_000)
    bamio.write_bam(path, blk, qual_seed=seed)
    return path


@pytest.mark.parametrize("fmt,min_shift", [("bai", 14), ("csi", 14), ("csi", 12)])
def test_long_reads_match_host(ctx, tmp_path, fmt, min_shift):
    path = _long_read_bam(str(tmp_path / "long.bam"))
    _check_host(ctx, path, fmt, min_shift)


@pytest.mark.parametrize("window", [70_000, 300_000, 1_000_003])
def test_small_windows_match_host(ctx, tmp_path, window):
    """windows of a few members: records straddle window edges and are carried over, some across several windows"""
    path = _long_read_bam(str(tmp_path / "long.bam"))
    st = _check_host(ctx, path, "bai", window=window)
    assert st["n_windows"] > 3
    edge = _edge_bam(str(tmp_path / "edge.bam"))
    assert _check_host(ctx, edge, "csi", window=window)["n_windows"] > 3


def test_built_index_answers_like_the_original(ctx, tmp_path):
    """BamFile over the built BAI and CSI: the records of merged_chunks that overlap a region, and fetch, as with write_bam's index"""
    blk = synth.generate(5, [2_000_000, 800_000, 1_500_000], 12.0, len_mean=20_000.0, len_sd=5_000.0)
    path, _ = bamio.write_bam(str(tmp_path / "q.bam"), blk, qual_seed=5)
    orig = bamio.BamFile(path, index_path=path + ".bai")
    rng = np.random.default_rng(3)
    for fmt in ("bai", "csi"):
        built = str(tmp_path / f"built.{fmt}")
        with open(built, "wb") as f:
            f.write(bamio.build_index(path, fmt, ctx=ctx))
        new = bamio.BamFile(path, index_path=built)
        for _ in range(60):
            name, ln = orig.contigs[int(rng.integers(0, len(orig.contigs)))]
            a = int(rng.integers(0, ln))
            b = min(ln, a + int(rng.integers(1, 200_000)))

            def overlapping(bam):
                out = set()
                for vb, ve in bam.merged_chunks(name, a, b):
                    for r in bam.records(vb, ve):
                        d = bamio.decode_record(r)
                        if d["ref_id"] == bam.name_to_id[name] and d["pos"] < b and d["pos"] + max(bamio.ref_span(d["cigar"]), 1) > a:
                            out.add((d["qname"], d["pos"]))
                return out
            assert overlapping(new) == overlapping(orig)
            assert [(r["qname"], r["pos"]) for r in new.fetch(name, a, b)] == [(r["qname"], r["pos"]) for r in orig.fetch(name, a, b)]
        new.close()
    orig.close()


with open(csc.EXPECTED) as _f:
    GOLD = json.load(_f)


@pytest.fixture(scope="module")
def inputs(tmp_path_factory, ctx):
    """every call_sample golden input with its index replaced by a BAI built on the device"""
    d = tmp_path_factory.mktemp("indexed_inputs")
    out = {}
    for name in {n for n, _ in csc.CASES.values()}:
        paths = csc.write_inputs(name, str(d / name))
        bam = paths["bam"]
        for ext in (".bai", ".csi"):
            if os.path.exists(bam + ext):
                os.remove(bam + ext)
        with open(bam + ".bai", "wb") as f:
            f.write(bamio.build_index(bam, "bai", ctx=ctx))
        out[name] = paths
    return out


@pytest.mark.parametrize("case", sorted(csc.CASES))
def test_call_sample_through_the_built_index(case, inputs, tmp_path):
    gold = GOLD["cases"][case]
    paths = inputs[gold["input"]]
    args = csc.case_args(case, paths, str(tmp_path / "out.vcf"), str(tmp_path / "out.snf"))
    cfg = sconfig.default_config(*args)
    for k, v in GOLD["stamp"].items():
        setattr(cfg, k, v)
    cfg.input = paths["bam"]
    n = call.call_sample(cfg)
    assert n == gold["n_written"]
    assert cfg.task_read_id_offset_mult == gold["task_read_id_offset_mult"]
    assert csc.vcf_digest((tmp_path / "out.vcf").read_text()) == gold["vcf"]


def _cli_refusal(path, caplog, args=()):
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="sniffles_b200.index"):
        code = index_cli.main([path, *args])
    errs = [r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR]
    assert code == 1 and len(errs) == 1
    assert not os.path.exists(path + ".bai") and not os.path.exists(path + ".csi")
    return errs[0]


def test_unsorted_bam_is_refused(tmp_path, caplog):
    blk = synth.generate(9, [1_000_000], 5.0, len_mean=20_000.0, len_sd=3_000.0)
    rec = blk.rec.copy()
    k = next(i for i in range(len(rec) // 2, len(rec) - 1) if rec[i]["pos"] < rec[i + 1]["pos"])
    rec[[k, k + 1]] = rec[[k + 1, k]]                 # two neighbours swapped (different positions)
    assert rec[k]["pos"] > rec[k + 1]["pos"]
    blk.rec = rec
    path, idx = bamio.write_bam(str(tmp_path / "unsorted.bam"), blk)
    os.remove(idx)
    name = bytes(blk.var[int(rec[k + 1]["var_off"]):int(rec[k + 1]["var_off"]) + int(rec[k + 1]["l_qname"])]).decode()
    for args in ((), ("-c",)):
        msg = _cli_refusal(path, caplog, args)
        assert f"record '{name}' (record {k + 2} of the file" in msg and "unsorted positions on reference #0" in msg, msg


def _members(path):
    with open(path, "rb") as f:
        z = f.read()
    return z, [o for o, *_ in bamio.bgzf_members(z)]


def test_corrupted_and_truncated_bams_are_refused(tmp_path, caplog):
    src = _long_read_bam(str(tmp_path / "src.bam"))
    z, starts = _members(src)
    k = len(starts) // 2
    bsize = starts[k + 1] - starts[k]
    bad = bytearray(z)
    bad[starts[k] + bsize - 8] ^= 0x5a                # the member's CRC-32: it inflates, but does not check
    path = str(tmp_path / "crc.bam")
    with open(path, "wb") as f:
        f.write(bytes(bad))
    msg = _cli_refusal(path, caplog)
    assert f"BGZF block at file offset {starts[k]}: CRC32 mismatch" in msg, msg
    path = str(tmp_path / "cut_member.bam")        # ends inside a member
    with open(path, "wb") as f:
        f.write(z[:starts[k] + bsize // 2])
    msg = _cli_refusal(path, caplog)
    assert f"truncated BGZF block at file offset {starts[k]}" in msg, msg
    path = str(tmp_path / "cut_record.bam")        # ends on a member boundary inside a record
    with open(path, "wb") as f:
        f.write(z[:starts[k]] + bamio._BGZF_EOF)
    msg = _cli_refusal(path, caplog, ("-c",))
    assert "truncated BAM file: the record at virtual offset" in msg, msg
    path = str(tmp_path / "garbage.bam")           # a member whose bytes are not records: the chain breaks, naming the record before
    first_data = starts[1]
    payload = bytes(range(256)) * 200
    with open(path, "wb") as f:
        f.write(z[:first_data] + bamio._bgzf_block(payload) + bamio._BGZF_EOF)
    msg = _cli_refusal(path, caplog)
    assert "not a valid BAM record" in msg or "the record chain breaks" in msg, msg
