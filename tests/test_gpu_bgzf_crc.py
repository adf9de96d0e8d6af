"""The device ingest verifies every BGZF block's CRC-32, as htslib does: valid members pass at every length and output alignment,
each damaged member is reported by index, and a block that still decodes to ISIZE bytes but to different bases (a changed byte of a
stored block) is rejected by snfb_load_bam and by a task, with device ingest and with the host reader."""
import os
import struct
import zlib

import numpy as np
import pytest

from sniffles_b200 import abi, bamio, binding, synth, tasks
from sniffles_b200 import config as sconfig
from test_gpu_ingest import _compare, _device_records

pytestmark = pytest.mark.gpu

HG002 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bams", "hg002.bam")
LENGTHS = [0, 1, 2, 3, 5, 7, 8, 15, 16, 17, 31, 32, 33, 255, 256, 4095, 4096, 4097, 65535, 65536]


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    c.set_config(abi.Config.from_sniffles(sconfig.default_config()))
    yield c
    c.close()


def _member(data: bytes, level: int):
    """one BGZF member with a correct trailer, or None when it would exceed BGZF's 64 KiB block size"""
    try:
        return bamio._bgzf_block(data, level)
    except ValueError:                                   # larger than 65536 bytes
        return None


@pytest.fixture(scope="module")
def members():
    """BGZF members of every length in LENGTHS at levels 0 and 6, back to back, so the blocks land at many output alignments.  A stored
    (level 0) member of 65535 or more bytes exceeds BGZF's 64 KiB block size and is left out."""
    rnd = np.random.default_rng(23)
    out = []
    for n in LENGTHS:
        # random bytes (stored even at level 6) or bases (Huffman-coded); the longest are bases so that level 6 fits a BGZF block
        data = bytes(rnd.choice(np.frombuffer(b"ACGTN", "u1"), n)) if n % 2 or n >= 65535 else rnd.integers(0, 256, n, dtype=np.uint8).tobytes()
        for level in (0, 6):
            m = _member(data, level)
            if m is not None:
                out.append((m, data))
    assert sum(len(d) >= 65535 for _, d in out) == 2 and len(out) == 2 * len(LENGTHS) - 2
    return out


def test_valid_members_pass_at_every_length_and_alignment(ctx, members):
    z = b"".join(m for m, _ in members)
    assert ctx.inflate_bgzf(np.frombuffer(z, "u1")) == b"".join(d for _, d in members)


def _flip_crc(members, bad):
    parts = []
    for j, (m, _) in enumerate(members):
        if j in bad:
            m = bytearray(m)
            m[len(m) - 8 + (j % 4)] ^= 1 << (j % 8)      # one bit of the CRC field
            m = bytes(m)
        parts.append(m)
    return np.frombuffer(b"".join(parts), "u1")


def test_each_bad_member_is_named(ctx, members):
    for j in range(len(members)):
        with pytest.raises(binding.SnfbError, match=rf"inflate: 1 BGZF block\(s\) failed to decode \(first: block {j}, code 10, CRC32 mismatch"):
            ctx.inflate_bgzf(_flip_crc(members, {j}))
    lo, hi = 5, len(members) - 3
    start = sum(len(m) for m, _ in members[:lo])
    with pytest.raises(binding.SnfbError, match=rf"inflate: 2 BGZF block\(s\) failed to decode \(first: block {lo}, code 10, CRC32 mismatch, at byte {start} "):
        ctx.inflate_bgzf(_flip_crc(members, {hi, lo}))
    assert ctx.inflate_bgzf(_flip_crc(members, set())) == b"".join(d for _, d in members)       # the context is still usable


def _equal_zlib_and_host_reader(ctx, path):
    z = open(path, "rb").read()
    want = b"".join(zlib.decompress(z[po:po + pl], -15) for _, po, pl, _ in bamio.bgzf_members(z))
    assert ctx.inflate_bgzf(np.frombuffer(z, "u1")) == want
    f = bamio.BamFile(path)
    regions = [(n, 0, L) for n, L in f.contigs]
    tables = bamio.pack_records(f.contigs, [], [(t, a, b, t) for t, (n, a, b) in enumerate(regions)])
    bgzf, spans = f.device_input(regions)
    _, rec, cig, var, seq = _device_records(ctx, bgzf, spans, tables)
    host, task_of = [], []
    for t, (n, a, b) in enumerate(regions):
        rs = list(f.fetch(n, a, b))
        host += rs
        task_of += [t] * len(rs)
    assert len(host) > 0
    _compare(rec, cig, var, seq, host, task_of)
    f.close()


def test_hg002_and_synthetic_bam_pass(ctx, tmp_path):
    _equal_zlib_and_host_reader(ctx, HG002)
    blk = synth.generate(77, [260_000, 150_000], 14.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=5000.0, phased_frac=0.5)
    path = str(tmp_path / "s.bam")
    bamio.write_bam(path, blk)
    _equal_zlib_and_host_reader(ctx, path)


def _corrupt_one_base(path: str, out: str):
    """Re-emit, at level 0, one block of a level-0 BAM that holds read bases, with one byte of a record's 4-bit sequence changed and
    the block's original CRC trailer kept: the DEFLATE stream, ISIZE and the record chain stay valid.  Returns (block index, contig)."""
    z = open(path, "rb").read()
    blocks = list(bamio.bgzf_members(z))
    raw = [zlib.decompress(z[po:po + pl], -15) for _, po, pl, _ in blocks]
    ubase = np.cumsum([0] + [len(d) for d in raw])
    stream = b"".join(raw)
    f = bamio.BamFile(path)
    v = f.first_record
    off = int(ubase[[b[0] for b in blocks].index(v >> 16)]) + (v & 0xffff)
    f.close()
    while True:                                          # the first record whose bases start in a block of the second half
        bs, ref_id = struct.unpack_from("<ii", stream, off)
        l_rn, n_cig, l_seq = stream[off + 12], struct.unpack_from("<H", stream, off + 16)[0], struct.unpack_from("<i", stream, off + 20)[0]
        s = off + 4 + 32 + l_rn + 4 * n_cig + 10
        k = int(np.searchsorted(ubase, s, side="right")) - 1
        if k >= len(blocks) // 2 and l_seq > 40:
            break
        off += 4 + bs
    data = bytearray(raw[k])
    data[s - int(ubase[k])] ^= 0x33                      # two bases of the read change, every nibble stays a legal base code
    start, po, pl, _ = blocks[k]
    c = zlib.compressobj(0, zlib.DEFLATED, -15)
    comp = c.compress(bytes(data)) + c.flush()
    assert len(comp) == pl                               # same layout: every index offset stays valid
    zz = bytearray(z)
    zz[po:po + pl] = comp
    open(out, "wb").write(bytes(zz))
    open(out + ".bai", "wb").write(open(path + ".bai", "rb").read())
    return k, ref_id


def test_changed_base_in_stored_block_is_rejected(ctx, tmp_path):
    blk = synth.generate(5, [300_000], 12.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=6000.0)
    good = str(tmp_path / "good.bam")
    bamio.write_bam(good, blk, level=0)
    bad = str(tmp_path / "bad.bam")
    k, rid = _corrupt_one_base(good, bad)
    f = bamio.BamFile(bad)
    name, L = f.contigs[rid]
    regions = [(name, 0, L)]
    tables = bamio.pack_records(f.contigs, [], [(rid, 0, L, 0)])
    bgzf, spans = f.device_input(regions)
    f.close()
    with pytest.raises(binding.SnfbError, match=rf"first: block \d+, code 10, CRC32 mismatch"):
        ctx.load_bam(bgzf, spans, tables)
    for device_ingest, err in ((True, binding.SnfbError), (False, ValueError)):
        t = tasks.CallTask(id=0, sv_id=0, contig=name, start=0, end=L, config=sconfig.default_config(), bam=bad, device_ingest=device_ingest)
        with pytest.raises(err, match="CRC32 mismatch"):
            t.execute()
    g = bamio.BamFile(good)                              # the untouched file still loads on the same context
    bgzf, spans = g.device_input(regions)
    assert ctx.load_bam(bgzf, spans, tables)["n_rec"] == len(blk.rec)
    g.close()
