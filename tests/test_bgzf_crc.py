"""BGZF CRC-32 without a GPU: the CRC of sniffles_b200/csrc/ingest_core.h (one-lane host build) against zlib at every length and
alignment, the combine step that joins the lanes' slices on the device, and the host reader (bamio) rejecting blocks whose trailer
does not match their data, as htslib does."""
import ctypes as C
import os
import random
import subprocess
import zlib

import numpy as np
import pytest

from sniffles_b200 import bamio, synth

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "native", "crc_host.cpp")


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("crc_host") / "libcrc_host.so")       # built outside the tree: the checkout may be read-only
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-o", so, _SRC])
    lib = C.CDLL(so)
    lib.crc_host_crc32.restype = C.c_uint32
    lib.crc_host_crc32.argtypes = [C.c_void_p, C.c_uint32]
    lib.crc_host_crc32_combine.restype = C.c_uint32
    lib.crc_host_crc32_combine.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    return lib


def _crc(L, buf: np.ndarray, off: int, n: int) -> int:
    return L.crc_host_crc32(buf.ctypes.data + off, n)


def test_crc_equals_zlib_at_every_length_and_alignment(L):
    rnd = random.Random(17)
    buf = np.frombuffer(bytes(rnd.getrandbits(8) for _ in range(65536 + 16)), "u1").copy()
    lengths = list(range(65)) + [4095, 4096, 4097, 65535, 65536] + [rnd.randint(1, 65536) for _ in range(20)]
    for n in lengths:
        for off in range(16):
            assert _crc(L, buf, off, n) == zlib.crc32(buf[off:off + n].tobytes()), (n, off)


def test_combined_slices_equal_crc_of_whole(L):
    rnd = np.random.default_rng(3)
    data = rnd.integers(0, 256, 65536, dtype=np.uint8)
    for trial in range(20):
        cuts = np.sort(rnd.integers(0, len(data) + 1, 15))
        if trial % 2:
            cuts[3:6] = cuts[3]                          # empty slices
        bounds = [0, *cuts.tolist(), len(data)]
        crc = 0
        for a, b in zip(bounds[:-1], bounds[1:]):
            crc = L.crc_host_crc32_combine(crc, _crc(L, data, a, b - a), b - a)
        assert crc == zlib.crc32(data.tobytes()), bounds


def _gf2_shift(crc: int, nbytes: int) -> int:
    """crc times x^(8 nbytes) mod P, by square-and-multiply computed here (independent of the powers table in ingest_core.h)"""
    P = 0xEDB88320

    def mul(a, b):
        p = 0
        for k in range(32):
            if a & (1 << (31 - k)):
                p ^= b
            b = (b >> 1) ^ (P if b & 1 else 0)
        return p
    xn, sq, e = 1 << 31, 1 << (31 - 8), nbytes   # x^0, x^8
    while e:
        if e & 1:
            xn = mul(sq, xn)
        sq, e = mul(sq, sq), e >> 1
    return mul(xn, crc)


def test_combine_over_every_power(L):
    """lengths up to 2^32 - 1 use all 32 precomputed powers; a run of zeros checks the step against zlib directly"""
    rnd = random.Random(5)
    for k in range(32):
        for n in (1 << k, (1 << k) | rnd.getrandbits(k) if k else 1, (1 << (k + 1)) - 1):
            a, b = rnd.getrandbits(32), rnd.getrandbits(32)
            assert L.crc_host_crc32_combine(a, b, n) == _gf2_shift(a, n) ^ b, (k, n)
    a = zlib.crc32(b"abc")
    for n in (1, 7, 1000, 65536, 1 << 20):
        assert L.crc_host_crc32_combine(a, zlib.crc32(bytes(n)), n) == zlib.crc32(bytes(n), a)


@pytest.fixture(scope="module")
def blk():
    return synth.generate(31, [200_000, 120_000], 10.0, len_mean=8000.0, len_sd=2000.0, sv_spacing=6000.0)


def _fetch_all(path, blk):
    f = bamio.BamFile(path)
    try:
        return [r for n in blk.contig_names for r in f.fetch(n, 0, f.get_reference_length(n))]
    finally:
        f.close()


def _data_block(z: bytes):
    """(start, payload offset, payload length, isize) of a record block in the middle of the file"""
    blocks = list(bamio.bgzf_members(z))
    assert len(blocks) > 4
    return blocks[len(blocks) // 2]


def test_fetch_checks_crc(tmp_path, blk):
    path = str(tmp_path / "ok.bam")
    bamio.write_bam(path, blk)
    recs = _fetch_all(path, blk)
    assert [r["pos"] for r in recs] == [int(p) for p in blk.rec["pos"]]
    z = bytearray(open(path, "rb").read())
    start, po, pl, _ = _data_block(bytes(z))
    z[po + pl] ^= 0x10                                    # one bit of the block's CRC field
    bad = str(tmp_path / "bad_crc.bam")
    open(bad, "wb").write(bytes(z))
    open(bad + ".bai", "wb").write(open(path + ".bai", "rb").read())
    with pytest.raises(ValueError, match=f"offset {start}: CRC32 mismatch"):
        _fetch_all(bad, blk)


def test_fetch_rejects_changed_stored_block(tmp_path, blk):
    """level 0: a changed byte of a stored block still inflates to ISIZE bytes; only the CRC tells"""
    path = str(tmp_path / "stored.bam")
    bamio.write_bam(path, blk, level=0)
    assert len(_fetch_all(path, blk)) == len(blk.rec)
    z = bytearray(open(path, "rb").read())
    _, po, pl, isz = _data_block(bytes(z))
    z[po + pl // 2] ^= 0x44
    got = zlib.decompress(bytes(z[po:po + pl]), -15)
    assert len(got) == isz and zlib.crc32(got) != int.from_bytes(z[po + pl:po + pl + 4], "little")
    bad = str(tmp_path / "stored_bad.bam")
    open(bad, "wb").write(bytes(z))
    open(bad + ".bai", "wb").write(open(path + ".bai", "rb").read())
    with pytest.raises(ValueError, match="CRC32 mismatch"):
        _fetch_all(bad, blk)
