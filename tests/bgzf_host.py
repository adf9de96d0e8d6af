"""Test helpers for the BGZF encoder: the one-thread g++ build of sniffles_b200/csrc/deflate_core.h (tests/native/deflate_host.cpp) as a
`compress(bytes) -> (members, coffsets)` callable with the signature of binding.Context.deflate_bgzf, the fixture VCF text, and the
inputs both the CPU and the GPU tests compress."""
import ctypes as C
import glob
import json
import os
import random
import subprocess
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "deflate_host.cpp")
BLOCK = 0xff00


def build(dirpath):
    so = os.path.join(str(dirpath), "libdeflate_host.so")      # built outside the tree: the checkout may be read-only
    subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-o", so, SRC])
    lib = C.CDLL(so)
    lib.deflate_host_bgzf.restype = C.c_int64
    lib.deflate_host_bgzf.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]

    def compress(data):
        data = bytes(data)
        nb = (len(data) + BLOCK - 1) // BLOCK
        src = np.frombuffer(data + b"\0", "u1")
        out = np.empty(max(nb * 65536, 1), "u1")
        coff = np.zeros(max(nb, 1), "<u8")
        n = lib.deflate_host_bgzf(src.ctypes.data, len(data), out.ctypes.data, len(out), coff.ctypes.data)
        assert n >= 0
        return out[:n].tobytes(), [int(x) for x in coff[:nb]]
    return compress


def fixture_vcf_lines():
    """every `vcf` and `vcf_ref` line of the golden fixtures (the reference writer's output)"""
    lines = []
    for p in sorted(glob.glob(os.path.join(HERE, "golden", "*.json"))):
        with open(p) as f:
            d = json.load(f)
        if isinstance(d, dict) and isinstance(d.get("tasks"), list):
            for t in d["tasks"]:
                lines += t.get("vcf", []) + t.get("vcf_ref", [])
    return lines


def fixture_vcf_text() -> bytes:
    return ("\n".join(fixture_vcf_lines()) + "\n").encode()


def tiled_vcf_text(n_bytes: int, seed: int) -> bytes:
    """at least n_bytes of fixture VCF lines tiled with seeded POS shifts (a large VCF of realistic lines)"""
    rnd = random.Random(seed)
    rows = [l.split("\t") for l in fixture_vcf_lines()]
    out, n, shift = [], 0, 0
    while n < n_bytes:
        for f in rows:
            line = "\t".join([f[0], str(int(f[1]) + shift + rnd.randrange(1000))] + f[2:]) + "\n"
            out.append(line)
            n += len(line)
        shift += 10_000_000
    return "".join(out).encode()


def near_window_text(seed=11, n=200_000) -> bytes:
    """random 64-byte phrases repeated at distances just below, at and above 32 KiB"""
    rnd = random.Random(seed)
    out = bytearray(rnd.getrandbits(8) for _ in range(40_000))
    while len(out) < n:
        d = rnd.choice((32_700, 32_767, 32_768, 32_769, 32_800))
        src = len(out) - d
        out += out[src:src + 64] + bytes(rnd.getrandbits(8) for _ in range(rnd.randrange(1, 300)))
    return bytes(out[:n])


def inputs():
    """name -> bytes: the block-size edge cases, random bytes (stored blocks), one repeated byte (distance-1 matches of 258), repeats near
    the 32 KiB window, and the fixture VCF text"""
    rnd = np.random.default_rng(5)
    text = fixture_vcf_text()
    return {"empty": b"", "one": b"A", "block": text[:BLOCK], "block+1": text[:BLOCK + 1],
            "random": rnd.integers(0, 256, 3 * BLOCK + 777, dtype=np.uint8).tobytes(), "repeat": b"\x07" * (2 * BLOCK + 4321),
            "window": near_window_text(), "vcf": text}


def members(z: bytes, coffsets):
    """the members of a compressed buffer, cut at the given offsets"""
    ends = list(coffsets[1:]) + [len(z)]
    return [z[a:b] for a, b in zip(coffsets, ends)]


def zlib_bgzf_size(data: bytes, level: int) -> int:
    """total size of zlib-compressed BGZF members of the same 0xff00 split (18-byte header + 8-byte trailer each)"""
    total = 0
    for k in range(0, len(data), BLOCK):
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        total += len(c.compress(data[k:k + BLOCK]) + c.flush()) + 26
    return total
