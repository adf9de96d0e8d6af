"""Test infrastructure: snfb_load_bam's pipeline replayed on the CPU with the one-lane host build of sniffles_b200/csrc/ingest_core.h
(tests/native/ingest_host.cpp) — the same DEFLATE decoder, record decoder and CIGAR16 converter the CUDA kernels instantiate with 32
lanes.  Lets the index / span logic of bamio.device_input and the decoders be checked without a GPU; the GPU tests compare the real
library with the host reader."""
import ctypes as C
import os
import subprocess

import numpy as np

from sniffles_b200 import abi, bamio

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "native", "ingest_host.cpp")
_SO = os.path.join(_HERE, "native", "libingest_host.so")
_CORE = [os.path.join(os.path.dirname(_HERE), "sniffles_b200", "csrc", f) for f in ("ingest_core.h", "cigar16.h")]
_L = None

RAWREC_DTYPE = np.dtype([("body", "<u8"), ("cig_src", "<u8"), ("seq_src", "<u8"), ("sa_src", "<u8"), ("body_len", "<u4"), ("n_cig", "<u4"), ("sa_len", "<u4"),
                         ("ref_id", "<i4"), ("pos", "<i4"), ("l_seq", "<i4"), ("nm", "<i4"), ("ps", "<i4"), ("task", "<u4"), ("flag", "<u2"), ("mapq", "u1"), ("aux_flags", "u1"),
                         ("hp", "u1"), ("l_qname", "u1"), ("status", "u1"), ("_pad", "u1", 5)])


def lib():
    global _L
    if _L is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(p) for p in [_SRC, *_CORE]):
            subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-Wall", "-o", _SO, _SRC])
        L = C.CDLL(_SO)
        L.ingest_host_inflate.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32)]
        L.ingest_host_sizeof_rawrec.restype = C.c_uint64
        L.ingest_host_parse.restype = C.c_int64
        L.ingest_host_parse.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64]
        L.ingest_host_c16.restype = C.c_int64
        L.ingest_host_c16.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint32, C.POINTER(C.c_int64)]
        assert L.ingest_host_sizeof_rawrec() == RAWREC_DTYPE.itemsize
        _L = L
    return _L


def inflate(comp: bytes, n_out: int, lead: int = 0):
    """raw DEFLATE -> (rc, bytes); `lead` junk bytes in front of the stream exercise the unaligned start"""
    buf = np.frombuffer(b"\xa5" * lead + comp + b"\0" * 16, "u1").copy()
    out = np.zeros(n_out + 8, "u1")
    ol = C.c_uint32(0)
    rc = lib().ingest_host_inflate(buf.ctypes.data, lead, lead + len(comp), out.ctypes.data, n_out, C.byref(ol))
    return rc, out[:ol.value].tobytes()


def load_bam(bgzf: np.ndarray, spans: np.ndarray, task_table: np.ndarray, evt_min: int = 11):
    """-> list of per-record dicts in output order (what snfb_load_bam packs), fields as bamio.decode_record + task + cigar16"""
    z = bgzf.tobytes()
    blocks = list(bamio.bgzf_members(z))
    starts = [b[0] for b in blocks]
    uoff, raw = [], bytearray()
    for k, (_, po, pl, isz) in enumerate(blocks):
        uoff.append(len(raw))
        rc, d = inflate(z[po:po + pl], isz, lead=k % 4)
        assert rc == 0 and len(d) == isz, (rc, len(d), isz)
        raw += d
    raw_len = len(raw)
    rawa = np.frombuffer(bytes(raw) + b"\0" * 64, "u1").copy()

    def resolve(c, u):
        if c == len(z):
            assert u == 0
            return raw_len
        k = starts.index(c)
        assert u <= blocks[k][3]
        return uoff[k] + u
    L = lib()
    out = []
    for sp in spans:
        ub, ue, t = resolve(int(sp["cbeg"]), int(sp["ubeg"])), resolve(int(sp["cend"]), int(sp["uend"])), int(sp["task"])
        n = L.ingest_host_parse(rawa.ctypes.data, raw_len, ub, ue, None, 0)
        assert n >= 0
        recs = np.zeros(max(n, 1), RAWREC_DTYPE)
        assert L.ingest_host_parse(rawa.ctypes.data, raw_len, ub, ue, recs.ctypes.data, n) == n
        tk = task_table[t]
        for r in recs[:n]:
            assert r["status"] == 0, "malformed record"
            if int(r["ref_id"]) != int(tk["contig"]) or int(r["pos"]) >= int(tk["end"]):
                continue
            ref = C.c_int64(0)
            words = L.ingest_host_c16(rawa.ctypes.data, int(r["cig_src"]), int(r["n_cig"]), None, evt_min, C.byref(ref))
            assert words >= 0
            if int(r["pos"]) + max(ref.value, 1) <= int(tk["start"]):
                continue
            c16 = np.zeros(((words + 7) // 8) * 8, "<u2")
            assert L.ingest_host_c16(rawa.ctypes.data, int(r["cig_src"]), int(r["n_cig"]), c16.ctypes.data, evt_min, C.byref(ref)) == words
            body, lq = int(r["body"]), int(r["l_qname"])
            af = int(r["aux_flags"])
            out.append(dict(task=t, pos=int(r["pos"]), flag=int(r["flag"]), mapq=int(r["mapq"]), l_seq=int(r["l_seq"]), qname=bytes(rawa[body + 32:body + 32 + lq]),
                            cigar=np.frombuffer(rawa[int(r["cig_src"]):int(r["cig_src"]) + 4 * int(r["n_cig"])].tobytes(), "<u4"),
                            seq=rawa[int(r["seq_src"]):int(r["seq_src"]) + (int(r["l_seq"]) + 1) // 2].copy(), cigar16=c16, n_words=int(words),
                            nm=int(r["nm"]) if af & abi.AUX_NM else None, hp=int(r["hp"]) if af & abi.AUX_HP else None, ps=int(r["ps"]) if af & abi.AUX_PS else None,
                            sa=bytes(rawa[int(r["sa_src"]):int(r["sa_src"]) + int(r["sa_len"])]) if af & abi.AUX_SA else None))
    return out
