"""snfb_deflate_bgzf on the device: byte-identical to the one-thread host build of deflate_core.h on every CPU input and on a 64 MB text
(many waves of thread blocks), inflated back by the library's own CRC-checked snfb_inflate_bgzf and by zlib, member offsets where the
members start, and a .vcf.gz + .tbi written through CallTask, VCFWriter and open_output."""
import copy
import ctypes as C
import gzip

import numpy as np
import pytest

import bgzf_host
from sniffles_b200 import bamio, binding, synth, tasks, vcf
from sniffles_b200 import config as sconfig
from test_bgzf_write import _linear, _query, _text_starts, parse_tbi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return bgzf_host.build(tmp_path_factory.mktemp("deflate_host"))


def _starts(z: bytes):
    return [o for o, *_ in bamio.bgzf_members(z)]


def _check(ctx, host, data):
    z, co = ctx.deflate_bgzf(data)
    assert data == b"" or "deflate" in [n for n, *_ in ctx.timings()]
    assert (z, co) == host(data)
    assert co == _starts(z)
    assert gzip.decompress(z + bamio._BGZF_EOF) == data
    assert ctx.inflate_bgzf(np.frombuffer(z, "u1")) == data if data else z == b""
    return z


@pytest.mark.parametrize("name", ["empty", "one", "block", "block+1", "random", "repeat", "window", "vcf"])
def test_identical_to_host_build(ctx, host, name):
    _check(ctx, host, bgzf_host.inputs()[name])


def test_64mb_text(ctx, host):
    data = bgzf_host.tiled_vcf_text(64 << 20, seed=29)
    assert len(data) >= 64 << 20
    z = _check(ctx, host, data)
    assert all(m[18] & 6 == 4 for m in bgzf_host.members(z, _starts(z))[:-1])        # dynamic Huffman blocks


def test_small_out_cap_is_refused(ctx):
    src = np.frombuffer(b"x" * 70_000, "u1")
    out = np.empty(65536, "u1")
    n = C.c_uint64()
    assert ctx._lib.snfb_deflate_bgzf(ctx._h, src.ctypes.data, len(src), out.ctypes.data, len(out), C.byref(n), None) != 0
    assert b"out_cap" in ctx._lib.snfb_last_error(ctx._h)


def test_call_task_to_indexed_vcf(tmp_path):
    blk = synth.generate(91, [260_000, 150_000], 20.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=6000.0, tr_frac=0.2)
    bam = str(tmp_path / "s.bam")
    bamio.write_bam(bam, blk)
    calls, contigs = [], []
    for t, name in enumerate(blk.contig_names):
        L = int(blk.contig[t]["length"])
        contigs.append((name, L))
        c, _ = tasks.CallTask(id=t, sv_id=0, contig=name, start=0, end=L, config=sconfig.default_config(), bam=bam, device_ingest=True).execute()
        calls += sorted(c, key=lambda x: x.pos)
    assert len(calls) > 10 and {c.svtype for c in calls} >= {"INS", "DEL"}
    ctx = tasks.device_context(0)
    out = {}
    for fname in ("calls.vcf", "calls.vcf.gz"):
        cfg = sconfig.SnifflesConfig("--input", bam, "--vcf", str(tmp_path / fname))
        with vcf.open_output(cfg, ctx) as h:
            w = vcf.VCFWriter(cfg, h)
            w.write_header(contigs)
            for c in calls:
                w.write_call(copy.deepcopy(c))
        out[fname] = open(tmp_path / fname, "rb").read()
    text = out["calls.vcf"]
    assert gzip.decompress(out["calls.vcf.gz"]) == text
    names, refs = parse_tbi(gzip.decompress(open(tmp_path / "calls.vcf.gz.tbi", "rb").read()))
    assert names == blk.contig_names
    starts = _text_starts(out["calls.vcf.gz"][:-len(bamio._BGZF_EOF)])
    for name, L in contigs:
        for beg in range(0, L, L // 50):
            assert _query(text, starts, names, refs, name, beg, beg + 20_000) == _linear(text, name, beg, beg + 20_000)
