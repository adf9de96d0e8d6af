"""Device BAM ingest (SURVEY 8 (f)3) on the GPU, through the C ABI: snfb_inflate_bgzf against zlib, snfb_load_bam against the host
reader (bamio.fetch + pack_records + snfb_pack_cigar16) record by record, and the whole path fed compressed bytes against the
same path fed the host-packed block and against the oracle."""
import zlib

import numpy as np
import pytest

import devcheck
from sniffles_b200 import abi, bamio, binding, synth
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bam(tmp_path_factory):
    blk = synth.generate(77, [260_000, 150_000, 90_000], 14.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=5000.0, phased_frac=0.5, tr_frac=0.2)
    path = str(tmp_path_factory.mktemp("ingest") / "t.bam")
    bamio.write_bam(path, blk)
    return blk, path


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    c.set_config(abi.Config.from_sniffles(sconfig.default_config()))
    yield c
    c.close()


def test_inflate_equals_zlib(bam, ctx):
    _, path = bam
    z = open(path, "rb").read()
    want = b"".join(zlib.decompress(z[po:po + pl], -15) for _, po, pl, _ in bamio.bgzf_members(z))
    got = ctx.inflate_bgzf(np.frombuffer(z, "u1"))
    assert got == want and len(got) > 5_000_000


def test_inflate_block_kinds(ctx):
    """stored / fixed / dynamic blocks, long codes, overlapping matches, empty members — every compressor setting zlib offers"""
    import random
    rnd = random.Random(3)
    datas = [b"", b"a", b"abc" * 3000, b"\0" * 65280, bytes(rnd.getrandbits(8) for _ in range(65280)), bytes(rnd.choice(b"ACGT") for _ in range(65280)), open(__file__, "rb").read()]
    datas += [bytes(rnd.randint(0, rnd.randint(1, 255)) for _ in range(rnd.randint(1, 65280))) for _ in range(10)]
    members, want = [], []
    for d in datas:
        for level in (0, 1, 6, 9):
            for strat in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE):
                m = bamio._bgzf_block(d, level, strat)
                if len(m) <= 65536:
                    members.append(m)
                    want.append(d)
    got = ctx.inflate_bgzf(np.frombuffer(b"".join(members), "u1"))
    assert got == b"".join(want) and len(members) > 200


def test_corrupt_block_fails_cleanly(bam, ctx):
    _, path = bam
    z = bytearray(open(path, "rb").read())
    blocks = list(bamio.bgzf_members(z))
    _, po, pl, _ = blocks[len(blocks) // 2]
    for k in range(po + 20, po + 60):
        z[k] ^= 0x5a
    with pytest.raises(binding.SnfbError, match="inflate"):
        ctx.inflate_bgzf(np.frombuffer(bytes(z), "u1"))
    assert len(ctx.inflate_bgzf(np.frombuffer(open(path, "rb").read(), "u1"))) > 0          # the context is still usable


def _device_records(ctx, bgzf, spans, tables):
    z = ctx.load_bam(bgzf, spans, tables)
    rec, cig, var, seq = ctx.ingest_fetch()
    assert len(rec) == z["n_rec"]
    return z, rec, cig, var, seq


def _compare(rec, cig, var, seq, host, task_of, evt_min=11):
    """device block vs the host reader's records, field by field, and the CIGAR16 words vs snfb_pack_cigar16"""
    assert len(rec) == len(host)
    if not host:
        return
    hrec = np.zeros(len(host), abi.REC_DTYPE)
    off = 0
    for i, h in enumerate(host):
        hrec[i]["cigar_off"], hrec[i]["n_cigar"] = off, len(h["cigar"])
        off += len(h["cigar"])
    rec16, c16 = binding.pack_cigar16(hrec, np.concatenate([h["cigar"] for h in host]), evt_min)
    for i, (r, h) in enumerate(zip(rec, host)):
        a = h["aux"]
        assert (int(r["task"]), int(r["pos"]), int(r["flag"]), int(r["mapq"]), int(r["l_seq"])) == (task_of[i], h["pos"], h["flag"], h["mapq"], h["l_seq"]), i
        vo, lq, sl = int(r["var_off"]), int(r["l_qname"]), int(r["sa_len"])
        assert var[vo:vo + lq].tobytes() == bytes(h["qname"])
        af = int(r["aux_flags"])
        assert (af & abi.AUX_NM != 0, af & abi.AUX_HP != 0, af & abi.AUX_PS != 0, af & abi.AUX_SA != 0) == ("NM" in a, "HP" in a, "PS" in a, "SA" in a)
        assert (int(r["nm"]), int(r["hp"]), int(r["ps"])) == (int(a.get("NM", 0)), int(a.get("HP", 0)) & 255, int(a.get("PS", 0)))
        assert var[vo + lq:vo + lq + sl].tobytes() == a.get("SA", b"")
        so, nb = int(r["seq_off"]), (h["l_seq"] + 1) // 2
        assert so % 16 == 0 and (seq[so:so + nb] == h["seq"]).all()
        co, n = int(r["cigar_off"]), int(r["n_cigar"])
        ho, hn = int(rec16[i]["cigar_off"]), int(rec16[i]["n_cigar"])
        assert co % 8 == 0 and n == hn and (cig[co:co + n] == c16[ho:ho + hn]).all() and not cig[co + n:co + ((n + 7) // 8) * 8].any(), i


def test_whole_contigs_equal_host_reader(bam, ctx):
    blk, path = bam
    f = bamio.BamFile(path)
    regions = [(n, 0, f.get_reference_length(n)) for n in blk.contig_names]
    tables = bamio.pack_records(f.contigs, [], [(t, a, b, t) for t, (n, a, b) in enumerate(regions)])
    bgzf, spans = f.device_input(regions)
    z, rec, cig, var, seq = _device_records(ctx, bgzf, spans, tables)
    host, task_of = [], []
    for t, (n, a, b) in enumerate(regions):
        rs = list(f.fetch(n, a, b))
        host += rs
        task_of += [t] * len(rs)
    assert z["n_rec"] == len(blk.rec) and z["n_raw"] >= z["n_rec"] and z["bgzf_bytes"] == len(bgzf)
    _compare(rec, cig, var, seq, host, task_of)
    f.close()


def test_regions_equal_host_fetch(bam, ctx):
    blk, path = bam
    f = bamio.BamFile(path)
    rnd = np.random.default_rng(11)
    regions = []
    for t in sorted(int(x) for x in rnd.integers(0, 3, 14)):
        L = f.get_reference_length(blk.contig_names[t])
        a = int(rnd.integers(0, L - 1000))
        regions.append((blk.contig_names[t], a, min(L, a + int(rnd.integers(1, 70000)))))
    regions.append((blk.contig_names[2], 89_000, 90_000))
    tables = bamio.pack_records(f.contigs, [], [(f.name_to_id[n], a, b, t) for t, (n, a, b) in enumerate(regions)])
    for split in (True, False):
        bgzf, spans = f.device_input(regions, split=split)
        _, rec, cig, var, seq = _device_records(ctx, bgzf, spans, tables)
        host, task_of = [], []
        for t, (n, a, b) in enumerate(regions):
            rs = list(f.fetch(n, a, b))
            host += rs
            task_of += [t] * len(rs)
        _compare(rec, cig, var, seq, host, task_of)
    f.close()


def test_long_cigar_and_wide_ops(tmp_path, ctx):
    n = 70000
    cigw = np.empty(n, "<u4"); cigw[0::2] = (3 << 4) | 0; cigw[1::2] = (1 << 4) | 2
    l_seq = 3 * (n // 2)
    wide = np.array([(5 << 4) | 4, (2047 << 4) | 0, (2048 << 4) | 2, (7 << 4) | 0, (9_000_000 << 4) | 3, (1 << 4) | 7, (3000 << 4) | 1, (1 << 4) | 8, (2 << 4) | 8, (40 << 4) | 1, (4000 << 4) | 4], "<u4")
    l2 = 5 + 2047 + 7 + 1 + 3000 + 1 + 2 + 40 + 4000
    rec = np.zeros(2, abi.REC_DTYPE)
    rec[0] = (0, 100, 0, 60, abi.AUX_NM, 0, 2, 0, 5, 0, n, l_seq, 0, 0, 0, 0, 0)
    rec[1] = (0, 200, 16, 33, abi.AUX_NM | abi.AUX_HP | abi.AUX_PS | abi.AUX_SA, 2, 3, 0, 77, 12345, len(wide), l2, 21, 0, n, (l_seq + 1) // 2, 2)
    contig = np.zeros(1, abi.CONTIG_DTYPE); contig[0] = (abi.fnv1a64(b"c"), 20_000_000, 0)
    task = np.zeros(1, abi.TASK_DTYPE); task[0] = (0, 0, 20_000_000, 20_000_000, 0, 0, 0, 0)
    var = np.frombuffer(b"rd" + b"abc" + b"c,500,+,100M50S,60,3;", "u1")
    blk = synth.RecordBlock(rec=rec, cigar=np.concatenate([cigw, wide]), var=var, seq=np.full((l_seq + 1) // 2 + (l2 + 1) // 2, 0x12, "u1"), task=task, contig=contig,
                            tr=np.zeros(0, "<i4"), contig_names=["c"])
    path = str(tmp_path / "long.bam")
    bamio.write_bam(path, blk)
    f = bamio.BamFile(path)
    bgzf, spans = f.device_input([("c", 0, 20_000_000)])
    _, r, cig, v, seq = _device_records(ctx, bgzf, spans, blk)
    host = list(f.fetch("c", 0, 20_000_000))
    assert len(host) == 2 and len(host[0]["cigar"]) == n
    _compare(r, cig, v, seq, host, [0, 0])
    f.close()


def test_path_from_compressed_bytes_equals_packed_block_and_oracle(bam):
    """lead -> cluster -> consensus over the block built on the device from BGZF bytes == over the host-packed block == the oracle"""
    import oracle.oracle as orc
    blk, path = bam
    f = bamio.BamFile(path)
    cfg = abi.Config.from_sniffles(sconfig.default_config())
    regions = [(n, 0, f.get_reference_length(n)) for n in blk.contig_names]
    bgzf, spans = f.device_input(regions)
    c = binding.Context(0)
    try:
        c.set_config(cfg)
        z = c.load_bam(bgzf, spans, blk)
        got = c.run()
        names = [t[0] for t in c.timings()]
    finally:
        c.close()
    assert z["n_rec"] == len(blk.rec) and "inflate" in names and "pack_records" in names
    want = orc.run(blk, cfg, 3, 4)
    devcheck.assert_same(want, got)
    assert len(got.cand) > 20
    f.close()


def test_empty_region_and_bad_spans(bam, ctx):
    blk, path = bam
    f = bamio.BamFile(path)
    L = f.get_reference_length(blk.contig_names[0])
    tables = bamio.pack_records(f.contigs, [], [(0, 0, L, 0)])
    z = ctx.load_bam(np.zeros(0, "u1"), np.zeros(0, abi.SPAN_DTYPE), tables)
    assert z["n_rec"] == 0
    res = ctx.run()
    assert len(res.cand) == 0
    bgzf, spans = f.device_input([(blk.contig_names[0], 0, L)])
    bad = spans.copy()
    bad["ubeg"][1] += 3                                   # not a record boundary
    with pytest.raises(binding.SnfbError, match="record chain|overlap"):
        ctx.load_bam(bgzf, bad, tables)
    bad = spans.copy()
    bad["cbeg"][1] += 1                                   # not a block start
    with pytest.raises(binding.SnfbError, match="virtual offset"):
        ctx.load_bam(bgzf, bad, tables)
    f.close()
