"""Device BAM ingest (SURVEY 8 (f)3), the parts checkable without a GPU: the DEFLATE decoder, the BAM record decoder and the CIGAR16
converter of sniffles_b200/csrc/ingest_core.h in their one-lane host build, against zlib and the host reader; and the index work of
bamio.device_input (merged chunks, spans cut at the linear index, compressed-block selection)."""
import os
import random
import zlib

import numpy as np
import pytest

import ingest_emul
from sniffles_b200 import abi, bamio, synth
from test_cigar16 import check_record


def _streams():
    rnd = random.Random(7)
    yield b""
    yield b"a"
    yield b"abc" * 3000
    yield b"\0" * 65280
    yield bytes(rnd.getrandbits(8) for _ in range(65280))
    yield bytes(rnd.choice(b"ACGT") for _ in range(65280))
    yield open(__file__, "rb").read()
    for _ in range(12):
        n, alpha = rnd.randint(1, 65280), rnd.randint(1, 255)
        yield bytes(rnd.randint(0, alpha) for _ in range(n))


def test_inflate_equals_zlib():
    """stored, fixed and dynamic blocks, long codes (more than 9 bits), run-length code lengths, overlapping matches"""
    n = 0
    for data in _streams():
        for level in (0, 1, 6, 9):
            for strat in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE):
                c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strat)
                comp = c.compress(data) + c.flush()
                rc, out = ingest_emul.inflate(comp, len(data), lead=n % 4)
                assert rc == 0 and out == data, (len(data), level, strat)
                n += 1
    assert n > 300


def test_inflate_rejects_corrupt_streams():
    data = open(__file__, "rb").read()
    comp = zlib.compress(data)[2:-4]
    rnd = random.Random(5)
    for _ in range(200):
        b = bytearray(comp)
        b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8)
        rc, out = ingest_emul.inflate(bytes(b), len(data))
        try:
            want = zlib.decompress(bytes(b), -15)
        except zlib.error:
            want = None
        if want is not None and len(want) == len(data):
            assert rc == 0 and out == want                 # a flip zlib tolerates (padding bits, an unused code) decodes the same way
        else:
            assert rc != 0 or out != data
    rc, _ = ingest_emul.inflate(comp, len(data) - 1)          # output smaller than the stream produces
    assert rc != 0
    rc, _ = ingest_emul.inflate(comp[:len(comp) // 2], len(data))      # truncated input
    assert rc != 0


@pytest.fixture(scope="module")
def bam(tmp_path_factory):
    blk = synth.generate(77, [260_000, 150_000, 90_000], 14.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=5000.0, phased_frac=0.5)
    path = str(tmp_path_factory.mktemp("ingest") / "t.bam")
    bamio.write_bam(path, blk)
    return blk, path


def _same(dev, host, evt_min=11):
    assert len(dev) == len(host)
    recs = [(0, h) for h in host]
    for d, h in zip(dev, host):
        assert (d["pos"], d["flag"], d["mapq"], d["l_seq"], d["qname"]) == (h["pos"], h["flag"], h["mapq"], h["l_seq"], bytes(h["qname"]))
        assert (d["cigar"] == h["cigar"]).all() and (d["seq"] == h["seq"]).all()
        a = h["aux"]
        assert (d["nm"], d["hp"], d["ps"], d["sa"]) == (a.get("NM"), a.get("HP"), a.get("PS"), a.get("SA"))
        # CIGAR16 words: decoded apart from the encoder, against the record's BAM ops; pad words behind the last op
        n = d["n_words"]
        check_record(d["cigar16"][:n], h["cigar"], evt_min)
        assert not d["cigar16"][n:].any()


def test_whole_contigs_equal_host_reader(bam):
    blk, path = bam
    f = bamio.BamFile(path)
    regions = [(n, 0, f.get_reference_length(n)) for n in blk.contig_names]
    bgzf, spans = f.device_input(regions)
    assert len(spans) > 3 * len(regions)                    # cut at the linear index: many parallel walks
    task = np.zeros(len(regions), abi.TASK_DTYPE)
    for t, (n, a, b) in enumerate(regions):
        task[t] = (t, a, b, b, t, 0, 0, 0)
    dev = ingest_emul.load_bam(bgzf, spans, task)
    for t, (n, a, b) in enumerate(regions):
        _same([d for d in dev if d["task"] == t], list(f.fetch(n, a, b)))
    assert len(dev) == len(blk.rec)
    f.close()


def test_regions_equal_host_fetch(bam):
    """region tasks: records that overlap two regions appear in both, unsplit spans give the same records as split ones"""
    blk, path = bam
    f = bamio.BamFile(path)
    rnd = np.random.default_rng(11)
    regions = []
    for _ in range(12):
        t = int(rnd.integers(0, 3))
        L = f.get_reference_length(blk.contig_names[t])
        a = int(rnd.integers(0, L - 1000))
        regions.append((blk.contig_names[t], a, min(L, a + int(rnd.integers(1, 70000)))))
    regions.append((blk.contig_names[0], 250_000, 260_000))
    task = np.zeros(len(regions), abi.TASK_DTYPE)
    for t, (n, a, b) in enumerate(regions):
        task[t] = (f.name_to_id[n], a, b, f.get_reference_length(n), t, 0, 0, 0)
    for split in (True, False):
        bgzf, spans = f.device_input(regions, split=split)
        dev = ingest_emul.load_bam(bgzf, spans, task)
        for t, (n, a, b) in enumerate(regions):
            _same([d for d in dev if d["task"] == t], list(f.fetch(n, a, b)))
    small, _ = f.device_input([(blk.contig_names[1], 40_000, 45_000)])
    assert len(small) < 0.25 * len(open(path, "rb").read())      # only the blocks a region touches are shipped
    f.close()


def test_long_cigar_and_wide_ops(tmp_path):
    """the CG:B,I escape (more than 65535 ops) and operations of 2^11 / 2^23 bases and more (extension words, group padding)"""
    n = 70000
    cig = np.empty(n, "<u4"); cig[0::2] = (3 << 4) | 0; cig[1::2] = (1 << 4) | 2
    l_seq = 3 * (n // 2)
    wide = np.array([(5 << 4) | 4, (2047 << 4) | 0, (2048 << 4) | 2, (7 << 4) | 0, (9_000_000 << 4) | 3, (1 << 4) | 7, (3000 << 4) | 1, (1 << 4) | 8, (2 << 4) | 8, (40 << 4) | 1, (4000 << 4) | 4], "<u4")
    l2 = 5 + 2047 + 7 + 1 + 3000 + 1 + 2 + 40 + 4000
    rec = np.zeros(2, abi.REC_DTYPE)
    rec[0] = (0, 100, 0, 60, abi.AUX_NM, 0, 2, 0, 5, 0, n, l_seq, 0, 0, 0, 0, 0)
    rec[1] = (0, 200, 16, 33, abi.AUX_NM | abi.AUX_HP | abi.AUX_PS | abi.AUX_SA, 2, 3, 0, 77, 12345, len(wide), l2, 21, 0, n, (l_seq + 1) // 2, 2)
    contig = np.zeros(1, abi.CONTIG_DTYPE); contig[0] = (abi.fnv1a64(b"c"), 20_000_000, 0)
    task = np.zeros(1, abi.TASK_DTYPE); task[0] = (0, 0, 20_000_000, 20_000_000, 0, 0, 0, 0)
    var = np.frombuffer(b"rd" + b"abc" + b"c,500,+,100M50S,60,3;", "u1")
    blk = synth.RecordBlock(rec=rec, cigar=np.concatenate([cig, wide]), var=var, seq=np.full((l_seq + 1) // 2 + (l2 + 1) // 2, 0x12, "u1"), task=task, contig=contig,
                            tr=np.zeros(0, "<i4"), contig_names=["c"])
    path = str(tmp_path / "long.bam")
    bamio.write_bam(path, blk)
    f = bamio.BamFile(path)
    bgzf, spans = f.device_input([("c", 0, 20_000_000)])
    dev = ingest_emul.load_bam(bgzf, spans, task)
    host = list(f.fetch("c", 0, 20_000_000))
    assert len(host) == 2 and len(host[0]["cigar"]) == n
    _same(dev, host)
    f.close()


def test_aux_fields_of_every_type(tmp_path):
    """records carrying every aux type of the SAM spec (A c C s S i I f Z H and B arrays of every subtype, as ONT / PacBio BAMs do:
    MM / ML / ip / pw ...) around the tags the path reads; integer tags in their narrow encodings; the device record decoder against the host reader"""
    import struct
    rnd = np.random.default_rng(9)

    def aux_blob(k):
        parts = [b"RGZ" + b"grp%d" % k + b"\0", b"XAA" + b"q", b"Xcc" + struct.pack("<b", -5), b"XfF".replace(b"F", b"f") + struct.pack("<f", 1.5)]
        parts.append(b"MLBC" + struct.pack("<I", 7 + k) + bytes(range(7 + k)))
        parts.append(b"pwBS" + struct.pack("<I", 3) + struct.pack("<3H", 1, 2, 3))
        parts.append(b"ipBs" + struct.pack("<I", 2) + struct.pack("<2h", -1, 2))
        parts.append(b"XiBi" + struct.pack("<I", 1) + struct.pack("<i", -7))
        parts.append(b"XIBI" + struct.pack("<I", 2) + struct.pack("<2I", 9, 10))
        parts.append(b"XFBf" + struct.pack("<I", 2) + struct.pack("<2f", 0.5, 2.5))
        parts.append(b"XbBc" + struct.pack("<I", 3) + bytes([1, 255, 3]))
        parts.append(b"MMZ" + b"C+m,5,12,0;" * (1 + k % 3) + b"\0")
        parts.append(b"XHH" + b"1AE301" + b"\0")
        nm = [b"NMC" + struct.pack("<B", 200), b"NMs" + struct.pack("<h", -3 + k), b"NMS" + struct.pack("<H", 40000), b"NMi" + struct.pack("<i", 123456), b"NMI" + struct.pack("<I", 77), b"NMc" + struct.pack("<b", 9)][k % 6]
        parts.insert(int(rnd.integers(0, len(parts))), nm)
        if k % 2:
            parts.insert(int(rnd.integers(0, len(parts))), b"HPC" + struct.pack("<B", 1 + k % 2))
            parts.insert(int(rnd.integers(0, len(parts))), b"PSi" + struct.pack("<i", 1000 + k))
        if k % 3 == 0:
            parts.insert(int(rnd.integers(0, len(parts))), b"SAZ" + b"ctg,%d,+,50M20S,60,1;" % (100 + k) + b"\0")
        return b"".join(parts)

    recs = []
    for k in range(40):
        qname = b"read_%d" % k + b"x" * (k % 7) + b"\0"
        cig = np.array([(10 + k << 4) | 4, (300 << 4) | 0, (15 << 4) | 1, (200 << 4) | 0], "<u4")
        l_seq = 10 + k + 300 + 15 + 200
        seq = bytes(rnd.integers(0, 256, (l_seq + 1) // 2, dtype=np.uint8))
        body = struct.pack("<iiBBHHHiiii", 0, 1000 + 50 * k, len(qname), 60, 4681, len(cig), 16 if k % 2 else 0, l_seq, -1, -1, 0) + qname + cig.tobytes() + seq + b"\x11" * l_seq + aux_blob(k)
        recs.append(struct.pack("<i", len(body)) + body)
    raw = b"".join(recs)
    want = [bamio.decode_record(r[4:]) for r in recs]
    L = ingest_emul.lib()
    rawa = np.frombuffer(raw + b"\0" * 64, "u1").copy()
    out = np.zeros(len(recs), ingest_emul.RAWREC_DTYPE)
    assert L.ingest_host_parse(rawa.ctypes.data, len(raw), 0, len(raw), out.ctypes.data, len(recs)) == len(recs)
    for r, h in zip(out, want):
        a = h["aux"]
        assert r["status"] == 0 and int(r["pos"]) == h["pos"] and int(r["l_seq"]) == h["l_seq"] and int(r["n_cig"]) == len(h["cigar"]) and int(r["flag"]) == h["flag"]
        af = int(r["aux_flags"])
        assert (af & abi.AUX_NM != 0, af & abi.AUX_HP != 0, af & abi.AUX_PS != 0, af & abi.AUX_SA != 0) == ("NM" in a, "HP" in a, "PS" in a, "SA" in a)
        assert int(r["nm"]) == int(a.get("NM", 0)) and int(r["hp"]) == int(a.get("HP", 0)) and int(r["ps"]) == int(a.get("PS", 0))
        assert bytes(rawa[int(r["sa_src"]):int(r["sa_src"]) + int(r["sa_len"])]) == a.get("SA", b"")
        assert bytes(rawa[int(r["body"]) + 32:int(r["body"]) + 32 + int(r["l_qname"])]) == bytes(h["qname"])
    # truncated / malformed records are reported, never walked out of bounds
    bad = bytearray(recs[0])
    bad[4 + 32 + len(b"read_0\0") + 16 + (525 + 1) // 2 + 525 + 2] = ord("?")       # the type byte of the first aux field
    o1 = np.zeros(1, ingest_emul.RAWREC_DTYPE)
    b2 = np.frombuffer(bytes(bad) + b"\0" * 64, "u1").copy()
    assert L.ingest_host_parse(b2.ctypes.data, len(bad), 0, len(bad), o1.ctypes.data, 1) == 1 and o1[0]["status"] == 1


def test_contig_shards_of_a_bam_partition_its_records(bam):
    """multi-GPU ingest (SURVEY 8e): contigs are LPT-assigned by the index's mapped-read counts; every rank ships only the BGZF blocks of its
    own contigs and the ranks' blocks together are exactly the file's records"""
    from sniffles_b200 import dist
    blk, path = bam
    f = bamio.BamFile(path)
    names = blk.contig_names
    owner = dist.lpt_assign([f.count_mapped(n) for n in names], 2)
    assert sorted(set(owner)) == [0, 1]
    total, shipped = 0, 0
    for rank in (0, 1):
        mine = [t for t in range(len(names)) if owner[t] == rank]
        regions = [(names[t], 0, f.get_reference_length(names[t])) for t in mine]
        task = np.zeros(len(mine), abi.TASK_DTYPE)
        for k, t in enumerate(mine):
            task[k] = (t, 0, regions[k][2], regions[k][2], t, 0, 0, 0)
        bgzf, spans = f.device_input(regions)
        dev = ingest_emul.load_bam(bgzf, spans, task)
        for k, t in enumerate(mine):
            _same([d for d in dev if d["task"] == k], list(f.fetch(names[t], 0, regions[k][2])))
        total += len(dev)
        shipped += len(bgzf)
    assert total == len(blk.rec)
    assert shipped < 1.2 * os.path.getsize(path)            # a block shared by two contigs' boundary may travel twice, nothing more
    f.close()
