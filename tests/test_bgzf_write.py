"""BGZF output without a GPU: the encoder of sniffles_b200/csrc/deflate_core.h in its one-thread g++ build (the bytes the device writes,
see test_gpu_bgzf_write.py) against zlib and the host BGZF reader, its ratio against zlib level 1, the BAI-layout index builder shared by
write_bam and the .tbi writer, tabix queries answered from a .tbi parsed here from the spec, and the .vcf.gz output handle."""
import gzip
import hashlib
import os
import random
import re
import struct
import zlib

import pytest

import bgzf_host
from sniffles_b200 import bamio, synth, vcf
from sniffles_b200 import config as sconfig

BLOCK = 0xff00


@pytest.fixture(scope="module")
def compress(tmp_path_factory):
    return bgzf_host.build(tmp_path_factory.mktemp("deflate_host"))


@pytest.fixture(scope="module")
def inputs():
    return bgzf_host.inputs()


def _check_members(z, coffsets, data):
    ms = bgzf_host.members(z, coffsets)
    assert len(ms) == (len(data) + BLOCK - 1) // BLOCK
    for k, m in enumerate(ms):
        chunk = data[k * BLOCK:(k + 1) * BLOCK]
        assert len(m) <= 65536
        assert m[:4] == b"\x1f\x8b\x08\x04" and m[12:16] == b"BC\x02\x00" and struct.unpack("<H", m[16:18])[0] == len(m) - 1
        assert zlib.decompress(m[18:-8], -15) == chunk
        assert struct.unpack("<II", m[-8:]) == (zlib.crc32(chunk), len(chunk))
    return ms


@pytest.mark.parametrize("name", ["empty", "one", "block", "block+1", "random", "repeat", "window", "vcf"])
def test_round_trip(compress, inputs, tmp_path, name):
    data = inputs[name]
    z, coffsets = compress(data)
    ms = _check_members(z, coffsets, data)
    assert gzip.decompress(z + bamio._BGZF_EOF) == data
    path = str(tmp_path / "x.gz")
    with open(path, "wb") as f:
        f.write(z + bamio._BGZF_EOF)
    r = bamio.BgzfReader(path)                         # checks every member's CRC-32 and ISIZE
    try:
        got, _ = r.read_from(0, len(data) + 1)
    finally:
        r.close()
    assert got == data
    if name == "random":                               # incompressible: stored blocks, each member 65280 + 5 + 26 bytes
        assert all(m[18] & 7 == 1 for m in ms) and max(len(m) for m in ms) == BLOCK + 31
    if name == "repeat":
        assert len(z) < 200 * len(ms)


def test_deterministic(compress, inputs):
    assert compress(inputs["vcf"]) == compress(inputs["vcf"])


def test_ratio_not_above_zlib_level_1(compress, inputs):
    data = inputs["vcf"]
    z, _ = compress(data)
    assert len(z) <= bgzf_host.zlib_bgzf_size(data, 1)


# ------------------------------------------------------------------------------------------------ write_bam after the index refactor
def test_write_bam_bytes_unchanged(tmp_path):
    """BAM / BAI / CSI bytes as the writer produced them before the BAI tables moved into bamio.bin_index and before the header and
    the records shared one placement step: a seeded block, the same in 100-byte blocks (the header spans two), a record larger than
    a BGZF block, and the benchmark's config-6 block (at a twentieth of its contig length) at levels 6 and 0"""
    from test_bamio import long_cigar_block
    seeded = synth.generate(31, [200_000, 120_000], 10.0, len_mean=8000.0, len_sd=2000.0, sv_spacing=6000.0)
    c6 = synth.generate(606, [75_000] * 4, 30.0, len_mean=15000.0, len_sd=6000.0, sv_spacing=8000.0, phased_frac=0.3, tr_frac=0.2)
    sha = lambda p: hashlib.sha256(open(p, "rb").read()).hexdigest()
    cases = [                                              # (block, write_bam arguments, BAM, BAI, CSI)
        (seeded, {}, "3e7667e27b50add1657dad351344613556fd6ef6bd5a95cd3f0e04792c6173ab",
         "dc7c958d85f87e9d2115da854ae640be1750b600f8a76b7b67f96b7f65fd0005", "df6a8826d2d1e2ea338dd24b0ddca739d59bc2c443f0abfb96ac8198c4cfeb88"),
        (seeded, dict(block_bytes=100), "20e822ae86af4dbd9658e9e78b5de32ff456d09fd11e823b3a97ad0a02b0340c",
         "205faa87aa0f85c62a36aaa2e6d5041475cf1e60dba0fec6312711b665d1bad3", "7f902495365c46893ed9c1d5f9db5c7c5a84cb9d0b0a505645b4bfd703ca93fa"),
        (long_cigar_block(), {}, "76231e29f22c1030016ac9cb3c663a36571f7c11cf86cbfb85919fd00b880c7f",
         "89faea55223bdd931bc7a919d92521ff344da72aaa4c57f8c507f8cddfcc7055", "84a5f6e7675cf0dea1a9fd78f197270efa7188120ecd3c73b4803615f65c8d77"),
        (c6, dict(level=6, qual_seed=7), "8534220ed4568b93d2ca4e188e6e12a6ab81d2a22300b8e4db3c1f72b0390d74",
         "695e250a26062270b6e52461c97ac5c27781d35c7b3913627f3403f7853da2d6", "b5370d7aaca84225502555f618ab0c3a2c89d00b9ff0afee699c5ced306b6b07"),
        (c6, dict(level=0, qual_seed=7), "0b5e09ce9ab52f822839a8def7a5e7ebd41075ab059e1c5ba43d392edc51fe6e",
         "3e2ab91e8481f93ae4899afbb7998fb2ccffe2a84ea6a54c853f12b110517392", "90203aa79feab924f39b4434427c7e0bb16758802bc856359f3713955a4390fe")]
    for k, (blk, kw, want_bam, want_bai, want_csi) in enumerate(cases):
        for index, want in (("bai", want_bai), ("csi", want_csi)):
            path = str(tmp_path / f"s{k}_{index}.bam")
            bamio.write_bam(path, blk, index=index, **kw)
            assert sha(path) == want_bam and sha(path + "." + index) == want, (k, index)


# ------------------------------------------------------------------------------------------------ tabix
def sorted_vcf_text() -> bytes:
    """the fixture lines sorted by contig (first appearance) and POS behind a header, plus lines for every INFO/END case"""
    lines = [l.split("\t") for l in bgzf_host.fixture_vcf_lines()]
    extra = [["chrX", "1000", ".", "N", "<DEL>", "60", "PASS", "END=5000;SVTYPE=DEL", "GT", "0/1"],           # END at INFO start
             ["chrX", "2000", ".", "N", "<INV>", "60", "PASS", "IMPRECISE;SVTYPE=INV;END=9000000", "GT", "0/1"],  # END far behind
             ["chrX", "3000", ".", "NNNN", "<DUP>", "60", "PASS", "PRECISE;END=1500", "GT", "0/1"],         # END <= POS: beg + 1
             ["chrX", "4000", ".", "NNN", "<DEL>", "60", "PASS", "PRECISE;END=.", "GT", "0/1"],            # END '.': REF length
             ["chrX", "4000", ".", "N", "<DUP>", "60", "PASS", "PRECISE;XEND=99999", "GT", "0/1"]]         # not INFO/END
    order = {}
    for f in lines + extra:
        order.setdefault(f[0], len(order))
    rows = sorted(lines + extra, key=lambda f: (order[f[0]], int(f[1])))
    head = ["##fileformat=VCFv4.2"] + [f"##contig=<ID={c}>" for c in order] + ["#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE"]
    return ("\n".join(head + ["\t".join(f) for f in rows]) + "\n").encode()


def interval(fields):
    """VCF line -> [beg, end) for the tabix VCF preset, written here from htslib's tbx_parse1 independently of bamio"""
    beg = int(fields[1]) - 1
    end = beg + len(fields[3])
    m = re.search(r"(?:^|;)END=([0-9]+)", fields[7])
    if m and not fields[7].startswith("END=.") and ";END=." not in fields[7]:
        e = int(m.group(1))
        end = e if e > beg else beg + 1
    return beg, end


def parse_tbi(body: bytes):
    """tabix spec: header, names, then per reference the bins (with chunks) and the linear index"""
    assert body[:4] == b"TBI\1"
    n_ref, fmt, col_seq, col_beg, col_end, meta, skip, l_nm = struct.unpack("<8i", body[4:36])
    assert (fmt, col_seq, col_beg, col_end, chr(meta), skip) == (2, 1, 2, 0, "#", 0)
    names = body[36:36 + l_nm].split(b"\0")[:-1]
    p, refs = 36 + l_nm, []
    for _ in range(n_ref):
        n_bin, = struct.unpack_from("<i", body, p)
        p += 4
        bins = {}
        for _ in range(n_bin):
            b, n_chunk = struct.unpack_from("<Ii", body, p)
            p += 8
            bins[b] = [struct.unpack_from("<QQ", body, p + 16 * k) for k in range(n_chunk)]
            p += 16 * n_chunk
        n_intv, = struct.unpack_from("<i", body, p)
        p += 4
        refs.append((bins, list(struct.unpack_from(f"<{n_intv}Q", body, p))))
        p += 8 * n_intv
    assert p == len(body)
    return [n.decode() for n in names], refs


def _text_starts(z: bytes):
    """coffset -> start of its data in the text, from the members of the written file"""
    starts, u = {}, 0
    for o, _, _, isize in bamio.bgzf_members(z):
        starts[o], u = u, u + isize
    return starts


def _query(text, starts, names, refs, contig, beg, end):
    """line starts (text offsets) of the lines overlapping [beg, end), found through the index as htslib's tbx_itr_queryi does"""
    bins, lin = refs[names.index(contig)]
    min_off = lin[min(beg >> 14, len(lin) - 1)] if lin else 0
    to_u = lambda v: starts[v >> 16] + (v & 0xffff)
    found = set()
    for b in bamio.reg2bins(beg, end):
        for c0, c1 in bins.get(b, []) if b != 37450 else []:
            if c1 <= min_off:
                continue
            u, stop = to_u(max(c0, min_off)), to_u(c1)
            while u < stop:
                e = text.index(b"\n", u) + 1
                f = text[u:e - 1].decode().split("\t")
                b0, b1 = interval(f)
                if f[0] == contig and b0 < end and b1 > beg:
                    found.add(u)
                u = e
    return found


def _linear(text, contig, beg, end):
    found, u = set(), 0
    for line in text.split(b"\n")[:-1]:
        if not line.startswith(b"#"):
            f = line.decode().split("\t")
            b0, b1 = interval(f)
            if f[0] == contig and b0 < end and b1 > beg:
                found.add(u)
        u += len(line) + 1
    return found


def test_tabix_queries_match_a_linear_scan(compress, tmp_path):
    text = sorted_vcf_text()
    out = vcf.BgzfIndexedOutput(str(tmp_path / "q.vcf.gz"), compress)
    out.write(text.decode())
    out.close()
    z = open(tmp_path / "q.vcf.gz", "rb").read()
    assert gzip.decompress(z) == text
    starts = _text_starts(z)
    assert len(starts) > 40
    names, refs = parse_tbi(gzip.decompress(open(tmp_path / "q.vcf.gz.tbi", "rb").read()))
    rows = [l.split(b"\t") for l in text.split(b"\n")[:-1] if not l.startswith(b"#")]
    assert names == list(dict.fromkeys(r[0].decode() for r in rows))
    span = {}
    for r in rows:
        b0, b1 = interval([x.decode() for x in r])
        c = r[0].decode()
        span[c] = max(span.get(c, 0), b1)
    rnd = random.Random(7)
    crossing = 0
    for q in range(500):
        contig = rnd.choice(names)
        beg = rnd.randrange(0, span[contig] + 1000)
        end = beg + rnd.choice((1, 10, 1000, 50_000, 3_000_000))
        got = _query(text, starts, names, refs, contig, beg, end)
        assert got == _linear(text, contig, beg, end), (contig, beg, end)
        crossing += sum((u // BLOCK) != (text.index(b"\n", u) // BLOCK) for u in got)
    assert crossing > 0                                     # some answers are lines that cross a block boundary
    for contig, beg, end in (("chrX", 8_000_000, 8_000_001), ("chrX", 1600, 1601), ("chrX", 4001, 4002)):
        assert _query(text, starts, names, refs, contig, beg, end) == _linear(text, contig, beg, end) != set()


def test_virtual_offsets_read_back(compress, tmp_path):
    text = sorted_vcf_text()
    z, coffsets = compress(text)
    body = bamio.tabix_index(text, coffsets)
    names, refs = parse_tbi(body)
    path = str(tmp_path / "v.gz")
    with open(path, "wb") as f:
        f.write(z + bamio._BGZF_EOF)
    r = bamio.BgzfReader(path)
    try:
        for bins, _ in refs:
            for b, ch in bins.items():
                for v0, v1 in (ch[:1] if b == 37450 else ch):          # the pseudo-bin's second pair holds record counts
                    got, _ = r.read_from(v0, 40)
                    u = coffsets.index(v0 >> 16) * BLOCK + (v0 & 0xffff)
                    assert got == text[u:u + 40] and (u == 0 or text[u - 1:u] == b"\n")
    finally:
        r.close()


@pytest.mark.parametrize("bad, what", [
    ("chr1\t500\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL\nchr1\t400\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL\n", "not sorted"),
    ("chr1\t500\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL\nchr2\t400\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL\nchr1\t900\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL\n", "reappears"),
    (f"chr1\t{(1 << 29) + 1}\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL\n", "2\\^29"),
    ("chr1\t5\t.\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL;END=600000000\n", "2\\^29")])
def test_rejected_input_writes_nothing(compress, tmp_path, bad, what):
    path = str(tmp_path / "bad.vcf.gz")
    out = vcf.BgzfIndexedOutput(path, compress)
    out.write("##fileformat=VCFv4.2\n" + bad)
    with pytest.raises(ValueError, match=what) as e:
        out.close()
    assert "line " in str(e.value)
    assert not os.path.exists(path) and not os.path.exists(path + ".tbi")


class _HostCtx:
    def __init__(self, compress):
        self.deflate_bgzf = compress


def test_open_output_end_to_end(compress, tmp_path):
    """VCFWriter through open_output: the .vcf.gz decompresses to exactly the text of the plain .vcf"""
    from test_vcf import final_calls
    from test_oracle_golden import NAMES, load_fixture
    from sniffles_b200 import abi
    import oracle.oracle as orc
    fx, blk = load_fixture(NAMES[0])
    cfg = sconfig.default_config(*fx["args"])
    res = orc.run(blk, abi.Config.from_sniffles(cfg), 3, 2, keep_rec_nm=True)
    calls = sorted((c for t in range(len(fx["tasks"])) for c in final_calls(fx, blk, res, cfg, t)), key=lambda c: (c.contig, c.pos))
    assert len(calls) > 5
    texts = {}
    for name in ("plain.vcf", "out.vcf.gz"):
        c = sconfig.SnifflesConfig("--input", "input.bam", "--vcf", str(tmp_path / name), *fx["args"])
        assert bool(c.vcf_output_bgz) == name.endswith(".gz")
        with vcf.open_output(c, _HostCtx(compress)) as h:
            w = vcf.VCFWriter(c, h)
            w.write_header([(n, int(x["length"])) for n, x in zip(blk.contig_names, blk.contig)])
            for call in calls:
                w.write_call(__import__("copy").deepcopy(call))
        texts[name] = open(tmp_path / name, "rb").read()
    assert texts["plain.vcf"].count(b"\n") > 5
    assert gzip.decompress(texts["out.vcf.gz"]) == texts["plain.vcf"]
    assert os.path.exists(tmp_path / "out.vcf.gz.tbi") and not os.path.exists(tmp_path / "plain.vcf.tbi")
