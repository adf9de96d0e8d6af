"""BGZF / BAM / BAI with the standard library — the host-side stand-in for htslib behind `bam.fetch(contig, start, end)`
(leadprov.py:488; the accessor contract is SURVEY.md §8a row A0).  Region fetches go through the BAI index (bins + linear
index, SAM spec §5.2), so a task only inflates the BGZF blocks its region touches.  A small writer (BAM + BAI from a packed
record block) exists for the tests and the benchmark inputs; it is not part of the product path.

Base qualities are never decoded; of the aux tags only NM, HP, PS, SA and the CG:B,I long-CIGAR escape are read."""
import bisect
import os
import struct
import zlib

import numpy as np

from . import abi
from .synth import RecordBlock

_AUX_SIZE = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4}
_AUX_FMT = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}
_BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


# ------------------------------------------------------------------------------------------------ BGZF
def bgzf_header(buf, o=0):
    """The BGZF member header at offset o of a bytes-like buffer (SAM spec §4.1: the gzip magic with FEXTRA, then the BC subfield)
    -> (bsize, payload offset, payload length): the member's total size and where in `buf` its raw DEFLATE data lies."""
    if buf[o:o + 4] != b"\x1f\x8b\x08\x04":
        raise ValueError("not a BGZF block")
    xlen = struct.unpack_from("<H", buf, o + 10)[0]
    e = o + 12
    while e + 4 <= o + 12 + xlen:
        slen = struct.unpack_from("<H", buf, e + 2)[0]
        if buf[e] == 66 and buf[e + 1] == 67:
            bsize = struct.unpack_from("<H", buf, e + 4)[0] + 1
            return bsize, o + 12 + xlen, bsize - 12 - xlen - 8
        e += 4 + slen
    raise ValueError("BGZF block without a BC field")


def bgzf_members(z):
    """(start, payload offset, payload length, ISIZE) of every member of a buffer of whole BGZF members"""
    o = 0
    while o < len(z):
        bsize, po, pl = bgzf_header(z, o)
        yield o, po, pl, struct.unpack_from("<I", z, o + bsize - 4)[0]
        o += bsize


class BgzfReader:
    """random access by BGZF virtual offset (coffset << 16 | uoffset)"""

    def __init__(self, path):
        self.f = open(path, "rb")
        self._cache = (None, b"", 0)           # (coffset, data, block length)

    def close(self):
        self.f.close()

    def member(self, coffset):
        """bgzf_header of the member at a file offset, with the payload offset relative to it; (0, 0, 0) at the end of the file"""
        self.f.seek(coffset)
        head = self.f.read(18)
        if len(head) < 18:
            return 0, 0, 0
        return bgzf_header(head + self.f.read(max(struct.unpack_from("<H", head, 10)[0] - 6, 0)))

    def _block(self, coffset):
        if self._cache[0] == coffset:
            return self._cache[1], self._cache[2]
        bsize, po, pl = self.member(coffset)
        if bsize == 0:
            return b"", 0
        self.f.seek(coffset + po)
        cdata = self.f.read(pl)
        trailer = self.f.read(8)
        data = zlib.decompress(cdata, -15)
        # the gzip trailer, checked as htslib checks it: a damaged block can still inflate to ISIZE bytes, but not to the same CRC-32
        crc, isize = struct.unpack("<II", trailer) if len(trailer) == 8 else (None, None)
        if isize != len(data):
            raise ValueError(f"BGZF block at file offset {coffset}: inflated size {len(data)} differs from ISIZE {isize}")
        if crc != zlib.crc32(data):
            raise ValueError(f"BGZF block at file offset {coffset}: CRC32 mismatch")
        self._cache = (coffset, data, bsize)
        return data, bsize

    def read_from(self, voffset, nbytes):
        """nbytes of uncompressed data starting at a virtual offset; returns (data, virtual offset after it)"""
        coff, uoff = voffset >> 16, voffset & 0xffff
        out = bytearray()
        while len(out) < nbytes:
            data, bsize = self._block(coff)
            if bsize == 0:
                break
            take = data[uoff:uoff + nbytes - len(out)]
            out += take
            uoff += len(take)
            if uoff >= len(data):
                coff, uoff = coff + bsize, 0
        return bytes(out), (coff << 16) | uoff


def _parse_aux(buf):
    tags, i, n = {}, 0, len(buf)
    while i + 3 <= n:
        tag, typ = buf[i:i + 2].decode(), chr(buf[i + 2])
        i += 3
        if typ in _AUX_FMT:
            sz = _AUX_SIZE[typ]
            tags[tag] = struct.unpack(_AUX_FMT[typ], buf[i:i + sz])[0]
            i += sz
        elif typ in ("A", "f"):
            i += _AUX_SIZE[typ]
        elif typ in ("Z", "H"):
            j = buf.index(b"\0", i)
            tags[tag] = buf[i:j]
            i = j + 1
        elif typ == "B":
            sub, cnt = chr(buf[i]), struct.unpack("<I", buf[i + 1:i + 5])[0]
            if tag == "CG" and sub == "I":
                tags["CG"] = np.frombuffer(buf[i + 5:i + 5 + 4 * cnt], "<u4").copy()
            i += 5 + _AUX_SIZE[sub] * cnt
        else:
            raise ValueError(f"unknown aux type {typ!r}")
    return tags


def decode_record(b):
    """one BAM alignment (without its block_size prefix) -> dict of the fields the path reads"""
    ref_id, pos, l_rn, mapq, _bin, n_cig, flag, l_seq, _nr, _np, _tl = struct.unpack("<iiBBHHHiiii", b[:32])
    o = 32
    qname = b[o:o + l_rn - 1]
    o += l_rn
    cigar = np.frombuffer(b[o:o + 4 * n_cig], "<u4").copy()
    o += 4 * n_cig
    seq = np.frombuffer(b[o:o + (l_seq + 1) // 2], "u1").copy()
    o += (l_seq + 1) // 2 + l_seq
    aux = _parse_aux(b[o:])
    # records with more than 65535 CIGAR ops carry the real CIGAR in CG:B,I behind a "<l_seq>S<reflen>N" placeholder (SAM spec §4.2.2;
    # htslib and pysam restore it transparently)
    if n_cig == 2 and "CG" in aux and (int(cigar[0]) & 15) == 4 and (int(cigar[0]) >> 4) == l_seq and (int(cigar[1]) & 15) == 3:
        cigar = aux["CG"]
    elif n_cig == 2 and (int(cigar[0]) & 15) == 4 and (int(cigar[0]) >> 4) == l_seq and (int(cigar[1]) & 15) == 3 and l_seq > 0:
        raise ValueError(f"record {qname!r}: placeholder CIGAR without a CG tag")
    return dict(ref_id=ref_id, pos=pos, mapq=mapq, flag=flag, l_seq=l_seq, qname=qname, cigar=cigar, seq=seq, aux=aux)


def ref_span(cigar):
    ops = cigar & 15
    return int(np.where(np.isin(ops, (0, 2, 3, 7, 8)), cigar >> 4, 0).sum())


# ------------------------------------------------------------------------------------------------ BAI
def reg2bins(beg, end, min_shift=14, depth=5):
    """bins overlapping [beg, end) in the binning scheme of SAM spec §5.3; the defaults are the BAI / TBI geometry"""
    end -= 1
    bins, t, s = [], 0, min_shift + 3 * depth
    for lvl in range(depth + 1):
        bins.extend(range(t + (beg >> s), t + (end >> s) + 1))
        t += 1 << (3 * lvl)
        s -= 3
    return bins


def _merge_ranges(ranges):
    """ascending (beg, end) ranges -> [beg, end] lists with every overlapping or touching run merged into one"""
    merged = []
    for a, b in ranges:
        if merged and a <= merged[-1][1]:
            merged[-1][1] = max(merged[-1][1], b)
        else:
            merged.append([a, b])
    return merged


def reg2bin(beg, end):
    end -= 1
    for shift, off in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return off + (beg >> shift)
    return 0


def read_header(bgzf):
    """the BAM header through a BgzfReader -> ([(contig name, length)], virtual offset of the first record)"""
    head, v = bgzf.read_from(0, 12)
    if head[:4] != b"BAM\1":
        raise ValueError("not a BAM file")
    l_text = struct.unpack("<i", head[4:8])[0]
    data, v = bgzf.read_from(0, 12 + l_text)
    if len(data) < 12 + l_text:
        raise ValueError("truncated BAM header")
    n_ref = struct.unpack("<i", data[8 + l_text:12 + l_text])[0]
    contigs = []
    for _ in range(n_ref):
        d, v = bgzf.read_from(v, 4)
        if len(d) < 4:
            raise ValueError("truncated BAM header")
        l_name = struct.unpack("<i", d)[0]
        d, v = bgzf.read_from(v, l_name + 4)
        if len(d) < l_name + 4:
            raise ValueError("truncated BAM header")
        contigs.append((d[:l_name - 1].decode(), struct.unpack("<i", d[l_name:l_name + 4])[0]))
    return contigs, v


def find_index(path):
    """the index BamFile opens for `path` when none is named: path.bai, path.csi or the .bai beside a .bam, the first that exists; None"""
    return next((p for p in (path + ".bai", path + ".csi", path[:-4] + ".bai" if path.endswith(".bam") else path + ".bai") if os.path.exists(p)), None)


class BamFile:
    """`fetch(contig, start, end)` over an indexed BAM; yields decoded records in file (coordinate) order"""

    def __init__(self, path, index_path=None):
        self.path = path
        self.bgzf = BgzfReader(path)
        self.contigs, self.first_record = read_header(self.bgzf)
        self.name_to_id = {n: i for i, (n, _) in enumerate(self.contigs)}
        if index_path is None:
            index_path = find_index(path) or path + ".bai"
        self.min_shift, self.depth = 14, 5
        self.index = self._load_csi(index_path) if index_path.endswith(".csi") else self._load_bai(index_path)
        self.meta_bin = ((1 << ((self.depth + 1) * 3)) - 1) // 7 + 1          # 37450 for the BAI layout

    def close(self):
        self.bgzf.close()

    @staticmethod
    def _load_bai(path):
        with open(path, "rb") as f:
            d = f.read()
        if d[:4] != b"BAI\1":
            raise ValueError("not a BAI index")
        n_ref = struct.unpack("<i", d[4:8])[0]
        p, refs = 8, []
        for _ in range(n_ref):
            n_bin = struct.unpack("<i", d[p:p + 4])[0]
            p += 4
            bins = {}
            for _ in range(n_bin):
                b, n_chunk = struct.unpack("<Ii", d[p:p + 8])
                p += 8
                bins[b] = [struct.unpack("<QQ", d[p + 16 * k:p + 16 * k + 16]) for k in range(n_chunk)]
                p += 16 * n_chunk
            n_intv = struct.unpack("<i", d[p:p + 4])[0]
            p += 4
            lin = list(struct.unpack(f"<{n_intv}Q", d[p:p + 8 * n_intv]))
            p += 8 * n_intv
            refs.append((bins, lin, None))
        return refs

    def _load_csi(self, path):
        """CSI (SAM spec §5.3 / CSIv1): a BGZF file; bins of a configurable geometry (min_shift, depth), every bin with the smallest virtual
        offset of a record overlapping its first window (`loffset`) instead of BAI's linear index"""
        with open(path, "rb") as f:
            z = f.read()
        d, o = b"", 0
        while o < len(z):                                # concatenated gzip members
            dec = zlib.decompressobj(31)
            d += dec.decompress(z[o:])
            o = len(z) - len(dec.unused_data)
        if d[:4] != b"CSI\1":
            raise ValueError("not a CSI index")
        self.min_shift, self.depth, l_aux = struct.unpack("<iii", d[4:16])
        p = 16 + l_aux
        n_ref = struct.unpack("<i", d[p:p + 4])[0]
        p += 4
        refs = []
        for _ in range(n_ref):
            n_bin = struct.unpack("<i", d[p:p + 4])[0]
            p += 4
            bins, loff = {}, {}
            for _ in range(n_bin):
                b, lo, n_chunk = struct.unpack("<IQi", d[p:p + 16])
                p += 16
                bins[b] = [struct.unpack("<QQ", d[p + 16 * k:p + 16 * k + 16]) for k in range(n_chunk)]
                loff[b] = lo
                p += 16 * n_chunk
            refs.append((bins, None, loff))
        return refs

    # ---- index queries shared by fetch and device_input
    def _min_offset(self, rid, start):
        """smallest virtual offset a record overlapping `start` can have: BAI's linear index, or CSI's per-bin loffset found the way
        htslib looks it up (the leaf bin of start, else the nearest earlier sibling / ancestor that exists)"""
        bins, lin, loff = self.index[rid]
        if lin is not None:
            w = start >> 14
            return lin[w] if w < len(lin) else (lin[-1] if lin else 0)
        first_leaf = ((1 << (3 * self.depth)) - 1) // 7
        b = first_leaf + (start >> self.min_shift)
        while b:
            if b in loff:
                return loff[b]
            parent = (b - 1) >> 3
            b = b - 1 if b > (parent << 3) + 1 else parent
        return loff.get(0, 0)

    def _anchors(self, rid):
        """record-aligned virtual offsets inside a contig's data: where the device ingest may cut its spans"""
        bins, lin, loff = self.index[rid]
        return sorted(set(lin if lin is not None else loff.values()))

    def get_reference_length(self, contig):
        return self.contigs[self.name_to_id[contig]][1]

    def count_mapped(self, contig):
        """mapped-read count of the pseudo-bin 37450 (what get_index_statistics reports), or None"""
        bins = self.index[self.name_to_id[contig]][0]
        ch = bins.get(self.meta_bin)
        return int(ch[1][0]) if ch and len(ch) > 1 else None

    def records(self, v, stop=1 << 64):
        """the raw records (without their block_size prefix) that start at virtual offsets from v up to `stop`, in file order"""
        while v < stop:
            d, v = self.bgzf.read_from(v, 4)
            if len(d) < 4:
                return
            bs = struct.unpack("<i", d)[0]
            b, v = self.bgzf.read_from(v, bs)
            if len(b) < bs:
                return
            yield b

    def fetch(self, contig, start, end):
        rid = self.name_to_id[contig]
        for vb, ve in self.merged_chunks(contig, start, end):
            for b in self.records(vb, ve):
                ref_id, pos = struct.unpack("<ii", b[:8])
                if ref_id > rid or pos >= end:
                    break
                if ref_id == rid:
                    r = decode_record(b)
                    if pos + max(ref_span(r["cigar"]), 1) > start:
                        yield r

    # ---- device ingest (snfb_load_bam): the index work stays on the host, the bytes stay compressed
    def merged_chunks(self, contig, start, end):
        """disjoint, ascending virtual-offset ranges holding every record `fetch(contig, start, end)` looks at (the BAI chunks of the
        region's bins behind the linear-index minimum, merged the way htslib merges them)"""
        rid = self.name_to_id[contig]
        bins = self.index[rid][0]
        min_off = self._min_offset(rid, max(start, 0))
        chunks = sorted(c for b in reg2bins(max(start, 0), max(end, start + 1), self.min_shift, self.depth) if b in bins and b != self.meta_bin
                        for c in bins[b] if c[1] > min_off)
        return [(a, b) for a, b in _merge_ranges((max(beg, min_off), stop) for beg, stop in chunks) if b > a]

    def device_input(self, regions, split=True, tags=None):
        """regions: [(contig, start, end)] = the tasks, in task order.  Returns (bgzf, spans): the compressed bytes of every BGZF block the
        regions need (file order, each block once) and abi.SPAN_DTYPE rows — the merged index chunks of each task, cut at the linear
        index's record-aligned offsets so that every ~16 kb window is its own parallel walk on the device.  tags: per query (task, region)
        for the spans (default: query k is task k, region 0); several queries of a task share its BGZF blocks, shipped once."""
        pieces = []                                      # (task, vbeg, vend, region)
        tags = tags if tags is not None else [(t, 0) for t in range(len(regions))]
        anchors_of = {}                                  # per contig, sorted once: each chunk bisects into them
        for (t, g), (contig, start, end) in zip(tags, regions):
            rid = self.name_to_id[contig]
            if split and rid not in anchors_of:
                anchors_of[rid] = self._anchors(rid)
            anchors = anchors_of.get(rid, [])
            for vb, ve in self.merged_chunks(contig, start, end):
                cuts = [vb] + anchors[bisect.bisect_right(anchors, vb):bisect.bisect_left(anchors, ve)] + [ve]
                pieces.extend((t, cuts[k], cuts[k + 1], g) for k in range(len(cuts) - 1))
        # file intervals [cb, ce) that hold the blocks of the pieces; a piece that ends inside a block needs that block too
        iv, bs_cache = [], {}
        for _, vb, ve, _ in pieces:
            cb, ce = vb >> 16, ve >> 16
            if ve & 0xffff:
                if ce not in bs_cache:
                    bs_cache[ce] = self.bgzf.member(ce)[0]
                ce += bs_cache[ce]
            iv.append((cb, ce))
        merged = _merge_ranges(sorted(iv))
        starts, base, parts = [], [], []
        off = 0
        for a, b in merged:
            self.bgzf.f.seek(a)
            d = self.bgzf.f.read(b - a)
            if len(d) != b - a:
                raise ValueError("truncated BAM file")
            starts.append(a)
            base.append(off)
            parts.append(d)
            off += len(d)
        bgzf = np.frombuffer(b"".join(parts), "u1") if parts else np.zeros(0, "u1")

        def to_buf(c):                                   # file offset of a block start (or of an interval's end) -> offset in bgzf
            k = bisect.bisect_right(starts, c) - 1
            if k < 0 or c > merged[k][1]:
                raise ValueError("virtual offset outside the loaded intervals")
            return base[k] + (c - starts[k])
        spans = np.zeros(len(pieces), abi.SPAN_DTYPE)
        for i, (t, vb, ve, g) in enumerate(pieces):
            spans[i] = (to_buf(vb >> 16), to_buf(ve >> 16), vb & 0xffff, ve & 0xffff, t, g)
        return bgzf, spans


def pack_records(contigs, recs, tasks, with_seq=True, tandem_repeats=None) -> RecordBlock:
    """records (already grouped by task, coordinate sorted inside a task) -> packed block of include/snfb.h.
    tasks: list of (contig index, start, end, task_id); recs: list of (task index, record dict[, region index])."""
    n = len(recs)
    rec = np.zeros(n, abi.REC_DTYPE)
    cig, var, seq = [], [], []
    co = vo = so = 0
    for i, (t, r, *g) in enumerate(recs):
        a = r["aux"]
        sa = a.get("SA", b"")
        flags = (abi.AUX_NM if "NM" in a else 0) | (abi.AUX_HP if "HP" in a else 0) | (abi.AUX_PS if "PS" in a else 0) | (abi.AUX_SA if "SA" in a else 0)
        if len(r["qname"]) > 255:
            raise ValueError("query name longer than 255 bytes")
        rec[i] = (t, r["pos"], r["flag"], r["mapq"], flags, int(a.get("HP", 0)) & 255, len(r["qname"]), 0,
                  int(a.get("NM", 0)), int(a.get("PS", 0)), len(r["cigar"]), r["l_seq"], len(sa), g[0] if g else 0, co, so, vo)
        cig.append(r["cigar"])
        var.append(np.frombuffer(r["qname"] + sa, "u1"))
        s = r["seq"] if with_seq else np.zeros((r["l_seq"] + 1) // 2, "u1")
        seq.append(s)
        co += len(r["cigar"])
        vo += len(r["qname"]) + len(sa)
        so += len(s)
    names = [c[0] for c in contigs]
    order = sorted(range(len(names)), key=lambda k: names[k].encode())
    rank = {k: i for i, k in enumerate(order)}
    ctg = np.zeros(len(contigs), abi.CONTIG_DTYPE)
    for k, (nm, ln) in enumerate(contigs):
        ctg[k] = (abi.fnv1a64(nm.encode()), ln, rank[k])
    task = np.zeros(len(tasks), abi.TASK_DTYPE)
    tr_flat, tr_off = [], 0
    for t, (c, start, end, tid) in enumerate(tasks):
        iv = sorted((tandem_repeats or {}).get(t, []))
        task[t] = (c, start, end, contigs[c][1], tid, tr_off, len(iv), 0)
        tr_flat.extend(x for ab in iv for x in ab)
        tr_off += len(iv)
    cat = lambda xs, dt: np.concatenate(xs).astype(dt) if xs else np.zeros(0, dt)
    return RecordBlock(rec=rec, cigar=cat(cig, "<u4"), var=cat(var, "u1"), seq=cat(seq, "u1"), task=task, contig=ctg,
                       tr=np.asarray(tr_flat, dtype="<i4"), contig_names=names, aligned_bp=0)


def bin_index(records, n_ref):
    """The BAI-layout tables of coordinate-sorted records (SAM spec §5.2; tabix uses the same layout): `records` yields (ref, beg, end, v0,
    v1) = the reference index, the 0-based half-open interval and the virtual offsets of the record's first byte and of the byte after it.
    Returns per reference (bins, linear index, stats): bins = {bin: [(v0, v1) chunks]} in order of first use, adjacent chunks of a bin
    merged; the linear index = per 16 kb window the smallest v0 of a record overlapping it, empty windows inheriting the previous offset;
    stats = [first v0, last v1, record count] (pseudo-bin 37450), first v0 None for a reference without records."""
    tabs = [({}, [], [None, None, 0]) for _ in range(n_ref)]
    for rid, pos, end, v0, v1 in records:
        bins, lin, st = tabs[rid]
        ch = bins.setdefault(reg2bin(pos, end), [])
        if ch and ch[-1][1] == v0:
            ch[-1] = (ch[-1][0], v1)
        else:
            ch.append((v0, v1))
        for w in range(pos >> 14, ((end - 1) >> 14) + 1):
            while len(lin) <= w:
                lin.append(0)
            if lin[w] == 0:
                lin[w] = v0
        st[0] = v0 if st[0] is None else st[0]
        st[1] = v1
        st[2] += 1
    for _, lin, _ in tabs:
        for w in range(1, len(lin)):                   # empty windows inherit the previous offset
            if lin[w] == 0:
                lin[w] = lin[w - 1]
    return tabs


def _bai_ref_bytes(bins, lin, st) -> bytes:
    """one reference of a BAI / TBI index: bins with their chunks, the pseudo-bin 37450, the linear index"""
    out = [struct.pack("<i", len(bins) + (1 if st[2] else 0))]
    for b, ch in bins.items():
        out.append(struct.pack("<Ii", b, len(ch)) + b"".join(struct.pack("<QQ", v0, v1) for v0, v1 in ch))
    if st[2]:
        out.append(struct.pack("<Ii", 37450, 2) + struct.pack("<QQ", st[0], st[1]) + struct.pack("<QQ", st[2], 0))
    out.append(struct.pack("<i", len(lin)) + struct.pack(f"<{len(lin)}Q", *lin))
    return b"".join(out)


_TBI_MAX = 1 << 29                                     # TBI's bins cover [0, 2^29)


def _vcf_interval(fields):
    """0-based half-open interval of a VCF line as htslib's tbx_parse1 derives it for the VCF preset (htslib tbx.c): beg = POS - 1;
    end = beg + len(REF), replaced by INFO END= (at the start of INFO or after a ';') when present and not '.', or by beg + 1 when that
    END <= beg"""
    beg = int(fields[1]) - 1
    end = beg + len(fields[3]) if len(fields) > 3 else beg + 1
    info = fields[7] if len(fields) > 7 else ""
    s = info[4:] if info.startswith("END=") else (info.split(";END=", 1)[1] if ";END=" in info else None)
    if s and s[0] != ".":
        k = 1 if s[0] in "+-" else 0
        while k < len(s) and s[k].isdigit():
            k += 1
        if k and s[:k] not in "+-":
            e = int(s[:k])
            end = e if e > beg else beg + 1
    return beg, end


def tabix_index(text: bytes, coffsets) -> bytes:
    """The uncompressed body of the .tbi index (tabix spec) of a VCF whose text was cut into BGZF members of 0xff00 bytes starting at
    the file offsets `coffsets` — what `pysam.tabix_index(..., preset="vcf")` writes.  Byte u of the text has the virtual offset
    coffsets[u // 0xff00] << 16 | u % 0xff00; the end of a text that fills its last block is (last block << 16 | 0xff00), as htslib's
    bgzf_tell reports it.  Lines starting with '#' are skipped; intervals follow _vcf_interval.  Raises ValueError, naming the line, for a
    contig that reappears after another one, a POS below the previous POS of the contig, or an interval beyond 2^29 — the input tabix
    refuses."""
    blk = 0xff00

    def voff(u):
        k = u // blk
        if k == len(coffsets) and k and u % blk == 0:
            return (coffsets[k - 1] << 16) | blk
        return (coffsets[k] << 16) | (u % blk)
    names, ids, placed = [], {}, []
    last_rid, last_beg = -1, -1
    u, n = 0, len(text)
    lineno = 0
    while u < n:
        e = text.find(b"\n", u)
        e = n if e < 0 else e + 1
        line = text[u:e].rstrip(b"\r\n")
        lineno += 1
        if line and not line.startswith(b"#"):
            f = line.decode().split("\t")
            try:
                beg, end = _vcf_interval(f)
            except (ValueError, IndexError):
                raise ValueError(f"line {lineno}: cannot parse the position of {line[:80]!r}") from None
            rid = ids.get(f[0])
            if rid is None:
                rid = ids[f[0]] = len(names)
                names.append(f[0])
            elif rid != last_rid:
                raise ValueError(f"line {lineno}: contig {f[0]!r} reappears after {names[last_rid]!r}: the VCF is not sorted ({line[:80]!r})")
            if rid == last_rid and beg < last_beg:
                raise ValueError(f"line {lineno}: POS {beg + 1} after POS {last_beg + 1} on {f[0]!r}: the VCF is not sorted ({line[:80]!r})")
            if beg < 0 or end > _TBI_MAX:
                raise ValueError(f"line {lineno}: interval {beg}..{end} on {f[0]!r} lies outside the 2^29 range of a TBI index ({line[:80]!r})")
            placed.append((rid, beg, end, voff(u), voff(e)))
            last_rid, last_beg = rid, beg
        u = e
    nm = b"".join(x.encode() + b"\0" for x in names)
    out = [b"TBI\1", struct.pack("<8i", len(names), 2, 1, 2, 0, ord("#"), 0, len(nm)), nm]   # n_ref, VCF preset: format, col_seq/beg/end, meta, skip
    out += [_bai_ref_bytes(*t) for t in bin_index(placed, len(names))]
    return b"".join(out)


# ------------------------------------------------------------------------------------------------ building an index (sniffles_b200.index)
# device memory per inflated byte of a window (the window's inflated and compressed bytes, the candidate masks and the chain's nodes) and
# the share of the free memory a window may plan on
INDEX_DEVICE_BYTES_PER_INFLATED_BYTE = 4
INDEX_FREE_MEMORY_SHARE = 0.8


def csi_depth(contigs, min_shift):
    """htslib's CSI depth for a BAM (bam_index): the fewest levels whose top bin covers the longest contig + 256"""
    max_len, depth, s = max((ln for _, ln in contigs), default=0) + 256, 0, 1 << min_shift
    while max_len > s:
        depth += 1
        s <<= 3
    return depth


def index_window_bytes(device=0):
    """the inflated bytes of one window of build_index: the device's free memory share over INDEX_DEVICE_BYTES_PER_INFLATED_BYTE"""
    import torch
    free, _ = torch.cuda.mem_get_info(device)
    return max(1 << 20, int(free * INDEX_FREE_MEMORY_SHARE / INDEX_DEVICE_BYTES_PER_INFLATED_BYTE))


def index_bytes(tab, n_ref, fmt, min_shift, depth) -> bytes:
    """the uncompressed index file of tables `tab` (the dict of binding.Context.index_bam): BAI (SAM spec §5.2) or the CSI body (§5.3).
    Bins are written in ascending order, each reference's pseudo-bin last; htslib writes them in its hash table's order, so two indexes
    compare as tables, not as bytes."""
    n_bins = ((1 << (3 * (depth + 1))) - 1) // 7
    meta = n_bins + 1
    keys = np.asarray(tab["bin_key"], dtype=np.uint64)
    ref_of = keys // np.uint64(n_bins)
    bin_of = keys % np.uint64(n_bins)
    cb = np.asarray(tab["chunk_bin"], dtype=np.int64)
    starts = np.searchsorted(cb, np.arange(len(keys) + 1))            # chunks are grouped by bin, in bin order
    live = np.diff(starts) > 0                                        # a bin that moved its chunks to its parent is not written
    out = [b"BAI\1" + struct.pack("<i", n_ref)] if fmt == "bai" else [b"CSI\1" + struct.pack("<iiii", min_shift, depth, 0, n_ref)]
    first = np.searchsorted(ref_of, np.arange(n_ref + 1, dtype=np.uint64))
    for t in range(n_ref):
        st = tab["ref"][t]
        has = int(st[0]) != 0xFFFFFFFFFFFFFFFF
        out.append(struct.pack("<i", int(live[first[t]:first[t + 1]].sum()) + has))
        for b in range(int(first[t]), int(first[t + 1])):
            c0, c1 = int(starts[b]), int(starts[b + 1])
            if c0 == c1:
                continue
            head = struct.pack("<Ii", int(bin_of[b]), c1 - c0) if fmt == "bai" else struct.pack("<IQi", int(bin_of[b]), int(tab["bin_loff"][b]), c1 - c0)
            pairs = np.empty((c1 - c0, 2), "<u8")
            pairs[:, 0], pairs[:, 1] = tab["chunk_beg"][c0:c1], tab["chunk_end"][c0:c1]
            out.append(head + pairs.tobytes())
        if has:
            head = struct.pack("<Ii", meta, 2) if fmt == "bai" else struct.pack("<IQi", meta, 0, 2)
            out.append(head + struct.pack("<QQQQ", int(st[0]), int(st[1]), int(st[2]), int(st[3])))
        if fmt == "bai":
            lo, hi = int(tab["lin_off"][t]), int(tab["lin_off"][t + 1])
            out.append(struct.pack("<i", hi - lo) + np.asarray(tab["lin"][lo:hi], "<u8").tobytes())
    out.append(struct.pack("<Q", int(tab["n_no_coor"])))
    return b"".join(out)


def build_index(path, fmt="bai", min_shift=14, device=0, window_bytes=None, ctx=None, stats=None) -> bytes:
    """The .bai / .csi file of the coordinate-sorted BAM at `path`, as `samtools index [-c [-m min_shift]]` builds it: the record
    boundaries, rows and tables on the GPU (snfb_index_bam), the file streamed through the device in windows of `window_bytes` inflated
    bytes (default: index_window_bytes); the host only serializes the tables, and a CSI is BGZF-compressed on the GPU.  Raises
    ValueError for a file that is not a BAM, binding.SnfbError (naming the record or the block) for one the device refuses.  stats: a dict
    that receives n_records, n_windows, device_bytes and device_ms."""
    from . import binding
    if fmt not in ("bai", "csi"):
        raise ValueError(f"unknown index format {fmt!r}")
    reader = BgzfReader(path)
    try:
        contigs, first = read_header(reader)
    finally:
        reader.close()
    min_shift, depth = (14, 5) if fmt == "bai" else (int(min_shift), csi_depth(contigs, int(min_shift)))
    own = ctx is None
    ctx = ctx or binding.Context(device)
    try:
        tab = ctx.index_bam(path, first, [ln for _, ln in contigs], min_shift, depth, window_bytes or index_window_bytes(device))
        body = index_bytes(tab, len(contigs), fmt, min_shift, depth)
        if fmt == "csi":
            body = ctx.deflate_bgzf(body)[0] + _BGZF_EOF
    finally:
        if own:
            ctx.close()
    if stats is not None:
        stats.update((k, tab[k]) for k in ("n_records", "n_windows", "device_bytes", "device_ms"))
    return body


# ------------------------------------------------------------------------------------------------ sorting a BAM (sniffles_b200.sort)
# device memory per inflated byte of the two budgets together: an input window takes INDEX_DEVICE_BYTES_PER_INFLATED_BYTE, an output bucket
# three (its bytes, the encoder's member slots, the packed members); the rest is left for the per-record keys, lengths and offsets
SORT_DEVICE_BYTES_PER_INFLATED_BYTE = 8


def sort_budget_bytes(device=0):
    """the default window_bytes and bucket_bytes of sort_bam: each the device's free memory share over SORT_DEVICE_BYTES_PER_INFLATED_BYTE"""
    import torch
    free, _ = torch.cuda.mem_get_info(device)
    return max(1 << 20, int(free * INDEX_FREE_MEMORY_SHARE / SORT_DEVICE_BYTES_PER_INFLATED_BYTE))


def read_header_bytes(bgzf):
    """the BAM header through a BgzfReader -> (its inflated bytes from the magic through the references, contigs, virtual offset of the
    first record)"""
    contigs, first = read_header(bgzf)
    l_text = struct.unpack("<i", bgzf.read_from(0, 8)[0][4:8])[0]
    n = 12 + l_text + sum(9 + len(name.encode()) for name, _ in contigs)
    return bgzf.read_from(0, n)[0], contigs, first


def sort_header(header: bytes) -> bytes:
    """the BAM header `header` as a coordinate sort writes it: the first text line, when it is @HD, gets SO:coordinate (its SO field
    replaced, or appended); without an @HD line, "@HD\\tVN:1.6\\tSO:coordinate" is put first.  Everything else is kept byte for byte."""
    l_text = struct.unpack("<i", header[4:8])[0]
    text, rest = header[8:8 + l_text], header[8 + l_text:]
    nl = text.find(b"\n")
    first, tail = (text, b"") if nl < 0 else (text[:nl], text[nl:])
    if first.startswith(b"@HD\t") or first == b"@HD":
        fields = first.split(b"\t")
        so = [k for k, f in enumerate(fields) if f.startswith(b"SO:")]
        if so:
            fields[so[0]] = b"SO:coordinate"
        else:
            fields.append(b"SO:coordinate")
        text = b"\t".join(fields) + tail
    else:
        text = b"@HD\tVN:1.6\tSO:coordinate\n" + text
    return header[:4] + struct.pack("<i", len(text)) + text + rest


def sort_bam(path, out_path, device=0, window_bytes=None, bucket_bytes=None, ctx=None, stats=None):
    """Write the BAM at `path` sorted by coordinate to `out_path`, as `samtools sort` orders it and cuts its BGZF members
    (snfb_sort_bam; the rules are in include/snfb.h and DESIGN §4): the input streamed through the device in windows of `window_bytes`
    inflated bytes for the keys, the output assembled and compressed on the device in buckets of `bucket_bytes` (defaults:
    sort_budget_bytes).  The header is sort_header's.  Raises ValueError for a file that is not a BAM, binding.SnfbError (naming the record
    or the block) for one the device refuses; out_path may then hold a partial file.  stats: a dict that receives n_records, n_windows,
    n_buckets, n_members, n_input_reads, bytes_in, bytes_out, device_bytes and the device milliseconds ms_keys, ms_sort, ms_layout,
    ms_scatter, ms_deflate (ms_layout_host: the host's member-cut loop)."""
    from . import binding
    reader = BgzfReader(path)
    try:
        header, contigs, first = read_header_bytes(reader)
    finally:
        reader.close()
    own = ctx is None
    ctx = ctx or binding.Context(device)
    try:
        budget = sort_budget_bytes(device) if window_bytes is None or bucket_bytes is None else 0
        view = ctx.sort_bam(path, out_path, sort_header(header), first, [ln for _, ln in contigs], window_bytes or budget, bucket_bytes or budget)
    finally:
        if own:
            ctx.close()
    if stats is not None:
        stats.update(view)
    return view


# ------------------------------------------------------------------------------------------------ writer (tests / benchmark inputs)
def _bgzf_block(data: bytes, level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY) -> bytes:
    """one BGZF member: the header with its BC subfield, the raw DEFLATE stream of `data` from zlib, the CRC-32 / ISIZE trailer"""
    c = zlib.compressobj(level, zlib.DEFLATED, -15, 8, strategy)
    comp = c.compress(data) + c.flush()
    if len(comp) + 26 > 65536:
        raise ValueError(f"a BGZF member holds at most 65536 bytes; this one would take {len(comp) + 26}")
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", len(comp) + 25) + comp
            + struct.pack("<II", zlib.crc32(data), len(data)))


def write_bam(path, blk: RecordBlock, block_bytes=0xff00, level=6, qual_seed=None, index="bai"):
    """packed block -> coordinate-sorted BAM + BAI (records keep the block's order; one contig per task).  Returns the paths.
    qual_seed: None writes the "qualities absent" bytes 0xff; an integer writes noisy phred values (what makes a real BAM hard to compress).
    index: "bai" or "csi" (the BAI bin geometry, min_shift 14 / depth 5, with per-bin loffsets derived from the linear index as htslib derives them)."""
    qrng = np.random.default_rng(qual_seed) if qual_seed is not None else None
    names = blk.contig_names
    text = b"@HD\tVN:1.6\tSO:coordinate\n" + b"".join(f"@SQ\tSN:{n}\tLN:{int(c['length'])}\n".encode() for n, c in zip(names, blk.contig))
    head = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(names))
    for n, c in zip(names, blk.contig):
        head += struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", int(c["length"]))
    out = open(path, "wb")
    buf, coff = bytearray(), 0
    placed = []                                        # (ref, beg, end, v0, v1) of every record

    def flush():
        nonlocal buf, coff
        if buf:
            blk_b = _bgzf_block(bytes(buf), level)
            out.write(blk_b)
            coff += len(blk_b)
            buf = bytearray()

    def put(data):
        """append to the BGZF stream -> virtual offsets of the first byte and of the byte after the end"""
        nonlocal buf
        if len(buf) + len(data) > block_bytes:
            flush()
        v0 = (coff << 16) | len(buf)
        if len(data) > block_bytes:                    # larger than one block: cut into block_bytes pieces, flushed as each fills
            for k in range(0, len(data), block_bytes):
                buf += data[k:k + block_bytes]
                if len(buf) >= block_bytes:
                    flush()
        else:
            buf += data
        return v0, (coff << 16) | len(buf)
    put(head)
    flush()
    for r in blk.rec:
        rid = int(blk.task[int(r["task"])]["contig"])
        co, nco = int(r["cigar_off"]), int(r["n_cigar"])
        cig = np.ascontiguousarray(blk.cigar[co:co + nco], dtype="<u4")
        vo, lq, sl = int(r["var_off"]), int(r["l_qname"]), int(r["sa_len"])
        qname = bytes(blk.var[vo:vo + lq]) + b"\0"
        sa = bytes(blk.var[vo + lq:vo + lq + sl])
        l_seq = int(r["l_seq"])
        seq = bytes(blk.seq[int(r["seq_off"]):int(r["seq_off"]) + (l_seq + 1) // 2])
        aux = b""
        af = int(r["aux_flags"])
        if af & abi.AUX_NM:
            aux += b"NMi" + struct.pack("<i", int(r["nm"]))
        if af & abi.AUX_HP:
            aux += b"HPC" + struct.pack("<B", int(r["hp"]))
        if af & abi.AUX_PS:
            aux += b"PSi" + struct.pack("<i", int(r["ps"]))
        if af & abi.AUX_SA:
            aux += b"SAZ" + sa + b"\0"
        pos = int(r["pos"])
        end = pos + max(ref_span(cig), 1)
        n_cig, cig_b = nco, cig.tobytes()
        if nco > 65535:                                # long CIGAR escape
            aux += b"CGBI" + struct.pack("<I", nco) + cig_b
            cig_b = struct.pack("<II", (l_seq << 4) | 4, ((end - pos) << 4) | 3)
            n_cig = 2
        body = struct.pack("<iiBBHHHiiii", rid, pos, len(qname), int(r["mapq"]), reg2bin(pos, end), n_cig, int(r["flag"]), l_seq, -1, -1, 0) \
            + qname + cig_b + seq + (b"\xff" * l_seq if qrng is None else np.clip(qrng.normal(22.0, 9.0, l_seq), 2, 50).astype("u1").tobytes()) + aux
        placed.append((rid, pos, end, *put(struct.pack("<i", len(body)) + body)))
    flush()
    out.write(_BGZF_EOF)
    out.close()
    tabs = bin_index(placed, len(names))
    if index == "csi":
        body = b"CSI\1" + struct.pack("<iii", 14, 5, 0) + struct.pack("<i", len(names))
        level_first = [((1 << (3 * l)) - 1) // 7 for l in range(6)]
        for bins, lin, st in tabs:
            body += struct.pack("<i", len(bins) + (1 if st[2] else 0))
            for b, ch in bins.items():
                lvl = max(l for l in range(6) if level_first[l] <= b)
                w = (b - level_first[lvl]) << (3 * (5 - lvl))
                body += struct.pack("<IQi", b, lin[w] if w < len(lin) else 0, len(ch)) + b"".join(struct.pack("<QQ", v0, v1) for v0, v1 in ch)
            if st[2]:
                body += struct.pack("<IQi", 37450, 0, 2) + struct.pack("<QQ", st[0], st[1]) + struct.pack("<QQ", st[2], 0)
        with open(path + ".csi", "wb") as f:
            for k in range(0, len(body), 0xff00):
                f.write(_bgzf_block(body[k:k + 0xff00], level))
            f.write(_BGZF_EOF)
        return path, path + ".csi"
    with open(path + ".bai", "wb") as f:
        f.write(b"BAI\1" + struct.pack("<i", len(names)) + b"".join(_bai_ref_bytes(*t) for t in tabs))
    return path, path + ".bai"
