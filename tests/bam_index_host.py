"""The host restatement of bamio.build_index's tables: the records walked one by one from the end of the header (the way BamFile.records
walks them), pushed into the bins and the linear index as htslib's hts_idx_push does, finished as hts_idx_finish does (update_loff: an
empty linear-index window takes the next window's offset; then compress_binning: the parent merge level by level from the leaves, the
chunks of a bin sorted and those starting in the block where the previous one ends merged).  Returns the dict that
binding.Context.index_bam returns, so bamio.index_bytes serializes both alike."""
import struct

import numpy as np

from sniffles_b200 import bamio

NONE = 0xFFFFFFFFFFFFFFFF


def _bin_level(b):
    level = 0
    while b:
        b, level = (b - 1) >> 3, level + 1
    return level


def _reg2bin(beg, end, min_shift, depth):
    end -= 1
    s, t = min_shift, ((1 << (3 * depth)) - 1) // 7
    for level in range(depth, 0, -1):
        if beg >> s == end >> s:
            return t + (beg >> s)
        s += 3
        t -= 1 << (3 * (level - 1))
    return 0


def rows(path, limit=None):
    """(contigs, [(tid, beg, end, v0, v1, mapped)] in file order); end = htslib's bam_endpos.  limit: stop after that many records"""
    reader = bamio.BgzfReader(path)
    try:
        contigs, v = bamio.read_header(reader)
        out = []
        while limit is None or len(out) < limit:
            d, v1 = reader.read_from(v, 4)
            if not d:
                break
            if len(d) < 4:
                raise ValueError(f"truncated record at virtual offset {v >> 16}:{v & 0xffff}")
            bs = struct.unpack("<i", d)[0]
            b, v2 = reader.read_from(v1, bs)
            if len(b) < bs:
                raise ValueError(f"truncated record at virtual offset {v >> 16}:{v & 0xffff}")
            tid, pos, l_rn, _mapq, _bin, n_cig, flag = struct.unpack("<iiBBHHH", b[:16])
            span = 0 if flag & 4 else bamio.ref_span(np.frombuffer(b[32 + l_rn:32 + l_rn + 4 * n_cig], "<u4"))
            out.append((tid, pos, pos + (span if span > 0 else 1), v, v2, not flag & 4))
            v = v2
        return contigs, out
    finally:
        reader.close()


def tables(contigs, recs, min_shift=14, depth=5):
    """htslib's index tables of `recs` (rows()): raises ValueError naming the record for an order the index refuses"""
    n_ref = len(contigs)
    n_bins = ((1 << (3 * (depth + 1))) - 1) // 7
    max_end = 1 << (min_shift + 3 * depth)
    bidx = [{} for _ in range(n_ref)]                 # bin -> [[u, v], ...]
    lidx = [[] for _ in range(n_ref)]
    meta = [None] * n_ref
    n_no_coor = 0
    last_tid = save_tid = -1
    last_bin = save_bin = None
    last_coor = -1
    last_off = off_beg = recs[0][3] if recs else 0
    save_off = last_off
    n_mapped = n_unmapped = 0
    for k, (tid, beg, end, v0, v1, mapped) in enumerate(recs):
        if tid >= 0 and end > max_end:
            raise ValueError(f"record {k + 1}: end {end} beyond the {max_end} positions of the index geometry")
        if tid != last_tid:
            if (last_tid == -1 and k and tid >= 0) or (tid >= 0 and tid < last_tid):
                raise ValueError(f"record {k + 1}: reference #{tid} after reference #{last_tid}")
            last_tid, last_bin = tid, None
        elif tid >= 0 and last_coor > beg:
            raise ValueError(f"record {k + 1}: unsorted positions on reference #{tid}: {beg + 1} after {last_coor + 1}")
        if tid >= 0:
            beg, end = max(beg, 0), (end if end > 0 else 1)
            for w in range(beg >> min_shift, ((end - 1) >> min_shift) + 1):
                lin = lidx[tid]
                while len(lin) <= w:
                    lin.append(None)
                if lin[w] is None:
                    lin[w] = last_off
        else:
            n_no_coor += 1
            beg, end = -1, 0
        b = _reg2bin(beg, end, min_shift, depth) if tid >= 0 else -1
        if last_bin != b:
            if save_bin is not None and save_tid >= 0:
                bidx[save_tid].setdefault(save_bin, []).append([save_off, last_off])
            if last_bin is None and save_bin is not None and save_tid >= 0:         # change of reference: its pseudo-bin
                meta[save_tid] = (off_beg, last_off, n_mapped, n_unmapped)
                n_mapped = n_unmapped = 0
                off_beg = last_off
            elif last_bin is None and save_bin is not None:
                n_mapped = n_unmapped = 0
                off_beg = last_off
            save_off, save_bin, last_bin, save_tid = last_off, b, b, tid
        if mapped:
            n_mapped += 1
        else:
            n_unmapped += 1
        last_off, last_coor = v1, beg
    if save_tid >= 0 and save_bin is not None:
        bidx[save_tid].setdefault(save_bin, []).append([save_off, last_off])
        meta[save_tid] = (off_beg, last_off, n_mapped, n_unmapped)
    ref = np.zeros((n_ref, 5), "<u8")
    keys, loffs, cb, cu, cv, lin_all, lin_off = [], [], [], [], [], [], [0]
    for t in range(n_ref):
        lin, bins = lidx[t], bidx[t]
        for w in range(len(lin) - 2, -1, -1):         # update_loff: an empty window takes the next window's offset (the last one is set)
            if lin[w] is None:
                lin[w] = lin[w + 1]
        loff = {}
        for b in bins:
            level = _bin_level(b)
            bot = (b - ((1 << (3 * level)) - 1) // 7) << (3 * (depth - level))
            loff[b] = lin[bot] if bot < len(lin) else 0
        for level in range(depth, 0, -1):              # compress_binning
            for b in sorted(x for x in list(bins) if _bin_level(x) == level):
                ch = sorted(bins[b])
                bins[b] = ch
                parent = (b - 1) >> 3
                if (ch[-1][1] >> 16) - (ch[0][0] >> 16) < 0x10000 and parent in bins:
                    bins[parent].extend(ch)
                    del bins[b]
        for b in sorted(bins):
            ch = sorted(bins[b])
            merged = [list(ch[0])]
            for u, v in ch[1:]:
                if merged[-1][1] >> 16 >= u >> 16:
                    merged[-1][1] = max(merged[-1][1], v)
                else:
                    merged.append([u, v])
            for u, v in merged:
                cb.append(len(keys))
                cu.append(u)
                cv.append(v)
            keys.append(t * n_bins + b)
            loffs.append(loff[b])
        ref[t] = (meta[t][0], meta[t][1], meta[t][2], meta[t][3], len(lin)) if meta[t] else (NONE, 0, 0, 0, len(lin))
        lin_all.extend(lin)
        lin_off.append(len(lin_all))
    return dict(ref=ref, lin_off=np.asarray(lin_off, "<u8"), lin=np.asarray(lin_all, "<u8"), bin_key=np.asarray(keys, "<u8"),
                bin_loff=np.asarray(loffs, "<u8"), chunk_bin=np.asarray(cb, "<u4"), chunk_beg=np.asarray(cu, "<u8"), chunk_end=np.asarray(cv, "<u8"),
                n_no_coor=n_no_coor, n_records=len(recs))


def host_index(path, fmt="bai", min_shift=14, limit=None):
    """(index file body, uncompressed, and the tables) of the BAM at `path`, by the host restatement"""
    contigs, recs = rows(path, limit)
    ms, depth = (14, 5) if fmt == "bai" else (min_shift, bamio.csi_depth(contigs, min_shift))
    tab = tables(contigs, recs, ms, depth)
    return bamio.index_bytes(tab, len(contigs), fmt, ms, depth), tab


def hg008_bam(path):
    """Write a BAM with the byte layout of the reference's test data hg008.bam, whose htslib-written index is tests/golden/bams/hg008.bam.csi:
    the same 218 contigs, the same 16 records (reference, position, flag, CIGAR, read-name and sequence lengths from hg008_bnd.npz), each
    with its original block_size, cut into BGZF members of the original inflated sizes, each member padded to its original total size with
    an extra gzip subfield.  Every record therefore sits at its original virtual offsets, and the file's index tables are htslib's.  Bases,
    qualities and tags are filler (the index never reads them), so the members compress far below their original sizes before the padding."""
    import json
    import os
    import zlib
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    with open(os.path.join(golden, "bams", "hg008_layout.json")) as f:
        lay = json.load(f)
    z = np.load(os.path.join(golden, "hg008_bnd.npz"))
    rec, cig, var, task, ctg = (z[f"hg008_{k}"] for k in ("rec", "cigar", "var", "task", "contig"))
    names = [str(x) for x in z["hg008_names"]]
    refs = b"".join(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", int(c["length"])) for n, c in zip(names, ctg))
    l_text = lay["members"][0][1] - 12 - len(refs)                   # the header fills the first member
    text = b"@HD\tVN:1.6\tSO:coordinate\n@CO\t"
    text += b"x" * (l_text - len(text) - 1) + b"\n"
    stream = [b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(names)) + refs]
    for r, bs in zip(rec, lay["block_size"]):
        c = cig[int(r["cigar_off"]):int(r["cigar_off"]) + int(r["n_cigar"])].astype("<u4")
        qname = bytes(var[int(r["var_off"]):int(r["var_off"]) + int(r["l_qname"])]) + b"\0"
        l_seq, pos = int(r["l_seq"]), int(r["pos"])
        end = pos + max(bamio.ref_span(c) if not int(r["flag"]) & 4 else 0, 1)
        body = struct.pack("<iiBBHHHiiii", int(task[int(r["task"])]["contig"]), pos, len(qname), int(r["mapq"]), bamio.reg2bin(pos, end), len(c),
                           int(r["flag"]), l_seq, -1, -1, 0) + qname + c.tobytes() + b"\x11" * ((l_seq + 1) // 2) + b"\x1e" * l_seq
        pad = bs - len(body)
        assert pad >= 4, "the record's tags leave room for one filler tag"
        stream.append(struct.pack("<i", bs) + body + b"XXZ" + b"A" * (pad - 4) + b"\0")
    data, out, u = b"".join(stream), [], 0
    assert len(data) == sum(isize for _, isize in lay["members"])
    for bsize, isize in lay["members"]:
        chunk = data[u:u + isize]
        u += isize
        comp = zlib.compress(chunk, 9)[2:-4]
        pad = bsize - 26 - len(comp)                                     # 18 header bytes with BC, 8 trailer bytes
        if pad:
            assert 4 <= pad <= 0xffff - 10, "a member must compress below its original size"
        extra = b"BC\x02\x00" + struct.pack("<H", bsize - 1) + ((b"ZZ" + struct.pack("<H", pad - 4) + b"\0" * (pad - 4)) if pad else b"")
        out.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff" + struct.pack("<H", len(extra)) + extra + comp
                   + struct.pack("<II", zlib.crc32(chunk), isize))
        assert len(out[-1]) == bsize
    with open(path, "wb") as f:
        f.write(b"".join(out))
    return path


def fixture_bam(name, tmp):
    """the path of an htslib-indexed fixture BAM: hg002.bam as committed, hg008.bam rewritten under `tmp` by hg008_bam; its index is
    tests/golden/bams/<name>.bam.csi either way"""
    import os
    if name == "hg008":
        return hg008_bam(os.path.join(str(tmp), "hg008.bam"))
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bams", name + ".bam")


def parse_index(data):
    """a .bai / .csi file (CSI BGZF-compressed or not) -> {"refs": [{bin: (loffset or None, [(u, v), ...])}], "lin": [[...]] or None,
    "n_no_coor", "min_shift", "depth"}: the tables, independent of the order the bins were written in"""
    import zlib
    if data[:2] == b"\x1f\x8b":
        d, o = b"", 0
        while o < len(data):
            dec = zlib.decompressobj(31)
            d += dec.decompress(data[o:])
            o = len(data) - len(dec.unused_data)
        data = d
    csi = data[:4] == b"CSI\1"
    if csi:
        min_shift, depth, l_aux = struct.unpack("<iii", data[4:16])
        p = 16 + l_aux
    else:
        assert data[:4] == b"BAI\1"
        min_shift, depth, p = 14, 5, 4
    n_ref = struct.unpack_from("<i", data, p)[0]
    p += 4
    refs, lins = [], []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", data, p)[0]
        p += 4
        bins = {}
        for _ in range(n_bin):
            if csi:
                b, lo, nc = struct.unpack_from("<IQi", data, p)
                p += 16
            else:
                (b, nc), lo = struct.unpack_from("<Ii", data, p), None
                p += 8
            bins[b] = (lo, [struct.unpack_from("<QQ", data, p + 16 * k) for k in range(nc)])
            p += 16 * nc
        refs.append(bins)
        if not csi:
            n_intv = struct.unpack_from("<i", data, p)[0]
            lins.append(list(struct.unpack_from(f"<{n_intv}Q", data, p + 4)))
            p += 4 + 8 * n_intv
    n_no_coor = struct.unpack_from("<Q", data, p)[0] if p + 8 <= len(data) else None
    return dict(refs=refs, lin=None if csi else lins, n_no_coor=n_no_coor, min_shift=min_shift, depth=depth)
