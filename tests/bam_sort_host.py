"""The host restatement of bamio.sort_bam: records read one by one with bamio's BGZF reader, sorted stably by samtools' coordinate key
(bam_sort.c bam1_cmp_core: tid as unsigned so -1 is last, then pos + 1, then the reverse-strand bit), the header's @HD line given
SO:coordinate, and the stream cut into BGZF members as htslib's writer cuts them (bam_hdr_write + bgzf_flush, then bam_write1 ->
bgzf_flush_try / bgzf_write at BGZF_BLOCK_SIZE 0xff00), each member compressed by zlib."""
import random
import struct
import zlib

from sniffles_b200 import bamio

BLOCK = 0xff00


def records(path):
    """(header bytes from the magic through the references, [raw record bytes with their block_size prefix] in file order)"""
    reader = bamio.BgzfReader(path)
    try:
        header, _contigs, v = bamio.read_header_bytes(reader)
        out = []
        while True:
            d, v1 = reader.read_from(v, 4)
            if not d:
                break
            bs = struct.unpack("<i", d)[0]
            b, v = reader.read_from(v1, bs)
            out.append(d + b)
        return header, out
    finally:
        reader.close()


def n_ref(header):
    l_text = struct.unpack_from("<i", header, 4)[0]
    return struct.unpack_from("<i", header, 8 + l_text)[0]


def key(rec, n_contig):
    """samtools' coordinate order as one integer (the device key)"""
    tid, pos = struct.unpack_from("<ii", rec, 4)
    flag = struct.unpack_from("<H", rec, 18)[0]
    return ((n_contig if tid < 0 else tid) << 33) | ((pos + 1) << 1) | ((flag >> 4) & 1)


def sort_records(header, recs):
    n = n_ref(header)
    return sorted(recs, key=lambda r: key(r, n))                      # Python's sort is stable


def header_text(header):
    l_text = struct.unpack_from("<i", header, 4)[0]
    return header[8:8 + l_text]


def rewrite_header(header):
    """SO:coordinate on the @HD line (replaced or appended), or a new @HD line first"""
    text = header_text(header)
    lines = text.split(b"\n")
    if lines[0].split(b"\t")[0] == b"@HD":
        f = [x for x in lines[0].split(b"\t") if not x.startswith(b"SO:")]
        k = next((i for i, x in enumerate(lines[0].split(b"\t")) if x.startswith(b"SO:")), None)
        f.insert(k if k is not None else len(f), b"SO:coordinate")
        lines[0] = b"\t".join(f)
        text = b"\n".join(lines)
    else:
        text = b"@HD\tVN:1.6\tSO:coordinate\n" + text
    return header[:4] + struct.pack("<i", len(text)) + text + header[8 + len(header_text(header)):]


def member_sizes(header_len, rec_lens):
    """inflated sizes of the members htslib writes for a header of header_len bytes and records of rec_lens (4 + block_size) bytes"""
    out = []
    left = header_len
    while left:
        out.append(min(left, BLOCK))
        left -= out[-1]
    cur = 0
    for r in rec_lens:
        if cur and cur + r > BLOCK:
            out.append(cur)
            cur = 0
        while r:
            take = min(r, BLOCK - cur)
            cur, r = cur + take, r - take
            if cur == BLOCK:
                out.append(cur)
                cur = 0
    if cur:
        out.append(cur)
    return out


def sorted_stream(path):
    """(inflated stream, member ISIZEs) of the sorted BAM"""
    header, recs = records(path)
    header = rewrite_header(header)
    recs = sort_records(header, recs)
    return header + b"".join(recs), member_sizes(len(header), [len(r) for r in recs])


def write_sorted(path, out_path):
    data, sizes = sorted_stream(path)
    with open(out_path, "wb") as f:
        u = 0
        for s in sizes:
            f.write(bamio._bgzf_block(data[u:u + s]))
            u += s
        f.write(bamio._BGZF_EOF)
    return out_path


def members(path):
    """(ISIZE, inflated bytes) of every member of a BGZF file, each checked against its CRC-32 and ISIZE"""
    z = open(path, "rb").read()
    out = []
    for o, po, pl, isize in bamio.bgzf_members(z):
        data = zlib.decompress(z[po:po + pl], -15)
        bsize = bamio.bgzf_header(z, o)[0]
        crc = struct.unpack_from("<I", z, o + bsize - 8)[0]
        assert len(data) == isize and zlib.crc32(data) == crc, f"member at {o}"
        out.append((isize, data))
    return out


def shuffled_bam(path, out_path, seed=1, sort_order=None):
    """the records of `path` in a seeded random order that keeps records of equal keys in their relative order, written with htslib's
    cuts; sort_order: the @HD SO value to put in the header (None keeps the header)"""
    header, recs = records(path)
    n = n_ref(header)
    rng = random.Random(seed)
    by_key = {}
    for r in recs:
        by_key.setdefault(key(r, n), []).append(r)
    slots = [k for k, rs in by_key.items() for _ in rs]
    rng.shuffle(slots)
    nxt = {k: iter(rs) for k, rs in by_key.items()}
    out = [next(nxt[k]) for k in slots]
    if sort_order is not None:
        text = header_text(header)
        lines = text.split(b"\n")
        if lines[0].startswith(b"@HD"):
            lines[0] = b"\t".join(x if not x.startswith(b"SO:") else b"SO:" + sort_order for x in lines[0].split(b"\t"))
        text = b"\n".join(lines)
        header = header[:4] + struct.pack("<i", len(text)) + text + header[8 + len(header_text(header)):]
    data = header + b"".join(out)
    with open(out_path, "wb") as f:
        u = 0
        for s in member_sizes(len(header), [len(r) for r in out]):
            f.write(bamio._bgzf_block(data[u:u + s]))
            u += s
        f.write(bamio._BGZF_EOF)
    return out_path
