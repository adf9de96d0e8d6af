"""The reference FASTA of `--reference`, held on the device: the `pysam.FastaFile` surface the reference touches (`fetch`, `references`,
`lengths`; leadprov.py:420-443, vcf.py:108-119 and 299-342) over a genome that snfb_load_reference unwraps on the GPU, plus its runs of
'N' for LeadProvider._mask_N_coverage.

  * The index is `path + ".fai"`.  A plain-text FASTA without one is indexed in memory by htslib's fai_build rules (the name is the header
    up to the first whitespace; every line of a sequence but the last has the same length; a duplicate name or a changed line length is an
    error naming the sequence).  No file is written (the reference writes one through pysam.faidx).
  * A BGZF FASTA needs its .fai (no .gzi): the BGZF member headers map each contig's byte range to the members that cover it, so only the
    loaded contigs' members are shipped and inflated (on the device, CRC-checked).  Plain gzip is refused, as pysam refuses it.
  * `fetch` resolves pysam's rules on the host and gathers on the device; `prefetch` serves a whole call set with one gather."""
import logging
import os
import struct

import numpy as np

from . import abi

class ReferenceError(ValueError):
    """the FASTA or its index cannot be used"""


FAI_DTYPE = np.dtype([("length", "<u8"), ("offset", "<u8"), ("linebases", "<u4"), ("linewidth", "<u4")])


def parse_fai(text):
    """.fai text -> (names, FAI_DTYPE rows).  Columns NAME LENGTH OFFSET LINEBASES LINEWIDTH (extra columns, as for FASTQ, ignored)."""
    names, rows = [], []
    for k, line in enumerate(text.splitlines()):
        if not line.strip():
            continue
        f = line.split("\t")
        if len(f) < 5:
            raise ReferenceError(f"malformed .fai line {k + 1}: {line!r}")
        try:
            rows.append((int(f[1]), int(f[2]), int(f[3]), int(f[4])))
        except ValueError:
            raise ReferenceError(f"malformed .fai line {k + 1}: {line!r}") from None
        if f[0] in names:
            raise ReferenceError(f"duplicate sequence name {f[0]!r} in the .fai")
        names.append(f[0])
    return names, np.array(rows, dtype=FAI_DTYPE) if rows else np.zeros(0, FAI_DTYPE)


def build_fai(data):
    """the index htslib's fai_build makes of a plain-text FASTA, vectorised over lines -> (names, FAI_DTYPE rows)"""
    a = np.frombuffer(data, "u1") if isinstance(data, (bytes, bytearray, memoryview)) else np.asarray(data, "u1")
    n = len(a)
    if n == 0:
        return [], np.zeros(0, FAI_DTYPE)
    nl = np.flatnonzero(a == 10)
    starts = np.concatenate(([0], nl + 1))
    ends = np.concatenate((nl, [n]))                     # exclusive, without the '\n'
    if starts[-1] == n:                                  # the file ends with '\n': no line after it
        starts, ends = starts[:-1], ends[:-1]
    has_cr = (ends > starts) & (a[np.maximum(ends - 1, 0)] == 13)
    bases = (ends - starts - has_cr).astype(np.int64)
    width = (ends - starts + 1).astype(np.int64)
    is_head = a[starts] == 62                            # '>'
    heads = np.flatnonzero(is_head)
    if len(heads) == 0 or np.any(bases[:heads[0]] > 0):
        raise ReferenceError("not a FASTA file: sequence data before the first '>' header")
    names, rows, seen = [], [], set()
    bounds = np.concatenate((heads, [len(starts)]))
    for h, nxt in zip(bounds[:-1], bounds[1:]):
        head = bytes(a[starts[h] + 1:ends[h]]).rstrip(b"\r")
        name = head.split(None, 1)[0].decode() if head.split() else ""
        if name in seen:
            raise ReferenceError(f"duplicate sequence name {name!r} in the FASTA")
        seen.add(name)
        lo, hi = h + 1, nxt
        b = bases[lo:hi]
        nz = np.flatnonzero(b > 0)
        if len(nz) == 0:                                 # no bases
            names.append(name)
            rows.append((0, int(starts[lo]) if lo < len(starts) else n, 0, 0))
            continue
        last = lo + int(nz[-1])                          # trailing empty lines end the sequence
        lb, lw = int(bases[lo]), int(width[lo])
        if lb == 0 or np.any(bases[lo:last] != lb) or np.any(width[lo:last] != lw) or int(bases[last]) > lb:
            raise ReferenceError(f"different line length in sequence {name!r}")
        names.append(name)
        rows.append((int(b.sum()), int(starts[lo]), lb, lw))
    return names, np.array(rows, dtype=FAI_DTYPE)


def _bgzf_kind(head):
    """'bgzf', 'gzip' or None for the first bytes of a file"""
    if head[:2] != b"\x1f\x8b":
        return None
    from . import bamio
    try:
        bamio.bgzf_header(head, 0)
        return "bgzf"
    except (ValueError, struct.error, IndexError):
        return "gzip"


def _raw_end(row):
    """exclusive raw offset after the last base of a contig"""
    L, lb, lw = int(row["length"]), int(row["linebases"]), int(row["linewidth"])
    if L == 0:
        return int(row["offset"])
    return int(row["offset"]) + ((L - 1) // lb) * lw + (L - 1) % lb + 1


def bgzf_plan(z, spans):
    """BGZF members covering each raw byte range: z = the file's bytes, spans = [(begin, end)] of the inflated stream.  Returns
    (shipped member bytes, per span its offset rebased to the inflated stream of the shipped members).  Only the members some span
    touches are shipped, in file order."""
    from . import bamio
    members = list(bamio.bgzf_members(z))
    co = np.array([m[0] for m in members] + [len(z)], dtype=np.int64)
    isz = np.array([m[3] for m in members], dtype=np.int64)
    ustart = np.concatenate(([0], np.cumsum(isz)))
    keep = np.zeros(len(members), bool)
    first = []
    for b, e in spans:
        if e <= b:
            first.append(-1)
            continue
        m0 = int(np.searchsorted(ustart, b, side="right")) - 1
        m1 = int(np.searchsorted(ustart, e, side="left"))       # members m0 .. m1 - 1 hold [b, e)
        if m0 < 0 or m1 > len(members):
            raise ReferenceError(f"the .fai names bytes {b}..{e} beyond the {int(ustart[-1])}-byte inflated file")
        keep[m0:m1] = True
        first.append(m0)
    idx = np.flatnonzero(keep)
    ship_ustart = np.zeros(len(members) + 1, np.int64)
    ship_ustart[idx] = np.concatenate(([0], np.cumsum(isz[idx])[:-1])) if len(idx) else []
    zb = z if isinstance(z, (bytes, bytearray)) else bytes(z)
    pieces, k = [], 0
    while k < len(idx):                                  # contiguous member runs as one slice each
        j = k
        while j + 1 < len(idx) and idx[j + 1] == idx[j] + 1:
            j += 1
        pieces.append(zb[co[idx[k]]:co[idx[j] + 1]])
        k = j + 1
    rebased = [0 if m0 < 0 else int(ship_ustart[m0] + (b - ustart[m0])) for (b, _), m0 in zip(spans, first)]
    return b"".join(pieces), rebased


class Reference:
    """`pysam.FastaFile` duck type over a genome resident on the device of `ctx` (binding.Context).  contigs: the names to load (None:
    all); fetching any other contig raises KeyError."""

    def __init__(self, path, ctx, contigs=None):
        self.path, self.ctx = str(path), ctx
        with open(self.path, "rb") as f:
            head = f.read(1 << 16)
        kind = _bgzf_kind(head)
        if kind == "gzip":
            raise ReferenceError(f"{self.path} is compressed with gzip, not BGZF: recompress it with bgzip")
        fai = self.path + ".fai"
        if os.path.exists(fai):
            with open(fai) as f:
                names, rows = parse_fai(f.read())
        elif kind == "bgzf":
            raise ReferenceError(f"{fai} is missing: a BGZF-compressed FASTA needs its .fai index (samtools faidx)")
        else:
            names, rows = build_fai(np.fromfile(self.path, dtype="u1"))
        self.references = tuple(names)
        self.lengths = tuple(int(x) for x in rows["length"])
        self._row = {n: rows[i] for i, n in enumerate(names)}
        self.loaded = [n for n in names if contigs is None or n in set(contigs)]
        self._slot = {n: k for k, n in enumerate(self.loaded)}
        spans = [(int(self._row[n]["offset"]), _raw_end(self._row[n])) for n in self.loaded]
        table = np.zeros(len(self.loaded), abi.REF_CONTIG_DTYPE)
        for k, n in enumerate(self.loaded):
            r = self._row[n]
            table[k] = (0, int(r["length"]), int(r["linebases"]), int(r["linewidth"]))
        if kind == "bgzf":
            with open(self.path, "rb") as f:
                z = f.read()
            data, offs = bgzf_plan(z, spans)
            table["offset"] = offs
        else:
            mm = np.memmap(self.path, dtype="u1", mode="r") if os.path.getsize(self.path) else np.zeros(0, "u1")
            lo = min((b for b, e in spans if e > b), default=0)
            hi = max((e for b, e in spans if e > b), default=0)
            data = np.ascontiguousarray(mm[lo:hi])
            table["offset"] = [b - lo if e > b else 0 for b, e in spans]
        try:
            runs, coff = ctx.load_reference(data, table, is_bgzf=kind == "bgzf")
        except Exception as e:
            msg = str(e)
            import re
            m = re.search(r"contig (\d+), line (\d+)", msg)
            if m:
                raise ReferenceError(f"{self.path}: sequence {self.loaded[int(m.group(1))]!r}, line {int(m.group(2)) + 1} of its bases does not match "
                                     f"{fai}: the index is stale or does not belong to this file ({msg})") from None
            raise
        self._runs = {n: runs[int(coff[k]):int(coff[k + 1])] for k, n in enumerate(self.loaded)}
        self._cache = {}

    # ---- pysam.FastaFile surface ----
    def _resolve(self, contig, start=None, end=None):
        """pysam / htslib faidx_fetch_seq rules -> (slot, start, end) with 0 <= start <= end <= length"""
        if contig not in self._row:
            raise KeyError(f"sequence {contig!r} not present in {self.path}")
        if contig not in self._slot:
            raise KeyError(f"sequence {contig!r} of {self.path} is not loaded on this device")
        L = int(self._row[contig]["length"])
        start = 0 if start is None else int(start)
        end = L if end is None else int(end)
        if start < 0:
            raise ValueError(f"start out of range ({start})")
        if start > end:
            raise ValueError(f"invalid coordinates: start ({start}) > stop ({end})")
        end = min(end, L)
        start = min(start, end)
        return self._slot[contig], start, end

    def _gather(self, keys):
        q = np.zeros(len(keys), abi.REF_QUERY_DTYPE)
        o = 0
        for i, (slot, s, e) in enumerate(keys):
            q[i] = (slot, 0, s, e - s, o)
            o += e - s
        out = self.ctx.fetch_reference(q) if o else np.zeros(0, "u1")
        raw = out.tobytes()
        return [raw[int(r["out_off"]):int(r["out_off"]) + int(r["length"])].decode("latin-1") for r in q]

    def fetch(self, contig, start=None, end=None):
        key = self._resolve(contig, start, end)
        if key[1] == key[2]:
            return ""
        got = self._cache.get(key)
        if got is None:
            got = self._cache[key] = self._gather([key])[0]
        return got

    def prefetch(self, intervals):
        """one snfb_fetch_reference call for every (contig, start, end) not cached yet; intervals `fetch` would refuse are skipped.
        Returns the number of bases gathered."""
        keys = set()
        for contig, start, end in intervals:
            try:
                k = self._resolve(contig, start, end)
            except (KeyError, ValueError):
                continue
            if k[1] < k[2] and k not in self._cache:
                keys.add(k)
        keys = sorted(keys)
        for k, s in zip(keys, self._gather(keys) if keys else []):
            self._cache[k] = s
        return sum(e - s for _, s, e in keys)

    # ---- the N mask ----
    def n_runs(self):
        """{contig: int32 [n, 2] (start, end)} of the maximal runs of 'N' (upper case only) of every loaded contig"""
        return dict(self._runs)

    def task_runs(self, contig, start, end):
        """the runs _mask_N_coverage applies to a task region [start, end) of `contig`, or None (with the reference's warning) when it
        cannot: the contig is missing from the FASTA (KeyError there), or shorter than the region's end (the fetched mask does not fit
        the region, leadprov.py:436-438).  The device clips the runs to the region."""
        try:
            if contig not in self._row:
                raise KeyError(f"sequence '{contig}' not present")
            if contig not in self._slot:
                raise KeyError(f"sequence '{contig}' not loaded on this device")
            L = int(self._row[contig]["length"])
            if L < end:
                raise ValueError(f"could not broadcast input array from shape ({max(0, L - start)},) into shape ({end - start},)")
        except (KeyError, ValueError) as e:
            logging.warning(f"Unable to mask N regions in coverage vector, reference could not be fetched: {e}")
            return None
        return self._runs[contig]


    def region_runs(self, contig, regions, length):
        """the runs _mask_N_coverage applies to a task with regions (leadprov.py:432-439): the mask is zero outside the regions and each
        region's slice mask[start:end] of the contig-long vector (`length` bases) takes fasta.fetch(contig, start, end).  So the runs are
        clipped to the regions.  One region whose fetch or slice assignment raises (the contig missing from the FASTA, or a fetch that
        does not fit its slice, numpy broadcasting a single base over it) leaves the whole task unmasked, with the reference's warning."""
        try:
            if contig not in self._row:
                raise KeyError(f"sequence '{contig}' not present")
            if contig not in self._slot:
                raise KeyError(f"sequence '{contig}' not loaded on this device")
            L = int(self._row[contig]["length"])
            runs = self._runs[contig]
            keep = []
            for s, e in regions:
                n_slice, n_fetch = max(0, min(e, length) - s), max(0, min(e, L) - s)
                if n_fetch != n_slice and n_fetch != 1:
                    raise ValueError(f"could not broadcast input array from shape ({n_fetch},) into shape ({n_slice},)")
                if n_fetch == 1 and n_slice > 1:          # one base broadcast over the slice: all N or none
                    k = int(np.searchsorted(runs[:, 1], s, side="right")) if len(runs) else 0
                    if k < len(runs) and runs[k, 0] <= s:
                        keep.append((s, min(e, length)))
                    continue
                keep.extend((max(int(a), s), min(int(b), e, length)) for a, b in runs if a < e and b > s)
        except (KeyError, ValueError) as e:
            logging.warning(f"Unable to mask N regions in coverage vector, reference could not be fetched: {e}")
            return None
        merged = []
        for a, b in sorted(x for x in keep if x[1] > x[0]):
            if merged and a <= merged[-1][1]:
                merged[-1][1] = max(merged[-1][1], b)
            else:
                merged.append([a, b])
        return np.asarray(merged, dtype=np.int32).reshape(-1, 2)


def mask_block(block, reference, regions=None):
    """the N-mask tables of a record block (RecordBlock.set_n_mask) from `reference` for each of its tasks; regions: {task index: [(start,
    end), ...]} for the tasks that have regions (Reference.region_runs)"""
    per = {}
    for t, task in enumerate(block.task):
        name = block.contig_names[int(task["contig"])]
        rg = (regions or {}).get(t)
        runs = reference.task_runs(name, int(task["start"]), int(task["end"])) if rg is None else reference.region_runs(name, rg, int(task["contig_len"]))
        if runs is not None and len(runs):
            per[t] = [(int(a), int(b)) for a, b in runs]
    block.set_n_mask(per)
    return block
