"""Seeded reference FASTA texts for the --reference tests and golden data, and the numpy restatement of their 'N' runs.

Every contig carries the cases the device N scan and the unwrap must get right: N runs at position 0 and at the contig end, across
60-column line breaks and across 64 KiB tile edges, single-base runs, an all-N stretch longer than a read, lower-case `n` (never masked),
lower-case soft-masked stretches and IUPAC codes."""
import hashlib

import numpy as np

IUPAC = b"RYSWKMBDHV"

# the golden blocks' FASTAs (tests/golden/reference): c2_ont_wgs_small has ctg1..ctg4 of 300, 260, 220 and 150 kb, phased_phase ctg1, ctg2
# of 260 and 140 kb.  ctg2 of c2 is missing, ctg3 of c2 is shorter than in the BAM (left unmasked), ctg1 of phased_phase longer (masked:
# the task region still fits), and a contig the BAM lacks is appended.
GOLDEN_FASTA = {
    "c2_ont_wgs_small": (2002, [("ctg1", 300_000), ("ctg3", 200_000), ("ctg4", 150_000), ("chrUn_extra", 7_000)]),
    "phased_phase": (2079, [("ctg1", 270_000), ("ctg2", 140_000), ("chrUn_extra", 7_000)]),
}


def contig_seq(rng, length, long_gap=30_000):
    """one contig's bases (bytes) with the cases listed above, placed where the length allows"""
    s = np.frombuffer(b"ACGT", "u1")[rng.integers(0, 4, length)].copy()
    if length == 0:
        return b""
    for _ in range(max(1, length // 20_000)):                     # soft-masked stretches
        a = int(rng.integers(0, length)); s[a:a + int(rng.integers(50, 3000))] |= 0x20
    for _ in range(max(1, length // 5_000)):                      # IUPAC codes
        s[int(rng.integers(0, length))] = IUPAC[int(rng.integers(0, len(IUPAC)))]
    for _ in range(max(1, length // 30_000)):                     # lower-case n stretches: not masked
        a = int(rng.integers(0, length)); s[a:a + int(rng.integers(1, 500))] = ord("n")
    runs = [(0, 37), (length - 113, length), (119, 122), (59, 61), (65_530, 65_545), (131_071, 131_073), (196_608, 196_609)]
    runs += [(int(p), int(p) + 1) for p in rng.integers(0, length, 6)]             # single bases
    runs += [(int(p), int(p) + int(rng.integers(2, 2000))) for p in rng.integers(0, length, max(1, length // 40_000))]
    if length > 4 * long_gap:
        a = length // 2 + 12_345; runs.append((a, a + long_gap))
    for a, b in runs:
        a, b = max(0, a), min(length, b)
        if a < b:
            s[a:b] = ord("N")
    return s.tobytes()


def genome(seed, contigs):
    """[(name, length)] -> [(name, bases)]"""
    rng = np.random.default_rng(seed)
    return [(n, contig_seq(rng, L)) for n, L in contigs]


def fasta_text(seqs, width=60, crlf=False, last_newline=True, header_extra=" synthetic"):
    """[(name, bases)] -> FASTA bytes wrapped at `width` columns"""
    nl = b"\r\n" if crlf else b"\n"
    out = []
    for name, s in seqs:
        out.append(b">" + name.encode() + header_extra.encode() + nl)
        out.extend(s[k:k + width] + nl for k in range(0, len(s), width))
    text = b"".join(out)
    return text if last_newline or not text.endswith(nl) else text[:-len(nl)]


def fai_text(seqs, width=60, crlf=False):
    """the .fai htslib writes for fasta_text(seqs, width, crlf)"""
    nl = 2 if crlf else 1
    o, rows = 0, []
    for name, s in seqs:
        o += 1 + len(name) + len(" synthetic") + nl
        lb = min(width, len(s))                           # a one-line sequence: its own length
        rows.append(f"{name}\t{len(s)}\t{o}\t{lb}\t{lb + nl if s else 0}")
        o += len(s) + nl * ((len(s) + width - 1) // width)
    return ("\n".join(rows) + "\n").encode()


def n_runs(bases):
    """int32 [n, 2] (start, end) of the maximal runs of b'N' (upper case only)"""
    a = np.frombuffer(bases, "u1") == 78
    d = np.diff(np.concatenate(([0], a.astype(np.int8), [0])))
    return np.stack([np.flatnonzero(d == 1), np.flatnonzero(d == -1)], axis=1).astype("<i4")


def task_runs(blk, seqs):
    """{task: [(a, b)]} N runs a --reference run loads for a block: a task's contig must be in the FASTA and reach the task's end,
    or the reference's _mask_N_coverage fails its fetch and leaves the task unmasked (leadprov.py:431-441)"""
    by_name = dict(seqs)
    out = {}
    for t, k in enumerate(blk.task):
        s = by_name.get(blk.contig_names[int(k["contig"])])
        if s is not None and len(s) >= int(k["end"]):
            out[t] = [tuple(map(int, r)) for r in n_runs(s)]
    return out


def coverage_bins(cv, binsize):
    """SNFile.annotate_block_coverages' means (snf.py:257-258): the vector zero-padded to a multiple of binsize, row means"""
    return np.pad(np.asarray(cv, np.int64), (0, -len(cv) % binsize)).reshape(-1, binsize).mean(axis=1)


def golden_fasta(name):
    """(FASTA bytes, [(contig, bases)]) of a golden block"""
    seed, contigs = GOLDEN_FASTA[name]
    seqs = genome(seed, contigs)
    return fasta_text(seqs), seqs


def sha256(data):
    return hashlib.sha256(data).hexdigest()


CAND_FIELDS = ("svtype", "pos", "end", "svlen", "support", "qual", "precise", "fwd", "rev", "cov")


def vcf_digest(line, keep=24):
    """a VCF line as the golden data stores it: CHROM .. FILTER and the sample column, REF and ALT cut to `keep` characters (plus their
    length), and the sha256 prefix of the whole line, so a comparison is still byte for byte"""
    f = line.split("\t")
    f = f[:7] + f[9:]
    for k in (3, 4):
        if len(f) > k and len(f[k]) > keep:
            f[k] = f"{f[k][:keep]}...({len(f[k])})"
    return ["\t".join(f), sha256(line.encode())[:16]]
