"""Seeded synthetic alignment blocks (SURVEY.md §8d shapes) — ctypes front end of
csrc/host/synth.c (libsnfb_host.so).  Test / bench input only."""
import ctypes as C
import os
from dataclasses import dataclass, field

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

GRCH38 = [248956422, 242193529, 198295559, 190214555, 181538259, 170805979, 159345973, 145138636,
          138394717, 133797422, 135086622, 133275309, 114364328, 107043718, 101991189, 90338345,
          83257441, 80373285, 58617616, 64444167, 46709983, 50818468, 156040895, 57227415]


class _Params(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_contig", C.c_int32), ("len_model", C.c_int32),
                ("contig_len", C.POINTER(C.c_int32)), ("coverage", C.c_double), ("len_mean", C.c_double),
                ("len_sd", C.c_double), ("len_min", C.c_int32), ("len_max", C.c_int32),
                ("op_mean_run", C.c_double), ("nm_rate", C.c_double), ("clip_prob", C.c_double),
                ("lowmapq_prob", C.c_double), ("secondary_prob", C.c_double), ("sv_spacing", C.c_double),
                ("phased_frac", C.c_double), ("tr_frac", C.c_double), ("ins_noise", C.c_double),
                ("mosaic", C.c_int32), ("with_seq", C.c_int32), ("ins_only", C.c_int32),
                ("sv_min", C.c_int32), ("sv_max", C.c_int32), ("threads", C.c_int32), ("_pad", C.c_int32),
                ("contig_mask", C.POINTER(C.c_uint8)), ("sample", C.c_uint64), ("site_keep", C.c_double)]


SITE_DTYPE = np.dtype([("contig", "<i4"), ("pos", "<i4"), ("svtype", "<i4"), ("size", "<i4"),
                       ("mate_contig", "<i4"), ("mate_pos", "<i4"), ("in_tr", "<i4"), ("hap", "<i4"),
                       ("vaf", "<f8")])


def host_lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libsnfb_host.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
        lib = C.CDLL(path)
        lib.snfb_synth_generate.restype = C.c_void_p
        lib.snfb_synth_generate.argtypes = [C.POINTER(_Params)]
        lib.snfb_synth_records.restype = C.POINTER(abi.Records)
        lib.snfb_synth_records.argtypes = [C.c_void_p]
        lib.snfb_synth_sites.restype = C.c_uint64
        lib.snfb_synth_sites.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        lib.snfb_synth_aligned_bp.restype = C.c_uint64
        lib.snfb_synth_aligned_bp.argtypes = [C.c_void_p]
        lib.snfb_synth_free.argtypes = [C.c_void_p]
        _LIB = lib
    return _LIB


@dataclass
class RecordBlock:
    """Packed alignment records of include/snfb.h as numpy arrays (host memory)."""
    rec: np.ndarray
    cigar: np.ndarray
    var: np.ndarray
    seq: np.ndarray
    task: np.ndarray
    contig: np.ndarray
    tr: np.ndarray
    contig_names: list = field(default_factory=list)
    aligned_bp: int = 0
    sites: np.ndarray = None
    _owner: object = None
    mask: np.ndarray = None            # optional reference N runs: int32 pairs (start, end), per task contiguous
    mask_task_off: np.ndarray = None   # uint32 [n_task + 1]
    rec16: np.ndarray = None           # CIGAR16 twin of rec / cigar (pack16); what the device path ships
    cigar16: np.ndarray = None

    def pack16(self):
        """Convert the BAM CIGAR words to CIGAR16 once (snfb_pack_cigar16, host code of libsnfb200)."""
        if self.cigar16 is None:
            from . import binding
            self.rec16, self.cigar16 = binding.pack_cigar16(self.rec, self.cigar)
        return self

    def as_struct(self, cigar16: bool = False) -> abi.Records:
        """cigar16=False: the BAM-word form (what the oracle reads); True: the CIGAR16 form the kernels stream."""
        r = abi.Records()
        if cigar16:
            self.pack16()
            rec, cig, r.cigar_fmt = self.rec16, self.cigar16, abi.CIGAR_16
        else:
            rec, cig, r.cigar_fmt = self.rec, self.cigar, abi.CIGAR_BAM32
        r.n_rec, r.n_cigar, r.n_var, r.n_seq = len(rec), len(cig), len(self.var), len(self.seq)
        r.rec, r.cigar = rec.ctypes.data, cig.ctypes.data
        r.var, r.seq = self.var.ctypes.data, self.seq.ctypes.data
        r.n_task, r.n_contig, r.n_tr, r.on_device = len(self.task), len(self.contig), len(self.tr) // 2, 0
        r.task, r.contig, r.tr = self.task.ctypes.data, self.contig.ctypes.data, self.tr.ctypes.data
        if self.mask is not None and len(self.mask):
            r.n_mask, r.mask, r.mask_task_off = len(self.mask) // 2, self.mask.ctypes.data, self.mask_task_off.ctypes.data
        return r

    def set_n_mask(self, per_task_intervals):
        """per_task_intervals: {task index: [(start, end), ...]} of reference 'N' runs (sorted, disjoint)."""
        off, flat = [0], []
        for t in range(len(self.task)):
            iv = sorted(per_task_intervals.get(t, []))
            flat.extend(x for ab in iv for x in ab)
            off.append(off[-1] + len(iv))
        self.mask = np.asarray(flat, dtype="<i4")
        self.mask_task_off = np.asarray(off, dtype="<u4")

    def nbytes(self) -> int:
        cig = self.cigar16 if self.cigar16 is not None else self.cigar
        return self.rec.nbytes + cig.nbytes + self.var.nbytes + self.seq.nbytes


class _Owner:
    def __init__(self, handle):
        self.handle = handle

    def __del__(self):
        try:
            host_lib().snfb_synth_free(self.handle)
        except Exception:
            pass


def generate(seed: int, contig_len, coverage: float, *, len_model=0, len_mean=15000.0, len_sd=0.6 * 1000,
             len_min=1000, len_max=200000, tech="ont", clip_prob=0.10, lowmapq_prob=0.05,
             secondary_prob=0.02, sv_spacing=120000.0, phased_frac=0.5, tr_frac=0.15, ins_noise=0.03,
             mosaic=False, with_seq=True, ins_only=False, sv_min=50, sv_max=5000, threads=0, contig_mask=None, sample=0, site_keep=0.0) -> RecordBlock:
    lib = host_lib()
    lens = (C.c_int32 * len(contig_len))(*[int(x) for x in contig_len])
    p = _Params()
    p.seed, p.n_contig, p.len_model, p.contig_len = int(seed), len(contig_len), int(len_model), lens
    p.coverage, p.len_mean, p.len_sd, p.len_min, p.len_max = coverage, len_mean, len_sd, int(len_min), int(len_max)
    p.op_mean_run, p.nm_rate = (80.0, 0.01) if tech == "ont" else (700.0, 0.001)
    p.clip_prob, p.lowmapq_prob, p.secondary_prob = clip_prob, lowmapq_prob, secondary_prob
    p.sv_spacing, p.phased_frac, p.tr_frac, p.ins_noise = sv_spacing, phased_frac, tr_frac, ins_noise
    p.mosaic, p.with_seq, p.ins_only = int(mosaic), int(with_seq), int(ins_only)
    p.sv_min, p.sv_max, p.threads = int(sv_min), int(sv_max), int(threads)
    p.sample, p.site_keep = int(sample), float(site_keep)
    mask = None
    if contig_mask is not None:
        mask = (C.c_uint8 * len(contig_len))(*[1 if m else 0 for m in contig_mask])
        p.contig_mask = C.cast(mask, C.POINTER(C.c_uint8))
    h = lib.snfb_synth_generate(C.byref(p))
    if not h:
        raise MemoryError("snfb_synth_generate failed")
    owner = _Owner(h)
    R = lib.snfb_synth_records(h).contents
    sp = C.c_void_p()
    ns = lib.snfb_synth_sites(h, C.byref(sp))
    blk = RecordBlock(
        rec=abi.view(R.rec, abi.REC_DTYPE, R.n_rec), cigar=abi.view(R.cigar, "<u4", R.n_cigar),
        var=abi.view(R.var, "u1", R.n_var), seq=abi.view(R.seq, "u1", R.n_seq),
        task=abi.view(R.task, abi.TASK_DTYPE, R.n_task), contig=abi.view(R.contig, abi.CONTIG_DTYPE, R.n_contig),
        tr=abi.view(R.tr, "<i4", R.n_tr * 2), contig_names=[f"ctg{i + 1}" for i in range(len(contig_len))],
        aligned_bp=int(lib.snfb_synth_aligned_bp(h)), sites=abi.view(sp.value, SITE_DTYPE, ns), _owner=owner)
    return blk


# ---- the BASELINE.json configurations (SURVEY.md §8d); `scale` shrinks contig lengths ----
def config_block(index: int, scale: float = 1.0, threads: int = 0, with_seq: bool = True, contig_mask=None, sample: int = 1) -> RecordBlock:
    seed = 1000 + index
    if index == 4:      # one of the 50 samples of the population shape: 30x ONT like config 2, shared sites, 60 % of them per sample
        return generate(seed, [max(200000, int(x * scale)) for x in GRCH38], 30.0, len_model=1, len_mean=15000.0,
                        len_sd=600.0, len_min=1000, len_max=200000, tech="ont", threads=threads, with_seq=with_seq, contig_mask=contig_mask,
                        sample=sample, site_keep=0.6)
    if index == 1:      # 1 Mb contig, ~200 ONT reads of ~100 kb @20x
        return generate(seed, [int(1_000_000 * scale)], 20.0, len_model=0, len_mean=100000.0, len_sd=10000.0,
                        len_min=1000, len_max=200000, tech="ont", sv_spacing=25000.0, threads=threads, with_seq=with_seq)
    if index == 2:      # 30x ONT WGS, lognormal 15 kb
        return generate(seed, [max(200000, int(x * scale)) for x in GRCH38], 30.0, len_model=1, len_mean=15000.0,
                        len_sd=600.0, len_min=1000, len_max=200000, tech="ont", threads=threads, with_seq=with_seq, contig_mask=contig_mask)
    if index == 3:      # 60x HiFi WGS, mosaic
        return generate(seed, [max(200000, int(x * scale)) for x in GRCH38], 60.0, len_model=0, len_mean=18000.0,
                        len_sd=3000.0, len_min=1000, len_max=60000, tech="hifi", mosaic=True, threads=threads,
                        with_seq=with_seq, contig_mask=contig_mask)
    if index == 5:      # INS-heavy: 5 Mb region, 5000 sites x 20 reads
        return generate(seed, [int(5_000_000 * scale)], 20.0, len_model=0, len_mean=20000.0, len_sd=2000.0,
                        len_min=5000, len_max=60000, tech="ont", sv_spacing=1000.0, ins_only=True, tr_frac=0.0,
                        clip_prob=0.0, sv_min=50, sv_max=5000, threads=threads, with_seq=with_seq)
    raise ValueError(f"no synthetic shape for BASELINE config {index}")


def genotype_targets(cand, n_task, contig_len, rng, n):
    """seeded force-calling targets as the int32 columns of snfb_gt_in (task, svtype, pos, svlen, bnd_is_first, mate_contig), ordered by
    task: half are candidates jittered inside and beyond the matching limits (exact copies included), half random decoys and edge cases
    (POS 0, the contig's last positions, bin edges, svlen 0, unsupported types, unknown mate contigs)"""
    rows = []
    for c in cand[rng.integers(0, len(cand), n // 2)]:
        j = int(rng.choice([0, 0, 5, 50, 300, 1200]))
        rows.append((int(c["task"]), int(c["svtype"]) if int(c["svtype"]) <= abi.BND else -1, int(c["pos"]) + int(rng.integers(-j, j + 1)),
                     int(c["svlen"]) + int(rng.integers(-j, j + 1)), int(c["bnd_is_first"]), int(c["bnd_mate_contig"]) if rng.random() < 0.9 else -1))
    for _ in range(n - len(rows)):
        t = int(rng.integers(0, n_task))
        L = int(contig_len[t])
        pos = int(rng.choice([rng.integers(0, L), -1, 0, L - 2, int(rng.integers(0, L // 5000)) * 5000 + int(rng.choice([0, 499, 500, 4500, 4501, 4999]))]))
        rows.append((t, int(rng.integers(-1, 5)), pos, int(rng.choice([0, rng.integers(-20000, 20000), 60])), int(rng.integers(0, 2)), int(rng.integers(-1, 3))))
    rows.sort(key=lambda r: r[0])          # stable: input order inside a task
    return np.array(rows, dtype=np.int64).T.astype(np.int32)
