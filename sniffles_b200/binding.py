"""ctypes binding of libsnfb200.so (include/snfb.h).  The library is CUDA-only: importing this
module works anywhere, but creating a `Context` requires a GPU and raises otherwise — there is
no CPU fallback for the lead -> cluster -> consensus path."""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsnfb200.so")
_LIB = None

EXPORTS = ["snfb_version", "snfb_sizeof", "snfb_hash_name", "snfb_ctx_create", "snfb_ctx_destroy", "snfb_last_error", "snfb_set_config",
           "snfb_load_records", "snfb_extract_leads", "snfb_cluster_call", "snfb_consensus", "snfb_run",
           "snfb_last_timings", "snfb_device_candidates", "snfb_device_alt", "snfb_launch_count",
           "snfb_pin_host", "snfb_unpin_host", "snfb_pack_cigar16", "snfb_rerun_count", "snfb_coverage_bins",
           "snfb_nccl_unique_id", "snfb_comm_init", "snfb_allgather_candidates", "snfb_selftest_sqrt_frac", "snfb_poa", "snfb_combine_groups", "snfb_combine_plan", "snfb_selftest_edit_distance",
           "snfb_load_bam", "snfb_set_regions", "snfb_ingest_sizes", "snfb_ingest_fetch", "snfb_inflate_bgzf", "snfb_deflate_bgzf",
           "snfb_genotype_targets", "snfb_load_reference", "snfb_reference_runs", "snfb_fetch_reference",
           "snfb_population_load", "snfb_population_match", "snfb_read_names", "snfb_set_consensus_slices",
           "snfb_index_bam", "snfb_sort_bam"]


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(the CUDA extension is required; there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.snfb_version.restype = C.c_int
        L.snfb_sizeof.restype = C.c_size_t
        L.snfb_sizeof.argtypes = [C.c_int]
        L.snfb_hash_name.restype = C.c_uint64
        L.snfb_hash_name.argtypes = [C.c_char_p, C.c_size_t]
        L.snfb_ctx_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
        L.snfb_ctx_destroy.argtypes = [C.c_void_p]
        L.snfb_last_error.restype = C.c_char_p
        L.snfb_last_error.argtypes = [C.c_void_p]
        L.snfb_set_config.argtypes = [C.c_void_p, C.POINTER(abi.Config)]
        L.snfb_load_records.argtypes = [C.c_void_p, C.POINTER(abi.Records)]
        L.snfb_load_bam.argtypes = [C.c_void_p, C.POINTER(abi.BamInput)]
        L.snfb_set_regions.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32]
        L.snfb_ingest_sizes.argtypes = [C.c_void_p, C.c_void_p]
        L.snfb_ingest_fetch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.snfb_inflate_bgzf.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
        L.snfb_deflate_bgzf.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p]
        L.snfb_extract_leads.argtypes = [C.c_void_p, C.POINTER(abi.LeadView)]
        L.snfb_cluster_call.argtypes = [C.c_void_p, C.POINTER(abi.CandView)]
        L.snfb_consensus.argtypes = [C.c_void_p, C.POINTER(abi.SeqView)]
        L.snfb_run.argtypes = [C.c_void_p, C.POINTER(abi.LeadView), C.POINTER(abi.CandView), C.POINTER(abi.SeqView)]
        L.snfb_last_timings.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.POINTER(C.c_uint64), C.c_int]
        L.snfb_device_candidates.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.snfb_device_alt.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.snfb_launch_count.restype = C.c_uint64
        L.snfb_launch_count.argtypes = [C.c_void_p]
        L.snfb_pin_host.argtypes = [C.c_void_p, C.c_size_t]
        L.snfb_unpin_host.argtypes = [C.c_void_p]
        L.snfb_rerun_count.restype = C.c_uint64
        L.snfb_rerun_count.argtypes = [C.c_void_p]
        L.snfb_set_consensus_slices.argtypes = [C.c_void_p, C.c_int]
        L.snfb_coverage_bins.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.snfb_nccl_unique_id.argtypes = [C.c_void_p]
        L.snfb_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.snfb_allgather_candidates.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.GatherView)]
        L.snfb_poa.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p]
        L.snfb_genotype_targets.argtypes = [C.c_void_p, C.POINTER(abi.GtIn), C.POINTER(abi.GtOut)]
        L.snfb_read_names.argtypes = [C.c_void_p, C.POINTER(abi.RnamesView)]
        L.snfb_index_bam.argtypes = [C.c_void_p, C.POINTER(abi.IndexInput), C.POINTER(abi.IndexView)]
        L.snfb_sort_bam.argtypes = [C.c_void_p, C.POINTER(abi.SortInput), C.POINTER(abi.SortView)]
        L.snfb_load_reference.argtypes = [C.c_void_p, C.POINTER(abi.RefInput)]
        L.snfb_reference_runs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        L.snfb_fetch_reference.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
        L.snfb_combine_groups.argtypes = [C.c_void_p, C.POINTER(abi.CombineIn), C.POINTER(abi.CombineOut)]
        L.snfb_combine_plan.argtypes = [C.c_void_p, C.POINTER(abi.CombinePlanIn), C.POINTER(abi.CombinePlanOut)]
        L.snfb_population_load.argtypes = [C.c_void_p, C.POINTER(abi.PopTable)]
        L.snfb_population_match.argtypes = [C.c_void_p, C.POINTER(abi.PopQuery), C.c_void_p]
        L.snfb_selftest_edit_distance.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
        L.snfb_selftest_sqrt_frac.restype = C.c_double
        L.snfb_selftest_sqrt_frac.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_int]
        L.snfb_pack_cigar16.restype = C.c_uint64
        L.snfb_pack_cigar16.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32]
        _LIB = L
    return _LIB


class SnfbError(RuntimeError):
    pass


def pack_cigar16(rec: np.ndarray, cigar32: np.ndarray, evt_min: int = 0):
    """BAM CIGAR words -> (rec16, cigar16) of include/snfb.h (host code of the library; needs no GPU)."""
    L = lib()
    rec = np.ascontiguousarray(rec)
    cigar32 = np.ascontiguousarray(cigar32, dtype="<u4")
    need = L.snfb_pack_cigar16(rec.ctypes.data, len(rec), cigar32.ctypes.data, None, None, 0, int(evt_min))
    if need == 0xFFFFFFFFFFFFFFFF:
        raise SnfbError("snfb_pack_cigar16: a CIGAR holds an operation the path does not know")
    rec16 = np.empty(len(rec), abi.REC_DTYPE)
    cigar16 = np.empty(int(need), "<u2")
    got = L.snfb_pack_cigar16(rec.ctypes.data, len(rec), cigar32.ctypes.data, rec16.ctypes.data, cigar16.ctypes.data, int(need), int(evt_min))
    if got != need:
        raise SnfbError("snfb_pack_cigar16 failed")
    return rec16, cigar16


class Result:
    """Host copies of one run's outputs (numpy, struct layouts of include/snfb.h)."""

    def __init__(self):
        self.leads = None
        self.task_read_count = None
        self.task_mean_nm = None
        self.rec_nm = None
        self.n_pass = 0
        self.soft_errors = 0
        self.cand = np.zeros(0, abi.CAND_DTYPE)
        self.cand_leads = np.zeros(0, abi.LEAD_DTYPE)
        self.rnames = np.zeros(0, "<u8")
        self.rn_off = np.zeros(1, "<u4")
        self.task_cov_mean = None
        self.alt = np.zeros(0, "u1")

    def alt_of(self, i):
        c = self.cand[i]
        if c["alt_off"] < 0:
            return None
        return self.alt[int(c["alt_off"]):int(c["alt_off"]) + int(c["alt_len"])].tobytes().decode()


class GatheredResult(Result):
    """Concatenation of every rank's candidates in rank order, offsets rebased into the merged arenas."""
    n_cand = n_alt_bytes = n_rnames = n_cand_leads = dev_bytes_per_rank = 0

    def in_emission_order(self):
        """indices that order the merged candidates by task id (sniffles:544-547), each rank's own order kept inside a task"""
        return np.argsort(self.cand["task"], kind="stable")


def nccl_unique_id() -> bytes:
    buf = C.create_string_buffer(128)
    if lib().snfb_nccl_unique_id(buf) != 0:
        raise SnfbError("snfb_nccl_unique_id: NCCL is not available")
    return buf.raw


class Context:
    """One CUDA device, one stream.  Not thread safe; create it in the process that uses it
    (after fork), never pickle it."""

    def __init__(self, device: int = 0):
        self._lib = lib()
        h = C.c_void_p()
        rc = self._lib.snfb_ctx_create(int(device), C.byref(h))
        if rc != 0 or not h:
            raise SnfbError(f"snfb_ctx_create(device={device}) failed with code {rc}: a CUDA device is required "
                            "(libsnfb200 has no CPU fallback)")
        self._h = h
        self.device = device
        self._block = None

    def close(self):
        if getattr(self, "_h", None):
            self._lib.snfb_ctx_destroy(self._h)
            self._h = None

    __del__ = close

    def _check(self, rc, what):
        if rc != 0:
            raise SnfbError(f"{what}: {self._lib.snfb_last_error(self._h).decode()}")

    def set_config(self, cfg: abi.Config):
        self._check(self._lib.snfb_set_config(self._h, C.byref(cfg)), "snfb_set_config")

    def load(self, block, seq_on_demand=False, cigar16=True):
        """block: sniffles_b200.synth.RecordBlock-like (numpy arenas) or an abi.Records struct.
        seq_on_demand: leave the 4-bit seq arena on the host and fetch only the slices the consensus stage needs.
        cigar16: ship the CIGAR16 form (packed once per block); False hands the BAM words to the library, which converts them."""
        rs = block if isinstance(block, abi.Records) else block.as_struct(cigar16=cigar16)
        if seq_on_demand:
            rs.on_device = 2
        self._block = block          # keep host arrays alive during the async copy
        self._check(self._lib.snfb_load_records(self._h, C.byref(rs)), "snfb_load_records")

    def set_regions(self, regions=None):
        """snfb_set_regions: abi.REGION_DTYPE rows (grouped by task) for the next load; None or empty clears the table"""
        r = np.ascontiguousarray(regions if regions is not None else np.zeros(0, abi.REGION_DTYPE), dtype=abi.REGION_DTYPE)
        self._regions = r
        self._check(self._lib.snfb_set_regions(self._h, r.ctypes.data if len(r) else None, len(r)), "snfb_set_regions")

    def load_bam(self, bgzf: np.ndarray, spans: np.ndarray, tables):
        """Device BAM ingest (snfb_load_bam): `bgzf` = whole BGZF blocks (uint8), `spans` = abi.SPAN_DTYPE rows (bamio.BamFile.device_input
        builds both from the BAI index), `tables` = anything with the task / contig / tr (/ mask) arrays of a RecordBlock.  The record block is
        built in device memory; returns the sizes dict of snfb_ingest_sizes."""
        bgzf = np.ascontiguousarray(bgzf, dtype="u1")
        spans = np.ascontiguousarray(spans, dtype=abi.SPAN_DTYPE)
        I = abi.BamInput()
        I.bgzf, I.n_bytes, I.span, I.n_span = bgzf.ctypes.data, len(bgzf), spans.ctypes.data, len(spans)
        I.n_task, I.n_contig, I.n_tr = len(tables.task), len(tables.contig), len(tables.tr) // 2
        I.task, I.contig, I.tr = tables.task.ctypes.data, tables.contig.ctypes.data, tables.tr.ctypes.data
        mask = getattr(tables, "mask", None)
        if mask is not None and len(mask):
            I.n_mask, I.mask, I.mask_task_off = len(mask) // 2, mask.ctypes.data, tables.mask_task_off.ctypes.data
        self._block = tables
        self._check(self._lib.snfb_load_bam(self._h, C.byref(I)), "snfb_load_bam")
        return self.ingest_sizes()

    def ingest_sizes(self):
        out = np.zeros(8, "<u8")
        if self._lib.snfb_ingest_sizes(self._h, out.ctypes.data) != 0:
            raise SnfbError("snfb_ingest_sizes: no block was built by snfb_load_bam on this context")
        return dict(zip(("n_rec", "n_cigar", "n_var", "n_seq", "n_raw", "n_blocks", "raw_bytes", "bgzf_bytes"), (int(x) for x in out)))

    def ingest_fetch(self):
        """host copies (rec, cigar16, var, seq) of the block snfb_load_bam built — tests and inspection"""
        z = self.ingest_sizes()
        rec, cig = np.zeros(z["n_rec"], abi.REC_DTYPE), np.zeros(z["n_cigar"], "<u2")
        var, seq = np.zeros(z["n_var"], "u1"), np.zeros(z["n_seq"], "u1")
        self._check(self._lib.snfb_ingest_fetch(self._h, rec.ctypes.data, cig.ctypes.data, var.ctypes.data, seq.ctypes.data), "snfb_ingest_fetch")
        return rec, cig, var, seq

    def inflate_bgzf(self, bgzf: np.ndarray) -> bytes:
        """whole BGZF blocks -> their inflated bytes, decoded on the device (snfb_inflate_bgzf)"""
        bgzf = np.ascontiguousarray(bgzf, dtype="u1")
        n = C.c_uint64()
        self._check(self._lib.snfb_inflate_bgzf(self._h, bgzf.ctypes.data, len(bgzf), None, 0, C.byref(n)), "snfb_inflate_bgzf")
        out = np.zeros(max(int(n.value), 1), "u1")
        self._check(self._lib.snfb_inflate_bgzf(self._h, bgzf.ctypes.data, len(bgzf), out.ctypes.data, len(out), C.byref(n)), "snfb_inflate_bgzf")
        return out[:int(n.value)].tobytes()

    def deflate_bgzf(self, data) -> tuple:
        """bytes -> (BGZF members, their byte offsets), compressed on the device (snfb_deflate_bgzf); no EOF marker is appended"""
        src = np.frombuffer(bytes(data), "u1")
        nb = (len(src) + 0xff00 - 1) // 0xff00
        out = np.empty(max(nb * 65536, 1), "u1")
        coff = np.zeros(max(nb, 1), "<u8")
        n = C.c_uint64()
        self._check(self._lib.snfb_deflate_bgzf(self._h, src.ctypes.data, len(src), out.ctypes.data, len(out), C.byref(n), coff.ctypes.data), "snfb_deflate_bgzf")
        return out[:int(n.value)].tobytes(), [int(x) for x in coff[:nb]]

    def run(self, want_leads=True, want_cands=True, want_seqs=True, copy=True) -> Result:
        lv, cv, sv = abi.LeadView(), abi.CandView(), abi.SeqView()
        rc = self._lib.snfb_run(self._h, C.byref(lv) if want_leads else None, C.byref(cv) if want_cands else None,
                                C.byref(sv) if want_seqs else None)
        self._check(rc, "snfb_run")
        return self._collect(lv if want_leads else None, cv if want_cands else None, sv if want_seqs else None, copy)

    def extract_leads(self, want=True):
        lv = abi.LeadView()
        self._check(self._lib.snfb_extract_leads(self._h, C.byref(lv) if want else None), "snfb_extract_leads")
        return self._collect(lv if want else None, None, None, True)

    def _collect(self, lv, cv, sv, copy) -> Result:
        r = Result()
        cp = (lambda a: a.copy()) if copy else (lambda a: a)
        nt = None
        if lv is not None:
            r.leads = cp(abi.view(lv.leads, abi.LEAD_DTYPE, lv.n_leads))
            nt = self._n_task()
            r.task_read_count = cp(abi.view(lv.task_read_count, "<u4", nt))
            r.task_mean_nm = cp(abi.view(lv.task_mean_nm, "<f8", nt))
            r.n_pass, r.soft_errors = int(lv.n_pass), int(lv.soft_errors)
            r._rec_nm_ptr = lv.rec_nm
        if cv is not None:
            nt = self._n_task()
            r.cand = cp(abi.view(cv.cand, abi.CAND_DTYPE, cv.n_cand))
            r.cand_leads = cp(abi.view(cv.cand_leads, abi.LEAD_DTYPE, cv.n_cand_leads))
            r.rn_off = cp(abi.view(cv.rnames_off, "<u4", cv.n_cand + 1))
            r.rnames = cp(abi.view(cv.rnames, "<u8", int(r.rn_off[-1]) if cv.n_cand else 0))
            r.task_cov_mean = cp(abi.view(cv.task_coverage_mean, "<f8", nt))
        if sv is not None:
            r.alt = cp(abi.view(sv.alt, "u1", sv.n_alt_bytes))
        return r

    def _n_task(self):
        b = self._block
        return int(b.n_task) if isinstance(b, abi.Records) else len(b.task)

    def timings(self):
        """[(name, ms, algorithmic_bytes)] of the last run, from CUDA events on the ctx stream."""
        names = (C.c_char_p * 64)()
        ms = (C.c_float * 64)()
        by = (C.c_uint64 * 64)()
        n = self._lib.snfb_last_timings(self._h, names, ms, by, 64)
        return [(names[i].decode(), float(ms[i]), int(by[i])) for i in range(n)]

    def launch_count(self):
        return int(self._lib.snfb_launch_count(self._h))

    def rerun_count(self):
        return int(self._lib.snfb_rerun_count(self._h))

    def set_consensus_slices(self, k: int):
        """snfb_set_consensus_slices: run stage C in k slices (1 to 8); the results are the same for every k"""
        self._check(self._lib.snfb_set_consensus_slices(self._h, int(k)), "snfb_set_consensus_slices")

    def coverage_bins(self, task: int, binsize: int) -> np.ndarray:
        """Mean coverage per `binsize` bases over the task's contig (snf.py:248-267); the SNF writer rounds them."""
        p = C.c_void_p()
        n = C.c_uint64()
        self._check(self._lib.snfb_coverage_bins(self._h, int(task), int(binsize), C.byref(p), C.byref(n)), "snfb_coverage_bins")
        return abi.view(p.value, "<f8", n.value).copy()

    def genotype_targets(self, task, svtype, pos, svlen, bnd_is_first, mate_contig, combine_match, combine_match_max):
        """Force calling on the device (snfb_genotype_targets) after `run` on this context.  Targets as int32 arrays,
        ordered by task then input order.  Returns (match, cov_start, cov_center, cov_end, bnd_no_prev): match = the candidate's index
        in the run's emission order (int64, -1 none); bnd_no_prev = 1 for a BND with no earlier non-BND target in its task."""
        cols = [np.ascontiguousarray(a, dtype="<i4") for a in (task, svtype, pos, svlen, bnd_is_first, mate_contig)]
        n = len(cols[0])
        if any(len(a) != n for a in cols):
            raise ValueError("genotype_targets: the target arrays differ in length")
        out = (np.full(n, -1, "<i8"),) + tuple(np.zeros(n, "<i4") for _ in range(4))
        I, O = abi.GtIn(), abi.GtOut()
        I.n = n
        I.task, I.svtype, I.pos, I.svlen, I.bnd_is_first, I.mate_contig = (a.ctypes.data for a in cols)
        I.combine_match, I.combine_match_max = int(combine_match), int(combine_match_max)
        O.match, O.cov_start, O.cov_center, O.cov_end, O.bnd_no_prev = (a.ctypes.data for a in out)
        self._check(self._lib.snfb_genotype_targets(self._h, C.byref(I), C.byref(O)), "snfb_genotype_targets")
        return out

    def read_names(self):
        """The supporting reads' names of the last run's candidates (snfb_read_names), after `run` on this context and before
        the next load.  Returns ReadNames: the names' bytes back to back (uint8) and their offsets (uint32, one per name of result.rnames
        plus the end), so candidate i owns names rn_off[i] .. rn_off[i + 1], each in the order of its hash list."""
        v = abi.RnamesView()
        self._check(self._lib.snfb_read_names(self._h, C.byref(v)), "snfb_read_names")
        return ReadNames(abi.view(v.text, "u1", v.n_text).copy(), abi.view(v.off, "<u4", v.n_names + 1).copy() if v.n_names else np.zeros(1, "<u4"),
                         int(v.collisions))

    def index_bam(self, path, first_record, contig_lengths, min_shift, depth, window_bytes):
        """The tables of a BAI / CSI index of the coordinate-sorted BAM at `path`, built on the device (snfb_index_bam).  first_record: the
        virtual offset after the header; contig_lengths: the header's; window_bytes: inflated bytes per window.  Returns a dict of numpy
        copies: ref [n_ref, 5] (first v0, last v1, mapped, unmapped, linear windows), lin_off, lin, bin_key (reference * n_bins + bin), bin_loff,
        chunk_bin, chunk_beg, chunk_end, and n_no_coor, n_records, n_windows, device_bytes, device_ms."""
        clen = np.ascontiguousarray(contig_lengths, dtype="<i8")
        I, V = abi.IndexInput(), abi.IndexView()
        I.path, I.first_record, I.contig_len, I.n_ref = os.fsencode(path), int(first_record), clen.ctypes.data, len(clen)
        I.min_shift, I.depth, I.window_bytes = int(min_shift), int(depth), int(window_bytes)
        self._check(self._lib.snfb_index_bam(self._h, C.byref(I), C.byref(V)), "snfb_index_bam")
        n_ref = len(clen)
        lin_off = abi.view(V.lin_off, "<u8", n_ref + 1).copy()
        out = dict(ref=abi.view(V.ref, "<u8", 5 * n_ref).reshape(n_ref, 5).copy() if n_ref else np.zeros((0, 5), "<u8"), lin_off=lin_off,
                   lin=abi.view(V.lin, "<u8", int(lin_off[-1])).copy(), bin_key=abi.view(V.bin_key, "<u8", V.n_bin).copy(),
                   bin_loff=abi.view(V.bin_loff, "<u8", V.n_bin).copy(), chunk_bin=abi.view(V.chunk_bin, "<u4", V.n_chunk).copy(),
                   chunk_beg=abi.view(V.chunk_beg, "<u8", V.n_chunk).copy(), chunk_end=abi.view(V.chunk_end, "<u8", V.n_chunk).copy())
        out.update(n_no_coor=int(V.n_no_coor), n_records=int(V.n_records), n_windows=int(V.n_windows), device_bytes=int(V.device_bytes),
                   device_ms=float(V.device_ms))
        return out

    def sort_bam(self, path, out_path, header, first_record, contig_lengths, window_bytes, bucket_bytes):
        """The BAM at `path` sorted by coordinate into `out_path` on the device (snfb_sort_bam).  header: the output's BAM header bytes;
        first_record: the input's virtual offset after its header; contig_lengths: the header's; window_bytes / bucket_bytes: inflated bytes
        per input window / output bucket.  Returns a dict of the view's counts and per-phase milliseconds."""
        clen = np.ascontiguousarray(contig_lengths, dtype="<i8")
        hdr = np.frombuffer(bytes(header), dtype="u1")
        I, V = abi.SortInput(), abi.SortView()
        I.path, I.out_path, I.header, I.header_len = os.fsencode(path), os.fsencode(out_path), hdr.ctypes.data, len(hdr)
        I.first_record, I.contig_len, I.n_ref = int(first_record), clen.ctypes.data, len(clen)
        I.window_bytes, I.bucket_bytes = int(window_bytes), int(bucket_bytes)
        self._check(self._lib.snfb_sort_bam(self._h, C.byref(I), C.byref(V)), "snfb_sort_bam")
        return {n: (float if t is C.c_double else int)(getattr(V, n)) for n, t in abi.SortView._fields_}

    def load_reference(self, data, contigs, is_bgzf=False):
        """Reference FASTA -> the unwrapped genome resident on this context, and its 'N' runs (snfb_load_reference).  data: the file's bytes
        (whole BGZF members when is_bgzf); contigs: abi.REF_CONTIG_DTYPE rows (raw offset rebased to `data`'s inflated stream, length,
        linebases, linewidth).  Returns (runs int32 [n, 2], contig_off uint64 [n_contig + 1]) as snfb_reference_runs gives them."""
        data = np.frombuffer(data, "u1") if isinstance(data, (bytes, bytearray, memoryview)) else np.ascontiguousarray(data, dtype="u1")
        contigs = np.ascontiguousarray(contigs, dtype=abi.REF_CONTIG_DTYPE)
        I = abi.RefInput()
        I.bytes, I.n_bytes, I.is_bgzf, I.n_contig, I.contig = data.ctypes.data, len(data), int(bool(is_bgzf)), len(contigs), contigs.ctypes.data
        self._ref_n_contig = len(contigs)
        self._check(self._lib.snfb_load_reference(self._h, C.byref(I)), "snfb_load_reference")
        return self.reference_runs()

    def reference_runs(self):
        """(runs int32 [n, 2], contig_off uint64 [n_contig + 1]) of the loaded reference (snfb_reference_runs), copied"""
        r, o, n = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._check(self._lib.snfb_reference_runs(self._h, C.byref(r), C.byref(o), C.byref(n)), "snfb_reference_runs")
        return abi.view(r.value, "<i4", 2 * n.value).reshape(-1, 2).copy(), abi.view(o.value, "<u8", 0 if not o.value else self._ref_n_contig + 1).copy()

    def fetch_reference(self, queries) -> np.ndarray:
        """resolved gathers from the loaded reference (snfb_fetch_reference): abi.REF_QUERY_DTYPE rows -> the output bytes (uint8)"""
        queries = np.ascontiguousarray(queries, dtype=abi.REF_QUERY_DTYPE)
        cap = int((queries["out_off"] + queries["length"]).max()) if len(queries) else 0
        out = np.zeros(max(cap, 1), "u1")
        self._check(self._lib.snfb_fetch_reference(self._h, queries.ctypes.data, len(queries), out.ctypes.data, cap), "snfb_fetch_reference")
        return out[:cap]

    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        """Join the NCCL communicator of the per-GPU processes (the 128-byte id comes from `nccl_unique_id()` on one rank)."""
        buf = C.create_string_buffer(bytes(unique_id), 128)
        self._check(self._lib.snfb_comm_init(self._h, buf, int(rank), int(nranks)), "snfb_comm_init")

    def allgather_candidates(self, with_leads=False, device_only=False, copy=True):
        """ONE NCCL all-gather of every rank's candidate records, ALT arena and read names (SURVEY 8e) -> GatheredResult."""
        gv = abi.GatherView()
        flags = (abi.GATHER_LEADS if with_leads else 0) | (abi.GATHER_DEVICE_ONLY if device_only else 0)
        self._check(self._lib.snfb_allgather_candidates(self._h, flags, C.byref(gv)), "snfb_allgather_candidates")
        g = GatheredResult()
        g.n_cand, g.n_alt_bytes, g.n_rnames, g.n_cand_leads = int(gv.n_cand), int(gv.n_alt_bytes), int(gv.n_rnames), int(gv.n_cand_leads)
        g.dev_bytes_per_rank = int(gv.dev_bytes_per_rank)
        if not device_only:
            cp = (lambda a: a.copy()) if copy else (lambda a: a)
            g.cand = cp(abi.view(gv.cand, abi.CAND_DTYPE, gv.n_cand))
            g.alt = cp(abi.view(gv.alt, "u1", gv.n_alt_bytes))
            g.rnames = cp(abi.view(gv.rnames, "<u8", gv.n_rnames))
            g.rn_off = cp(abi.view(gv.rnames_off, "<u4", gv.n_cand + 1))
            g.cand_leads = cp(abi.view(gv.cand_leads, abi.LEAD_DTYPE, gv.n_cand_leads)) if with_leads else np.zeros(0, abi.LEAD_DTYPE)
        return g

    def poa(self, jobs):
        """Partial-order alignment jobs on the device (snfb_poa; LocalAsm's two spoa calls, local_asm.py:287-291).
        jobs: dicts with seqs (list of bytes), mode (0 consensus / 1 two-row MSA), min_cov, scores (m, n, g, e, q, c), band.
        Returns per job: bytes (mode 0), (row_a, row_b) with b'-' gaps (mode 1), or None when the job failed."""
        n = len(jobs)
        if n == 0:
            return []
        J = (abi.PoaJob * n)()
        flat, offs, out_off = [], [], 0
        seq_off = 0
        for k, jb in enumerate(jobs):
            seqs = [bytes(x) for x in jb["seqs"]]
            total = sum(len(x) for x in seqs)
            J[k].seq_off, J[k].offs_off, J[k].n_seq = seq_off, len(offs), len(seqs)
            o = 0
            for x in seqs:
                offs.append(o)
                o += len(x)
            offs.append(o)
            flat.extend(seqs)
            seq_off += total
            J[k].min_cov = int(jb.get("min_cov", 1))
            J[k].m, J[k].n, J[k].g, J[k].e, J[k].q, J[k].c = [int(x) for x in jb["scores"]]
            J[k].band = int(min(jb.get("band", 1 << 28), 1 << 28))
            J[k].mode = int(jb.get("mode", 0))
            cap = total + 16
            J[k].out_cap, J[k].out_off = cap, out_off
            out_off += cap * (2 if J[k].mode == 1 else 1)
        sq = np.frombuffer(b"".join(flat), "u1").copy() if seq_off else np.zeros(1, "u1")
        of = np.asarray(offs, dtype="<i4")
        out = np.zeros(max(out_off, 1), "u1")
        ln = np.zeros(n, "<i4")
        self._check(self._lib.snfb_poa(self._h, J, n, sq.ctypes.data, seq_off, of.ctypes.data, len(of), out.ctypes.data, out_off, ln.ctypes.data), "snfb_poa")
        res = []
        dec = lambda r: bytes(45 if x == 255 else x for x in r)
        for k in range(n):
            L = int(ln[k])
            if L < 0:
                res.append(None)
            elif J[k].mode == 0:
                res.append(out[J[k].out_off:J[k].out_off + L].tobytes())
            else:
                a = out[J[k].out_off:J[k].out_off + L]
                b = out[J[k].out_off + J[k].out_cap:J[k].out_off + J[k].out_cap + L]
                res.append((dec(a), dec(b)))
        return res

    def combine_groups(self, plan, config, arrays=None):
        """The grouping of multi-sample combine on the device (snfb_combine_groups; cluster.resolve_block_groups + the chunk loop of
        CombineTask.execute).  plan: combine.Plan.  Returns (cand_group, emit_chunk, emit_ord, cov_non[n_cand][n_samples])."""
        from . import combine
        a = arrays if arrays is not None else combine.plan_arrays(plan, config)
        n, S = len(a["pos"]), a["n_samples"]
        out = (np.zeros(max(n, 1), "<u4"), np.full(max(n, 1), -1, "<i4"), np.zeros(max(n, 1), "<u4"), np.full((max(n, 1), S), -1, "<i4"))
        if n == 0:
            return out
        I, O = abi.CombineIn(), abi.CombineOut()
        I.n_chain, I.n_chunk, I.n_cand, I.n_samples = len(a["chains"]), len(a["chunks"]), n, S
        for k in ("chains", "chunks", "pos", "svlen", "sample", "mate_contig", "mate_pos", "block_start", "cov"):
            setattr(I, k, a[k].ctypes.data)
        _combine_params(I, a, config)
        O.cand_group, O.emit_chunk, O.emit_ord, O.cov_non = (x.ctypes.data for x in out)
        self._check(self._lib.snfb_combine_groups(self._h, C.byref(I), C.byref(O)), "snfb_combine_groups")
        return out

    def combine_plan(self, flat, config):
        """The chunk plan of combine mode and the grouping on the device (snfb_combine_plan).  flat: the columns of combine.FlatPass
        (task, row, svtype, support, pos, svlen, sample, mate_contig, mate_pos, ALT arena, coverage tables) in the reference's iteration
        order.  Returns a dict: perm (slot -> flat index), chains and chunks in plan_arrays' layout, and the four outputs of combine_groups."""
        n = len(flat["pos"])
        S = flat["n_samples"]
        cap = max(n, 1)
        perm, chains, chunks = np.zeros(cap, "<u4"), np.zeros((cap, 6), "<u4"), np.zeros((cap, 6), "<i4")
        out = (np.zeros(cap, "<u4"), np.full(cap, -1, "<i4"), np.zeros(cap, "<u4"), np.full((cap, S), -1, "<i4"))
        I, O = abi.CombinePlanIn(), abi.CombinePlanOut()
        I.n_flat, I.n_task = n, flat["n_task"]
        for k in ("task", "row", "svtype", "support"):
            setattr(I, k, flat[k].ctypes.data)
        I.support_threshold, I.bin_min_size = int(config.combine_support_threshold), int(config.combine_min_size)
        I.bin_max_candidates, I.exhaustive = max(25, int(len(config.snf_input_info) * 0.5)), int(bool(config.combine_exhaustive))      # parallel.py:458
        G = I.group
        G.n_cand, G.n_samples = n, S
        for k in ("pos", "svlen", "sample", "mate_contig", "mate_pos", "block_start", "cov"):
            setattr(G, k, flat[k].ctypes.data)
        _combine_params(G, flat, config)
        O.perm, O.chains, O.chunks = perm.ctypes.data, chains.ctypes.data, chunks.ctypes.data
        O.group.cand_group, O.group.emit_chunk, O.group.emit_ord, O.group.cov_non = (x.ctypes.data for x in out)
        self._check(self._lib.snfb_combine_plan(self._h, C.byref(I), C.byref(O)), "snfb_combine_plan")
        m = int(O.n_cand)
        return dict(perm=perm[:m], chains=chains[:O.n_chain], chunks=chunks[:O.n_chunk], cand_group=out[0][:m], emit_chunk=out[1][:m], emit_ord=out[2][:m],
                    cov_non=out[3][:m])

    def population_load(self, contig, block, svtype, pos, svlen, alts):
        """The population table on the device (snfb_population_load): per variant in file order its contig index (-1: not among the
        run's contigs), block key, svtype 0..4, pos, svlen and ALT bytes.  It replaces any table loaded before."""
        cols = [np.ascontiguousarray(v, "<i4") for v in (contig, block, svtype, pos, svlen)]
        arena = alt_arena(alts)
        T = abi.PopTable()
        T.n = len(cols[0])
        T.contig, T.block, T.svtype, T.pos, T.svlen = (v.ctypes.data for v in cols)
        T.alt, T.alt_off, T.alt_len, T.n_alt_bytes = arena[0].ctypes.data, arena[1].ctypes.data, arena[2].ctypes.data, len(arena[0]) - 1
        self._check(self._lib.snfb_population_load(self._h, C.byref(T)), "snfb_population_load")

    def population_match(self, contig, svtype, pos, svlen, alts, combine_match, combine_match_max, combine_pctseq, block_size):
        """PopulationSNF.get_population_AF on the device for one batch of calls (snfb_population_match): per call the file-order index of
        the matching population variant, -1 for none, -2 where the reference would divide by a zero svlen"""
        cols = [np.ascontiguousarray(v, "<i4") for v in (contig, svtype, pos, svlen)]
        n = len(cols[0])
        if n == 0:
            return np.zeros(0, "<i4")
        arena = alt_arena(alts)
        Q = abi.PopQuery()
        Q.n = n
        Q.contig, Q.svtype, Q.pos, Q.svlen = (v.ctypes.data for v in cols)
        Q.alt, Q.alt_off, Q.alt_len, Q.n_alt_bytes = arena[0].ctypes.data, arena[1].ctypes.data, arena[2].ctypes.data, len(arena[0]) - 1
        Q.combine_match, Q.combine_match_max, Q.block_size = int(combine_match), int(combine_match_max), int(block_size)
        Q.combine_pctseq = float(combine_pctseq or 0.0)
        best = np.zeros(n, "<i4")
        self._check(self._lib.snfb_population_match(self._h, C.byref(Q), best.ctypes.data), "snfb_population_match")
        return best

    def edit_distances(self, pairs):
        """device edit distance of (bytes, bytes) pairs (snfb_selftest_edit_distance)"""
        n = len(pairs)
        if n == 0:
            return np.zeros(0, "<i4")
        flat = [x for p in pairs for x in p]
        lens = np.array([len(x) for x in flat], "<u4")
        offs = np.zeros(len(flat), "<u8")
        offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
        by = np.frombuffer(b"".join(bytes(x) for x in flat) + b"\0", "u1").copy()
        ao, bo, al, bl = (np.ascontiguousarray(v) for v in (offs[0::2], offs[1::2], lens[0::2], lens[1::2]))
        out = np.zeros(n, "<i4")
        self._check(self._lib.snfb_selftest_edit_distance(self._h, by.ctypes.data, len(by), ao.ctypes.data, al.ctypes.data, bo.ctypes.data, bl.ctypes.data, n, out.ctypes.data), "snfb_selftest_edit_distance")
        return out

    def device_alt(self):
        p = C.c_void_p()
        n = C.c_uint64()
        self._check(self._lib.snfb_device_alt(self._h, C.byref(p), C.byref(n)), "snfb_device_alt")
        return p.value, int(n.value)

    def device_candidates(self):
        p = C.c_void_p()
        n = C.c_uint64()
        self._check(self._lib.snfb_device_candidates(self._h, C.byref(p), C.byref(n)), "snfb_device_candidates")
        return p.value, int(n.value)


class ReadNames:
    """The read names of a run's candidates (Context.read_names): text (uint8) and off (uint32, [n_names + 1]) with name k =
    text[off[k]:off[k + 1]], in the order of the run's rnames hashes; collisions = leads whose name differs from the one kept for their hash."""

    def __init__(self, text, off, collisions=0):
        self.text, self.off, self.collisions = text, off, collisions
        self._str = self._off = None

    def per_candidate(self, rn_off, lo, hi):
        """[list of str] for candidates lo .. hi - 1 (rn_off: the run's rnames offsets).  The text is decoded once, as ASCII (the SAM
        specification's QNAME alphabet), and every name is a slice of that one string."""
        if self._str is None:
            self._str, self._off = self.text.tobytes().decode("ascii"), self.off.tolist()
        s, off = self._str, self._off
        return [[s[off[k]:off[k + 1]] for k in range(int(rn_off[i]), int(rn_off[i + 1]))] for i in range(lo, hi)]


def alt_arena(alts):
    """[bytes] -> (arena with one spare byte, u64 offsets, u32 lengths)"""
    lens = np.fromiter((len(a) for a in alts), "<u4", len(alts))
    offs = np.zeros(len(alts), "<u8")
    if len(alts):
        offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    return np.frombuffer(b"".join(alts) + b"\0", np.uint8).copy(), offs, lens


def _combine_params(I, a, config):
    """the coverage geometry, the grouping parameters and (with --combine-pctseq != 0) the ALT arena of an snfb_combine_in"""
    I.n_cov_block, I.bins_per_block, I.cov_binsize = len(a["block_start"]), a["bins_per_block"], a["cov_binsize"]
    I.combine_match, I.combine_match_max, I.cluster_merge_bnd = int(config.combine_match), int(config.combine_match_max), int(config.cluster_merge_bnd)
    I.combine_separate_intra, I.combine_overlap_abs = int(bool(config.combine_separate_intra)), int(config.combine_overlap_abs)
    I.combine_pctseq = float(getattr(config, "combine_pctseq", 0.0) or 0.0)
    if I.combine_pctseq != 0.0:
        I.alt, I.alt_off, I.alt_len, I.n_alt_bytes = a["alt"].ctypes.data, a["alt_off"].ctypes.data, a["alt_len"].ctypes.data, len(a["alt"])
