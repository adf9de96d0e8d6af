"""ctypes / numpy mirrors of the C structs in include/snfb.h (single source of truth is
the header; tests/test_abi.py checks sizes and offsets against the compiled library)."""
import ctypes as C

import numpy as np

INS, DEL, DUP, INV, BND, SINGLE_LEFT, SINGLE_RIGHT = range(7)
SVTYPE_NAMES = ["INS", "DEL", "DUP", "INV", "BND", "SINGLE_LEFT", "SINGLE_RIGHT"]  # sv.py:31-33 order
SOURCE_NAMES = ["INLINE", "SPLIT_PRIM", "SPLIT_SUP", "BND_SA"]
AUX_NM, AUX_HP, AUX_PS, AUX_SA = 1, 2, 4, 8
CIGAR_BAM32, CIGAR_16 = 0, 1

LF_REVERSE, LF_IS_SA, LF_SVLEN_NONE, LF_BND_FIRST, LF_BND_REVERSE, LF_HAS_SEQ = (1 << 5, 1 << 6, 1 << 7, 1 << 8, 1 << 9, 1 << 10)

REC_DTYPE = np.dtype([
    ("task", "<i4"), ("pos", "<i4"), ("flag", "<u2"), ("mapq", "u1"), ("aux_flags", "u1"),
    ("hp", "u1"), ("l_qname", "u1"), ("_pad0", "<u2"), ("nm", "<i4"), ("ps", "<i4"),
    ("n_cigar", "<u4"), ("l_seq", "<i4"), ("sa_len", "<u4"), ("region", "<u4"),
    ("cigar_off", "<u8"), ("seq_off", "<u8"), ("var_off", "<u8")])
assert REC_DTYPE.itemsize == 64

TASK_DTYPE = np.dtype([("contig", "<i4"), ("start", "<i4"), ("end", "<i4"), ("contig_len", "<i4"),
                       ("task_id", "<i4"), ("tr_off", "<i4"), ("tr_n", "<i4"), ("_pad", "<i4")])
CONTIG_DTYPE = np.dtype([("name_hash", "<u8"), ("length", "<i4"), ("lex_rank", "<i4")])

LEAD_DTYPE = np.dtype([
    ("rec", "<u4"), ("ref_start", "<i4"), ("ref_end", "<i4"), ("qry_start", "<i4"), ("qry_end", "<i4"),
    ("svlen", "<i4"), ("seq_off", "<i4"), ("seq_len", "<i4"), ("read_len", "<i4"), ("mate_pos", "<i4"),
    ("mate_contig", "<i4"), ("nm_sa", "<i4"), ("flags", "<u4"), ("task", "<u2"), ("k", "<u2"),
    ("qname_hash", "<u8")])
assert LEAD_DTYPE.itemsize == 64

CAND_DTYPE = np.dtype([
    ("task", "<i4"), ("svtype", "<i4"), ("pos", "<i4"), ("end", "<i4"), ("svlen", "<i4"), ("support", "<i4"),
    ("qual", "<i4"), ("precise", "<i4"), ("fwd", "<i4"), ("rev", "<i4"), ("support_long", "<i4"),
    ("support_sa", "<i4"), ("cov_upstream", "<i4"), ("cov_start", "<i4"), ("cov_center", "<i4"),
    ("cov_end", "<i4"), ("cov_downstream", "<i4"), ("hap_counts", "<i4", (6,)), ("sa_count", "<i4"),
    ("sa_total", "<i4"), ("bnd_mate_contig", "<i4"), ("bnd_mate_pos", "<i4"), ("bnd_is_first", "<i4"),
    ("bnd_is_reverse", "<i4"), ("n_strands", "<i4"), ("support_inline", "<i4"), ("lead_off", "<i4"),
    ("lead_n", "<i4"), ("long_off", "<i4"), ("long_n", "<i4"), ("alt_off", "<i4"), ("alt_len", "<i4"),
    ("hp_top", "<i4"), ("hp_support", "<i4"), ("hp_other", "<i4"), ("ps_top", "<i4"), ("ps_top_null", "<i4"),
    ("ps_support", "<i4"), ("ps_other", "<i4"), ("cluster_seed", "<i4"), ("resplit_bin", "<i4"),
    ("stdev_pos", "<f8"), ("stdev_len", "<f8"), ("nm_mean", "<f8")], align=True)


class Records(C.Structure):
    _fields_ = [("n_rec", C.c_uint64), ("n_cigar", C.c_uint64), ("n_var", C.c_uint64), ("n_seq", C.c_uint64),
                ("rec", C.c_void_p), ("cigar", C.c_void_p), ("var", C.c_void_p), ("seq", C.c_void_p),
                ("n_task", C.c_uint32), ("n_contig", C.c_uint32), ("n_tr", C.c_uint32), ("on_device", C.c_uint32),
                ("task", C.c_void_p), ("contig", C.c_void_p), ("tr", C.c_void_p),
                ("n_mask", C.c_uint32), ("cigar_fmt", C.c_uint32), ("mask", C.c_void_p), ("mask_task_off", C.c_void_p),
                ("cigar_evt_min", C.c_uint32), ("_pad2", C.c_uint32)]


SPAN_DTYPE = np.dtype([("cbeg", "<u8"), ("cend", "<u8"), ("ubeg", "<u4"), ("uend", "<u4"), ("task", "<u4"), ("region", "<u4")])      # snfb_bam_span
REGION_DTYPE = np.dtype([("task", "<i4"), ("start", "<i4"), ("end", "<i4"), ("_pad", "<i4")])      # snfb_region
assert SPAN_DTYPE.itemsize == 32


class BamInput(C.Structure):                                    # snfb_bam_input
    _fields_ = [("bgzf", C.c_void_p), ("n_bytes", C.c_uint64), ("span", C.c_void_p), ("n_span", C.c_uint64),
                ("n_task", C.c_uint32), ("n_contig", C.c_uint32), ("n_tr", C.c_uint32), ("n_mask", C.c_uint32),
                ("task", C.c_void_p), ("contig", C.c_void_p), ("tr", C.c_void_p), ("mask", C.c_void_p), ("mask_task_off", C.c_void_p)]


class Config(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "mapq", "min_alignment_length", "exclude_flags", "minsvlen", "minsvlen_screen", "long_ins_length",
        "detect_large_ins", "dev_seq_cache_maxlen", "max_splits_base", "dev_keep_lowqual_splits",
        "qc_nm_measure", "phase", "cluster_binsize", "cluster_merge_pos", "cluster_merge_bnd",
        "cluster_resplit_binsize", "repeat", "dev_min_leads_cluster", "dev_no_resplit", "dev_no_resplit_repeat",
        "consensus_max_reads_bin", "consensus_min_reads", "consensus_kmer_len", "consensus_kmer_skip_base",
        "no_consensus", "symbolic", "precise", "coverage_binsize", "coverage_updown_bins", "_pad")] + [
        (n, C.c_double) for n in ("max_splits_kb", "cluster_r", "cluster_repeat_h", "cluster_repeat_h_max",
                                  "cluster_merge_len", "consensus_kmer_skip_seqlen_mult")]

    @classmethod
    def from_sniffles(cls, cfg) -> "Config":
        """Flatten a reference-style SnifflesConfig namespace (config.py:449-619)."""
        c = cls()
        c.mapq = int(cfg.mapq)
        c.min_alignment_length = int(cfg.min_alignment_length)
        c.exclude_flags = int(cfg.exclude_flags) if getattr(cfg, "exclude_flags", None) else 0
        c.minsvlen = int(cfg.minsvlen)
        c.minsvlen_screen = int(cfg.minsvlen_screen)
        c.long_ins_length = int(cfg.long_ins_length)
        c.detect_large_ins = int(bool(cfg.detect_large_ins))
        c.dev_seq_cache_maxlen = int(cfg.dev_seq_cache_maxlen)
        c.max_splits_base = int(cfg.max_splits_base)
        c.dev_keep_lowqual_splits = int(bool(cfg.dev_keep_lowqual_splits))
        c.qc_nm_measure = int(bool(cfg.qc_nm_measure))
        c.phase = int(bool(cfg.phase))
        c.cluster_binsize = int(cfg.cluster_binsize)
        c.cluster_merge_pos = int(cfg.cluster_merge_pos)
        c.cluster_merge_bnd = int(cfg.cluster_merge_bnd)
        c.cluster_resplit_binsize = int(cfg.cluster_resplit_binsize)
        c.repeat = int(bool(cfg.repeat))
        c.dev_min_leads_cluster = int(cfg.dev_min_leads_cluster)
        c.dev_no_resplit = int(bool(cfg.dev_no_resplit))
        c.dev_no_resplit_repeat = int(bool(cfg.dev_no_resplit_repeat))
        c.consensus_max_reads_bin = int(cfg.consensus_max_reads_bin)
        c.consensus_min_reads = int(cfg.consensus_min_reads)
        c.consensus_kmer_len = int(cfg.consensus_kmer_len)
        c.consensus_kmer_skip_base = int(cfg.consensus_kmer_skip_base)
        c.no_consensus = int(bool(cfg.no_consensus))
        c.symbolic = int(bool(cfg.symbolic))
        c.precise = int(cfg.precise)
        c.coverage_binsize = int(cfg.coverage_binsize)
        c.coverage_updown_bins = int(cfg.coverage_updown_bins)
        c.max_splits_kb = float(cfg.max_splits_kb)
        c.cluster_r = float(cfg.cluster_r)
        c.cluster_repeat_h = float(cfg.cluster_repeat_h)
        c.cluster_repeat_h_max = float(cfg.cluster_repeat_h_max)
        c.cluster_merge_len = float(cfg.cluster_merge_len)
        c.consensus_kmer_skip_seqlen_mult = float(cfg.consensus_kmer_skip_seqlen_mult)
        return c


class LeadView(C.Structure):
    _fields_ = [("n_leads", C.c_uint64), ("leads", C.c_void_p), ("n_pass", C.c_uint64),
                ("task_read_count", C.c_void_p), ("task_mean_nm", C.c_void_p), ("rec_nm", C.c_void_p),
                ("soft_errors", C.c_uint64)]


class CandView(C.Structure):
    _fields_ = [("n_cand", C.c_uint64), ("cand", C.c_void_p), ("n_cand_leads", C.c_uint64),
                ("cand_leads", C.c_void_p), ("rnames", C.c_void_p), ("rnames_off", C.c_void_p),
                ("task_coverage_mean", C.c_void_p), ("unverified_breaks", C.c_uint64)]


class SeqView(C.Structure):
    _fields_ = [("n_alt_bytes", C.c_uint64), ("alt", C.c_void_p)]


GATHER_LEADS, GATHER_DEVICE_ONLY = 1, 2


class PoaJob(C.Structure):
    _fields_ = [("seq_off", C.c_uint64), ("offs_off", C.c_uint32), ("n_seq", C.c_uint32), ("min_cov", C.c_int32)] + [(k, C.c_int32) for k in ("m", "n", "g", "e", "q", "c", "band")] + [
        ("mode", C.c_uint32), ("out_cap", C.c_uint32), ("out_off", C.c_uint64)]


class CombineIn(C.Structure):                                   # snfb_combine_in
    _fields_ = [("n_chain", C.c_uint32), ("n_chunk", C.c_uint32), ("n_cand", C.c_uint32), ("n_samples", C.c_uint32),
                ("chains", C.c_void_p), ("chunks", C.c_void_p), ("pos", C.c_void_p), ("svlen", C.c_void_p), ("sample", C.c_void_p),
                ("mate_contig", C.c_void_p), ("mate_pos", C.c_void_p),
                ("n_cov_block", C.c_uint32), ("bins_per_block", C.c_int32), ("cov_binsize", C.c_int32), ("pad", C.c_int32),
                ("block_start", C.c_void_p), ("cov", C.c_void_p),
                ("combine_match", C.c_int32), ("combine_match_max", C.c_int32), ("cluster_merge_bnd", C.c_int32),
                ("combine_separate_intra", C.c_int32), ("combine_overlap_abs", C.c_int32), ("pad2", C.c_int32),
                ("combine_pctseq", C.c_double), ("alt", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p), ("n_alt_bytes", C.c_uint64)]


class CombineOut(C.Structure):                                  # snfb_combine_out
    _fields_ = [("cand_group", C.c_void_p), ("emit_chunk", C.c_void_p), ("emit_ord", C.c_void_p), ("cov_non", C.c_void_p)]


class CombinePlanIn(C.Structure):                               # snfb_combine_plan_in
    _fields_ = [("n_flat", C.c_uint32), ("n_task", C.c_uint32), ("task", C.c_void_p), ("row", C.c_void_p), ("svtype", C.c_void_p), ("support", C.c_void_p),
                ("support_threshold", C.c_int32), ("bin_min_size", C.c_int32), ("bin_max_candidates", C.c_int32), ("exhaustive", C.c_int32),
                ("group", CombineIn)]


class CombinePlanOut(C.Structure):                              # snfb_combine_plan_out
    _fields_ = [("n_cand", C.c_uint32), ("n_chain", C.c_uint32), ("n_chunk", C.c_uint32), ("pad", C.c_uint32),
                ("perm", C.c_void_p), ("chains", C.c_void_p), ("chunks", C.c_void_p), ("group", CombineOut)]


class PopTable(C.Structure):                                    # snfb_pop_table
    _fields_ = [("n", C.c_uint32), ("pad", C.c_uint32), ("contig", C.c_void_p), ("block", C.c_void_p), ("svtype", C.c_void_p), ("pos", C.c_void_p),
                ("svlen", C.c_void_p), ("alt", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p), ("n_alt_bytes", C.c_uint64)]


class PopQuery(C.Structure):                                    # snfb_pop_query
    _fields_ = [("n", C.c_uint32), ("pad", C.c_uint32), ("contig", C.c_void_p), ("svtype", C.c_void_p), ("pos", C.c_void_p), ("svlen", C.c_void_p),
                ("alt", C.c_void_p), ("alt_off", C.c_void_p), ("alt_len", C.c_void_p), ("n_alt_bytes", C.c_uint64),
                ("combine_match", C.c_int32), ("combine_match_max", C.c_int32), ("block_size", C.c_int32), ("pad2", C.c_int32),
                ("combine_pctseq", C.c_double)]


class GatherView(C.Structure):
    _fields_ = [("n_cand", C.c_uint64), ("cand", C.c_void_p), ("n_alt_bytes", C.c_uint64), ("alt", C.c_void_p),
                ("n_rnames", C.c_uint64), ("rnames", C.c_void_p), ("rnames_off", C.c_void_p),
                ("n_cand_leads", C.c_uint64), ("cand_leads", C.c_void_p), ("rank_n_cand", C.c_void_p),
                ("dev_buffer", C.c_void_p), ("dev_bytes_per_rank", C.c_uint64)]


class GtIn(C.Structure):                                        # snfb_gt_in
    _fields_ = [("n", C.c_uint64), ("task", C.c_void_p), ("svtype", C.c_void_p), ("pos", C.c_void_p), ("svlen", C.c_void_p),
                ("bnd_is_first", C.c_void_p), ("mate_contig", C.c_void_p), ("combine_match", C.c_int32), ("combine_match_max", C.c_int32)]


class GtOut(C.Structure):                                       # snfb_gt_out
    _fields_ = [("match", C.c_void_p), ("cov_start", C.c_void_p), ("cov_center", C.c_void_p), ("cov_end", C.c_void_p), ("bnd_no_prev", C.c_void_p)]


class IndexInput(C.Structure):                                  # snfb_index_input
    _fields_ = [("path", C.c_char_p), ("first_record", C.c_uint64), ("contig_len", C.c_void_p), ("n_ref", C.c_uint32),
                ("min_shift", C.c_int32), ("depth", C.c_int32), ("_pad", C.c_int32), ("window_bytes", C.c_uint64)]


class IndexView(C.Structure):                                   # snfb_index_view
    _fields_ = [(n, C.c_void_p) for n in ("ref", "lin_off", "lin", "bin_key", "bin_loff", "chunk_bin", "chunk_beg", "chunk_end")] + \
               [(n, C.c_uint64) for n in ("n_bin", "n_chunk", "n_no_coor", "n_records", "n_windows", "device_bytes")] + [("device_ms", C.c_double)]


class SortInput(C.Structure):                                   # snfb_sort_input
    _fields_ = [("path", C.c_char_p), ("out_path", C.c_char_p), ("header", C.c_void_p), ("header_len", C.c_uint64), ("first_record", C.c_uint64),
                ("contig_len", C.c_void_p), ("n_ref", C.c_uint32), ("_pad", C.c_uint32), ("window_bytes", C.c_uint64), ("bucket_bytes", C.c_uint64)]


class SortView(C.Structure):                                    # snfb_sort_view
    _fields_ = [(n, C.c_uint64) for n in ("n_records", "n_windows", "n_buckets", "n_members", "n_input_reads", "bytes_in", "bytes_out", "device_bytes")] + \
               [(n, C.c_double) for n in ("ms_keys", "ms_sort", "ms_layout", "ms_scatter", "ms_deflate", "ms_layout_host")]


class RnamesView(C.Structure):                                  # snfb_rnames_view
    _fields_ = [("n_names", C.c_uint64), ("n_text", C.c_uint64), ("text", C.c_void_p), ("off", C.c_void_p), ("collisions", C.c_uint64)]


REF_CONTIG_DTYPE = np.dtype([("offset", "<u8"), ("length", "<u8"), ("linebases", "<u4"), ("linewidth", "<u4")])       # snfb_ref_contig
REF_QUERY_DTYPE = np.dtype([("contig", "<u4"), ("_pad", "<u4"), ("start", "<u8"), ("length", "<u8"), ("out_off", "<u8")])  # snfb_ref_query


class RefInput(C.Structure):                                    # snfb_ref_input
    _fields_ = [("bytes", C.c_void_p), ("n_bytes", C.c_uint64), ("is_bgzf", C.c_uint32), ("n_contig", C.c_uint32), ("contig", C.c_void_p)]


def view(ptr, dtype, n):
    """numpy array over library-owned memory (no copy); empty array for n == 0 / NULL."""
    dtype = np.dtype(dtype)
    if not ptr or n == 0:
        return np.zeros(0, dtype)
    buf = (C.c_uint8 * (int(n) * dtype.itemsize)).from_address(ptr)
    return np.frombuffer(buf, dtype=dtype, count=int(n))


def fnv1a64(name: bytes) -> int:
    """snfb_hash_name: FNV-1a 64 over the contig name bytes."""
    h = 0xcbf29ce484222325
    for b in name:
        h = ((h ^ b) * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return h
