/*
 * snfb.h — C ABI of libsnfb200.so: the H100-native lead -> cluster -> consensus hot path
 * of Sniffles2, callable through ctypes from the Python host (sniffles_b200/binding.py).
 *
 * Every entry point replaces a Python call site of the reference (paths relative to
 * /root/reference/src/sniffles/):
 *
 *   snfb_load_records      <- pysam `bam.fetch()` iteration + AlignedSegment accessors
 *                             (leadprov.py:488, accessor list SURVEY.md §2)
 *   snfb_load_bam          <- the same call site fed COMPRESSED BAM bytes: htslib's BGZF inflate, record decode, region
 *                             filter and long-CIGAR (CG) escape behind `bam.fetch(contig, start, end)` run on the device
 *                             (parallel.py:95-98, leadprov.py:488; SURVEY §8 (f)3)
 *   snfb_extract_leads     <- LeadProvider.build_leadtab / iter_region / read_iterindels /
 *                             Lead.for_bnd / read_itersplits (leadprov.py:445-670),
 *                             sv.classify_splits (sv.py:649-782); call site parallel.py:90-102
 *   snfb_cluster_call      <- cluster.resolve + merge_inner + resplit + resplit_bnd
 *                             (cluster.py:85-353), sv.call_from / resolve_bnd (sv.py:497-639),
 *                             postprocessing.coverage (postprocessing.py:69-130);
 *                             call site Task.call_candidates parallel.py:104-127
 *   snfb_consensus         <- postprocessing.annotate_sv INS branch (postprocessing.py:33-66)
 *                             + consensus.novel_from_reads (consensus.py:280-394);
 *                             call site Task.finalize_candidates parallel.py:145
 *   snfb_poa               <- spoa.poa as LocalAsm.assembly calls it (local_asm.py:287-291); call site parallel.py:186-196
 *   snfb_coverage_bins     <- SNFile.annotate_block_coverages' reshape-mean of lead_provider.coverage
 *                             (snf.py:248-267)
 *   snfb_load_reference / snfb_reference_runs / snfb_fetch_reference
 *                          <- pysam.FastaFile behind LeadProvider._mask_N_coverage (leadprov.py:420-443) and
 *                             VCF.open_reference / write_call (vcf.py:108-119, 299-342)
 *   snfb_read_names        <- the query names behind SVCall.rnames (sv.py:520-525, 555), written as RNAMES by --output-rnames
 *   snfb_allgather_candidates <- the parent collecting every worker's finished task results before VCF
 *                             emission (sniffles:544-547, parallel.py:270-271), as one NCCL all-gather
 *
 * Conventions: all functions return 0 on success, non-zero on error (message via
 * snfb_last_error).  No exceptions, no Python or torch types.  Views are library-owned
 * pinned host buffers, valid until the next call on the same ctx.  A ctx is bound to
 * one CUDA device and is not thread safe.  There is NO CPU fallback: if no CUDA device
 * is usable snfb_ctx_create fails.
 */
#ifndef SNFB_H
#define SNFB_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SNFB_ABI_VERSION 3

/* SV types in the reference's ALL_TYPES order (sv.py:31-33); the emission order of
 * candidates follows this order (parallel.py:106). */
enum { SNFB_INS = 0, SNFB_DEL = 1, SNFB_DUP = 2, SNFB_INV = 3, SNFB_BND = 4,
       SNFB_SINGLE_LEFT = 5, SNFB_SINGLE_RIGHT = 6, SNFB_NTYPES = 7 };
/* Lead.source (leadprov.py:46) */
enum { SNFB_SRC_INLINE = 0, SNFB_SRC_SPLIT_PRIM = 1, SNFB_SRC_SPLIT_SUP = 2, SNFB_SRC_BND_SA = 3 };

/* snfb_records.on_device */
#define SNFB_MEM_HOST 0u
#define SNFB_MEM_DEVICE 1u
#define SNFB_MEM_HOST_SEQ_ON_DEMAND 2u

/* snfb_records.cigar_fmt
 *
 * SNFB_CIGAR_BAM32: the BAM record's own words, len<<4|op (op: MIDNSHP=X = 0..8), 4 bytes per op.
 *
 * SNFB_CIGAR_16 (what the kernels read; snfb_pack_cigar16 produces it): 2-byte words, half the PCIe and HBM bytes.
 *   base word       bit 15 = 0, bit 14 = E, bits 11..13 = class, bits 0..10 = length & 0x7ff
 *                   class: 0 P (and the zero-length pad word 0x0000), 1 I, 2 D, 3 M/=/X, 4 H, 5 S, 6 N
 *                   (bit 11: the op advances the read, bit 12: it advances the reference)
 *                   E: the op is an I / D / S of at least the block's event length (snfb_records.cigar_evt_min, default
 *                   SNFB_CIGAR16_EVT_MIN = 11: every SV signature and every indel the NM correction counts).  The streaming kernel
 *                   only sums lengths and ORs this bit; a configuration that looks at shorter events re-flags the arena on the device.
 *   extension word  bit 15 = 1, bits 12..14 = level (1 or 2), bits 0..11 = payload: adds payload << (11 + 12 * (level - 1)) to the
 *                   length of the base word it follows (level 1, then level 2; lengths up to 2^28 as in BAM)
 *   A base word and its extension words never straddle a 16-byte boundary and every record starts on one; the gaps and
 *   the tail of the arena are filled with pad words, so a 16-byte load never needs masking.
 *   M, = and X are one class: the path never tells them apart (leadprov.py:137-142 OPLIST). */
#define SNFB_CIGAR_BAM32 0u
#define SNFB_CIGAR_16 1u
#define SNFB_CIGAR16_EVT_MIN 11u

/* aux_flags bits of snfb_rec */
#define SNFB_AUX_NM 1u
#define SNFB_AUX_HP 2u
#define SNFB_AUX_PS 4u
#define SNFB_AUX_SA 8u

/* One packed alignment record: the fields of a BAM record the path reads (SURVEY §8a A0),
 * fixed 64 bytes so a warp fetches it with one coalesced request.  Base qualities are
 * never shipped.  Variable-length parts live in three arenas of the block:
 *   cigar[cigar_off .. +n_cigar)   CIGAR words in the block's cigar_fmt (SNFB_CIGAR_*)
 *   var[var_off .. +l_qname)       query name bytes (no NUL), followed by
 *   var[var_off+l_qname .. +sa_len) the SA:Z tag text (no NUL)
 *   seq[seq_off .. +(l_seq+1)/2)   BAM 4-bit bases ("=ACMGRSVTWYHKDBN"), high nibble first
 */
typedef struct snfb_rec {
    int32_t  task;        /* index into the task table (one task per contig/region)   */
    int32_t  pos;         /* 0-based reference_start                                    */
    uint16_t flag;        /* SAM flag                                                   */
    uint8_t  mapq;
    uint8_t  aux_flags;   /* SNFB_AUX_*                                                 */
    uint8_t  hp;          /* HP:i tag value (0 when absent); must be 0,1,2              */
    uint8_t  l_qname;
    uint16_t _pad0;
    int32_t  nm;          /* NM:i tag value                                             */
    int32_t  ps;          /* PS:i tag value                                             */
    uint32_t n_cigar;     /* words of this record (CIGAR16: pad words inside included)   */
    int32_t  l_seq;       /* query_length (bases stored in seq)                         */
    uint32_t sa_len;
    uint32_t region;      /* index into the region table (snfb_set_regions); ignored while that table is empty */
    uint64_t cigar_off;   /* in words of the block's cigar_fmt (CIGAR16: a multiple of 8) */
    uint64_t seq_off;     /* in bytes                                                   */
    uint64_t var_off;     /* in bytes                                                   */
} snfb_rec;

/* One unit of work = what the reference hands to one CallTask (parallel.py:47-60):
 * a contig and one region on it.  Clusters never cross tasks. */
typedef struct snfb_task {
    int32_t contig;       /* index into the contig table                               */
    int32_t start;        /* region.start                                              */
    int32_t end;          /* region.end (exclusive)                                    */
    int32_t contig_len;   /* bam.get_reference_length(contig)                          */
    int32_t task_id;      /* Task.id (only used for ids on the host)                   */
    int32_t tr_off;       /* first tandem-repeat interval of this task in tr[]         */
    int32_t tr_n;         /* number of intervals (sorted by start, already padded)     */
    int32_t _pad;
} snfb_task;

/* Reference names: the SA tag names its mate contig as a string (leadprov.py:82);
 * the library resolves it through FNV-1a 64 hashes of the names and needs the
 * lexicographic rank of each name for util.most_common_top ties (util.py:101-103). */
typedef struct snfb_contig {
    uint64_t name_hash;   /* snfb_hash_name(name)                                      */
    int32_t  length;
    int32_t  lex_rank;    /* rank of the name among all contig names, byte-wise order  */
} snfb_contig;

typedef struct snfb_records {
    uint64_t n_rec;
    uint64_t n_cigar;     /* words in the cigar arena (CIGAR16: a multiple of 8, padded)  */
    uint64_t n_var;       /* bytes       */
    uint64_t n_seq;       /* bytes       */
    const snfb_rec* rec;
    const void*     cigar;   /* uint32_t[] (SNFB_CIGAR_BAM32) or uint16_t[] (SNFB_CIGAR_16) */
    const uint8_t*  var;
    const uint8_t*  seq;
    uint32_t n_task;
    uint32_t n_contig;
    uint32_t n_tr;
    uint32_t on_device;   /* SNFB_MEM_*: 0 host arenas (copied), 1 device arenas (no copy), 2 host arenas with the seq arena
                             left on the host: only the base slices the consensus stage asks for are fetched ("seq on demand") */
    const snfb_task*   task;
    const snfb_contig* contig;
    const int32_t*     tr;    /* n_tr pairs (start,end), per task sorted (util.py:121-147) */
    /* optional: reference 'N' runs per task for LeadProvider._mask_N_coverage (leadprov.py:420-443, only with --reference):
     * n_mask half-open pairs (start,end), sorted and disjoint inside a task; task t owns mask[mask_task_off[t] .. mask_task_off[t+1]).
     * snfb_load_records / snfb_load_bam refuse a task whose runs have start > end or overlap / precede the run before them. */
    uint32_t n_mask;
    uint32_t cigar_fmt;   /* SNFB_CIGAR_*; BAM32 host arenas are converted on the host inside snfb_load_records (device arenas must be CIGAR16) */
    const int32_t*  mask;
    const uint32_t* mask_task_off;   /* [n_task + 1]; may be NULL when n_mask == 0 */
    uint32_t cigar_evt_min;          /* CIGAR16: the event length the E bits were set for (0 = SNFB_CIGAR16_EVT_MIN) */
    uint32_t _pad2;
} snfb_records;

/* Flat POD of the reference's config values that the path reads (config.py:449-619). */
typedef struct snfb_config {
    int32_t mapq;                      /* config.py:533-534  */
    int32_t min_alignment_length;      /* config.py:535-536  */
    int32_t exclude_flags;             /* 0 = None           */
    int32_t minsvlen;                  /* config.py:508-514  */
    int32_t minsvlen_screen;           /* config.py:517      */
    int32_t long_ins_length;           /* 2500               */
    int32_t detect_large_ins;          /* bool               */
    int32_t dev_seq_cache_maxlen;      /* 50000              */
    int32_t max_splits_base;           /* 3                  */
    int32_t dev_keep_lowqual_splits;   /* bool               */
    int32_t qc_nm_measure;             /* config.py:596-599  */
    int32_t phase;                     /* bool               */
    int32_t cluster_binsize;           /* 100                */
    int32_t cluster_merge_pos;         /* 150                */
    int32_t cluster_merge_bnd;         /* 1000               */
    int32_t cluster_resplit_binsize;   /* 20                 */
    int32_t repeat;                    /* --repeat           */
    int32_t dev_min_leads_cluster;     /* config.py:607-611  */
    int32_t dev_no_resplit;
    int32_t dev_no_resplit_repeat;
    int32_t consensus_max_reads_bin;   /* 10                 */
    int32_t consensus_min_reads;       /* 4                  */
    int32_t consensus_kmer_len;        /* 6 (only 6 is supported on device) */
    int32_t consensus_kmer_skip_base;  /* 3                  */
    int32_t no_consensus;
    int32_t symbolic;
    int32_t precise;                   /* 25                 */
    int32_t coverage_binsize;          /* = cluster_binsize  */
    int32_t coverage_updown_bins;      /* 5                  */
    int32_t _pad;
    double  max_splits_kb;             /* 0.1                */
    double  cluster_r;                 /* 2.5                */
    double  cluster_repeat_h;          /* 1.5                */
    double  cluster_repeat_h_max;      /* 1000               */
    double  cluster_merge_len;         /* 0.22 / 0.27 mosaic */
    double  consensus_kmer_skip_seqlen_mult; /* 1/500        */
} snfb_config;

/* Lead as written by the device (64 B).  One lead = one reference `Lead`
 * (leadprov.py:34-55) that landed inside its task's region (leadprov.py:464-466). */
typedef struct snfb_lead {
    uint32_t rec;          /* index of the alignment record (stands in for read_id)   */
    int32_t  ref_start;
    int32_t  ref_end;
    int32_t  qry_start;
    int32_t  qry_end;
    int32_t  svlen;        /* undefined when SNFB_LF_SVLEN_NONE                        */
    int32_t  seq_off;      /* offset into the read's query_sequence, -1 = no sequence  */
    int32_t  seq_len;      /* length of the sequence slice                             */
    int32_t  read_len;     /* query_alignment_length for INLINE leads, else 0          */
    int32_t  mate_pos;     /* BND: bnd_info.mate_ref_start                             */
    int32_t  mate_contig;  /* BND: contig-table index of bnd_info.mate_contig          */
    int32_t  nm_sa;        /* BND: NM field of the SA entry (leadprov.py:119)          */
    uint32_t flags;        /* SNFB_LF_*                                                */
    uint16_t task;
    uint16_t k;            /* ordinal of the lead inside its read (A9 ordering)        */
    uint64_t qname_hash;   /* FNV-style 64-bit hash of query_name                      */
} snfb_lead;

#define SNFB_LF_TYPE(f)      ((f) & 7u)
#define SNFB_LF_SOURCE(f)    (((f) >> 3) & 3u)
#define SNFB_LF_REVERSE      (1u << 5)   /* strand == "-"                     */
#define SNFB_LF_IS_SA        (1u << 6)   /* read.is_supplementary             */
#define SNFB_LF_SVLEN_NONE   (1u << 7)   /* svlen is None ("long INS")        */
#define SNFB_LF_BND_FIRST    (1u << 8)
#define SNFB_LF_BND_REVERSE  (1u << 9)
#define SNFB_LF_HAS_SEQ      (1u << 10)  /* seq is not None                   */
#define SNFB_LF_NM_NONE      (1u << 11)  /* BND lead of a read without NM tag */
#define SNFB_LF_MAPQ(f)      (((f) >> 16) & 255u)
#define SNFB_LF_HAP(f)       (((f) >> 24) & 3u)

typedef struct snfb_lead_view {
    uint64_t n_leads;
    const snfb_lead* leads;        /* in bin order: (task, svtype, bin, record, k)     */
    uint64_t n_pass;               /* LeadProvider.read_count summed over tasks        */
    const uint32_t* task_read_count;  /* [n_task]                                       */
    const double*   task_mean_nm;     /* [n_task] config.average_regional_nm (leadprov.py:577) */
    const double*   rec_nm;        /* [n_rec] per-read nm (leadprov.py:524), -1 if none */
    uint64_t soft_errors;          /* malformed SA entries etc. (never fatal)          */
} snfb_lead_view;

/* One SV candidate = one reference SVCall as it leaves Task.call_candidates
 * (sv.py:561-598 + postprocessing.coverage), before QC/genotyping. */
typedef struct snfb_cand {
    int32_t  task;
    int32_t  svtype;
    int32_t  pos;
    int32_t  end;
    int32_t  svlen;
    int32_t  support;
    int32_t  qual;
    int32_t  precise;
    int32_t  fwd;
    int32_t  rev;
    int32_t  support_long;       /* INS: SUPPORT_LONG                                  */
    int32_t  support_sa;         /* DEL: SUPPORT_SA                                    */
    int32_t  cov_upstream, cov_start, cov_center, cov_end, cov_downstream;
    int32_t  hap_counts[6];      /* cluster.hap_counts (cluster.py:255-260)            */
    int32_t  sa_count;           /* cluster.sa_counts[0] (cluster.py:79-82)            */
    int32_t  sa_total;           /* denominator of sa_counts[1]                        */
    int32_t  bnd_mate_contig;
    int32_t  bnd_mate_pos;
    int32_t  bnd_is_first;
    int32_t  bnd_is_reverse;
    int32_t  n_strands;          /* len(set(lead.strand))                              */
    int32_t  support_inline;     /* distinct qnames among INLINE leads (sv.py:195)     */
    int32_t  lead_off;           /* first lead of this candidate in cand_leads[]       */
    int32_t  lead_n;
    int32_t  long_off;           /* INS: cluster.leads_long in cand_leads[]            */
    int32_t  long_n;
    int32_t  alt_off;            /* INS consensus: offset into alt[] (after snfb_consensus), -1 none */
    int32_t  alt_len;
    int32_t  hp_top, hp_support, hp_other;     /* phase_sv aggregates (postprocessing.py:626-654) */
    int32_t  ps_top, ps_top_null, ps_support, ps_other;
    int32_t  cluster_seed;       /* first bin of the merged cluster                    */
    int32_t  resplit_bin;        /* id suffix of cluster.resplit (cluster.py:151)      */
    double   stdev_pos;
    double   stdev_len;          /* NaN when absent (BND)                              */
    double   nm_mean;            /* -1 unless qc_nm_measure                            */
} snfb_cand;

typedef struct snfb_cand_view {
    uint64_t n_cand;
    const snfb_cand* cand;          /* in reference emission order: task, svtype, cluster */
    uint64_t n_cand_leads;
    const snfb_lead* cand_leads;    /* post merge_inner/resplit leads, reference order    */
    const uint64_t*  rnames;        /* distinct qname hashes per candidate, CSR below     */
    const uint32_t*  rnames_off;    /* [n_cand+1]                                          */
    const double*    task_coverage_mean; /* [n_task] coverage_average_total (postprocessing.py:130) */
    uint64_t unverified_breaks;     /* chain cuts whose independence check failed in the final run (0: a failed cut is redone with whole chains) */
} snfb_cand_view;

typedef struct snfb_seq_view {
    uint64_t n_alt_bytes;
    const uint8_t* alt;             /* ASCII, indexed by snfb_cand.alt_off/alt_len        */
} snfb_seq_view;

typedef struct snfb_ctx snfb_ctx;

int         snfb_version(void);
/* sizeof of the ABI structs, for binding self-checks: 0 rec, 1 task, 2 contig, 3 records, 4 config, 5 lead, 6 cand, 7 gather_view,
 * 8 gt_in, 9 gt_out, 10 ref_contig, 11 ref_input, 12 ref_query, 13 region, 14 combine_plan_in, 15 combine_plan_out, 16 pop_table,
 * 17 pop_query, 18 rnames_view */
size_t      snfb_sizeof(int which);
uint64_t    snfb_hash_name(const char* s, size_t n);
int         snfb_ctx_create(int device, snfb_ctx** out);
void        snfb_ctx_destroy(snfb_ctx* ctx);
const char* snfb_last_error(snfb_ctx* ctx);
int         snfb_set_config(snfb_ctx* ctx, const snfb_config* cfg);
int         snfb_load_records(snfb_ctx* ctx, const snfb_records* block);
int         snfb_extract_leads(snfb_ctx* ctx, snfb_lead_view* out);   /* out may be NULL: stay on device */
int         snfb_cluster_call(snfb_ctx* ctx, snfb_cand_view* out);
int         snfb_consensus(snfb_ctx* ctx, snfb_seq_view* out);
/* all three stages back to back.  Sizes live in device counters and every buffer has a capacity kept in the ctx, so the
 * stream is never drained between stages: the host reads the counters once on a side stream (while the consensus kernels
 * run) to size the device -> host copies, and once at the end.  A run whose capacities were too small (the first run on
 * a ctx, or a block unlike the previous one) is repeated with capacities that fit; snfb_rerun_count counts those.
 * The views (any may be NULL) are filled after the final synchronisation. */
int         snfb_run(snfb_ctx* ctx, snfb_lead_view* leads, snfb_cand_view* cands, snfb_seq_view* seqs);
/* ---- device BAM ingest (SURVEY §8 (f)3): compressed BGZF bytes in, the packed record block built in device memory ----
 * `bgzf` holds whole BGZF blocks back to back (host memory; any selection of a file's blocks, in file order).  A span is a
 * record-aligned range of the inflated stream that belongs to one task, given the way a BAI index gives it: (byte offset of a
 * BGZF block inside `bgzf`, offset inside that block's inflated data) for its begin and its end — i.e. a BAM virtual offset with
 * the file offset rebased to `bgzf`.  cend == n_bytes with uend == 0 means "to the end of the buffer".  Spans are listed task by
 * task in file order and must not overlap (merge the index chunks first, as htslib does); cutting a span at any record-aligned
 * offset (the linear index of the BAI provides one per 16 kb window) only adds parallelism.  The library inflates every block
 * (16 lanes of a warp per block), follows the block_size chain of every span, decodes the records, keeps those `bam.fetch(contig, start,
 * end)` would return for the span's task (task.contig is the BAM reference id), restores CIGARs of more than 65535 operations
 * from the CG:B,I tag, and writes snfb_rec + CIGAR16 + names/SA + 4-bit bases exactly as snfb_load_records expects them.
 * Every block is checked as htslib checks it: its DEFLATE stream must decode, to exactly ISIZE bytes, whose CRC-32 equals the
 * block's trailer; a failing block fails the call and the error names the lowest failing block, its code and its byte offset in
 * `bgzf` (code 10 = CRC32 mismatch: a damaged block that still decodes).  Tables (tasks, contigs,
 * tandem repeats, N mask) have the meaning they have in snfb_records. */
typedef struct snfb_bam_span {
    uint64_t cbeg, cend;      /* byte offsets of BGZF block starts inside bgzf[] */
    uint32_t ubeg, uend;      /* offsets inside those blocks' inflated data */
    uint32_t task;
    uint32_t region;          /* index into the region table (snfb_set_regions); ignored while that table is empty */
} snfb_bam_span;
typedef struct snfb_bam_input {
    const uint8_t* bgzf; uint64_t n_bytes;
    const snfb_bam_span* span; uint64_t n_span;
    uint32_t n_task, n_contig, n_tr, n_mask;
    const snfb_task* task; const snfb_contig* contig; const int32_t* tr; const int32_t* mask; const uint32_t* mask_task_off;
} snfb_bam_input;
int         snfb_load_bam(snfb_ctx* ctx, const snfb_bam_input* in);
/* ---- regions (--regions / --region): LeadProvider.build_leadtab over a task's list of regions (leadprov.py:445-470) ----
 * A task keeps one contig and clusters as one unit; its regions are segments of its records.  For each region in table order the
 * reference runs bam.fetch(contig, start, end), keeps the reads with start <= reference_start < end and records a lead only when
 * start <= lead.ref_start < end of the region it came from.  A read two regions take is read twice: two records, two read ids, its
 * coverage and NM counted twice.  config.average_regional_nm is the mean over the LAST region's reads only (nm_sum is reset per
 * iter_region, leadprov.py:475-577).
 * The table applies to the next snfb_load_records / snfb_load_bam on the context only: a load not preceded by this call has no table
 * (n = 0 is the same), and then snfb_rec.region / snfb_bam_span.region are ignored and every task is its own single region
 * [task.start, task.end).  With a table:
 *   - regions are grouped by task, in the task's order (start > end or start < 0 is refused: the host fails that task instead);
 *   - snfb_rec.region (host records) and snfb_bam_span.region (device ingest) name a region of the record's / span's own task;
 *     records come grouped by (task, region, BAM order) and spans by (task, region), each region's spans in file order;
 *   - the record filters, the fetch overlap test of the ingest and the lead filters use the record's region;
 *   - task.start / task.end only clip the N mask: the host clips the runs to the regions and passes [0, contig_len].
 * When some task has more than one region, the block is not coordinate sorted inside that task (a region's fetch also returns the
 * reads that start before it and overlap it); stage A then builds a coordinate-ordered copy of (pos, end, flags) with a stable radix
 * sort on (task, pos) (timing mark "cov_order") that every coverage reader uses. */
typedef struct snfb_region { int32_t task, start, end, _pad; } snfb_region;
int         snfb_set_regions(snfb_ctx* ctx, const snfb_region* regions, uint32_t n);
/* what the last snfb_load_bam built: out[0] records, out[1] CIGAR16 words, out[2] var bytes, out[3] seq bytes, out[4] raw records seen,
 * out[5] BGZF blocks, out[6] inflated bytes, out[7] compressed bytes */
int         snfb_ingest_sizes(snfb_ctx* ctx, uint64_t out[8]);
/* copies the block snfb_load_bam built back to the host (tests / inspection); any pointer may be NULL */
int         snfb_ingest_fetch(snfb_ctx* ctx, snfb_rec* rec, uint16_t* cigar16, uint8_t* var, uint8_t* seq);
/* inflate whole BGZF blocks on the device and return the inflated stream (tests / inspection).  Returns 0 and *out_len = bytes;
 * out may be NULL to get the size only. */
int         snfb_inflate_bgzf(snfb_ctx* ctx, const uint8_t* bgzf, uint64_t n_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_len);
/* compress host bytes in[0 .. n_in) into BGZF on the device and return the members in host memory (what `bgzip` / pysam.tabix_index
 * write for a .vcf.gz): the input is cut into blocks of 0xff00 bytes (the last may be shorter), each an independent gzip member with the
 * BC extra field, one DEFLATE block (stored, fixed or dynamic Huffman, whichever is smallest) and the CRC-32 + ISIZE trailer.  The bytes
 * are a pure function of the input.  out_cap must be at least ceil(n_in / 0xff00) * 65536; *out_len = bytes written; coffset[k] (may be
 * NULL) = byte offset of member k in out.  The BGZF EOF marker is not appended.  Device buffers belong to the context and grow on
 * demand; n_in is limited to 65535 blocks (~4 GiB) per call.  Records a "deflate" timing mark (snfb_last_timings). */
int         snfb_deflate_bgzf(snfb_ctx* ctx, const uint8_t* in, uint64_t n_in, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* coffset);

/* The tables of a BAI (min_shift 14, depth 5) or CSI index of a coordinate-sorted BAM, built on the device with no index to start from
 * (what `samtools index` computes; SAM spec §5).  The file streams through the device in windows of whole BGZF members of at most
 * window_bytes inflated bytes (at least one member): each window is inflated and CRC-checked, its record starts found from the carried
 * entry offset by pointer jumping over the offsets that pass a strict record test, one row per record computed (reference, begin,
 * bam_endpos, virtual offsets, mapped) and the sort order checked.  The tables are then built from all rows: bins by reg2bin, chunks as runs
 * of the same (reference, bin), htslib's finishing rules (a bin spanning < 0x10000 compressed bytes moves its chunks to an existing parent,
 * level by level from the leaves; chunks starting in the block where the previous one ends merge), the linear index at min_shift (an
 * empty window takes the next window's offset, as htslib's update_loff fills it) and the per-bin loffset, the per-reference pseudo-bin.  Fails (snfb_last_error names the record or the block) on a file that is not BGZF,
 * a block that fails to inflate or its CRC-32, a broken record chain, a truncated file, unsorted records, or (BAI) an end beyond 2^29. */
typedef struct snfb_index_input {
    const char* path;             /* the BAM file                                                                 */
    uint64_t first_record;        /* virtual offset of the first record (the end of the header)                  */
    const int64_t* contig_len;    /* n_ref contig lengths from the header                                        */
    uint32_t n_ref;
    int32_t min_shift, depth;     /* bin geometry: 14 / 5 for a BAI                                               */
    int32_t _pad;
    uint64_t window_bytes;        /* inflated bytes per window                                                   */
} snfb_index_input;
typedef struct snfb_index_view {  /* library-owned, valid until the next snfb_index_bam on the context           */
    const uint64_t* ref;          /* [n_ref][5]: first v0 (~0: no record), last v1, mapped, unmapped, linear-index windows */
    const uint64_t* lin_off;      /* [n_ref + 1]: reference t's linear index is lin[lin_off[t] .. lin_off[t + 1])  */
    const uint64_t* lin;
    const uint64_t* bin_key;      /* [n_bin] ascending: reference * n_bins + bin, n_bins = ((1 << 3 (depth + 1)) - 1) / 7; every bin
                                   * that held records, so one whose chunks moved to its parent has none */
    const uint64_t* bin_loff;     /* [n_bin] CSI loffset of the bin                                               */
    const uint32_t* chunk_bin;    /* [n_chunk] index into bin_key; chunks grouped by bin, ascending offsets inside one */
    const uint64_t* chunk_beg;
    const uint64_t* chunk_end;
    uint64_t n_bin, n_chunk, n_no_coor, n_records, n_windows, device_bytes;   /* device_bytes: device buffers held at the widest point */
    double device_ms;             /* the device's time in the call (CUDA events around each phase of work it was given)        */
} snfb_index_view;
int         snfb_index_bam(snfb_ctx* ctx, const snfb_index_input* in, snfb_index_view* out);

/* The BAM at `path` sorted by coordinate into out_path, as `samtools sort` writes it (samtools bam_sort.c: bam1_cmp_core for the order;
 * htslib bam_hdr_write / bam_write1 -> bgzf_flush_try / bgzf_write, BGZF_BLOCK_SIZE 0xff00, for the member cuts).
 *   Order: tid compared as unsigned (tid -1, no coordinate, last), then pos + 1, then the reverse-strand bit (flag 0x10), then input order.
 *     The device key is (tid' << 33) | ((pos + 1) << 1) | rev with tid' = n_ref for tid -1; one stable radix sort over only the key's
 *     bits, values = input ordinals.
 *   Records are copied verbatim (bin, mate fields and tags are not recomputed).  The output header is the caller's `header` bytes (the
 *     BAM header from the magic through the references; sniffles_b200.bamio.sort_header sets @HD SO:coordinate and changes nothing else).
 *   Member cuts: the header fills members of 0xff00 bytes and is flushed; a record of 4 + block_size bytes first closes the current member
 *     when that member is non-empty and the record would overflow it, then fills members of 0xff00 bytes, each closed when full; the last
 *     partial member is closed and the 28-byte EOF marker appended.  The members are compressed by the device encoder (not zlib), so the
 *     file is not byte-equal to samtools'; its inflated stream and member sizes are, and its bytes are a pure function of the input
 *     whatever the budgets.
 * Device pipeline: the keys pass streams the input in windows of whole members of at most window_bytes inflated bytes, exactly as
 * snfb_index_bam does (inflate + CRC, carry, the record chain), and writes each record's key, length and inflated offset; the sort; the
 * layout (one host loop over the sorted lengths cuts the members; buckets are runs of whole members starting at a record start, of at
 * most bucket_bytes inflated bytes, or one record's members when it alone is larger); then per bucket the windows holding its records are
 * read again, their records' bytes scattered into the bucket's buffer by a warp per record, the members compressed from device memory (at
 * most 65535 per launch) and appended to the file.  Fails (snfb_last_error names the record or the block) on the inputs snfb_index_bam
 * refuses except the order (a record whose tid < -1, tid >= n_ref or pos < -1 fails the strict record test and breaks the chain), on 2^32
 * records or more, and when out_path cannot be written. */
typedef struct snfb_sort_input {
    const char* path;             /* the BAM file                                                                 */
    const char* out_path;         /* the file written (created or truncated)                                     */
    const uint8_t* header;        /* the output's BAM header: magic, l_text, text, n_ref, the references          */
    uint64_t header_len;
    uint64_t first_record;        /* virtual offset of the input's first record (the end of its header)          */
    const int64_t* contig_len;    /* n_ref contig lengths from the header                                        */
    uint32_t n_ref, _pad;
    uint64_t window_bytes;        /* inflated bytes per input window                                             */
    uint64_t bucket_bytes;        /* inflated output bytes per bucket                                            */
} snfb_sort_input;
typedef struct snfb_sort_view {
    uint64_t n_records, n_windows, n_buckets, n_members;  /* n_windows: windows of the keys pass                  */
    uint64_t n_input_reads;       /* window reads of the input: the keys pass's and those of every bucket pass     */
    uint64_t bytes_in, bytes_out; /* file bytes read (both passes), file bytes written (with the EOF marker)      */
    uint64_t device_bytes;        /* device buffers held at the widest point                                     */
    double ms_keys, ms_sort, ms_layout, ms_scatter, ms_deflate;   /* device time per phase (CUDA events)          */
    double ms_layout_host;        /* the host's member-cut loop over the sorted lengths                          */
} snfb_sort_view;
int         snfb_sort_bam(snfb_ctx* ctx, const snfb_sort_input* in, snfb_sort_view* out);
/* device-time accounting of the last run: per-kernel milliseconds from CUDA events on
 * the ctx stream; names[i] is a static string.  Returns the number of entries. */
int         snfb_last_timings(snfb_ctx* ctx, const char** names, float* ms, uint64_t* bytes, int cap);
/* device pointer + count of the candidate buffer (for the NCCL all-gather done by the
 * Python host through torch.distributed) */
int         snfb_device_candidates(snfb_ctx* ctx, void** dptr, uint64_t* n_cand);
int         snfb_device_alt(snfb_ctx* ctx, void** dptr, uint64_t* n_bytes);
/* number of kernels launched by the library on this ctx since it was created */
uint64_t    snfb_launch_count(snfb_ctx* ctx);
/* number of times a run was repeated because a buffer capacity was too small or a chain cut had to be undone */
uint64_t    snfb_rerun_count(snfb_ctx* ctx);
/* the number of slices (1 to 8, default 2) stage C runs in: candidates cut to about equal consensus work, each slice's ALT bytes copied
 * to the host while the next slice runs.  The results do not depend on it; it changes the launches and the copy schedule. */
int         snfb_set_consensus_slices(snfb_ctx* ctx, int k);
/* mean coverage of consecutive `binsize`-base bins over the whole contig of one task, as the SNF writer stores it
 * (snf.py:248-267: the coverage vector zero-padded to a multiple of binsize, row means; the writer rounds them).  With an N mask
 * loaded, positions inside the task's runs (clipped to the task region) count 0, as in the masked vector (leadprov.py:470).
 * *out is a library-owned buffer of *n_bins doubles, valid until the next call on the ctx.  Needs snfb_extract_leads
 * (or snfb_run) first. */
int         snfb_coverage_bins(snfb_ctx* ctx, uint32_t task, int binsize, const double** out, uint64_t* n_bins);
/* ---- force calling (--genotype-vcf; GenotypeTask.execute, parallel.py:300-369) ----
 * Runs after snfb_run (or snfb_cluster_call) on the same context and changes nothing that call produced.  Targets are SoA host arrays,
 * ordered by task and then by input order (a BND target takes the `end` of the previous non-BND target of its task, as
 * postprocessing.coverage does).  svtype is SNFB_INS .. SNFB_BND, or -1 for a type the reference does not bin (not matched, still
 * probed).  mate_contig is a contig-table index, -1 for a name the BAM header lacks (never matches).  A target is matched against the
 * candidates of its task, svtype and 5000-bp bin (plus the neighbouring bin within 500 bp of an edge), SINGLE_* excluded:
 * non-BND: dist = |dpos| + ||svlen_t| - |svlen_c|| with min(|svlen_t|, |svlen_c|) > 0, dist <= combine_match * sqrt(minlen) and
 * dist <= combine_match_max; BND: dist = |dpos| <= cluster_merge_bnd (snfb_config) and equal mate contigs.  The smallest distance wins,
 * ties go to the earlier candidate.  Outputs per target (host arrays): the candidate's index in the run's emission order (-1 none), the
 * start / center / end coverage probes, and bnd_no_prev = 1 for a BND with no earlier non-BND target in its task (the reference's
 * UnboundLocalError: that task fails).  Records a "genotype" timing mark. */
typedef struct snfb_gt_in {
    uint64_t n;
    const int32_t* task; const int32_t* svtype; const int32_t* pos; const int32_t* svlen; const int32_t* bnd_is_first; const int32_t* mate_contig;
    int32_t combine_match, combine_match_max;
} snfb_gt_in;
typedef struct snfb_gt_out {
    int64_t* match;
    int32_t* cov_start; int32_t* cov_center; int32_t* cov_end; int32_t* bnd_no_prev;
} snfb_gt_out;
int         snfb_genotype_targets(snfb_ctx* ctx, const snfb_gt_in* in, snfb_gt_out* out);

/* ---- multi-GPU: one process per GPU, contigs sharded over the ranks, ONE all-gather of the per-rank candidate buffers ----
 * snfb_nccl_unique_id fills the 128 bytes of an ncclUniqueId on one rank; the host hands them to every rank (any transport),
 * then every rank calls snfb_comm_init.  snfb_allgather_candidates runs after snfb_run on every rank: it packs the rank's
 * candidate records, ALT arena, read names (and, with SNFB_GATHER_LEADS, the candidates' leads) into one buffer, all-gathers
 * the buffers over NCCL on the ctx stream, and returns the concatenation in rank order with lead_off / long_off / alt_off and
 * the rnames offsets rebased into the merged arrays (so a candidate of any rank indexes the merged arenas).  Ranks own
 * disjoint tasks; the caller orders by task id for emission (sniffles:544-547).  The view is library-owned pinned host
 * memory (dev_* are the same arrays in device memory), valid until the next call. */
#define SNFB_GATHER_LEADS 1u
#define SNFB_GATHER_DEVICE_ONLY 2u     /* leave the result in device memory (no device -> host copy; host pointers are NULL) */
typedef struct snfb_gather_view {
    uint64_t n_cand;        const snfb_cand* cand;
    uint64_t n_alt_bytes;   const uint8_t*  alt;
    uint64_t n_rnames;      const uint64_t* rnames;     const uint32_t* rnames_off;   /* [n_cand + 1] */
    uint64_t n_cand_leads;  const snfb_lead* cand_leads;                              /* 0 / NULL without SNFB_GATHER_LEADS */
    const uint64_t* rank_n_cand;                                                      /* [nranks] */
    const void* dev_buffer; uint64_t dev_bytes_per_rank;                              /* the gathered device buffer (nranks slots) */
} snfb_gather_view;
int         snfb_nccl_unique_id(void* out128);
int         snfb_comm_init(snfb_ctx* ctx, const void* unique_id128, int rank, int nranks);
int         snfb_allgather_candidates(snfb_ctx* ctx, uint32_t flags, snfb_gather_view* out);
/* ---- local assembly (LocalAsm, local_asm.py:254-304; gate parallel.py:186-196): the partial-order alignment the reference hands to pyspoa ----
 * A job is either mode 0: consensus of n_seq sequences = poa(read windows, local, min_coverage) (local_asm.py:287), or mode 1: the two-row
 * MSA of (sequence 0, sequence 1) = poa([consensus, ref], local, genmsa, m, n, g, e, q, c) (local_asm.py:289-291).  Sequences are bytes
 * compared for equality only; rows of an MSA use 255 for '-'.  out_len[k] = length / number of columns, -1 when the graph outgrew its
 * bounds, -2 when the job does not fit the scratch.  The algorithm is the one restated in oracle/poa_oracle.c (parity with pyspoa unpinned). */
typedef struct snfb_poa_job {
    uint64_t seq_off;        /* first byte of the job's sequences in seqs[]                                        */
    uint32_t offs_off;       /* index in offs[] of the job's n_seq + 1 offsets (relative to seq_off, ascending)    */
    uint32_t n_seq;
    int32_t  min_cov;        /* mode 0: round(0.5 n) (local_asm.py:285)                                            */
    int32_t  m, n, g, e, q, c;  /* match, mismatch, gap open / extend, second affine piece open / extend             */
    int32_t  band;           /* half width of the band around a node's column (>= the longest sequence: no band)   */
    uint32_t mode;
    uint32_t out_cap;        /* bytes per output row                                                               */
    uint64_t out_off;        /* mode 0: one row at out[out_off], mode 1: two rows of out_cap bytes                 */
} snfb_poa_job;
int         snfb_poa(snfb_ctx* ctx, const snfb_poa_job* jobs, uint32_t n_jobs, const uint8_t* seqs, uint64_t n_seq_bytes, const int32_t* offs, uint64_t n_offs,
                     uint8_t* out, uint64_t out_bytes, int32_t* out_len);
/* ---- multi-sample combine (SURVEY 8(f)1): the grouping of CombineTask.execute (parallel.py:443-572) -----------------------------------
 * The host reads the SNF blocks and lays the candidates out the way the reference visits them: a CHAIN is one (task, svtype) — its groups are
 * carried from chunk to chunk and from block to block (groups_keep, parallel.py:475,563) —, a CHUNK is one call of
 * cluster.resolve_block_groups (cluster.py:356-390): the candidates of the bins accumulated up to bin_max_candidates, already in the order
 * sorted(key=support, reverse=True) gives them.  The device runs every chain: nearest-group assignment with the reference's distance and
 * limits, SVGroup.from_candidate / add_candidate running means (sv.py:265-321), after each chunk the coverage of the samples a group does not
 * include (max over the chunks it lives through, parallel.py:538-552) and the keep / call split (parallel.py:554-557).
 * Outputs, per candidate: its group slot; per group slot (slot = chain.cand_off + order of creation): the chunk at whose end it was called
 * (n_chunk = kept to the end of the chain, -1 = unused slot), its position among the groups called then, the non-included coverages.
 * group.align_call (sv.py:282-292): with combine_pctseq != 0 and the ALT strings given, a candidate joins the nearest eligible group only if
 * (len_mean - editDistance(ALT of the group's first candidate, its ALT)) / len_mean > combine_pctseq — edlib.align's default global edit
 * distance, computed on the device (bit-vector blocks, one warp per pair).  combine_pctseq = 0 (or alt = NULL) is the reference's behaviour
 * without edlib / with --combine-pctseq 0: every pair passes. */
typedef struct snfb_combine_chain { uint32_t cand_off, n_cand, chunk_off, n_chunk, is_bnd, pad; } snfb_combine_chain;
typedef struct snfb_combine_chunk { int32_t cand_off, n_cand, curr_bin, size, cov_block, pad; } snfb_combine_chunk;   /* cov_block: row of cov[] of the block being read, -1 none */
typedef struct snfb_combine_in {
    uint32_t n_chain, n_chunk, n_cand, n_samples;
    const snfb_combine_chain* chains; const snfb_combine_chunk* chunks;
    const int32_t* pos; const int32_t* svlen; const uint32_t* sample;        /* per candidate; sample = index into the sample list   */
    const int32_t* mate_contig; const int32_t* mate_pos;                     /* BND chains only (any consistent contig numbering)     */
    uint32_t n_cov_block; int32_t bins_per_block, cov_binsize, pad;
    const int64_t* block_start;                                              /* [n_cov_block]                                         */
    const int32_t* cov;                                                      /* [n_cov_block][n_samples][bins_per_block]; -1 = the sample has no such block / key */
    int32_t combine_match, combine_match_max, cluster_merge_bnd, combine_separate_intra, combine_overlap_abs, pad2;
    double  combine_pctseq;
    const uint8_t* alt; const uint64_t* alt_off; const uint32_t* alt_len; uint64_t n_alt_bytes;   /* per candidate ALT bytes: alt[alt_off[i] .. + alt_len[i]) */
} snfb_combine_in;
typedef struct snfb_combine_out {
    uint32_t* cand_group;     /* [n_cand]                 */
    int32_t*  emit_chunk;     /* [n_cand] per group slot  */
    uint32_t* emit_ord;       /* [n_cand] per group slot  */
    int32_t*  cov_non;        /* [n_cand][n_samples]; -1 where the sample is included (never probed) */
} snfb_combine_out;
int         snfb_combine_groups(snfb_ctx* ctx, const snfb_combine_in* in, snfb_combine_out* out);
/* ---- the chunk plan of combine mode on the device, then the grouping (CombineTask.execute, parallel.py:484-572) ----
 * The host decodes the SNF blocks of one or more tasks into flat columns, in the reference's iteration order: task, block, svtype,
 * sample, part, list position.  `group` carries the per-candidate columns pos, svlen, sample, mate_contig, mate_pos and the ALT arena in
 * that flat order (n_cand = n_flat), the coverage tables and the grouping parameters, as snfb_combine_groups reads them; its chains,
 * chunks, n_chain and n_chunk are not read.  task is the task's index (< n_task <= 2^24), row the coverage row of the candidate's
 * (task, block), rows being numbered in (task, block) order; svtype 0..4 is INS DEL DUP INV BND.  The device
 *   - drops candidates with support < support_threshold,
 *   - sorts the rest stably on (task, svtype, block, bin), bin = int(pos / bin_min_size) * bin_min_size (the bins dict of one block),
 *   - cuts each (task, block, svtype) run into chunks: whole bins, closed at bin_max_candidates (unless exhaustive) or at the last bin,
 *   - sorts each chunk stably by support, descending (cluster.py:361),
 *   - builds the chain and chunk tables in device memory (chunk.cov_block = row, pads 0) and runs the grouping of snfb_combine_groups.
 * Outputs, each with room for n_flat entries: n_cand kept candidates; perm[slot] = the flat index in slot `slot`; the n_chain chains and
 * n_chunk chunks in the layout snfb_combine_groups reads; group: its four outputs per slot.  Timing marks "combine_plan", "combine_groups". */
typedef struct snfb_combine_plan_in {
    uint32_t n_flat, n_task;
    const uint32_t* task; const uint32_t* row; const int32_t* svtype; const int32_t* support;
    int32_t support_threshold, bin_min_size, bin_max_candidates, exhaustive;
    snfb_combine_in group;
} snfb_combine_plan_in;
typedef struct snfb_combine_plan_out {
    uint32_t n_cand, n_chain, n_chunk, pad;
    uint32_t* perm; snfb_combine_chain* chains; snfb_combine_chunk* chunks;
    snfb_combine_out group;
} snfb_combine_plan_out;
int         snfb_combine_plan(snfb_ctx* ctx, const snfb_combine_plan_in* in, snfb_combine_plan_out* out);
/* ---- population allele frequencies of combined calls (--combine-population, snfp.py) ----
 * snfb_population_load  <- PopulationSNF.open + get_all_blocks (sniffles:433-435, parallel.py:454-455, snf.py:235-243): the variants of a
 *                          population SNF, in file order, each with its contig index (-1 when the name is not among the run's contigs; such
 *                          a variant is never matched), the start of the block it is stored under (the index key, not recomputed from pos),
 *                          svtype 0..4 (INS DEL DUP INV BND), pos, svlen and its ALT bytes alt[alt_off[i] .. + alt_len[i]).  Only the
 *                          first part of a block is given, as get_all_blocks reads only read_blocks(...)[0].  The table is keyed on the
 *                          device, sorted stably on (contig, block, svtype) and stays resident on the context until the next load, which
 *                          replaces it, or snfb_ctx_destroy.  Timing mark: population_load.
 * snfb_population_match <- PopulationSNF.get_population_AF (snfp.py:131-155) with PopulationVariant.match (snfp.py:91-107) for one batch of
 *                          calls (contig index or -1, svtype, pos, svlen, ALT bytes): the call's list is the variants of key (contig,
 *                          int(pos / block_size) * block_size, svtype); a variant matches when dist = |pos_p - pos_c| + ||svlen_p| -
 *                          |svlen_c|| <= combine_match * sqrt(min(|svlen_p|, |svlen_c|)) and dist <= combine_match_max, and, for INS with
 *                          combine_pctseq != 0, (svlen_p - editDistance(ALT_p, ALT_c)) / svlen_p > combine_pctseq (edlib.align defaults).
 *                          best[q] = the file-order index of the variant with the strictly smallest distance, ties to the earlier one in
 *                          list order; -1 when none matches; -2 when an INS variant with svlen_p == 0 reaches the alignment test, where the
 *                          reference divides by zero.  Timing mark: population_match. */
typedef struct snfb_pop_table {
    uint32_t n, pad;
    const int32_t* contig; const int32_t* block; const int32_t* svtype; const int32_t* pos; const int32_t* svlen;
    const uint8_t* alt; const uint64_t* alt_off; const uint32_t* alt_len; uint64_t n_alt_bytes;
} snfb_pop_table;
typedef struct snfb_pop_query {
    uint32_t n, pad;
    const int32_t* contig; const int32_t* svtype; const int32_t* pos; const int32_t* svlen;
    const uint8_t* alt; const uint64_t* alt_off; const uint32_t* alt_len; uint64_t n_alt_bytes;
    int32_t combine_match, combine_match_max, block_size, pad2;
    double  combine_pctseq;
} snfb_pop_query;
int         snfb_population_load(snfb_ctx* ctx, const snfb_pop_table* in);
int         snfb_population_match(snfb_ctx* ctx, const snfb_pop_query* in, int32_t* best);
/* ---- read names (--output-rnames: the RNAMES of sv.py:520-525, 555) ----
 * Runs after snfb_run (or snfb_cluster_call) on the same context, on the candidates and the record block it left there, and changes nothing
 * that call produced.  Name k is the query name of snfb_cand_view.rnames[k]: for each candidate, each of its distinct qname hashes is
 * resolved through the first of the candidate's leads (cand_leads[lead_off .. + lead_n + long_n)) that carries it, to that lead's record's
 * var[var_off .. + l_qname).  Names come in the order of the hash list (per candidate ascending by hash), so candidate c owns names
 * rnames_off[c] .. rnames_off[c + 1] and name k is text[off[k] .. off[k + 1]).  `collisions` counts the leads whose own name differs from
 * the name kept for their hash (two reads with one 64-bit hash); a hash that none of the candidate's leads carries fails the call.  The view
 * is library-owned pinned host memory, valid until the next call on the context.  Timing marks: rnames_resolve, rnames_copy. */
typedef struct snfb_rnames_view {
    uint64_t n_names;               /* = the run's snfb_cand_view rnames count */
    uint64_t n_text;                /* bytes of text */
    const uint8_t*  text;           /* the names back to back, as the records store them (no separator, no NUL) */
    const uint32_t* off;            /* [n_names + 1] */
    uint64_t collisions;
} snfb_rnames_view;
int         snfb_read_names(snfb_ctx* ctx, snfb_rnames_view* out);
/* self-check of the exact statistics.stdev arithmetic (host build of the routine the kernels use): the correctly rounded sqrt(P / Q) for
 * P = p_hi * 2^64 + p_lo; slow != 0 selects the limb-by-limb restatement of CPython's _float_sqrt_of_frac, 0 the verified fast path */
double      snfb_selftest_sqrt_frac(uint64_t p_hi, uint64_t p_lo, uint64_t q, int slow);
/* self-check of the device edit distance behind group.align_call: n_pairs pairs (a_off/a_len, b_off/b_len into bytes[]), distances to out[] */
int         snfb_selftest_edit_distance(snfb_ctx* ctx, const uint8_t* bytes, uint64_t n_bytes, const uint64_t* a_off, const uint32_t* a_len, const uint64_t* b_off, const uint32_t* b_len, uint32_t n_pairs, int32_t* out);
/* ---- the reference FASTA (--reference) on the device ----
 * snfb_load_reference  <- pysam.FastaFile(config.reference) as LeadProvider._mask_N_coverage and VCF.open_reference open it
 *                         (leadprov.py:420-443, vcf.py:108-119): the bytes of the file (plain text, or whole BGZF members back to back with
 *                         is_bgzf = 1, inflated and CRC-checked on the device as snfb_load_bam does) and per contig its .fai geometry with
 *                         the raw offset rebased to those bytes (their inflated stream for BGZF).  Contig c becomes the newline-free bases
 *                         raw[offset + (p / linebases) * linewidth + p % linebases], p < length, kept byte for byte (case, IUPAC codes).
 *                         Every line that more sequence follows must end in "\n" (linewidth = linebases + 1) or "\r\n" (+ 2) and no base
 *                         may be a line break; otherwise the call fails naming the contig index and the line of the first violation (a
 *                         stale .fai, which htslib would read as wrong bases).  The maximal runs of 'N' (upper case only: leadprov.py:439
 *                         compares with 78) are computed on the device.  The genome stays resident on the context, replacing any earlier
 *                         one, until the next call or snfb_ctx_destroy; the raw stream is not kept.  Timing marks: h2d_ref, inflate
 *                         (BGZF), ref_unwrap, ref_nruns.
 * snfb_reference_runs  <- the `mask == 78` of _mask_N_coverage (leadprov.py:439): the runs as int32 (start, end) pairs, sorted per contig,
 *                         contig c owning runs[contig_off[c] .. contig_off[c + 1]); library-owned host arrays valid until the next call on
 *                         the context.  They enter a block through the N-mask tables of snfb_records / snfb_bam_input.
 * snfb_fetch_reference <- FastaFile.fetch(contig, start, end) of VCF.write_call (vcf.py:304-338): n resolved queries, one gather on the device
 *                         and one device -> host copy into out (query k fills out[out_off .. + length)).  The caller applies pysam's rules
 *                         (clipping, empty and invalid intervals) first: a query outside its contig fails the call. */
typedef struct snfb_ref_contig {
    uint64_t offset;          /* raw byte offset of the first base (the .fai OFFSET, rebased to the bytes given)   */
    uint64_t length;          /* bases (.fai LENGTH, < 2^31)                                                       */
    uint32_t linebases;       /* bases per line (.fai LINEBASES; may be 0 only when length is 0)                   */
    uint32_t linewidth;       /* bytes per line with its terminator (.fai LINEWIDTH)                               */
} snfb_ref_contig;
typedef struct snfb_ref_input {
    const uint8_t* bytes; uint64_t n_bytes;
    uint32_t is_bgzf;         /* 0 plain text, 1 whole BGZF members                                                */
    uint32_t n_contig;
    const snfb_ref_contig* contig;
} snfb_ref_input;
typedef struct snfb_ref_query {
    uint32_t contig; uint32_t _pad;
    uint64_t start, length;   /* 0 <= start, start + length <= the contig's length                                 */
    uint64_t out_off;
} snfb_ref_query;
int         snfb_load_reference(snfb_ctx* ctx, const snfb_ref_input* in);
int         snfb_reference_runs(snfb_ctx* ctx, const int32_t** runs, const uint64_t** contig_off, uint64_t* n_runs);
int         snfb_fetch_reference(snfb_ctx* ctx, const snfb_ref_query* q, uint64_t n, uint8_t* out, uint64_t out_cap);
/* BAM CIGAR words -> CIGAR16 (host code, OpenMP; no GPU needed).  rec_out receives copies of rec_in with cigar_off / n_cigar
 * rewritten for the 16-bit arena.  Call with out16 == NULL to get the number of 16-bit words the arena needs (a multiple
 * of 8); returns that number, or UINT64_MAX when a record holds an op the path does not know (B) or out_cap is too small.
 * evt_min: event length of the E bits (0 = SNFB_CIGAR16_EVT_MIN). */
uint64_t    snfb_pack_cigar16(const snfb_rec* rec_in, uint64_t n_rec, const uint32_t* cigar32, snfb_rec* rec_out, uint16_t* out16, uint64_t out_cap, uint32_t evt_min);
/* page-lock / unlock caller-owned host memory so that snfb_load_records copies at full PCIe rate */
int         snfb_pin_host(void* p, size_t bytes);
int         snfb_unpin_host(void* p);

#ifdef __cplusplus
}
#endif
#endif /* SNFB_H */
