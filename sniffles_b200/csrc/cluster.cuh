// cluster.cuh — stage B: leads -> bins -> clusters -> SV candidates.
//
// Data flow (all counts stay in device memory, no host round trips):
//   scatter canonical (record,k) order -> stable radix sort by (task,svtype,bin)        [A9 ordering]
//   bins -> kept bins (>= dev_min_leads_cluster non-"long" leads)                         cluster.py:248-275
//   the kept leads are gathered into kept order once: a cluster is then a contiguous range of 64-byte leads
//   chains of kept bins are cut at gaps no merge criterion can bridge; every piece runs
//   the reference's order-dependent merge automaton independently (one thread each)      cluster.py:278-308
//   per cluster, one warp (or block) with the leads staged in shared memory by a bulk copy:
//     merge_inner, resplit / resplit_bnd                                                  cluster.py:85-216
//     per sub-cluster sv.call_from / resolve_bnd, phase aggregates                        sv.py:497-639
//   compaction of the staged results into reference emission order
//   coverage probes without a per-base array                                              postprocessing.py:69-130
#pragma once
#include "common.cuh"
#include "extract.cuh"

namespace cluster {

constexpr int TYPE_SHIFT = 26;               // key = task << 29 | svtype << 26 | bin
constexpr int TASK_SHIFT = 29;
constexpr uint32_t NONE = 0xffffffffu;
constexpr int SMALL_CAP = 48;               // clusters up to this size: the dense warp-per-cluster kernel
constexpr int WARP_CAP = 128;               // mid-sized clusters, still one warp each (from a list); larger clusters take a whole block
constexpr int BLOCK_CAP = 1024;             // leads one block stages in shared memory; larger clusters work in global scratch

struct B {
    // inputs
    snfb_lead* leads; const snfb_rec* rec; const snfb_task* task; const snfb_contig* contig; const int32_t* tr; const int32_t* tr_pmax;
    const int32_t* rec_pos; const int32_t* rec_end; const uint8_t* rec_flags; const double* rec_nm; const uint32_t* rec_nlead; const uint32_t* rec_lead_off;
    const uint32_t* task_first; const uint32_t* task_last; const int32_t* task_maxspan;
    const int32_t* mask; const uint32_t* mask_task_off;      // reference 'N' runs (may be null)
    uint32_t n_task; unsigned long long n_bound;     // capacity of every per-lead array (launch size)
    DevCounters* ctr;
    snfb_config cfg;
    int cut_gap;                                      // chains are cut at gaps larger than this (INT_MAX: never)
    // sort buffers
    uint64_t* key0; uint32_t* val0; uint64_t* key1; uint32_t* val1;
    const uint64_t* skey; const uint32_t* sval;       // sorted result
    // bins
    uint32_t* flag; uint32_t* scan;                   // generic flag / scan arrays (n_bound)
    uint32_t* bin_start; uint32_t* bin_nl; uint32_t* bin_nlong; uint32_t* bin_kept; uint32_t* bin_hap;
    uint32_t* kl_off; uint32_t* kll_off; uint32_t* kb_idx;
    // kept leads: slot lists, then the 64-byte leads themselves gathered into kept order (a cluster is a contiguous byte range)
    uint32_t* kl; uint32_t* kll; snfb_lead* kleads; snfb_lead* klleads;
    uint32_t* kb_bin; uint32_t* kb_lead_off; uint32_t* kb_lead_n; uint32_t* kb_long_off; uint32_t* kb_long_n; int32_t* kb_seed; uint32_t* kb_chain; uint8_t* kb_repeat;
    // segments and clusters
    uint32_t* seg_start;
    uint32_t* c_next; uint32_t* c_last; double* c_sd; double* c_mean; uint8_t* c_rep;
    double* seg_sd_last; double* seg_maxsd_first;
    uint32_t* cl_first; uint32_t* cl_last; uint8_t* cl_rep;
    uint32_t* big_list; uint32_t* mid_list;      // clusters with more than WARP_CAP / SMALL_CAP leads
    // global workspace of the clusters too large for shared memory, indexed in kept-lead space
    uint64_t* g_khi; uint64_t* g_klo; uint32_t* g_u32;
    // per-lead results of the cluster kernel
    uint32_t* ord;                  // kept-lead indices in merge_inner iteration order (absolute)
    // staging in kept-lead space: a cluster's sub-clusters, their leads and read names, before the compaction into reference order
    snfb_lead* st_leads; uint32_t* st_plo; uint32_t* st_pn; uint64_t* st_rn; snfb_cand* cand_tmp; uint8_t* sub_valid;
    uint32_t* cl_nsub; uint32_t* cl_nvalid; uint32_t* cl_nlead; uint32_t* cl_nrn; uint32_t* cl_cand_base; uint32_t* cl_lead_base; uint32_t* cl_rn_base;
    // candidates
    snfb_cand* cand; snfb_lead* cand_leads; uint32_t* out_plo; uint32_t* out_pn; uint64_t* rnames; uint32_t* rn_off_out;
    unsigned long long cand_cap, cand_lead_cap, rn_cap;
    uint32_t* scan_tmp;
};

__device__ __forceinline__ int lf_type(uint32_t f) { return (int)(f & 7u); }

// ---------------------------------------------------------------- in-thread heap sort (rare serial paths only)
__device__ inline void hsort1(uint64_t* a, long n) {                  // ascending, unsigned
    if (n < 2) return;
    for (long start = n / 2 - 1; start >= 0; --start) {
        long r = start; uint64_t v = a[r];
        for (;;) { long c = 2 * r + 1; if (c >= n) break; if (c + 1 < n && a[c] < a[c + 1]) ++c; if (!(v < a[c])) break; a[r] = a[c]; r = c; }
        a[r] = v;
    }
    for (long end = n - 1; end > 0; --end) {
        uint64_t v = a[end]; a[end] = a[0]; long r = 0;
        for (;;) { long c = 2 * r + 1; if (c >= end) break; if (c + 1 < end && a[c] < a[c + 1]) ++c; if (!(v < a[c])) break; a[r] = a[c]; r = c; }
        a[r] = v;
    }
}
__device__ __forceinline__ uint64_t bias64(long long v) { return (uint64_t)v ^ 0x8000000000000000ull; }
__device__ __forceinline__ long long unbias64(uint64_t v) { return (long long)(v ^ 0x8000000000000000ull); }

// ---------------------------------------------------------------- canonical order + sort keys
__global__ void k_scatter_keys(B b) {
    const unsigned long long n_slots = b.ctr->n_slots < b.n_bound ? b.ctr->n_slots : b.n_bound;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n_slots; i += (unsigned long long)gridDim.x * blockDim.x) {
        const snfb_lead* l = &b.leads[i];
        if (l->rec == extract::HOLE) continue;         // unused slot of a retired allocation chunk
        const unsigned long long r = (unsigned long long)b.rec_lead_off[l->rec] + l->k;
        if (r >= b.n_bound) continue;                  // capacity exceeded: the run is repeated with a larger one
        const uint64_t bin = (uint64_t)(l->ref_start / b.cfg.cluster_binsize);
        b.key0[r] = ((uint64_t)l->task << TASK_SHIFT) | ((uint64_t)lf_type(l->flags) << TYPE_SHIFT) | bin;
        b.val0[r] = (uint32_t)i;
    }
}

__global__ void k_bin_heads(B b) {
    const unsigned long long n = b.ctr->n_leads < b.n_bound ? b.ctr->n_leads : b.n_bound;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        b.flag[i] = (i == 0 || b.skey[i] != b.skey[i - 1]) ? 1u : 0u;
}
// flag/scan -> start index of every bin; bin_start[n_bins] = n
__global__ void k_bin_build(B b) {
    const unsigned long long n = b.ctr->n_leads < b.n_bound ? b.ctr->n_leads : b.n_bound;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x)
        if (b.flag[i]) b.bin_start[b.scan[i]] = (uint32_t)i;
    if (blockIdx.x == 0 && threadIdx.x == 0) b.bin_start[b.ctr->n_bins] = (uint32_t)n;
}
// per-bin statistics: hap counts, split into leads / leads_long, seq dropping (leadprov.py:400-418)
__global__ void k_bin_stats(B b) {
    const unsigned long long nb = b.ctr->n_bins;
    for (unsigned long long bi = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; bi < nb; bi += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t lo = b.bin_start[bi], hi = b.bin_start[bi + 1];
        uint32_t hc[3] = { 0, 0, 0 }; uint32_t nl = 0, nlong = 0;
        for (uint32_t i = lo; i < hi; ++i) {
            snfb_lead* l = &b.leads[b.sval[i]]; uint32_t f = l->flags;
            if ((int)(i - lo) >= b.cfg.consensus_max_reads_bin && (f & SNFB_LF_HAS_SEQ)) { f &= ~SNFB_LF_HAS_SEQ; l->flags = f; l->seq_off = -1; l->seq_len = 0; }
            hc[SNFB_LF_HAP(f)]++;
            if (lf_type(f) == SNFB_INS && (f & SNFB_LF_SVLEN_NONE)) ++nlong; else ++nl;
        }
        const bool kept = (int)nl >= b.cfg.dev_min_leads_cluster;
        b.bin_kept[bi] = kept; b.bin_nl[bi] = kept ? nl : 0; b.bin_nlong[bi] = kept ? nlong : 0;
        for (int h = 0; h < 3; ++h) b.bin_hap[bi * 3 + h] = hc[h] > 65535u ? 65535u : hc[h];
    }
}
// tandem repeat flag of a seed (cluster.py:240-246): first interval whose running max end reaches the seed
__device__ inline bool within_tr(const B& b, const snfb_task& tk, int seed) {
    if (tk.tr_n <= 0 || b.tr == nullptr) return false;
    const int32_t* pm = b.tr_pmax + tk.tr_off; int lo = 0, hi = tk.tr_n;
    while (lo < hi) { int mid = (lo + hi) >> 1; if (pm[mid] >= seed) hi = mid; else lo = mid + 1; }
    int j = lo < tk.tr_n ? lo : tk.tr_n - 1;
    const int32_t* t = b.tr + 2 * (size_t)(tk.tr_off + j);
    return t[0] < seed && seed < t[1];
}
__global__ void k_kbin_build(B b) {
    const unsigned long long nb = b.ctr->n_bins;
    for (unsigned long long bi = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; bi < nb; bi += (unsigned long long)gridDim.x * blockDim.x) {
        if (!b.bin_kept[bi]) continue;
        const uint32_t kb = b.kb_idx[bi]; const uint32_t lo = b.bin_start[bi], hi = b.bin_start[bi + 1];
        uint32_t a = b.kl_off[bi], c = b.kll_off[bi];
        b.kb_bin[kb] = (uint32_t)bi; b.kb_lead_off[kb] = a; b.kb_lead_n[kb] = b.bin_nl[bi]; b.kb_long_off[kb] = c; b.kb_long_n[kb] = b.bin_nlong[bi];
        for (uint32_t i = lo; i < hi; ++i) { const uint32_t s = b.sval[i]; const uint32_t f = b.leads[s].flags;
            if (lf_type(f) == SNFB_INS && (f & SNFB_LF_SVLEN_NONE)) b.kll[c++] = s; else b.kl[a++] = s; }
        const uint64_t key = b.skey[lo]; const int seed = (int)(key & ((1ull << TYPE_SHIFT) - 1)) * b.cfg.cluster_binsize;
        const uint32_t chain = (uint32_t)(key >> TYPE_SHIFT);
        b.kb_seed[kb] = seed; b.kb_chain[kb] = chain;
        b.kb_repeat[kb] = (within_tr(b, b.task[chain >> 3], seed) || b.cfg.repeat) ? 1 : 0;
    }
}

// the kept leads themselves, gathered once into kept order: from here on a cluster's leads are one contiguous byte range
__global__ void k_gather_kept(B b) {
    const unsigned long long nk = b.ctr->n_kl, nl = b.ctr->n_kll;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nk + nl; i += (unsigned long long)gridDim.x * blockDim.x) {
        const bool lng = i >= nk; const unsigned long long j = lng ? i - nk : i;
        const uint4* s = reinterpret_cast<const uint4*>(b.leads + (lng ? b.kll[j] : b.kl[j])); uint4* d = reinterpret_cast<uint4*>((lng ? b.klleads : b.kleads) + j);
        const uint4 x0 = s[0], x1 = s[1], x2 = s[2], x3 = s[3]; d[0] = x0; d[1] = x1; d[2] = x2; d[3] = x3;
    }
}

// ---------------------------------------------------------------- chain segmentation
__host__ __device__ __forceinline__ int break_gap(const snfb_config& cfg) {
    double g = cfg.cluster_repeat_h_max > (double)cfg.cluster_merge_bnd ? cfg.cluster_repeat_h_max : (double)cfg.cluster_merge_bnd;
    return g > 2.0e9 ? 2000000000 : (int)g;
}
__global__ void k_seg_heads(B b) {
    const unsigned long long nk = b.ctr->n_kbins;
    const int bg = b.cut_gap;
    for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < nk; k += (unsigned long long)gridDim.x * blockDim.x)
        b.flag[k] = (k == 0 || b.kb_chain[k] != b.kb_chain[k - 1] || ((long long)b.kb_seed[k] - ((long long)b.kb_seed[k - 1] + b.cfg.cluster_binsize)) > (long long)bg) ? 1u : 0u;
}
__global__ void k_seg_build(B b) {
    const unsigned long long nk = b.ctr->n_kbins;
    for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < nk; k += (unsigned long long)gridDim.x * blockDim.x)
        if (b.flag[k]) b.seg_start[b.scan[k]] = (uint32_t)k;
    if (blockIdx.x == 0 && threadIdx.x == 0) b.seg_start[b.ctr->n_segs] = (uint32_t)nk;
}

// Cluster.compute_metrics over the kept leads [lo,hi) (cluster.py:48-61)
__device__ inline void compute_metrics(const B& b, uint32_t lo, uint32_t hi, double* mean_svlen, double* sd) {
    const long len = (long)hi - lo; const long n = len < 100 ? len : 100;
    if (n == 0) { *mean_svlen = 0; *sd = 0; return; }
    if (n == 1) { *mean_svlen = (double)b.kleads[lo].svlen; *sd = 0; return; }
    const long step = len / n;      // int(len / n)
    long long sum = 0; long m = 0; const long long base = b.kleads[lo].ref_start; u128 sxx = 0; __int128 sx = 0;
    for (long i = 0; i < len; i += step) { const snfb_lead* l = &b.kleads[lo + i]; sum += l->svlen; const __int128 d = (__int128)((long long)l->ref_start - base); sx += d; sxx += (u128)(d * d); ++m; }
    *mean_svlen = __ddiv_rn((double)sum, (double)n);
    *sd = sqrt_frac_rn((u128)m * sxx - (u128)(sx * sx), (uint64_t)m * (uint64_t)(m - 1));
}

// the merge automaton of cluster.resolve on one chain piece (cluster.py:278-308)
__global__ void k_merge(B b) {
    const unsigned long long ns = b.ctr->n_segs;
    const snfb_config& cfg = b.cfg;
    for (unsigned long long s = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; s < ns; s += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t k0 = b.seg_start[s], k1 = b.seg_start[s + 1];
        const uint32_t chain = b.kb_chain[k0]; const int svtype = (int)(chain & 7u);
        const bool first_piece = (k0 == 0) || b.kb_chain[k0 - 1] != chain;     // global index 0 of the chain lives here
        for (uint32_t k = k0; k < k1; ++k) {
            b.c_next[k] = k + 1 < k1 ? k + 1 : NONE; b.c_last[k] = k; b.c_rep[k] = b.kb_repeat[k];
            compute_metrics(b, b.kb_lead_off[k], b.kb_lead_off[k] + b.kb_lead_n[k], &b.c_mean[k], &b.c_sd[k]);
        }
        double maxsd_first = b.c_sd[k0];
        // i walks the linked list; `prev` is tracked so that i-1 is available; idx is the position inside the piece
        uint32_t cur = k0, prev = NONE; long idx = 0;
        while (b.c_next[cur] != NONE) {
            const uint32_t nx = b.c_next[cur];
            const int cur_end = b.kb_seed[b.c_last[cur]] + cfg.cluster_binsize, nx_end = b.kb_seed[b.c_last[nx]] + cfg.cluster_binsize;
            const long long inner = (long long)b.kb_seed[nx] - cur_end, outer = (long long)nx_end - b.kb_seed[cur];
            const double msd = b.c_sd[cur] < b.c_sd[nx] ? b.c_sd[cur] : b.c_sd[nx];
            bool merge = (double)inner <= __dmul_rn(msd, cfg.cluster_r);
            if (!merge && (cfg.repeat || b.c_rep[cur] || b.c_rep[nx])) {
                double lim = __dmul_rn(__dadd_rn(fabs(b.c_mean[cur]), fabs(b.c_mean[nx])), cfg.cluster_repeat_h);
                if (cfg.cluster_repeat_h_max < lim) lim = cfg.cluster_repeat_h_max;
                merge = (double)outer <= lim;
            }
            if (!merge) merge = svtype == SNFB_BND && inner <= cfg.cluster_merge_bnd;
            if (merge) {
                b.c_next[cur] = b.c_next[nx]; b.c_last[cur] = b.c_last[nx]; b.c_rep[cur] = b.c_rep[cur] | b.c_rep[nx];
                compute_metrics(b, b.kb_lead_off[cur], b.kb_lead_off[b.c_last[cur]] + b.kb_lead_n[b.c_last[cur]], &b.c_mean[cur], &b.c_sd[cur]);
                if (cur == k0 && b.c_sd[cur] > maxsd_first) maxsd_first = b.c_sd[cur];
                // i = max(0, i-2) + 1 in chain-global indices.  Pieces after the first sit at global index >= 1,
                // where the rule reduces to "step back one cluster if there is one inside the piece".
                if (first_piece) { if (idx >= 2) { /* i-1 */ cur = prev; --idx; prev = NONE; if (idx > 0) { uint32_t p = k0; while (b.c_next[p] != cur) p = b.c_next[p]; prev = p; } }
                                   else if (idx == 0) { prev = cur; cur = b.c_next[cur]; idx = 1; if (cur == NONE) break; }
                                   /* idx == 1 stays */ }
                else { if (idx >= 1) { cur = prev; --idx; prev = NONE; if (idx > 0) { uint32_t p = k0; while (b.c_next[p] != cur) p = b.c_next[p]; prev = p; } } }
            } else { prev = cur; cur = nx; ++idx; }
        }
        // verification data for the assumed chain cuts
        uint32_t last = k0; while (b.c_next[last] != NONE) last = b.c_next[last];
        b.seg_sd_last[s] = b.c_sd[last]; b.seg_maxsd_first[s] = maxsd_first;
        // mark surviving cluster heads
        for (uint32_t k = k0; k < k1; ++k) b.flag[k] = 0;
        for (uint32_t k = k0; k != NONE; k = b.c_next[k]) b.flag[k] = 1;
    }
}
// a cut between pieces is only valid if the stdev criterion could never have bridged it
__global__ void k_verify_cuts(B b) {
    const unsigned long long ns = b.ctr->n_segs;
    for (unsigned long long s = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x + 1; s < ns; s += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t k0 = b.seg_start[s];
        if (b.kb_chain[k0] != b.kb_chain[k0 - 1]) continue;
        const long long gap = (long long)b.kb_seed[k0] - (b.kb_seed[k0 - 1] + b.cfg.cluster_binsize);
        const double a = b.seg_sd_last[s - 1], c = b.seg_maxsd_first[s]; const double m = a < c ? a : c;
        if ((double)gap <= __dmul_rn(m, b.cfg.cluster_r)) atomicAdd(&b.ctr->unverified_breaks, 1ULL);
    }
}
__global__ void k_cluster_build(B b) {
    const unsigned long long nk = b.ctr->n_kbins;
    if (blockIdx.x == 0 && threadIdx.x == 0) b.ctr->n_small_taken = 0;        // the work queue of k_cluster_warp<SMALL_CAP>
    for (unsigned long long k = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; k < nk; k += (unsigned long long)gridDim.x * blockDim.x)
        if (b.flag[k]) {
            const uint32_t c = b.scan[k], kl_ = b.c_last[k]; b.cl_first[c] = (uint32_t)k; b.cl_last[c] = kl_; b.cl_rep[c] = b.c_rep[k];
            const uint32_t n = b.kb_lead_off[kl_] + b.kb_lead_n[kl_] - b.kb_lead_off[k];
            if (n > (uint32_t)WARP_CAP) b.big_list[atomicAdd(&b.ctr->n_big, 1ULL)] = c;
            else if (n > (uint32_t)SMALL_CAP) b.mid_list[atomicAdd(&b.ctr->n_mid, 1ULL)] = c;
        }
}

// ================================================================================================
// Per-cluster processing: cluster.merge_inner (cluster.py:85-122), cluster.resplit (125-161), cluster.resplit_bnd (164-216),
// then per sub-cluster sv.call_from / resolve_bnd (sv.py:497-639), get_sa_count (cluster.py:79-82) and the phase aggregates
// (postprocessing.py:626-654) — one kernel, one cooperating thread group per cluster:
//   * a warp for clusters of up to WARP_CAP leads, a 256-thread block for larger ones;
//   * the cluster's leads are one contiguous byte range of `kleads`; the group stages that range into shared memory with
//     one bulk copy (cp.async.bulk + mbarrier) and works on it there; clusters beyond BLOCK_CAP leads read their leads
//     from global memory and keep their key arrays in a global workspace (same code, other pointers);
//   * every sort is a cooperative bitonic network over (key, index) pairs in the workspace — index as the low key makes
//     it stable, so the reference's first-seen / stable-sort orders are reproduced;
//   * the order-dependent automata (resplit's merge with the negative index, tie rules) run on one thread over the
//     workspace arrays.
// Results go to a staging area indexed in kept-lead space; k_emit_cands compacts them into reference emission order.
// ================================================================================================
namespace coop {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                 :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}

// ---- thread groups ----
struct WarpG {
    static constexpr bool is_warp = true;
    __device__ __forceinline__ int maxi(int v) const { return __reduce_max_sync(FULL, v); }
    __device__ __forceinline__ int tid() const { return (int)(threadIdx.x & 31u); }
    __device__ __forceinline__ int nthr() const { return 32; }
    __device__ __forceinline__ void sync() const { __syncwarp(); }
    __device__ __forceinline__ long long sum(long long v) const {
        #pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        return v;
    }
    __device__ __forceinline__ void sum128(unsigned long long& hi, unsigned long long& lo) const {
        #pragma unroll
        for (int o = 16; o; o >>= 1) { const unsigned long long oh = __shfl_xor_sync(FULL, hi, o), ol = __shfl_xor_sync(FULL, lo, o); const unsigned long long nl = lo + ol; hi += oh + (nl < lo ? 1ull : 0ull); lo = nl; }
    }
    __device__ __forceinline__ int excl(bool f, int* total) const { const unsigned m = __ballot_sync(FULL, f); *total = __popc(m); return __popc(m & lanemask_lt()); }
    __device__ __forceinline__ unsigned long long bcast(unsigned long long v) const { return __shfl_sync(FULL, v, 0); }
};
struct BlockG {
    static constexpr bool is_warp = false;
    unsigned long long* red;      // shared scratch: 72 entries
    __device__ inline int maxi(int v) const {
        v = __reduce_max_sync(FULL, v);
        const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
        if ((threadIdx.x & 31) == 0) red[w] = (unsigned long long)(long long)v;
        __syncthreads();
        int t = (int)(long long)red[0]; for (int i = 1; i < nw; ++i) { const int x = (int)(long long)red[i]; if (x > t) t = x; }
        __syncthreads();
        return t;
    }
    __device__ __forceinline__ int tid() const { return (int)threadIdx.x; }
    __device__ __forceinline__ int nthr() const { return (int)blockDim.x; }
    __device__ __forceinline__ void sync() const { __syncthreads(); }
    __device__ inline long long sum(long long v) const {
        #pragma unroll
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
        const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
        if ((threadIdx.x & 31) == 0) red[w] = (unsigned long long)v;
        __syncthreads();
        long long t = 0; for (int i = 0; i < nw; ++i) t += (long long)red[i];
        __syncthreads();
        return t;
    }
    __device__ inline void sum128(unsigned long long& hi, unsigned long long& lo) const {
        #pragma unroll
        for (int o = 16; o; o >>= 1) { const unsigned long long oh = __shfl_xor_sync(FULL, hi, o), ol = __shfl_xor_sync(FULL, lo, o); const unsigned long long nl = lo + ol; hi += oh + (nl < lo ? 1ull : 0ull); lo = nl; }
        const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
        if ((threadIdx.x & 31) == 0) { red[2 * w] = hi; red[2 * w + 1] = lo; }
        __syncthreads();
        unsigned long long th = 0, tl = 0; for (int i = 0; i < nw; ++i) { const unsigned long long nl = tl + red[2 * i + 1]; th += red[2 * i] + (nl < tl ? 1ull : 0ull); tl = nl; }
        __syncthreads();
        hi = th; lo = tl;
    }
    __device__ inline int excl(bool f, int* total) const {
        const unsigned m = __ballot_sync(FULL, f);
        const int w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
        if ((threadIdx.x & 31) == 0) red[w] = (unsigned long long)__popc(m);
        __syncthreads();
        int base = 0, tot = 0; for (int i = 0; i < nw; ++i) { const int v = (int)red[i]; if (i < w) base += v; tot += v; }
        __syncthreads();
        *total = tot; return base + __popc(m & lanemask_lt());
    }
    __device__ inline unsigned long long bcast(unsigned long long v) const {
        if (threadIdx.x == 0) red[70] = v;
        __syncthreads();
        const unsigned long long r = red[70];
        __syncthreads();
        return r;
    }
};
template <class G> __device__ __forceinline__ long long bcast_ll(const G& g, long long v) { return (long long)g.bcast((unsigned long long)v); }
template <class G> __device__ __forceinline__ double bcast_f8(const G& g, double v) { return __longlong_as_double((long long)g.bcast((unsigned long long)__double_as_longlong(v))); }

// ---- bitonic network with ascending comparators only: positions >= n behave as +infinity and are never touched, so the
//      arrays need exactly n entries.  Keys must be distinct for a deterministic result (callers put the index in the low key).
__device__ __forceinline__ bool lt2(uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl) { return ah < bh || (ah == bh && al < bl); }
template <class G> __device__ __noinline__ void sort2(const G& g, uint64_t* hi, uint64_t* lo, int n) {    // ascending by (hi, lo)
    if (n < 2) return;
    if (G::is_warp && n <= 32) {                      // one element per lane: its rank is the number of smaller elements (register shuffles, no network)
        const int i = g.tid(); const uint64_t xh = i < n ? hi[i] : 0, xl = i < n ? lo[i] : 0; int rank = 0;
        for (int j = 0; j < n; ++j) { const uint64_t yh = __shfl_sync(FULL, xh, j), yl = __shfl_sync(FULL, xl, j); rank += lt2(yh, yl, xh, xl) ? 1 : 0; }
        g.sync();
        if (i < n) { hi[rank] = xh; lo[rank] = xl; }
        g.sync();
        return;
    }
    int lp = 1; while ((1 << lp) < n) ++lp;
    const int half = 1 << (lp - 1);
    for (int lk = 1; lk <= lp; ++lk) {
        {   const int lh = lk - 1, km1 = (1 << lk) - 1;
            for (int i = g.tid(); i < half; i += g.nthr()) { const int l = ((i >> lh) << lk) + (i & ((1 << lh) - 1)), r = l ^ km1;
                if (r < n) { const uint64_t ah = hi[l], al = lo[l], bh = hi[r], bl = lo[r]; if (lt2(bh, bl, ah, al)) { hi[l] = bh; lo[l] = bl; hi[r] = ah; lo[r] = al; } } }
            g.sync(); }
        for (int lj = lk - 2; lj >= 0; --lj) {
            for (int i = g.tid(); i < half; i += g.nthr()) { const int l = ((i >> lj) << (lj + 1)) + (i & ((1 << lj) - 1)), r = l + (1 << lj);
                if (r < n) { const uint64_t ah = hi[l], al = lo[l], bh = hi[r], bl = lo[r]; if (lt2(bh, bl, ah, al)) { hi[l] = bh; lo[l] = bl; hi[r] = ah; lo[r] = al; } } }
            g.sync();
        }
    }
}
template <class G> __device__ __noinline__ void sort1(const G& g, uint64_t* a, int n) {                     // ascending, unsigned (ties are equal values: order-free)
    if (n < 2) return;
    if (G::is_warp && n <= 32) {
        const int i = g.tid(); const uint64_t x = i < n ? a[i] : 0; int rank = 0;
        for (int j = 0; j < n; ++j) { const uint64_t y = __shfl_sync(FULL, x, j); rank += (y < x || (y == x && j < i)) ? 1 : 0; }
        g.sync();
        if (i < n) a[rank] = x;
        g.sync();
        return;
    }
    int lp = 1; while ((1 << lp) < n) ++lp;
    const int half = 1 << (lp - 1);
    for (int lk = 1; lk <= lp; ++lk) {
        {   const int lh = lk - 1, km1 = (1 << lk) - 1;
            for (int i = g.tid(); i < half; i += g.nthr()) { const int l = ((i >> lh) << lk) + (i & ((1 << lh) - 1)), r = l ^ km1;
                if (r < n) { const uint64_t x = a[l], y = a[r]; if (y < x) { a[l] = y; a[r] = x; } } }
            g.sync(); }
        for (int lj = lk - 2; lj >= 0; --lj) {
            for (int i = g.tid(); i < half; i += g.nthr()) { const int l = ((i >> lj) << (lj + 1)) + (i & ((1 << lj) - 1)), r = l + (1 << lj);
                if (r < n) { const uint64_t x = a[l], y = a[r]; if (y < x) { a[l] = y; a[r] = x; } } }
            g.sync();
        }
    }
}
// positions p of [0, n) with pred(p) true, in order, into out[]; returns their number (to every thread).  Ends with a sync.
template <class G, class F> __device__ inline int compact(const G& g, int n, uint32_t* out, F pred) {
    int carry = 0;
    for (int base = 0; base < n; base += g.nthr()) {
        const int p = base + g.tid(); const bool f = p < n && pred(p);
        int tot; const int e = g.excl(f, &tot);
        if (f) out[carry + e] = (uint32_t)p;
        carry += tot;
    }
    g.sync();
    return carry;
}
// number of distinct values of a sorted array (all threads get it)
template <class G> __device__ inline int count_distinct_sorted(const G& g, const uint64_t* a, int n) {
    long long c = 0; for (int i = g.tid(); i < n; i += g.nthr()) c += (i == 0 || a[i] != a[i - 1]) ? 1 : 0;
    return (int)g.sum(c);
}
// exact sample stdev of the biased-int64 values a[0..m): statistics.stdev through P = m Sxx - Sx^2, Q = m (m - 1) (common.cuh)
template <class G> __device__ __noinline__ double stdev_sorted(const G& g, const uint64_t* a, long m) {
    if (m < 2) return 0.0;
    const long long base = unbias64(a[0]);
    long long sx = 0; u128 sxx = 0;
    for (long i = g.tid(); i < m; i += g.nthr()) { const long long d = unbias64(a[i]) - base; sx += d; sxx += (u128)((__int128)d * d); }
    sx = g.sum(sx);
    unsigned long long h = (unsigned long long)(sxx >> 64), l = (unsigned long long)sxx; g.sum128(h, l);
    double r = 0.0;
    if (g.tid() == 0) { const u128 S = ((u128)h << 64) | l; const __int128 s1 = (__int128)sx; r = sqrt_frac_rn((u128)m * S - (u128)(s1 * s1), (uint64_t)m * (uint64_t)(m - 1)); }
    return bcast_f8(g, r);
}
// util.stdev(util.trim(v)) on a sorted array (util.py:25-27, 82-88)
template <class G> __device__ inline double stdev_trim_sorted(const G& g, const uint64_t* a, long n) {
    const long trim_n = (long)__dmul_rn(__ddiv_rn((double)n, 100.0), 25.0);
    const long lo = trim_n > 0 ? trim_n : 0, m = trim_n > 0 ? n - 2 * trim_n : n;
    return stdev_sorted(g, a + lo, m);
}

// util.center = median_modes over a sorted (biased) array (util.py:49-58): the upper median of the distinct values whose multiplicity is
// within 2 of the largest one.  Cooperative: run heads, run lengths, the qualifying runs.  s0 / s1: scratch of n entries each.
template <class G> __device__ __noinline__ long long center_sorted(const G& g, const uint64_t* a, int n, uint32_t* s0, uint32_t* s1) {
    const int nh = compact(g, n, s0, [&](int i) { return i == 0 || a[i] != a[i - 1]; });
    int mx = 0; for (int h = g.tid(); h < nh; h += g.nthr()) { const int c = (int)((h + 1 < nh ? s0[h + 1] : (uint32_t)n) - s0[h]); if (c > mx) mx = c; }
    const int maxc = g.maxi(mx);
    const int m = compact(g, nh, s1, [&](int h) { return maxc - (int)((h + 1 < nh ? s0[h + 1] : (uint32_t)n) - s0[h]) < 3; });
    const long long r = unbias64(a[s0[s1[m / 2]]]);
    g.sync();
    return r;
}

constexpr int NU32 = 15;
struct WS { const snfb_lead* L; uint64_t* khi; uint64_t* klo; uint32_t* u[NU32]; };

}  // namespace coop

__device__ inline int cmp_decstr(long long a, long long b) {     // strcmp(str(a), str(b)) for the PS tie break
    char x[24], y[24]; int nx = 0, ny = 0;
    { unsigned long long v = a < 0 ? (unsigned long long)(-a) : (unsigned long long)a; char t[24]; int k = 0; do { t[k++] = (char)('0' + v % 10); v /= 10; } while (v); if (a < 0) x[nx++] = '-'; while (k) x[nx++] = t[--k]; }
    { unsigned long long v = b < 0 ? (unsigned long long)(-b) : (unsigned long long)b; char t[24]; int k = 0; do { t[k++] = (char)('0' + v % 10); v /= 10; } while (v); if (b < 0) y[ny++] = '-'; while (k) y[ny++] = t[--k]; }
    for (int i = 0; i < nx && i < ny; ++i) if (x[i] != y[i]) return x[i] < y[i] ? -1 : 1;
    return nx == ny ? 0 : (nx < ny ? -1 : 1);
}

template <class G>
__device__ void process_cluster(const G& g, const B& b, const uint32_t c, const coop::WS& ws) {
    using namespace coop;
    const snfb_config& cfg = b.cfg;
    const uint32_t kf = b.cl_first[c], kl_ = b.cl_last[c];
    const uint32_t lo = b.kb_lead_off[kf], hi = b.kb_lead_off[kl_] + b.kb_lead_n[kl_];
    const int n = (int)(hi - lo);
    const uint32_t chain = b.kb_chain[kf]; const int svtype = (int)(chain & 7u); const int task = (int)(chain >> 3);
    const uint32_t llo = b.kb_long_off[kf], lhi = b.kb_long_off[kl_] + b.kb_long_n[kl_];
    const bool has_long = svtype == SNFB_INS; const int nlong = has_long ? (int)(lhi - llo) : 0;
    const snfb_lead* L = ws.L; const snfb_lead* LL = b.klleads + llo;
    uint64_t* khi = ws.khi; uint64_t* klo = ws.klo;
    uint32_t* ordv = ws.u[0]; uint32_t* ml_plo = ws.u[1]; uint32_t* ml_pn = ws.u[2]; int32_t* ml_svlen = reinterpret_cast<int32_t*>(ws.u[3]); int32_t* ml_seqlen = reinterpret_cast<int32_t*>(ws.u[4]);
    uint32_t* ml_has = ws.u[5]; uint32_t* subl = ws.u[6]; uint32_t* t_lo = ws.u[7]; uint32_t* t_n = ws.u[8]; int32_t* t_bin = reinterpret_cast<int32_t*>(ws.u[9]);
    uint32_t* sA = ws.u[10]; uint32_t* sB = ws.u[11]; uint32_t* sC = ws.u[12]; uint32_t* sD = ws.u[13]; uint32_t* sE = ws.u[14];
    const int tid = g.tid(), nthr = g.nthr();
    int nm = 0;
    // ------------------------------------------------------------ merge_inner
    if (svtype == SNFB_INS || svtype == SNFB_DEL) {
        const int thr = b.cl_rep[c] ? -1 : cfg.cluster_merge_pos;
        // groups by qname in first-seen order: sort (hash, idx); a run's first entry carries the smallest idx
        for (int i = tid; i < n; i += nthr) { khi[i] = L[i].qname_hash; klo[i] = (uint64_t)i; }
        g.sync();
        sort2(g, khi, klo, n);
        for (int p = tid; p < n; p += nthr) if (p == 0 || khi[p] != khi[p - 1]) { const uint32_t f = (uint32_t)klo[p]; for (int q = p; q < n && khi[q] == khi[p]; ++q) sA[klo[q]] = f; }
        g.sync();
        for (int i = tid; i < n; i += nthr) { const int rs = L[i].ref_start; khi[i] = ((uint64_t)sA[i] << 32) | (uint32_t)(rs ^ 0x80000000); klo[i] = (uint64_t)i; }
        g.sync();
        sort2(g, khi, klo, n);
        for (int r = tid; r < n; r += nthr) { const uint32_t i = (uint32_t)klo[r]; ordv[r] = i; b.ord[lo + r] = lo + i; }
        g.sync();
        // a lead starts a merged lead unless it folds into its predecessor of the same read (cluster.py:100-118): the test only looks
        // at the predecessor (the strand of a merged lead is the strand of all its parts whenever the test applies)
        nm = compact(g, n, ml_plo, [&](int q) {
            if (q == 0 || (uint32_t)(khi[q] >> 32) != (uint32_t)(khi[q - 1] >> 32)) return true;
            if (thr == -1) return false;
            const snfb_lead* to = &L[ordv[q]]; const snfb_lead* la = &L[ordv[q - 1]];
            const bool mg = ((abs(to->ref_start - la->ref_end) < thr || abs(to->ref_start - la->ref_start) < thr) && (abs(to->qry_start - la->qry_end) < thr || abs(to->qry_start - la->qry_start) < thr))
                            && ((to->flags & SNFB_LF_REVERSE) == (la->flags & SNFB_LF_REVERSE));
            return !mg; });
        for (int m = tid; m < nm; m += nthr) {
            const int q0 = (int)ml_plo[m], q1 = m + 1 < nm ? (int)ml_plo[m + 1] : n;
            long long sv = 0, sl = 0; bool hs = true;
            for (int q = q0; q < q1; ++q) { const snfb_lead* l = &L[ordv[q]]; sv += l->svlen; if (l->flags & SNFB_LF_HAS_SEQ) sl += l->seq_len; else hs = false; }
            ml_pn[m] = (uint32_t)(q1 - q0); ml_svlen[m] = (int)sv; ml_has[m] = hs ? 1u : 0u; ml_seqlen[m] = hs ? (int)sl : 0;
        }
        g.sync();
    } else {
        for (int i = tid; i < n; i += nthr) { const snfb_lead* l = &L[i]; ordv[i] = (uint32_t)i; b.ord[lo + i] = lo + i; ml_plo[i] = (uint32_t)i; ml_pn[i] = 1; ml_svlen[i] = l->svlen; ml_has[i] = (l->flags & SNFB_LF_HAS_SEQ) ? 1u : 0u; ml_seqlen[i] = l->seq_len; }
        nm = n;
        g.sync();
    }
    #define ML_LEAD(mi) (L[ordv[ml_plo[(mi)]]])
    // ------------------------------------------------------------ sub-clusters
    int nsub = 0;
    if (svtype == SNFB_BND && !(cfg.dev_no_resplit || nm <= 1)) {
        const int thr = cfg.cluster_merge_bnd;
        // groups by (mate_contig, is_first) in first-seen order, then by mate position bin inside a group (cluster.py:164-216)
        for (int i = tid; i < nm; i += nthr) { const snfb_lead* l = &ML_LEAD(i); khi[i] = ((uint64_t)(uint32_t)(l->mate_contig + 2) << 1) | ((l->flags & SNFB_LF_BND_FIRST) ? 1u : 0u); klo[i] = (uint64_t)i; }
        g.sync();
        sort2(g, khi, klo, nm);
        for (int p = tid; p < nm; p += nthr) if (p == 0 || khi[p] != khi[p - 1]) { const uint32_t f = (uint32_t)klo[p]; for (int q = p; q < nm && khi[q] == khi[p]; ++q) sA[klo[q]] = f; }
        g.sync();
        for (int i = tid; i < nm; i += nthr) { const int mp = ML_LEAD(i).mate_pos; const int pb = thr > 0 ? (mp / thr) * thr : 0; khi[i] = ((uint64_t)sA[i] << 32) | (uint32_t)(pb ^ 0x80000000); klo[i] = (uint64_t)i; }
        g.sync();
        sort2(g, khi, klo, nm);
        for (int i = tid; i < nm; i += nthr) subl[i] = (uint32_t)klo[i];
        nsub = compact(g, nm, t_lo, [&](int i) {
            if (i == 0) return true;
            const bool newgrp = (uint32_t)(khi[i] >> 32) != (uint32_t)(khi[i - 1] >> 32);
            const long long pbc = (int)((uint32_t)khi[i] ^ 0x80000000), pbp = (int)((uint32_t)khi[i - 1] ^ 0x80000000);
            return newgrp || (pbc != pbp && pbc - pbp > thr); });
        for (int j = tid; j < nsub; j += nthr) { t_n[j] = (j + 1 < nsub ? t_lo[j + 1] : (uint32_t)nm) - t_lo[j]; t_bin[j] = -1; }
        g.sync();
    } else if (svtype == SNFB_BND || cfg.dev_no_resplit_repeat || cfg.dev_no_resplit) {
        for (int i = tid; i < nm; i += nthr) subl[i] = (uint32_t)i;
        if (tid == 0) { t_lo[0] = 0; t_n[0] = (uint32_t)nm; t_bin[0] = -1; }
        nsub = 1;
        g.sync();
    } else {
        // resplit (cluster.py:125-161): distinct svlen bins ascending, then the order-dependent merge with python's negative index
        const int rb = cfg.cluster_resplit_binsize;
        for (int i = tid; i < nm; i += nthr) { const int sv = ml_svlen[i]; const int a = sv < 0 ? -sv : sv; khi[i] = (uint64_t)((a / rb) * rb); klo[i] = (uint64_t)i; }
        g.sync();
        sort2(g, khi, klo, nm);
        uint32_t* seg_first = sA; uint32_t* seg_end = sB; uint32_t* seg_next = sC; uint32_t* nc = sD; uint32_t* tail = sE;
        const int nb = compact(g, nm, seg_first, [&](int i) { return i == 0 || khi[i] != khi[i - 1]; });
        for (int k = tid; k < nb; k += nthr) { seg_end[k] = k + 1 < nb ? seg_first[k + 1] : (uint32_t)nm; seg_next[k] = NONE; tail[k] = (uint32_t)k; nc[k] = (uint32_t)k; }
        g.sync();
        int ns = 0;
        if (tid == 0) {
            long len = nb, i = 1;
            while (len > 1 && i < len) {
                const long li = i - 1 < 0 ? len - 1 : i - 1;
                const long long last = (long long)khi[seg_first[nc[li]]], curr = (long long)khi[seg_first[nc[i]]];
                double thr = __dmul_rn((double)(curr < last ? curr : last), cfg.cluster_merge_len); if ((double)cfg.minsvlen > thr) thr = (double)cfg.minsvlen;
                const long long d = curr - last < 0 ? last - curr : curr - last;
                if ((double)d <= thr) {
                    seg_next[tail[nc[i]]] = nc[li]; tail[nc[i]] = tail[nc[li]];          // bins[curr].extend(bins[last])
                    for (long k = li; k + 1 < len; ++k) nc[k] = nc[k + 1]; --len;        // pop(i-1)
                    i = i - 2 > 0 ? i - 2 : 0;
                } else ++i;
            }
            long w = 0;
            for (long k = 0; k < len; ++k) {
                const long start = w;
                for (uint32_t sg = nc[k]; sg != NONE; sg = seg_next[sg]) for (uint32_t q = seg_first[sg]; q < seg_end[sg]; ++q) subl[w++] = (uint32_t)klo[q];
                t_lo[ns] = (uint32_t)start; t_n[ns] = (uint32_t)(w - start); t_bin[ns] = (int)khi[seg_first[nc[k]]]; ++ns;
            }
        }
        nsub = (int)g.bcast((unsigned long long)ns);
        g.sync();
    }
    // ------------------------------------------------------------ per sub-cluster: sv.call_from and friends
    uint64_t* w = khi; uint64_t* w2 = klo;
    uint32_t nvalid = 0, nlead_out = 0, nrn_out = 0;
    for (int j = 0; j < nsub; ++j) {
        const int slo = (int)t_lo[j]; const int ns = (int)t_n[j];
        const uint32_t sidx = lo + (uint32_t)j;           // staging slot of this sub-cluster
        if (tid == 0) b.sub_valid[sidx] = 0;
        if (ns == 0) continue;
        #define SUB_ML(i) (subl[slo + (i)])
        #define SUB_LEAD(i) (L[sl[(i)]])
        // svlen = center(svlens); each lead's place in L is resolved here once (sl), so the loops below read a lead through one index
        uint32_t* sl = sC;
        for (int i = tid; i < ns; i += nthr) { const uint32_t mi = SUB_ML(i); sl[i] = ordv[ml_plo[mi]]; w[i] = bias64(ml_svlen[mi]); }
        g.sync();
        sort1(g, w, ns);
        const long long svlen = center_sorted(g, w, ns, sA, sB);
        const bool single = svtype == SNFB_SINGLE_LEFT || svtype == SNFB_SINGLE_RIGHT;
        if (!single && svtype != SNFB_BND && (svlen < 0 ? -svlen : svlen) < cfg.minsvlen_screen) { g.sync(); continue; }
        double sd_len = __longlong_as_double(0x7ff8000000000000LL);
        if (svtype != SNFB_BND) sd_len = stdev_trim_sorted(g, w, ns);
        g.sync();
        for (int i = tid; i < ns; i += nthr) w[i] = bias64(SUB_LEAD(i).ref_start);
        g.sync();
        sort1(g, w, ns);
        const long long ref_start = center_sorted(g, w, ns, sA, sB);
        const double sd_pos = stdev_trim_sorted(g, w, ns);
        g.sync();
        const bool precise = svtype != SNFB_BND ? (__dadd_rn(sd_pos, sd_len) < (double)cfg.precise) : (sd_pos < (double)cfg.precise);
        long long svstart, svend;
        if (svtype == SNFB_INS) { svstart = svend = ref_start; }
        else if (svtype == SNFB_DEL) { svstart = ref_start + svlen; svend = ref_start; }
        else { svstart = ref_start; svend = svstart + (svlen < 0 ? -svlen : svlen); }
        long long mq = 0, fwd = 0, sa = 0, nsplit = 0;
        for (int i = tid; i < ns; i += nthr) { const uint32_t f = SUB_LEAD(i).flags; mq += SNFB_LF_MAPQ(f); fwd += !(f & SNFB_LF_REVERSE); sa += (f & SNFB_LF_IS_SA) != 0; nsplit += SNFB_LF_SOURCE(f) != SNFB_SRC_INLINE; }
        for (int i = tid; i < nlong; i += nthr) sa += (LL[i].flags & SNFB_LF_IS_SA) != 0;
        mq = g.sum(mq); fwd = g.sum(fwd); sa = g.sum(sa); nsplit = g.sum(nsplit);
        // support = distinct qnames (+ leads_long for long insertions); the sorted distinct hashes stay in w2[0..nq)
        for (int i = tid; i < ns; i += nthr) w[i] = SUB_LEAD(i).qname_hash;
        g.sync();
        sort1(g, w, ns);
        int nq = compact(g, ns, sA, [&](int i) { return i == 0 || w[i] != w[i - 1]; });
        for (int i = tid; i < nq; i += nthr) w2[i] = w[sA[i]];
        g.sync();
        long long support = nq, support_long = 0;
        const bool use_long = svtype == SNFB_INS && svlen >= cfg.long_ins_length;
        if (use_long) {
            long long sl2 = 0, extra = 0;
            if (tid == 0) for (int i = 0; i < nlong; ++i) { const uint64_t h = LL[i].qname_hash; bool dup = false;
                for (int q = 0; q < i; ++q) if (LL[q].qname_hash == h) { dup = true; break; }
                if (dup) continue; ++sl2;
                int lo2 = 0, hi2 = nq; while (lo2 < hi2) { const int mid = (lo2 + hi2) >> 1; if (w2[mid] < h) lo2 = mid + 1; else hi2 = mid; }
                if (!(lo2 < nq && w2[lo2] == h)) ++extra; }
            support_long = bcast_ll(g, sl2); support += bcast_ll(g, extra);
        }
        double nm_mean = -1.0;
        if (cfg.qc_nm_measure) {       // util.mean(v.nm): python's sum() is Neumaier-compensated (bltinmodule.c); sequential by definition
            double r = 0.0;
            if (tid == 0) { double sm = 0.0, cc = 0.0;
                for (int i = 0; i < ns; ++i) { const snfb_lead* l = &SUB_LEAD(i); const double x = lf_type(l->flags) == SNFB_BND ? (double)l->nm_sa : b.rec_nm[l->rec];
                    const double tt = __dadd_rn(sm, x); if (fabs(sm) >= fabs(x)) cc = __dadd_rn(cc, __dadd_rn(__dadd_rn(sm, -tt), x)); else cc = __dadd_rn(cc, __dadd_rn(__dadd_rn(x, -tt), sm)); sm = tt; }
                if (cc != 0.0 && isfinite(cc)) sm = __dadd_rn(sm, cc);
                r = __ddiv_rn(sm, (double)ns); }
            nm_mean = bcast_f8(g, r);
        }
        int nfinal = ns; int bnd_contig = -1, bnd_pos = 0, bnd_first = 0, bnd_rev = 0;
        if (svtype == SNFB_BND) {      // resolve_bnd (sv.py:625-639): keep the leads of the modal mate contig (ties: smallest name)
            for (int i = tid; i < ns; i += nthr) { const int mc = SUB_LEAD(i).mate_contig; uint32_t k = 0; for (int q = 0; q < ns; ++q) k += SUB_LEAD(q).mate_contig == mc; sB[i] = k; }
            g.sync();
            int best = -2;
            if (tid == 0) { long bestc = 0; int bestrank = 0;
                for (int i = 0; i < ns; ++i) { const int mc = SUB_LEAD(i).mate_contig; const long k = sB[i]; const int rk = mc >= 0 ? b.contig[mc].lex_rank : 1 << 30;
                    if (k > bestc || (k == bestc && rk < bestrank)) { best = mc; bestc = k; bestrank = rk; } } }
            best = (int)bcast_ll(g, best);
            // stable filter of the sub-cluster's order
            const int m = compact(g, ns, sA, [&](int i) { return SUB_LEAD(i).mate_contig == best; });
            for (int i = tid; i < m; i += nthr) { sB[i] = SUB_ML(sA[i]); sD[i] = sl[sA[i]]; }
            g.sync();
            for (int i = tid; i < m; i += nthr) { subl[slo + i] = sB[i]; sl[i] = sD[i]; }
            g.sync();
            long long nf = 0, nr = 0;
            for (int i = tid; i < m; i += nthr) { const snfb_lead* l = &SUB_LEAD(i); w[i] = bias64(l->mate_pos); w2[i] = l->qname_hash; nf += (l->flags & SNFB_LF_BND_FIRST) != 0; nr += (l->flags & SNFB_LF_BND_REVERSE) != 0; }
            nf = g.sum(nf); nr = g.sum(nr);
            g.sync();
            sort1(g, w, m);
            const long long mp = center_sorted(g, w, m, sA, sB);
            bnd_contig = best; bnd_pos = (int)mp; bnd_first = nf > m - nf; bnd_rev = nr > m - nr;
            sort1(g, w2, m);
            nq = compact(g, m, sA, [&](int i) { return i == 0 || w2[i] != w2[i - 1]; });
            for (int i = tid; i < nq; i += nthr) w[i] = w2[sA[i]];
            g.sync();
            for (int i = tid; i < nq; i += nthr) w2[i] = w[i];
            g.sync();
            support = nq; nfinal = m;
        }
        // ---- candidate record (without its place in the output, which k_emit_cands assigns)
        const uint32_t st0 = lo + (uint32_t)slo;          // staging offset of this sub-cluster's leads and names
        int nstr_f = 0, nstr_r = 0; long long ninl = 0;
        for (int i = tid; i < nfinal; i += nthr) {
            const uint32_t mi = SUB_ML(i); snfb_lead X = L[sl[i]];
            X.svlen = ml_svlen[mi];
            if (ml_has[mi]) { X.flags |= SNFB_LF_HAS_SEQ; X.seq_len = ml_seqlen[mi]; } else { X.flags &= ~SNFB_LF_HAS_SEQ; X.seq_len = 0; X.seq_off = -1; }
            extract::store_lead(b.st_leads + st0 + i, X);
            b.st_plo[st0 + i] = lo + ml_plo[mi]; b.st_pn[st0 + i] = ml_pn[mi];
            if (X.flags & SNFB_LF_REVERSE) nstr_r = 1; else nstr_f = 1;
            w[i] = SNFB_LF_SOURCE(X.flags) == SNFB_SRC_INLINE ? X.qname_hash : 0xffffffffffffffffull;     // inline names first after the sort
            ninl += SNFB_LF_SOURCE(X.flags) == SNFB_SRC_INLINE;
        }
        nstr_f = g.sum(nstr_f) > 0; nstr_r = g.sum(nstr_r) > 0; ninl = g.sum(ninl);
        for (int i = tid; i < nq; i += nthr) b.st_rn[st0 + i] = w2[i];
        g.sync();
        sort1(g, w, nfinal);
        const int support_inline = count_distinct_sorted(g, w, (int)ninl);
        g.sync();
        // phase aggregates: reads_phases = {read_id: (hap, phase_set)}, the last lead of a record wins (postprocessing.py:626-654)
        for (int i = tid; i < nfinal; i += nthr) w[i] = ((uint64_t)SUB_LEAD(i).rec << 32) | (uint32_t)i;
        g.sync();
        sort1(g, w, nfinal);
        long long hc0 = 0, hc1 = 0, hc2 = 0;
        const int np = compact(g, nfinal, sA, [&](int i) { return !(i + 1 < nfinal && (w[i + 1] >> 32) == (w[i] >> 32)); });
        for (int i = tid; i < np; i += nthr) {
            const snfb_lead* l = &SUB_LEAD((uint32_t)w[sA[i]]);
            const bool bnd = lf_type(l->flags) == SNFB_BND; const int h = bnd ? 0 : (int)SNFB_LF_HAP(l->flags);
            hc0 += h == 0; hc1 += h == 1; hc2 += h == 2;
            const snfb_rec* r = &b.rec[l->rec]; const bool isnull = bnd || !(r->aux_flags & SNFB_AUX_PS);
            w2[i] = isnull ? 0xffffffffffffffffull : bias64(r->ps);
        }
        hc0 = g.sum(hc0); hc1 = g.sum(hc1); hc2 = g.sum(hc2);
        g.sync();
        sort1(g, w2, np);
        if (tid == 0) {
            snfb_cand cd; memset(&cd, 0, sizeof cd);
            cd.task = task; cd.svtype = svtype; cd.pos = (int)svstart; cd.end = (int)svend; cd.svlen = (int)svlen; cd.support = (int)support;
            cd.qual = (int)__ddiv_rn((double)mq, (double)ns); cd.precise = precise; cd.fwd = (int)fwd; cd.rev = (int)(ns - fwd);
            cd.stdev_pos = sd_pos; cd.stdev_len = sd_len; cd.support_long = (int)support_long; cd.nm_mean = nm_mean;
            cd.sa_count = (int)sa; cd.sa_total = (int)(ns + nlong);
            if (svtype == SNFB_DEL) cd.support_sa = (int)nsplit;
            cd.bnd_mate_contig = bnd_contig; cd.bnd_mate_pos = bnd_pos; cd.bnd_is_first = bnd_first; cd.bnd_is_reverse = bnd_rev;
            { const uint32_t bi = b.kb_bin[kf]; for (int h = 0; h < 3; ++h) cd.hap_counts[h] = (int)b.bin_hap[(size_t)bi * 3 + h]; }   // REF part is filled by k_coverage
            cd.cluster_seed = b.kb_seed[kf]; cd.resplit_bin = t_bin[j];
            cd.n_strands = nstr_f + nstr_r; cd.support_inline = support_inline;
            cd.lead_off = (int)st0; cd.lead_n = nfinal; cd.long_off = nq /* staged names */; cd.long_n = (has_long && svtype != SNFB_BND) ? nlong : 0; cd.alt_off = -1; cd.alt_len = 0;
            const long long hc[3] = { hc0, hc1, hc2 };
            int ht = 0; for (int h = 1; h < 3; ++h) if (hc[h] > 0 && hc[h] >= hc[ht]) ht = h;
            cd.hp_top = ht; cd.hp_support = (int)hc[ht]; cd.hp_other = (int)(hc0 + hc1 + hc2 - hc[ht]);
            long bc = 0; uint64_t bv = 0; bool have = false; long nonnull = 0;
            for (long i = 0; i < np;) { long q = i; while (q < np && w2[q] == w2[i]) ++q; const long cnt = q - i; const bool isnull = w2[i] == 0xffffffffffffffffull; if (!isnull) nonnull += cnt;
                bool gt;
                if (!have) gt = true; else if (cnt != bc) gt = cnt > bc; else { const bool bn = bv == 0xffffffffffffffffull; if (isnull != bn) gt = isnull; else gt = cmp_decstr(unbias64(w2[i]), unbias64(bv)) > 0; }
                if (gt) { bc = cnt; bv = w2[i]; have = true; } i = q; }
            cd.ps_top_null = bv == 0xffffffffffffffffull; cd.ps_top = cd.ps_top_null ? 0 : (int)unbias64(bv); cd.ps_support = (int)bc; cd.ps_other = (int)(nonnull - (cd.ps_top_null ? 0 : bc));
            b.cand_tmp[sidx] = cd; b.sub_valid[sidx] = 1;
        }
        ++nvalid; nlead_out += (uint32_t)nfinal + ((has_long && svtype != SNFB_BND) ? (uint32_t)nlong : 0u); nrn_out += (uint32_t)support;
        g.sync();
        #undef SUB_ML
        #undef SUB_LEAD
    }
    #undef ML_LEAD
    if (tid == 0) { b.cl_nsub[c] = (uint32_t)nsub; b.cl_nvalid[c] = nvalid; b.cl_nlead[c] = nlead_out; b.cl_nrn[c] = nrn_out; }
}

// workspace carved out of a shared-memory region: leads | khi | klo | NU32 arrays of `cap` entries
__device__ __forceinline__ coop::WS smem_ws(uint8_t* base, int cap) {
    coop::WS ws; ws.L = reinterpret_cast<const snfb_lead*>(base);
    ws.khi = reinterpret_cast<uint64_t*>(base + (size_t)cap * 64); ws.klo = ws.khi + cap;
    uint32_t* u = reinterpret_cast<uint32_t*>(ws.klo + cap);
    #pragma unroll
    for (int k = 0; k < coop::NU32; ++k) ws.u[k] = u + (size_t)k * cap;
    return ws;
}
__host__ __device__ constexpr size_t ws_bytes(int cap) { return (size_t)cap * (64 + 16 + 4 * coop::NU32); }

// one warp per cluster, the cluster's leads staged in the warp's slice of shared memory.  Two instantiations: clusters of at most
// SMALL_CAP leads (the bulk: 8 warps per block, 4 blocks per SM) and the mid-sized ones up to WARP_CAP from a list.
template <int CAP, int WARPS> struct CwCfg { static constexpr size_t smem = WARPS * ws_bytes(CAP) + 64; };
template <int CAP, int WARPS, bool LIST>
__global__ void __launch_bounds__(WARPS * 32, LIST ? 1 : 4) k_cluster_warp(const __grid_constant__ B b) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = lane_id();
    uint8_t* base = smem + (size_t)warp * ws_bytes(CAP);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + WARPS * ws_bytes(CAP)) + warp;
    const coop::WS ws = smem_ws(base, CAP);
    if (lane == 0) { coop::mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncwarp();
    unsigned phase = 0;
    const unsigned long long n_items = LIST ? b.ctr->n_mid : b.ctr->n_clusters;
    const unsigned long long nw = (unsigned long long)gridDim.x * WARPS;
    coop::WarpG g;
    // the dense kernel takes clusters from a queue (their cost varies with their size), asking for the next one before working on this one
    unsigned long long q = LIST ? (unsigned long long)blockIdx.x * WARPS + warp : __shfl_sync(FULL, lane == 0 ? atomicAdd(&b.ctr->n_small_taken, 1ULL) : 0ULL, 0);
    for (; q < n_items; ) {
        unsigned long long next = 0;
        if (LIST) next = q + nw; else if (lane == 0) next = atomicAdd(&b.ctr->n_small_taken, 1ULL);
        const uint32_t c = LIST ? b.mid_list[q] : (uint32_t)q;
        const uint32_t kf = b.cl_first[c], kl_ = b.cl_last[c];
        const uint32_t lo = b.kb_lead_off[kf], n = b.kb_lead_off[kl_] + b.kb_lead_n[kl_] - lo;
        if (LIST || n <= (uint32_t)CAP) {                     // larger ones: the list kernels take them
            __syncwarp();                                     // the previous cluster's reads of the staged leads are done
            if (lane == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                coop::mbar_expect_tx(bar, n * 64u); coop::bulk_g2s(base, b.kleads + lo, n * 64u, bar);
            }
            coop::mbar_wait(bar, phase); phase ^= 1u;
            process_cluster(g, b, c, ws);
        }
        q = LIST ? next : __shfl_sync(FULL, next, 0);
    }
}
constexpr int CWS_WARPS = 8, CWM_WARPS = 4;
constexpr int CB_THREADS = 256;
constexpr size_t CB_SMEM = ws_bytes(BLOCK_CAP) + 72 * 8 + 64;
// one block per cluster of more than WARP_CAP leads (from big_list)
__global__ void __launch_bounds__(CB_THREADS) k_cluster_block(const __grid_constant__ B b) {
    extern __shared__ __align__(128) uint8_t smem[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem + ws_bytes(BLOCK_CAP));
    coop::BlockG g; g.red = reinterpret_cast<unsigned long long*>(bar + 1);
    if (threadIdx.x == 0) { coop::mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
    __syncthreads();
    unsigned phase = 0;
    const unsigned long long nbig = b.ctr->n_big;
    for (unsigned long long q = blockIdx.x; q < nbig; q += gridDim.x) {
        const uint32_t c = b.big_list[q];
        const uint32_t kf = b.cl_first[c], kl_ = b.cl_last[c];
        const uint32_t lo = b.kb_lead_off[kf], n = b.kb_lead_off[kl_] + b.kb_lead_n[kl_] - lo;
        __syncthreads();
        coop::WS ws;
        if (n <= (uint32_t)BLOCK_CAP) {
            ws = smem_ws(smem, BLOCK_CAP);
            if (threadIdx.x == 0) { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); coop::mbar_expect_tx(bar, n * 64u); coop::bulk_g2s(smem, b.kleads + lo, n * 64u, bar); }
            coop::mbar_wait(bar, phase); phase ^= 1u;
        } else {                                              // global workspace, private to the cluster's range of kept-lead space
            ws.L = b.kleads + lo; ws.khi = b.g_khi + lo; ws.klo = b.g_klo + lo;
            #pragma unroll
            for (int k = 0; k < coop::NU32; ++k) ws.u[k] = b.g_u32 + (size_t)k * b.n_bound + lo;
        }
        process_cluster(g, b, c, ws);
    }
}

// ---- compaction into reference emission order (task, svtype, cluster, sub-cluster): one warp per cluster copies its valid
//      sub-clusters' candidate records, leads (+ the cluster's leads_long) and read names to their final places
__global__ void __launch_bounds__(128) k_emit_cands(const __grid_constant__ B b) {
    const unsigned long long ncl = b.ctr->n_clusters;
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const int lane = lane_id();
    for (unsigned long long c = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < ncl; c += nw) {
        if (b.cl_nvalid[c] == 0) continue;
        const uint32_t kf = b.cl_first[c]; const uint32_t lo = b.kb_lead_off[kf]; const uint32_t llo = b.kb_long_off[kf];
        uint32_t id = b.cl_cand_base[c], lout = b.cl_lead_base[c], rout = b.cl_rn_base[c];
        const uint32_t nsub = b.cl_nsub[c];
        for (uint32_t j = 0; j < nsub; ++j) {
            if (!b.sub_valid[lo + j]) continue;
            snfb_cand cd = b.cand_tmp[lo + j];
            const uint32_t st0 = (uint32_t)cd.lead_off; const int n = cd.lead_n, nq = cd.long_off, nl = cd.long_n;
            if (id >= b.cand_cap || (unsigned long long)lout + n + nl > b.cand_lead_cap || (unsigned long long)rout + cd.support > b.rn_cap) { if (lane == 0) atomicAdd(&b.ctr->scratch_overflow, 1ULL); ++id; lout += n + nl; rout += cd.support; continue; }
            // leads: 16 bytes per lane and step
            { const uint4* s = reinterpret_cast<const uint4*>(b.st_leads + st0); uint4* d = reinterpret_cast<uint4*>(b.cand_leads + lout);
              for (int i = lane; i < n * 4; i += 32) d[i] = s[i]; }
            { const uint4* s = reinterpret_cast<const uint4*>(b.klleads + llo); uint4* d = reinterpret_cast<uint4*>(b.cand_leads + lout + n);
              for (int i = lane; i < nl * 4; i += 32) d[i] = s[i]; }
            for (int i = lane; i < n; i += 32) { b.out_plo[lout + i] = b.st_plo[st0 + i]; b.out_pn[lout + i] = b.st_pn[st0 + i]; }
            for (int i = lane; i < nl; i += 32) { b.out_plo[lout + n + i] = NONE; b.out_pn[lout + n + i] = 0; }
            for (int i = lane; i < nq && i < cd.support; i += 32) b.rnames[rout + i] = b.st_rn[st0 + i];
            __syncwarp();
            if (lane == 0) {
                if (cd.svtype == SNFB_INS && cd.svlen >= b.cfg.long_ins_length && cd.support > nq) {
                    // union with leads_long: append the extra hashes, then keep the list sorted (rare)
                    int o = nq < cd.support ? nq : cd.support;
                    for (int i = 0; i < nl && o < cd.support; ++i) { const uint64_t h = b.klleads[llo + i].qname_hash; bool dup = false; for (int q = 0; q < o; ++q) if (b.rnames[rout + q] == h) { dup = true; break; } if (!dup) b.rnames[rout + o++] = h; }
                    hsort1(b.rnames + rout, o);
                }
                cd.lead_off = (int)lout; cd.long_off = (int)(lout + n);
                b.cand[id] = cd; b.rn_off_out[id] = rout;
            }
            ++id; lout += n + nl; rout += cd.support;
        }
    }
}

// coverage restricted by haplotype at one position: reads with start <= p < end (leadprov.py:510).
// Warp-cooperative: records are coordinate sorted, so the covering reads start inside
// (p - longest reference span, p]; the lanes split that window.
__device__ inline void cover_count_warp(const B& b, int t, long long p, uint32_t out[3]) {
    out[0] = out[1] = out[2] = 0;
    const uint32_t lo = b.task_first[t], hi = b.task_last[t];
    if (lo >= hi) return;
    uint32_t a = lo, z = hi;                     // first record with pos > p
    while (a < z) { uint32_t mid = a + ((z - a) >> 1); if ((long long)b.rec_pos[mid] <= p) a = mid + 1; else z = mid; }
    const long long span = b.task_maxspan[t];
    uint32_t c0 = 0, c1 = 0, c2 = 0;
    for (long long i = (long long)a - 1 - lane_id(); i >= (long long)lo; i -= 32) {
        const long long ps = b.rec_pos[i]; if (ps + span <= p) break;
        const uint8_t f = b.rec_flags[i];
        if ((f & extract::RF_PASS) && (long long)b.rec_end[i] > p) { const int h = (f >> 2) & 3; c0 += h == 0; c1 += h == 1; c2 += h == 2; }
    }
    out[0] = __reduce_add_sync(FULL, c0); out[1] = __reduce_add_sync(FULL, c1); out[2] = __reduce_add_sync(FULL, c2);
}
__device__ inline void cov_at_warp(const B& b, int t, long long idx, int* out) {     // numpy indexing of the uint16 coverage vector
    const long long L = b.task[t].contig_len;
    if (idx < 0) idx += L;
    if (idx < 0 || idx >= L) return;             // IndexError: the field keeps its default 0
    if (b.mask) {                                 // _mask_N_coverage: positions inside a reference 'N' run read 0 (leadprov.py:439)
        uint32_t lo = b.mask_task_off[t], hi = b.mask_task_off[t + 1];
        while (lo < hi) { const uint32_t mid = lo + ((hi - lo) >> 1); if ((long long)b.mask[2 * mid + 1] <= idx) lo = mid + 1; else hi = mid; }
        if (lo < b.mask_task_off[t + 1] && (long long)b.mask[2 * lo] <= idx && idx >= b.task[t].start && idx < b.task[t].end) { *out = 0; return; }   // the mask is fetched per region (leadprov.py:436-438)
    }
    uint32_t c[3]; cover_count_warp(b, t, idx, c); *out = (int)((c[0] + c[1] + c[2]) & 0xffffu);
}

// what postprocessing.coverage reads of one call
struct CovSv { int task, svtype; long long pos, svlen; int bnd_is_first; };
// postprocessing.coverage's probe positions (postprocessing.py:69-130) of call i of a list ordered by task: p = upstream, start, center,
// end, downstream.  `at(j)` returns call j; `prev(i)` the index of the last non-BND call of i's task before i, or -1.  A BND takes the
// `end` left over from that call; with none the reference raises UnboundLocalError, and this returns false with end = start.  Any
// svtype other than INS / BND (also an unsupported one, < 0) takes the interval branch.
template <class At, class Prev> __device__ inline bool cov_probes(long long i, At at, Prev prev, long long bs, long long ud, long long p[5]) {
    const CovSv c = at(i); long long start = c.pos, end; bool ok = true;
    if (c.svtype == SNFB_INS) end = start + 1;
    else if (c.svtype == SNFB_BND) {
        if (c.bnd_is_first) start -= 1;
        const long long j = prev(i);
        if (j >= 0) { const CovSv q = at(j); end = q.svtype == SNFB_INS ? q.pos + 1 : q.pos + (q.svlen < 0 ? -q.svlen : q.svlen); }
        else { end = start; ok = false; }
    } else end = c.pos + (c.svlen < 0 ? -c.svlen : c.svlen);
    if (c.svtype == SNFB_INS || c.svtype == SNFB_BND) { p[1] = start - bs; p[2] = start; p[3] = end + bs; }
    else { p[1] = start; p[2] = (long long)__ddiv_rn((double)(start + end), 2.0); p[3] = end - bs; }
    p[0] = start - ud; p[4] = end + ud;
    return ok;
}

// postprocessing.coverage (postprocessing.py:69-130) including the `end` that leaks from the previous call,
// plus the hap-REF counts of the cluster's first bin (cluster.py:255-260).  One warp per candidate.
__global__ void k_coverage(B b) {
    const unsigned long long nc = b.ctr->n_cand < b.cand_cap ? b.ctr->n_cand : b.cand_cap;
    const long long bs = b.cfg.coverage_binsize, ud = (long long)b.cfg.coverage_binsize * b.cfg.coverage_updown_bins;
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const auto at = [&](long long j) { const snfb_cand& q = b.cand[j]; return CovSv{ q.task, q.svtype, q.pos, q.svlen, q.bnd_is_first }; };
    const auto prev = [&](long long i) {          // candidates of a task hold few BNDs in a row: walk back
        const int t = b.cand[i].task; long long j = i - 1; while (j >= 0 && b.cand[j].task == t && b.cand[j].svtype == SNFB_BND) --j;
        return j >= 0 && b.cand[j].task == t ? j : -1ll; };
    for (unsigned long long i = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nc; i += nw) {
        snfb_cand* c = &b.cand[i]; const int t = c->task;
        long long p[5];
        if (!cov_probes((long long)i, at, prev, bs, ud, p) && lane_id() == 0) atomicAdd(&b.ctr->soft_errors, 1ULL);
        int v[5] = { 0, 0, 0, 0, 0 };          // upstream, start, center, end, downstream
        for (int k = 0; k < 5; ++k) cov_at_warp(b, t, p[k], &v[k]);
        uint32_t hr[3]; const int cb = b.cfg.cluster_binsize; cover_count_warp(b, t, (long long)(c->cluster_seed / cb) * cb + cb - 1, hr);
        if (lane_id() == 0) {
            c->cov_upstream = v[0]; c->cov_start = v[1]; c->cov_center = v[2]; c->cov_end = v[3]; c->cov_downstream = v[4];
            for (int h = 0; h < 3; ++h) c->hap_counts[3 + h] = (int)(hr[h] > 65535u ? 65535u : hr[h]);
        }
    }
}

// run m of task t as the coverage vector sees it: the mask is fetched per region (leadprov.py:436-438) and slices clip to [0, L)
__device__ inline void mask_run(const B& b, int t, unsigned long long m, long long* a, long long* e) {
    const long long L = b.task[t].contig_len;
    *a = b.mask[2 * m]; *e = b.mask[2 * m + 1];
    if (*a < b.task[t].start) *a = b.task[t].start; if (*e > b.task[t].end) *e = b.task[t].end; if (*a < 0) *a = 0; if (*e > L) *e = L;
}
// the passing reads of task t that overlap [a, e): each lane visits its share and calls f(o0, o1) with the overlap, the read's end
// clipped to the contig as the coverage slice is (leadprov.py:510).  Records are coordinate sorted, so they start in (a - longest span, e).
template <class F> __device__ inline void pass_overlaps_warp(const B& b, int t, long long a, long long e, F f) {
    const uint32_t lo = b.task_first[t], hi = b.task_last[t];
    if (a >= e || lo >= hi) return;
    const long long L = b.task[t].contig_len;
    uint32_t x = lo, z = hi;                     // first record with pos >= e
    while (x < z) { const uint32_t mid = x + ((z - x) >> 1); if ((long long)b.rec_pos[mid] < e) x = mid + 1; else z = mid; }
    const long long span = b.task_maxspan[t];
    for (long long i = (long long)x - 1 - lane_id(); i >= (long long)lo; i -= 32) {
        const long long ps = b.rec_pos[i]; if (ps + span <= a) break;
        if (!(b.rec_flags[i] & extract::RF_PASS)) continue;
        long long re = b.rec_end[i]; if (re > L) re = L;
        const long long o0 = ps > a ? ps : a, o1 = re < e ? re : e;
        if (o1 > o0) f(o0, o1);
    }
}

// _mask_N_coverage for the contig mean: subtract the read bases that fall inside reference 'N' runs.  One warp per run.
__global__ void k_mask_bp(B b, const uint32_t* __restrict__ mask_task, uint32_t n_mask, unsigned long long* task_cov_bp) {
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long m = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; m < n_mask; m += nw) {
        const int t = (int)mask_task[m]; long long a, e; mask_run(b, t, m, &a, &e);
        unsigned long long sum = 0;
        pass_overlaps_warp(b, t, a, e, [&](long long o0, long long o1) { sum += (unsigned long long)(o1 - o0); });
        #pragma unroll
        for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(FULL, sum, o);
        if (lane_id() == 0 && sum) atomicAdd(&task_cov_bp[t], 0ull - sum);
    }
}

// _mask_N_coverage for the SNF coverage means (snfb_coverage_bins): the same read bases subtracted from the `binsize`-base bin sums of
// task t that they fall in.  One warp per run.
__global__ void k_mask_bins(B b, int t, int binsize, unsigned long long* acc) {
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const uint32_t m0 = b.mask_task_off[t], m1 = b.mask_task_off[t + 1];
    for (unsigned long long m = m0 + (((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5); m < m1; m += nw) {
        long long a, e; mask_run(b, t, m, &a, &e);
        pass_overlaps_warp(b, t, a, e, [&](long long o0, long long o1) {
            for (long long bb = o0 / binsize; bb <= (o1 - 1) / binsize; ++bb) {
                const long long s0 = bb * binsize, s1 = s0 + binsize;
                const long long x0 = o0 > s0 ? o0 : s0, x1 = o1 < s1 ? o1 : s1;
                atomicAdd(&acc[bb], 0ull - (unsigned long long)(x1 - x0));
            }
        });
    }
}

}  // namespace cluster
