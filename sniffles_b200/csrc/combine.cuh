// combine.cuh — SURVEY §8(f)1: the grouping of multi-sample combine mode.
//   cluster.resolve_block_groups      cluster.py:356-390   (greedy nearest-group assignment, candidates by support)
//   SVGroup.from_candidate/add_candidate  sv.py:265-321    (running means, updated with the reference's operation order)
//   CombineTask.execute, the chunk loop   parallel.py:518-563 (coverage of non-included samples, keep / call split)
// The grouping is sequential along one (task, svtype) chain — the groups kept at the end of a chunk are the first groups the next chunk
// sees, across blocks — and independent between chains: one warp per chain, lanes over the active groups (distance + first-minimum
// reduction) and over the samples (coverage update).  All float decisions are in double with explicit _rn operations, in the
// reference's order.
#pragma once
#include "common.cuh"
#include "edit_distance.cuh"

namespace combine {

struct P {
    const snfb_combine_chain* chains; const snfb_combine_chunk* chunks; uint32_t n_chain, n_chunk, n_cand, n_samples, words;
    const int32_t* pos; const int32_t* svlen; const uint32_t* sample; const int32_t* mate_contig; const int32_t* mate_pos;
    const long long* block_start; const int32_t* cov; int bins_per_block, cov_binsize;
    int combine_match, combine_match_max, cluster_merge_bnd, separate_intra, overlap_abs;
    // per group slot (slot = chain.cand_off + local group id; a chain never has more groups than candidates)
    double* g_pos; double* g_len; double* g_mate; uint32_t* g_n; int32_t* g_mc; uint32_t* g_incl;   // g_incl: [slot][words] sample bitset
    uint32_t* act;                                 // [n_cand] active group list of the chain, at chain.cand_off
    uint32_t* cand_group; int32_t* emit_chunk; uint32_t* emit_ord; int32_t* cov_non;
    unsigned int* next_chain;
    // group.align_call (sv.py:282-292): pctseq > 0 switches it on.  alt: the candidates' ALT strings; g_first: the candidate that opened the group;
    // ex_stamp[g] == c + 1: group g failed the alignment test for candidate c; hs: per warp, max_alt bytes of carries between passes
    double pctseq; const uint8_t* alt; const unsigned long long* alt_off; const uint32_t* alt_len; uint32_t* g_first; uint32_t* ex_stamp; int8_t* hs; uint32_t max_alt;
};

__global__ void __launch_bounds__(128) k_combine(const P p) {
    const int lane = lane_id();
    for (;;) {
        uint32_t ci = 0; if (lane == 0) ci = atomicAdd(p.next_chain, 1u);
        ci = __shfl_sync(FULL, ci, 0);
        if (ci >= p.n_chain) break;
        const snfb_combine_chain ch = p.chains[ci];
        uint32_t* act = p.act + ch.cand_off; uint32_t n_act = 0, n_groups = 0;
        const uint32_t W = p.words;
        for (uint32_t k = 0; k < ch.n_chunk; ++k) {
            const snfb_combine_chunk ck = p.chunks[ch.chunk_off + k];
            // ---- resolve_block_groups over the chunk's candidates (already in support order)
            for (uint32_t c = ck.cand_off; c < ck.cand_off + ck.n_cand; ++c) {
                const int cpos = p.pos[c], clen = p.svlen[c]; const uint32_t smp = p.sample[c];
                const int cmc = ch.is_bnd ? p.mate_contig[c] : 0, cmp = ch.is_bnd ? p.mate_pos[c] : 0;
                const double alen = (double)(clen < 0 ? -(long long)clen : (long long)clen);
                double bd; uint32_t bi;
                for (;;) {
                    bd = __longlong_as_double(0x7ff0000000000000ll); bi = 0xffffffffu;
                    for (uint32_t a0 = 0; a0 < n_act; a0 += 32) {
                        const uint32_t a = a0 + lane;
                        if (a < n_act) {
                            const uint32_t g = act[a]; const double gp = p.g_pos[g];
                            double dist; bool ok;
                            if (ch.is_bnd) {
                                dist = __dadd_rn(fabs(__dsub_rn(gp, (double)cpos)), fabs(__dsub_rn(p.g_mate[g], (double)cmp)));
                                ok = dist <= (double)(p.cluster_merge_bnd * 2) && p.g_mc[g] == cmc;
                            } else {
                                const double gl = fabs(p.g_len[g]);
                                dist = __dadd_rn(fabs(__dsub_rn(gp, (double)cpos)), fabs(__dsub_rn(gl, alen)));
                                const double minlen = gl < alen ? gl : alen;
                                ok = minlen > 0.0 && dist <= __dmul_rn((double)p.combine_match, __dsqrt_rn(minlen)) && dist <= (double)p.combine_match_max && p.ex_stamp[g] != c + 1u;
                            }
                            if (ok && dist < bd && (!p.separate_intra || !((p.g_incl[(size_t)g * W + (smp >> 5)] >> (smp & 31)) & 1u))) { bd = dist; bi = a; }
                        }
                    }
                    // first minimum in list order: smallest distance, then smallest list index
                    #pragma unroll
                    for (int o = 16; o > 0; o >>= 1) {
                        const double od = __shfl_xor_sync(FULL, bd, o); const uint32_t oi = __shfl_xor_sync(FULL, bi, o);
                        if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
                    }
                    if (bi == 0xffffffffu || ch.is_bnd || !(p.pctseq != 0.0)) break;
                    // the nearest eligible group must also align (only groups that pass can become the best one, so testing them nearest first is the reference's result)
                    const uint32_t g = act[bi], fc = p.g_first[g];
                    const int d = edit_distance_warp(p.alt + p.alt_off[fc], (int)p.alt_len[fc], p.alt + p.alt_off[c], (int)p.alt_len[c], p.hs + (size_t)(blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * p.max_alt);
                    const double lm = p.g_len[g];
                    if (__ddiv_rn(__dsub_rn(lm, (double)d), lm) > p.pctseq) break;
                    if (lane == 0) p.ex_stamp[g] = c + 1u;
                    __syncwarp();
                }
                uint32_t g;
                if (bi == 0xffffffffu) {                          // SVGroup.from_candidate
                    g = ch.cand_off + n_groups;
                    if (lane == 0) {
                        p.g_pos[g] = (double)cpos; p.g_len[g] = alen; p.g_mate[g] = (double)cmp; p.g_mc[g] = cmc; p.g_n[g] = 1u; act[n_act] = g; p.g_first[g] = c; p.ex_stamp[g] = 0u;
                        p.emit_chunk[g] = (int32_t)p.n_chunk; p.emit_ord[g] = 0u;
                    }
                    for (uint32_t w = lane; w < W; w += 32) p.g_incl[(size_t)g * W + w] = (w == (smp >> 5)) ? (1u << (smp & 31)) : 0u;
                    for (uint32_t s = lane; s < p.n_samples; s += 32) p.cov_non[(size_t)g * p.n_samples + s] = -1;
                    ++n_groups; ++n_act;
                } else {                                          // SVGroup.add_candidate
                    g = act[bi];
                    if (lane == 0) {
                        const uint32_t n = p.g_n[g]; const double dn = (double)n, dn1 = (double)(n + 1u);
                        p.g_pos[g] = __ddiv_rn(__dadd_rn(__dmul_rn(p.g_pos[g], dn), (double)cpos), dn1);
                        p.g_len[g] = __ddiv_rn(__dadd_rn(__dmul_rn(p.g_len[g], dn), alen), dn1);
                        if (ch.is_bnd) p.g_mate[g] = __ddiv_rn(__dadd_rn(__dmul_rn(p.g_mate[g], dn), (double)cmp), dn1);
                        p.g_n[g] = n + 1u;
                        p.g_incl[(size_t)g * W + (smp >> 5)] |= 1u << (smp & 31);
                    }
                }
                if (lane == 0) p.cand_group[c] = g;
                __syncwarp();
            }
            // ---- end of chunk: coverage of the samples a group does not include, then keep / call
            const double lim = fmax(__dmul_rn((double)ck.size, 0.5), (double)p.overlap_abs);
            uint32_t n_keep = 0, n_call = 0;
            for (uint32_t a0 = 0; a0 < n_act; a0 += 32) {
                const uint32_t a = a0 + lane; const bool v = a < n_act;
                const uint32_t g = v ? act[a] : 0u; const double gp = v ? p.g_pos[g] : 0.0;
                // coverage: the lanes of the warp take the samples of one group at a time
                for (uint32_t j = 0; j < 32u && a0 + j < n_act; ++j) {
                    const uint32_t gj = __shfl_sync(FULL, g, j); const double pj = __shfl_sync(FULL, gp, j);
                    const long long cb = (long long)__ddiv_rn(pj, (double)p.cov_binsize) * p.cov_binsize;
                    long long kbin = -1;
                    if (ck.cov_block >= 0) { const long long off = cb - p.block_start[ck.cov_block]; if (off >= 0 && off < (long long)p.bins_per_block * p.cov_binsize) kbin = off / p.cov_binsize; }
                    for (uint32_t s = lane; s < p.n_samples; s += 32) {
                        if ((p.g_incl[(size_t)gj * W + (s >> 5)] >> (s & 31)) & 1u) continue;
                        int cv = 0;
                        if (kbin >= 0) { const int t = p.cov[((size_t)ck.cov_block * p.n_samples + s) * p.bins_per_block + kbin]; if (t >= 0) cv = t; }
                        int32_t* d = &p.cov_non[(size_t)gj * p.n_samples + s]; if (cv > *d) *d = cv;
                    }
                }
                const bool keep = v && fabs(__dsub_rn(gp, (double)ck.curr_bin)) < lim;
                const unsigned km = __ballot_sync(FULL, keep), cm = __ballot_sync(FULL, v && !keep);
                __syncwarp();
                if (keep) act[n_keep + __popc(km & lanemask_lt())] = g;          // compaction in place: n_keep + rank <= a
                else if (v) { p.emit_chunk[g] = (int32_t)(ch.chunk_off + k); p.emit_ord[g] = n_call + __popc(cm & lanemask_lt()); }
                n_keep += __popc(km); n_call += __popc(cm);
                __syncwarp();
            }
            n_act = n_keep;
        }
        // groups still kept at the end of the chain are called last, in list order (parallel.py:565-566)
        for (uint32_t a = lane; a < n_act; a += 32) { const uint32_t g = act[a]; p.emit_chunk[g] = (int32_t)p.n_chunk; p.emit_ord[g] = a; }
        for (uint32_t g = ch.cand_off + n_groups + lane; g < ch.cand_off + ch.n_cand; g += 32) p.emit_chunk[g] = -1;     // unused slots
        __syncwarp();
    }
}

// ---- the chunk plan (parallel.py:484-527) over flat candidates, for snfb_combine_plan ----
// Flat candidates come in the reference's iteration order (task, block, svtype, sample, part, list position).  The kept ones are sorted
// stably on (task, svtype, block, bin) by two LSD radix sorts (bin first): within one (task, block, svtype) segment that is the order in
// which the reference's bins dict hands them out.  One thread per segment then cuts the chunks, and a third stable sort on (chunk, support
// descending) gives each chunk the order of sorted(key=support, reverse=True) (cluster.py:361).  Segments of one (task, svtype) are
// consecutive after the sort: they form that chain.

// int(pos / bin_min) * bin_min: C's integer division truncates toward zero as int() does, and the double quotient of two int32 values
// lies at least 1 / bin_min from any integer it is not equal to, far more than its rounding error, so both truncate alike
__device__ __forceinline__ int32_t plan_bin(int32_t pos, int32_t bin_min) { return (pos / bin_min) * bin_min; }
__device__ __forceinline__ uint32_t biased(int32_t v) { return (uint32_t)v ^ 0x80000000u; }      // signed order as unsigned order

__global__ void k_plan_keep(const int32_t* __restrict__ support, uint32_t n, int32_t thr, uint32_t* __restrict__ keep) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) keep[i] = support[i] >= thr ? 1u : 0u;
}
// the kept candidates, in flat order, keyed by their bin
__global__ void k_plan_compact(const uint32_t* __restrict__ keep, const uint32_t* __restrict__ at, uint32_t n, const int32_t* __restrict__ pos, int32_t bin_min,
                               uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        if (keep[i]) { key[at[i]] = biased(plan_bin(pos[i], bin_min)); val[at[i]] = i; }
}
// (task, svtype, coverage row): rows are numbered in (task, block) order, so the row orders the blocks of a task
__global__ void k_plan_segkey(const uint32_t* __restrict__ val, uint32_t n, const uint32_t* __restrict__ task, const int32_t* __restrict__ svtype,
                              const uint32_t* __restrict__ row, uint64_t* __restrict__ key) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t v = val[j]; key[j] = ((uint64_t)task[v] << 35) | ((uint64_t)svtype[v] << 32) | row[v];
    }
}
// first position of each segment (same key) and of each chain (same task and svtype)
__global__ void k_plan_heads(const uint64_t* __restrict__ key, uint32_t n, uint32_t* __restrict__ seg_head, uint32_t* __restrict__ chain_head) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        seg_head[j] = (j == 0 || key[j] != key[j - 1]) ? 1u : 0u;
        chain_head[j] = (j == 0 || (key[j] >> 32) != (key[j - 1] >> 32)) ? 1u : 0u;
    }
}
__global__ void k_plan_seg_start(const uint32_t* __restrict__ seg_head, const uint32_t* __restrict__ seg_id, uint32_t n, uint32_t* __restrict__ seg_start) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) if (seg_head[j]) seg_start[seg_id[j]] = j;
}
// the chunk cut of one segment (parallel.py:518-527): bins are added whole; a chunk closes once it holds bin_max candidates (unless
// exhaustive) or at the segment's last bin.  Without chunk_off it counts the chunks of each segment; with it, it writes them and the chunk
// of every position.
__global__ void k_plan_cut(const uint32_t* __restrict__ seg_start, uint32_t n_seg, uint32_t n, const uint32_t* __restrict__ val, const int32_t* __restrict__ pos,
                           const uint64_t* __restrict__ key, int32_t bin_min, int32_t bin_max, int exhaustive, uint32_t* __restrict__ seg_nchunk,
                           const uint32_t* __restrict__ chunk_off, snfb_combine_chunk* __restrict__ chunks, uint32_t* __restrict__ chunk_of) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n_seg; s += gridDim.x * blockDim.x) {
        const uint32_t b = seg_start[s], e = s + 1 < n_seg ? seg_start[s + 1] : n;
        uint32_t k = chunk_off ? chunk_off[s] : 0u, nk = 0, c0 = b, nbins = 0;
        for (uint32_t j = b; j < e; ++j) {
            const int32_t bin = plan_bin(pos[val[j]], bin_min);
            if (j + 1 < e && plan_bin(pos[val[j + 1]], bin_min) == bin) continue;
            ++nbins;
            if ((!exhaustive && (int64_t)(j + 1 - c0) >= bin_max) || j + 1 == e) {
                if (chunk_off) {
                    chunks[k + nk] = snfb_combine_chunk{ (int32_t)c0, (int32_t)(j + 1 - c0), bin, (int32_t)(nbins * (uint32_t)bin_min), (int32_t)(uint32_t)key[b], 0 };
                    for (uint32_t q = c0; q <= j; ++q) chunk_of[q] = k + nk;
                }
                ++nk; c0 = j + 1; nbins = 0;
            }
        }
        if (!chunk_off) seg_nchunk[s] = nk;
    }
}
__global__ void k_plan_chains(const uint32_t* __restrict__ chain_head, const uint32_t* __restrict__ chain_id, const uint64_t* __restrict__ key, const uint32_t* __restrict__ chunk_of,
                              uint32_t n, snfb_combine_chain* __restrict__ chains) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
        if (chain_head[j]) chains[chain_id[j]] = snfb_combine_chain{ j, 0u, chunk_of[j], 0u, ((key[j] >> 32) & 7u) == 4u ? 1u : 0u, 0u };   // 4: BND
}
__global__ void k_plan_chain_len(snfb_combine_chain* __restrict__ chains, uint32_t n_chain, uint32_t n, uint32_t n_chunk) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_chain; c += gridDim.x * blockDim.x) {
        chains[c].n_cand = (c + 1 < n_chain ? chains[c + 1].cand_off : n) - chains[c].cand_off;
        chains[c].n_chunk = (c + 1 < n_chain ? chains[c + 1].chunk_off : n_chunk) - chains[c].chunk_off;
    }
}
// (chunk, support descending): a stable sort on it is sorted(chunk, key=support, reverse=True) inside every chunk
__global__ void k_plan_supkey(const uint32_t* __restrict__ val, const uint32_t* __restrict__ chunk_of, uint32_t n, const int32_t* __restrict__ support, uint64_t* __restrict__ key) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) key[j] = ((uint64_t)chunk_of[j] << 32) | (0xffffffffu - biased(support[val[j]]));
}
// the per-candidate columns of k_combine, in slot order
__global__ void k_plan_gather(const uint32_t* __restrict__ val, uint32_t n, const int32_t* __restrict__ pos, const int32_t* __restrict__ svlen, const uint32_t* __restrict__ sample,
                              const int32_t* __restrict__ mate_contig, const int32_t* __restrict__ mate_pos, const unsigned long long* __restrict__ alt_off, const uint32_t* __restrict__ alt_len,
                              int32_t* __restrict__ o_pos, int32_t* __restrict__ o_svlen, uint32_t* __restrict__ o_sample, int32_t* __restrict__ o_mc, int32_t* __restrict__ o_mp,
                              unsigned long long* __restrict__ o_alt_off, uint32_t* __restrict__ o_alt_len) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t v = val[j];
        o_pos[j] = pos[v]; o_svlen[j] = svlen[v]; o_sample[j] = sample[v]; o_mc[j] = mate_contig[v]; o_mp[j] = mate_pos[v];
        if (alt_off) { o_alt_off[j] = alt_off[v]; o_alt_len[j] = alt_len[v]; }
    }
}

// self-check: one warp per pair
__global__ void k_edit_selftest(const uint8_t* bytes, const unsigned long long* a_off, const uint32_t* a_len, const unsigned long long* b_off, const uint32_t* b_len, uint32_t n_pairs, int8_t* hs, uint32_t max_len, int* out) {
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t i = w; i < n_pairs; i += nw) {
        const int d = edit_distance_warp(bytes + a_off[i], (int)a_len[i], bytes + b_off[i], (int)b_len[i], hs + (size_t)w * max_len);
        if (lane_id() == 0) out[i] = d;
        __syncwarp();
    }
}

}  // namespace combine
