// population.cuh — population allele frequencies of combined calls (--combine-population):
//   PopulationSNF.get_population_AF   snfp.py:131-155   (the variant list of the call's (contig, block, svtype), strictly smallest distance wins)
//   PopulationVariant.match           snfp.py:91-107    (position / length test, then for INS the alignment test)
// The population table is sorted once by (contig, block, svtype) with the stable radix sort of prims.cuh, so each key's variants stay in
// list order.  A query is one warp: a binary search finds its key range, the lanes stride over it.
#pragma once
#include "common.cuh"
#include "edit_distance.cuh"

namespace population {

// (contig, svtype, block): contig < 2^24, svtype 0..4, the block start biased to unsigned order.  A variant whose contig is not among
// the run's contigs gets the contig n_contig, past the last one the table knows; k_pop_match answers a query on a contig >= n_contig
// with no match, without a search.
__device__ __forceinline__ uint64_t key_of(uint32_t contig, int32_t svtype, int32_t block) {
    return ((uint64_t)contig << 35) | ((uint64_t)(uint32_t)svtype << 32) | (uint64_t)((uint32_t)block ^ 0x80000000u);
}

__global__ void k_pop_keys(const int32_t* __restrict__ contig, const int32_t* __restrict__ block, const int32_t* __restrict__ svtype, uint32_t n,
                           uint32_t absent, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        key[i] = key_of(contig[i] < 0 ? absent : (uint32_t)contig[i], svtype[i], block[i]); val[i] = i;
    }
}
// the columns the match reads, in sorted order
__global__ void k_pop_gather(const uint32_t* __restrict__ val, uint32_t n, const int32_t* __restrict__ pos, const int32_t* __restrict__ svlen,
                             const unsigned long long* __restrict__ alt_off, const uint32_t* __restrict__ alt_len,
                             int32_t* __restrict__ o_pos, int32_t* __restrict__ o_svlen, unsigned long long* __restrict__ o_alt_off, uint32_t* __restrict__ o_alt_len) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
        const uint32_t v = val[j];
        o_pos[j] = pos[v]; o_svlen[j] = svlen[v]; o_alt_off[j] = alt_off[v]; o_alt_len[j] = alt_len[v];
    }
}

struct P {
    // the resident table, sorted by key; idx: the variant's file-order index
    const uint64_t* key; const uint32_t* idx; const int32_t* pos; const int32_t* svlen; const unsigned long long* alt_off; const uint32_t* alt_len;
    const uint8_t* alt; uint32_t n_var, n_contig;      // n_contig: 1 + the largest contig index of the table
    // one batch of queries
    const int32_t* q_contig; const int32_t* q_svtype; const int32_t* q_pos; const int32_t* q_svlen;
    const uint8_t* q_alt; const unsigned long long* q_alt_off; const uint32_t* q_alt_len; uint32_t n_q;
    int combine_match, combine_match_max, block_size; double pctseq;
    int8_t* hs; uint32_t max_alt;      // per warp, max_alt bytes of edit-distance carries
    int32_t* best;
};

__device__ __forceinline__ uint32_t lower_bound(const uint64_t* key, uint32_t n, uint64_t k) {
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (key[mid] < k) lo = mid + 1; else hi = mid; }
    return lo;
}

__device__ __forceinline__ long long iabs64(long long v) { return v < 0 ? -v : v; }

// (dist, slot) of the lanes' candidates -> the warp's first minimum; INT64_MAX / 0xffffffff when no lane has one
__device__ __forceinline__ void warp_min(long long& bd, uint32_t& bi) {
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const long long od = __shfl_xor_sync(FULL, bd, o); const uint32_t oi = __shfl_xor_sync(FULL, bi, o);
        if (od < bd || (od == bd && oi < bi)) { bd = od; bi = oi; }
    }
}

__global__ void __launch_bounds__(128) k_pop_match(const P p) {
    const int lane = lane_id();
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    int8_t* hs = p.hs + (size_t)w * p.max_alt;
    for (uint32_t q = w; q < p.n_q; q += nw) {
        const int32_t qc = p.q_contig[q];
        int32_t result = -1;
        if (qc >= 0 && (uint32_t)qc < p.n_contig) {
            const int32_t qpos = p.q_pos[q], qt = p.q_svtype[q];
            // str(int(pos / snf_block_size) * snf_block_size): C truncation, as plan_bin in combine.cuh argues
            const uint64_t k = key_of((uint32_t)qc, qt, (qpos / p.block_size) * p.block_size);
            const uint32_t lo = lower_bound(p.key, p.n_var, k), hi = lower_bound(p.key, p.n_var, k + 1);
            const long long qlen = iabs64((long long)p.q_svlen[q]);
            const bool align = qt == 0 && p.pctseq != 0.0;            // 0: INS
            // the position / length test of one slot: its distance, or -1 when rejected
            auto dist_of = [&](uint32_t j) -> long long {
                const long long plen = iabs64((long long)p.svlen[j]);
                const long long d = iabs64((long long)p.pos[j] - (long long)qpos) + iabs64(plen - qlen);
                const double thr = __dmul_rn((double)p.combine_match, __dsqrt_rn((double)(plen < qlen ? plen : qlen)));
                return ((double)d > thr || d > (long long)p.combine_match_max) ? -1 : d;
            };
            long long bd = INT64_MAX; uint32_t bi = 0xffffffffu; bool zero_len = false;
            for (uint32_t j = lo + lane; j < hi; j += 32) {
                const long long d = dist_of(j);
                if (d < 0) continue;
                if (align && p.svlen[j] == 0) zero_len = true;
                if (d < bd) { bd = d; bi = j; }           // lanes visit their slots in ascending order: the first of equal distances stays
            }
            warp_min(bd, bi);
            if (align && __any_sync(FULL, zero_len)) {
                // the reference divides by this variant's svlen whatever the other variants do: its worker stops on the division
                result = -2;
            } else if (!align) {
                if (bi != 0xffffffffu) result = (int32_t)p.idx[bi];
            } else {
                // Variants that pass the position test are aligned in ascending (distance, list index) order and the first that also passes
                // the alignment test is the answer.  The reference keeps the strictly smallest distance over the whole list, ties to the
                // earlier variant, among the variants that pass both tests; every variant visited before the first to pass has a smaller
                // distance, or the same distance and a smaller list index, and failed, so none of them can be the reference's answer, and
                // every variant after it is no better.  The warp aligns one pair where the reference aligns every candidate.
                while (bi != 0xffffffffu) {
                    const long long plen = (long long)p.svlen[bi];
                    const int d = edit_distance_warp(p.alt + p.alt_off[bi], (int)p.alt_len[bi], p.q_alt + p.q_alt_off[q], (int)p.q_alt_len[q], hs);
                    if (!(__ddiv_rn((double)(plen - d), (double)plen) <= p.pctseq)) { result = (int32_t)p.idx[bi]; break; }
                    // the next candidate: the smallest (distance, slot) above the one that failed
                    const long long fd = bd; const uint32_t fi = bi;
                    bd = INT64_MAX; bi = 0xffffffffu;
                    for (uint32_t j = lo + lane; j < hi; j += 32) {
                        const long long d = dist_of(j);
                        if (d < 0 || d < fd || (d == fd && j <= fi)) continue;
                        if (d < bd) { bd = d; bi = j; }
                    }
                    warp_min(bd, bi);
                }
            }
        }
        if (lane == 0) p.best[q] = result;
        __syncwarp();
    }
}

}  // namespace population
