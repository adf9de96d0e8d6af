// bam_sort.cuh — a BAM sorted by coordinate (samtools sort's order), records moved on the device (snfb_sort_bam).
// The input streams through the same windows as the index build (bam_index.cuh: inflate + CRC, carry, the record chain), then:
//
//   k_keys      one thread per chain record: the sort key (tid' << 33 | (pos + 1) << 1 | reverse strand, tid' = n_ref for tid -1),
//               the record's length 4 + block_size and its global inflated offset.  The chain runs once; the bucket passes never run it.
//   (radix sort) the keys, stable, values = input ordinals
//   k_gather_len  sorted lengths (the host cuts the members from them: htslib's writer rule is sequential)
//   k_place     each record's output offset back by ordinal; the bucket it falls in; per input window, the range of buckets its records
//               fall in (a bucket pass re-reads only the windows whose range holds it)
//   k_scatter   one warp per record of a re-read window: the window's part of every record of the current bucket, into the bucket's buffer
//               (16-byte stores once the destination is aligned, funnel-shifted from aligned 4-byte loads)
// and the bucket's members go through the BGZF encoder (bgzf_write.cuh) with an explicit member table.
#pragma once
#include "common.cuh"
#include "ingest_core.h"

namespace bamsort {

using ingest::ld32u; using ingest::ld16u;

__global__ void k_keys(const uint8_t* __restrict__ R, const uint32_t* __restrict__ cand, const uint32_t* __restrict__ is_rec, const uint32_t* __restrict__ rec_idx,
                       uint32_t n, unsigned long long base, int n_ref, uint64_t* __restrict__ key, uint32_t* __restrict__ len, unsigned long long* __restrict__ src) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        if (!is_rec[i]) continue;
        const unsigned long long p = cand[i];
        const uint32_t bs = ld32u(R, p), flag = ld16u(R, p + 18);
        const int tid = (int)ld32u(R, p + 4), pos = (int)ld32u(R, p + 8);
        const uint64_t t = tid < 0 ? (uint64_t)n_ref : (uint64_t)tid;
        const uint32_t r = rec_idx[i];
        key[r] = t << 33 | (uint64_t)(uint32_t)(pos + 1) << 1 | (uint64_t)((flag >> 4) & 1u);
        len[r] = 4u + bs; src[r] = base + p;
    }
}

__global__ void k_iota(uint32_t* __restrict__ v, unsigned long long n) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) v[i] = (uint32_t)i;
}

__global__ void k_gather_len(const uint32_t* __restrict__ ord, const uint32_t* __restrict__ len, unsigned long long n, uint32_t* __restrict__ slen) {
    for (unsigned long long s = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; s < n; s += (unsigned long long)gridDim.x * blockDim.x) slen[s] = len[ord[s]];
}

// the last index k with a[k] <= x over ascending a[0..n) (a[0] <= x)
__device__ __forceinline__ uint32_t last_le(const unsigned long long* a, uint32_t n, unsigned long long x) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (a[mid] <= x) lo = mid; else hi = mid; }
    return lo;
}

// dest[ord[s]] = dest_sorted[s]; win_lo / win_hi (start ~0u / 0): per window (inflated starts win_beg[0..n_win)), the lowest and highest
// bucket (output starts bkt_beg[0..n_bkt)) of the records whose bytes lie in it
__global__ void k_place(const uint32_t* __restrict__ ord, const unsigned long long* __restrict__ dest_sorted, unsigned long long n, const unsigned long long* __restrict__ src,
                        const uint32_t* __restrict__ len, const unsigned long long* __restrict__ bkt_beg, uint32_t n_bkt, const unsigned long long* __restrict__ win_beg, uint32_t n_win,
                        unsigned long long* __restrict__ dest, uint32_t* __restrict__ win_lo, uint32_t* __restrict__ win_hi) {
    for (unsigned long long s = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; s < n; s += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t o = ord[s];
        const unsigned long long d = dest_sorted[s], a = src[o];
        dest[o] = d;
        const uint32_t b = last_le(bkt_beg, n_bkt, d);
        const uint32_t w1 = last_le(win_beg, n_win, a + len[o] - 1);
        for (uint32_t w = last_le(win_beg, n_win, a); w <= w1; ++w) { atomicMin(&win_lo[w], b); atomicMax(&win_hi[w], b); }
    }
}

// records o0 .. o1 - 1 (input ordinals) intersect the window R = inflated bytes [g0, g0 + L); each one whose output offset is in
// [b0, b1) has its part in the window copied to out[dest - b0 + (part start - record start)].  R has 64 readable bytes past L.
__global__ void __launch_bounds__(256) k_scatter(const uint8_t* __restrict__ R, unsigned long long g0, unsigned long long L, uint32_t o0, uint32_t o1,
                                                 const unsigned long long* __restrict__ src, const uint32_t* __restrict__ len, const unsigned long long* __restrict__ dest,
                                                 unsigned long long b0, unsigned long long b1, uint8_t* __restrict__ out) {
    const int lane = lane_id();
    for (uint32_t o = o0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5); o < o1; o += (gridDim.x * blockDim.x) >> 5) {
        const unsigned long long d = dest[o];
        if (d < b0 || d >= b1) continue;
        const unsigned long long a = src[o], e = a + len[o];
        const unsigned long long lo = a > g0 ? a : g0, hi = e < g0 + L ? e : g0 + L;
        if (lo >= hi) continue;
        const uint8_t* s = R + (lo - g0);
        uint8_t* t = out + (d - b0) + (lo - a);
        const unsigned long long n = hi - lo;
        const unsigned long long head = ((16 - ((uintptr_t)t & 15)) & 15) < n ? ((16 - ((uintptr_t)t & 15)) & 15) : n;
        if ((unsigned long long)lane < head) t[lane] = s[lane];
        const unsigned long long n16 = (n - head) >> 4;
        const uint8_t* s1 = s + head; uint4* t1 = reinterpret_cast<uint4*>(t + head);
        const uintptr_t sa = (uintptr_t)s1;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(sa & ~(uintptr_t)3); const uint32_t sh = (uint32_t)(sa & 3) * 8;
        for (unsigned long long j = lane; j < n16; j += 32) {
            const uint32_t* q = w + 4 * j;
            const uint32_t x0 = q[0], x1 = q[1], x2 = q[2], x3 = q[3], x4 = sh ? q[4] : 0u;
            uint4 v;
            v.x = __funnelshift_r(x0, x1, sh); v.y = __funnelshift_r(x1, x2, sh); v.z = __funnelshift_r(x2, x3, sh); v.w = __funnelshift_r(x3, x4, sh);
            t1[j] = v;
        }
        for (unsigned long long j = head + 16 * n16 + lane; j < n; j += 32) t[j] = s[j];
    }
}

}  // namespace bamsort
