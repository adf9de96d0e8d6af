// prims.cuh — hand-written device primitives: exclusive scan and a stable LSD radix sort
// (u64 keys, u32 payload).  Element counts live in device memory (`n_ptr`); kernels are
// launched for an upper bound and exit early, so no host synchronisation is needed.
#pragma once
#include "common.cuh"

namespace prims {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v) {
    #pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(FULL, v, o); if (lane_id() >= o) v += t; }
    return v;
}

// block-wide exclusive scan of one value per thread (256 threads); returns exclusive prefix, total in *total
__device__ inline uint32_t block_excl_scan(uint32_t v, uint32_t* total) {
    __shared__ uint32_t wsum[8];
    __shared__ uint32_t tot;
    uint32_t inc = warp_incl_scan(v);
    int w = threadIdx.x >> 5;
    if (lane_id() == 31) wsum[w] = inc;
    __syncthreads();
    if (threadIdx.x < 32) {
        uint32_t x = threadIdx.x < 8 ? wsum[threadIdx.x] : 0;
        uint32_t xi = warp_incl_scan(x);
        if (threadIdx.x < 8) wsum[threadIdx.x] = xi - x;
        if (threadIdx.x == 7) tot = xi;
    }
    __syncthreads();
    uint32_t r = inc - v + wsum[w];
    *total = tot;
    __syncthreads();
    return r;
}

// The scans take blockIdx.y as a column: column y is in / out + y * stride, its tile sums tile_sum + y * gridDim.x, its total total_out[y].
// pass 1: per-tile sums
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_reduce(const uint32_t* __restrict__ in, uint32_t* __restrict__ tile_sum,
                                                              const unsigned long long* __restrict__ n_ptr, unsigned long long n_bound, size_t stride) {
    unsigned long long n = n_ptr ? *n_ptr : n_bound; if (n > n_bound) n = n_bound;
    in += blockIdx.y * stride; tile_sum += (size_t)blockIdx.y * gridDim.x;
    unsigned long long base = (unsigned long long)blockIdx.x * SCAN_TILE;
    uint32_t s = 0;
    #pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) { unsigned long long j = base + (unsigned long long)i * SCAN_THREADS + threadIdx.x; if (j < n) s += in[j]; }
    uint32_t tot; block_excl_scan(s, &tot);
    if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}
// pass 2: exclusive scan of the tile sums by one block; writes the grand total to *total_out (64-bit)
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_tiles(uint32_t* __restrict__ tile_sum, int ntiles, unsigned long long* total_out) {
    uint32_t carry = 0; tile_sum += (size_t)blockIdx.x * ntiles;
    for (int b = 0; b < ntiles; b += SCAN_THREADS) {
        int j = b + threadIdx.x; uint32_t v = j < ntiles ? tile_sum[j] : 0; uint32_t tot;
        uint32_t e = block_excl_scan(v, &tot);
        if (j < ntiles) tile_sum[j] = e + carry;
        carry += tot;
    }
    if (threadIdx.x == 0 && total_out) total_out[blockIdx.x] = carry;
}
// pass 3: per-tile exclusive scan plus tile offset.  Thread t owns SCAN_ITEMS consecutive elements.
__global__ void __launch_bounds__(SCAN_THREADS) k_scan_down(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, const uint32_t* __restrict__ tile_sum,
                                                            const unsigned long long* __restrict__ n_ptr, unsigned long long n_bound, size_t stride) {
    unsigned long long n = n_ptr ? *n_ptr : n_bound; if (n > n_bound) n = n_bound;
    in += blockIdx.y * stride; out += blockIdx.y * stride; tile_sum += (size_t)blockIdx.y * gridDim.x;
    unsigned long long base = (unsigned long long)blockIdx.x * SCAN_TILE + (unsigned long long)threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS]; uint32_t s = 0;
    #pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) { v[i] = base + i < n ? in[base + i] : 0; s += v[i]; }
    uint32_t tot; uint32_t e = block_excl_scan(s, &tot) + tile_sum[blockIdx.x];
    #pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) { if (base + i < n) out[base + i] = e; e += v[i]; }
}

// exclusive scans of `cols` columns in[y * stride + 0..n) into out (may alias in), in the same three launches; the totals (u64) to
// total_out[0..cols) if not null.  tmp must hold cols * ceil(n_bound / SCAN_TILE) u32.  Launches are counted in `launches`.
inline void exclusive_scan_cols(uint64_t& launches, const uint32_t* in, uint32_t* out, size_t stride, int cols, uint32_t* tmp, const unsigned long long* n_ptr,
                                unsigned long long n_bound, unsigned long long* total_out, cudaStream_t st) {
    if (n_bound == 0) { if (total_out) cudaMemsetAsync(total_out, 0, 8 * cols, st); return; }
    int ntiles = (int)((n_bound + SCAN_TILE - 1) / SCAN_TILE);
    launch(launches, k_scan_reduce, dim3(ntiles, cols), SCAN_THREADS, 0, st, in, tmp, n_ptr, n_bound, stride);
    launch(launches, k_scan_tiles, cols, SCAN_THREADS, 0, st, tmp, ntiles, total_out);
    launch(launches, k_scan_down, dim3(ntiles, cols), SCAN_THREADS, 0, st, in, out, tmp, n_ptr, n_bound, stride);
}
inline void exclusive_scan(uint64_t& launches, const uint32_t* in, uint32_t* out, uint32_t* tmp, const unsigned long long* n_ptr, unsigned long long n_bound,
                           unsigned long long* total_out, cudaStream_t st) {
    exclusive_scan_cols(launches, in, out, 0, 1, tmp, n_ptr, n_bound, total_out, st);
}
inline size_t scan_tmp_elems(unsigned long long n_bound) { return (size_t)((n_bound + SCAN_TILE - 1) / SCAN_TILE) + 1; }

// ---------------------------------------------------------------- stable LSD radix sort
constexpr int RS_THREADS = 256;
constexpr int RS_ITEMS = 8;
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;

__global__ void __launch_bounds__(RS_THREADS) k_radix_hist(const uint64_t* __restrict__ keys, uint32_t* __restrict__ hist, const unsigned long long* __restrict__ n_ptr,
                                                           unsigned long long n_bound, int shift, int nblk) {
    __shared__ uint32_t h[256];
    unsigned long long n = *n_ptr; if (n > n_bound) n = n_bound;
    unsigned long long base = (unsigned long long)blockIdx.x * RS_TILE;
    h[threadIdx.x] = 0;
    __syncthreads();
    if (base < n) {
        #pragma unroll
        for (int i = 0; i < RS_ITEMS; ++i) { unsigned long long j = base + (unsigned long long)i * RS_THREADS + threadIdx.x; if (j < n) atomicAdd(&h[(keys[j] >> shift) & 255], 1u); }
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * nblk + blockIdx.x] = h[threadIdx.x];
}

__global__ void __launch_bounds__(RS_THREADS) k_radix_scatter(const uint64_t* __restrict__ kin, const uint32_t* __restrict__ vin, uint64_t* __restrict__ kout, uint32_t* __restrict__ vout,
                                                              const uint32_t* __restrict__ offs, const unsigned long long* __restrict__ n_ptr, unsigned long long n_bound, int shift, int nblk) {
    __shared__ uint32_t cnt[8][256];
    unsigned long long n = *n_ptr; if (n > n_bound) n = n_bound;
    unsigned long long tile0 = (unsigned long long)blockIdx.x * RS_TILE;
    if (tile0 >= n) return;
    int w = threadIdx.x >> 5, l = lane_id();
    for (int i = threadIdx.x; i < 8 * 256; i += RS_THREADS) (&cnt[0][0])[i] = 0;
    __syncthreads();
    uint64_t k[RS_ITEMS]; uint32_t v[RS_ITEMS]; uint32_t lr[RS_ITEMS];
    unsigned long long wbase = tile0 + (unsigned long long)w * 32 * RS_ITEMS;
    #pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        unsigned long long j = wbase + (unsigned long long)r * 32 + l;
        bool valid = j < n;
        k[r] = valid ? kin[j] : 0; v[r] = valid ? vin[j] : 0;
        uint32_t d = (uint32_t)(k[r] >> shift) & 255u;
        uint32_t m = __match_any_sync(FULL, valid ? d : (256u + (uint32_t)l));
        uint32_t rank = __popc(m & lanemask_lt());
        uint32_t base = valid ? cnt[w][d] : 0;
        __syncwarp();
        if (valid && rank == 0) cnt[w][d] = base + __popc(m);
        __syncwarp();
        lr[r] = base + rank;
    }
    __syncthreads();
    {   // exclusive scan over warps for digit = threadIdx.x, seeded with the global offset of (digit, block)
        uint32_t s = offs[(size_t)threadIdx.x * nblk + blockIdx.x];
        #pragma unroll
        for (int ww = 0; ww < 8; ++ww) { uint32_t t = cnt[ww][threadIdx.x]; cnt[ww][threadIdx.x] = s; s += t; }
    }
    __syncthreads();
    #pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        unsigned long long j = wbase + (unsigned long long)r * 32 + l;
        if (j < n) { uint32_t d = (uint32_t)(k[r] >> shift) & 255u; uint32_t pos = cnt[w][d] + lr[r]; kout[pos] = k[r]; vout[pos] = v[r]; }
    }
}

struct RadixTemp { uint32_t* hist; uint32_t* scan_tmp; };
inline size_t radix_hist_elems(unsigned long long n_bound) { return (size_t)256 * (size_t)((n_bound + RS_TILE - 1) / RS_TILE) + 256; }

// sorts (k0,v0) by the key bits [0, bits); result ends in (k0,v0) when `*in_first` is true, else in (k1,v1).  Launches are counted in `launches`.
inline void radix_sort(uint64_t& launches, uint64_t* k0, uint32_t* v0, uint64_t* k1, uint32_t* v1, RadixTemp tmp, const unsigned long long* n_ptr, unsigned long long n_bound,
                       int bits, bool* in_first, cudaStream_t st) {
    *in_first = true;
    if (n_bound == 0) return;
    int nblk = (int)((n_bound + RS_TILE - 1) / RS_TILE);
    for (int shift = 0; shift < bits; shift += 8) {
        const uint64_t* ki = *in_first ? k0 : k1; const uint32_t* vi = *in_first ? v0 : v1;
        uint64_t* ko = *in_first ? k1 : k0; uint32_t* vo = *in_first ? v1 : v0;
        launch(launches, k_radix_hist, nblk, RS_THREADS, 0, st, ki, tmp.hist, n_ptr, n_bound, shift, nblk);
        exclusive_scan(launches, tmp.hist, tmp.hist, tmp.scan_tmp, nullptr, (unsigned long long)256 * nblk, nullptr, st);
        launch(launches, k_radix_scatter, nblk, RS_THREADS, 0, st, ki, vi, ko, vo, tmp.hist, n_ptr, n_bound, shift, nblk);
        *in_first = !*in_first;
    }
}

}  // namespace prims
