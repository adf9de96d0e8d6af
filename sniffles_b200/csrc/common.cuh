// common.cuh — shared device helpers of libsnfb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <math.h>
#include "../../include/snfb.h"

#define FULL 0xffffffffu

// SMs of the H100 SXM: persistent and grid-stride launches are sized in multiples of it
constexpr int NUM_SMS = 132;

#define CUDA_TRY(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ctx_fail(ctx, #x, cudaGetErrorString(e_)); return 1; } } while (0)

// every kernel of the library is launched here, so the launch counter n (snfb_launch_count) counts exactly the launches made
template <class... P, class... A> inline void launch(uint64_t& n, void (*k)(P...), dim3 g, dim3 b, size_t smem, cudaStream_t st, A... a) { k<<<g, b, smem, st>>>(a...); ++n; }

typedef unsigned __int128 u128;

// ---------------------------------------------------------------- device-side run state
// Counters written by kernels; copied to the host once per stage.
struct DevCounters {
    unsigned long long n_leads;        // number of leads (sum of the per-record counts)
    unsigned long long n_pass;         // reads passing the filters
    unsigned long long soft_errors;    // malformed SA entries etc.
    unsigned long long lead_overflow;  // leads dropped because the lead buffer was full
    unsigned long long unsorted;       // records out of coordinate order inside a task
    unsigned long long n_bins, n_kbins, n_segs, n_clusters, n_sub, n_cand, n_cand_leads, n_rnames;
    unsigned long long unverified_breaks;
    unsigned long long n_alt_bytes, n_seq_bytes, scratch_overflow;
    unsigned long long n_slots;        // high-water mark of the lead slot allocator (>= n_leads: warps reserve chunks)
    unsigned long long n_ev, n_sa;     // event slots handed out by the CIGAR walk (SV signatures + retired holes) / records with an SA tag
    unsigned long long n_kl, n_kll;    // kept leads / kept "long" leads
    unsigned long long n_big, n_mid;   // clusters handled by a whole block / by the mid-sized warp kernel
    unsigned long long ordinal_overflow;   // reads with more than 65535 leads (the ordinal is a 16-bit field)
    unsigned long long bad_records;    // records whose offsets point outside the block's arenas or tables (snfb_load_records fails)
    unsigned long long n_items, n_tiles, n_req, n_req_units;   // consensus work items / vote tiles / seq-on-demand requests
    unsigned long long n_small_taken;  // clusters handed out by the dense warp-per-cluster kernel's work queue (reset by k_cluster_build)
};

// ---------------------------------------------------------------- small utilities
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
// stores a struct whose size is a multiple of 16 bytes with 16-byte stores.  The bytes are taken with memcpy, not through a cast
// pointer: a cast breaks strict aliasing, and the compiler may then read the vectors before the fields are written.
template <class T> __device__ __forceinline__ void store16(void* dst, const T& v) {
    static_assert(sizeof(T) % 16 == 0, "store16: size must be a multiple of 16 bytes");
    uint4 t[sizeof(T) / 16]; memcpy(t, &v, sizeof(T));
    #pragma unroll
    for (int k = 0; k < (int)(sizeof(T) / 16); ++k) reinterpret_cast<uint4*>(dst)[k] = t[k];
}
__device__ __forceinline__ unsigned lanemask_lt() { unsigned m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// FNV-1a 64 of a contig name (snfb_hash_name); serial, names are a few bytes
__device__ __forceinline__ uint64_t fnv1a64(const uint8_t* s, int n) {
    uint64_t h = 0xcbf29ce484222325ull;
    for (int i = 0; i < n; ++i) { h ^= s[i]; h *= 0x100000001b3ull; }
    return h;
}

// Query-name hash: each 8-byte word is mixed with its index and the results are summed, so
// the lanes of a warp hash words independently (leadprov only ever compares names for equality).
__device__ __forceinline__ uint64_t qname_word(uint64_t w, uint32_t idx) {
    uint64_t z = w + 0x9E3779B97F4A7C15ull * (uint64_t)(idx + 1);
    return mix64(z);
}
__device__ __forceinline__ uint64_t qname_finish(uint64_t h) {
    h = (h ^ (h >> 33)) * 0xff51afd7ed558ccdull; h = (h ^ (h >> 33)) * 0xc4ceb9fe1a85ec53ull; return h ^ (h >> 33);
}
__device__ inline uint64_t qname_hash_warp(const uint8_t* s, int n) {   // all 32 lanes; n <= 255
    int l = lane_id(); uint64_t acc = 0;
    if (l * 8 < n) {
        uint64_t w = 0; int m = n - l * 8 < 8 ? n - l * 8 : 8;
        for (int j = 0; j < m; ++j) w |= (uint64_t)s[l * 8 + j] << (8 * j);
        acc = qname_word(w, (uint32_t)l);
    }
    #pragma unroll
    for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(FULL, acc, o);
    return qname_finish(acc + (0x9E3779B97F4A7C15ull ^ (uint64_t)n));
}

// ---------------------------------------------------------------- exact statistics.stdev
// RN(sqrt(P/Q)) for P < 2^128, 0 < Q < 2^63: the value CPython 3.12's statistics.stdev returns
// for integer data with P = n*Sxx - Sx^2 and Q = n*(n-1) (statistics.py _float_sqrt_of_frac).
__host__ __device__ inline int clz64_hd(uint64_t x) {
#ifdef __CUDA_ARCH__
    return __clzll((long long)x);
#else
    return x ? __builtin_clzll(x) : 64;
#endif
}
__host__ __device__ inline int bitlen_u128(u128 x) {
    uint64_t hi = (uint64_t)(x >> 64), lo = (uint64_t)x;
    return hi ? 128 - clz64_hd(hi) : (lo ? 64 - clz64_hd(lo) : 0);
}
// the reference algorithm, limb by limb: numerator shifted to 111+ significant quotient bits, long division, integer square root,
// round-to-odd, one final rounding (statistics.py _float_sqrt_of_frac).  Slow (a 288-bit long division): only the fallback of the fast path below.
__host__ __device__ inline double sqrt_frac_rn_slow(u128 P, uint64_t Q) {
    if (P == 0) return 0.0;
    int bl = bitlen_u128(P) - bitlen_u128((u128)Q);
    int s = 111 - bl; if (s < 0) s = 0; if (s & 1) ++s;
    // numerator P << s in 32-bit limbs (at most 128 + 112 bits)
    uint32_t num[9];
    for (int i = 0; i < 9; ++i) num[i] = 0;
    int w = s >> 5, o = s & 31;
    for (int i = 0; i < 4; ++i) {
        uint64_t limb = (uint64_t)((P >> (32 * i)) & 0xFFFFFFFFu) << o;
        // disjoint bit ranges: or-ing is exact
        if (w + i < 9) num[w + i] |= (uint32_t)limb;
        if (w + i + 1 < 9) num[w + i + 1] |= (uint32_t)(limb >> 32);
    }
    // long division by Q (Q < 2^63 so rem*2^32 + limb fits in u128)
    uint32_t quo[9]; u128 rem = 0;
    for (int i = 8; i >= 0; --i) { u128 cur = (rem << 32) | num[i]; u128 q = cur / Q; quo[i] = (uint32_t)q; rem = cur - q * Q; }
    u128 V = ((u128)quo[3] << 96) | ((u128)quo[2] << 64) | ((u128)quo[1] << 32) | quo[0];
    double vf = (double)(uint64_t)(V >> 64) * 18446744073709551616.0 + (double)(uint64_t)V;
    uint64_t a = (uint64_t)sqrt(vf);
    // fix up to the exact integer square root
    while ((u128)a * a > V) --a;
    while ((u128)(a + 1) * (a + 1) <= V) ++a;
    bool sticky = ((u128)a * a != V) || rem != 0;
    a |= (uint64_t)sticky;
    return ldexp((double)a, -(s >> 1));     // u64 -> double is round-to-nearest-even: the single rounding
}
// ---- fast path: a floating-point guess, then an EXACT check that it is the correctly rounded value: x = P / Q lies between the squares of the
//      midpoints to the neighbouring doubles.  The comparisons are done in 256-bit integers, so the result is the same bit pattern as above.
struct U256 { uint64_t w[4]; };
__host__ __device__ inline U256 mul_128_64(u128 a, uint64_t b) {
    const u128 lo = (u128)(uint64_t)a * b; const u128 hi = (u128)(uint64_t)(a >> 64) * b + (uint64_t)(lo >> 64);
    U256 r; r.w[0] = (uint64_t)lo; r.w[1] = (uint64_t)hi; r.w[2] = (uint64_t)(hi >> 64); r.w[3] = 0; return r;
}
__host__ __device__ inline int cmp256(const U256& a, const U256& b) {
    for (int i = 3; i >= 0; --i) if (a.w[i] != b.w[i]) return a.w[i] < b.w[i] ? -1 : 1;
    return 0;
}
// sign of (m * 2^e)^2 * Q - P for m < 2^55; 2 when the operands do not fit the 256-bit comparison (the caller falls back)
__host__ __device__ inline int cmp_mid_sq(uint64_t m, int e, u128 P, uint64_t Q) {
    const U256 A = mul_128_64((u128)m * m, Q);
    if (e >= 0) return 2;
    const int s = -2 * e;
    if (bitlen_u128(P) + s > 255) return -1;          // P * 2^s has more bits than A can have (A < 2^174): A is smaller
    U256 R; R.w[0] = R.w[1] = R.w[2] = R.w[3] = 0;
    const int ws = s >> 6, bs = s & 63; const uint64_t lo = (uint64_t)P, hi = (uint64_t)(P >> 64);
    if (ws < 4) R.w[ws] = lo << bs;
    if (ws + 1 < 4) R.w[ws + 1] = (hi << bs) | (bs ? lo >> (64 - bs) : 0ull);
    if (ws + 2 < 4) R.w[ws + 2] = bs ? hi >> (64 - bs) : 0ull;
    return cmp256(A, R);
}
__host__ __device__ inline double bits_to_f8(long long b) {
#ifdef __CUDA_ARCH__
    return __longlong_as_double(b);
#else
    double d; memcpy(&d, &b, 8); return d;
#endif
}
__host__ __device__ inline long long f8_to_bits(double d) {
#ifdef __CUDA_ARCH__
    return __double_as_longlong(d);
#else
    long long b; memcpy(&b, &d, 8); return b;
#endif
}
__host__ __device__ inline double sqrt_frac_rn(u128 P, uint64_t Q) {
    if (P == 0) return 0.0;
    const double pf = (double)(uint64_t)(P >> 64) * 18446744073709551616.0 + (double)(uint64_t)P;
    double d = sqrt(pf / (double)Q);
    for (int it = 0; it < 6; ++it) {
        const long long bits = f8_to_bits(d); const int ex = (int)((bits >> 52) & 0x7ff);
        if (ex == 0 || ex == 0x7ff || bits < 0) break;
        const uint64_t M = ((uint64_t)bits & ((1ull << 52) - 1)) | (1ull << 52); const int E = ex - 1075;      // d = M * 2^E
        // midpoints to the neighbouring doubles (below a power of two the spacing halves)
        const bool pow2 = M == (1ull << 52);
        const int c_lo = pow2 ? cmp_mid_sq(4 * M - 1, E - 2, P, Q) : cmp_mid_sq(2 * M - 1, E - 1, P, Q);
        if (c_lo == 2) break;
        if (c_lo > 0) { d = bits_to_f8(bits - 1); continue; }                          // the lower midpoint is already above sqrt(x): d is too large
        if (c_lo == 0) return (M & 1) ? bits_to_f8(bits - 1) : d;                       // exactly half way: ties to even
        const int c_hi = cmp_mid_sq(2 * M + 1, E - 1, P, Q);
        if (c_hi == 2) break;
        if (c_hi < 0) { d = bits_to_f8(bits + 1); continue; }                          // the upper midpoint is below sqrt(x): d is too small
        if (c_hi == 0) return (M & 1) ? bits_to_f8(bits + 1) : d;
        return d;
    }
    return sqrt_frac_rn_slow(P, Q);
}

// exact sample stdev of int values v[0..n) accessed through a functor (values fit in int32)
template <class F>
__device__ inline double stdev_ints(long n, F get) {
    if (n < 2) return 0.0;
    long long base = get(0); u128 sxx = 0; __int128 sx = 0;
    for (long i = 0; i < n; ++i) { __int128 d = (__int128)((long long)get(i) - base); sx += d; sxx += (u128)(d * d); }
    u128 P = (u128)n * sxx - (u128)(sx * sx);
    return sqrt_frac_rn(P, (uint64_t)n * (uint64_t)(n - 1));
}

// python-style int(x / b) * b for 0 <= x, b > 0 (float division then truncation == floor for these ranges)
__device__ __forceinline__ int bin_floor(int x, int b) { return (x / b) * b; }
