// bam_index.cuh — the BAI / CSI index of a coordinate-sorted BAM (SAM spec §5), built from the device ingest with no index to start from.
// A window is a run of whole BGZF members inflated by ingest::k_inflate, preceded by the bytes of the record the previous window could not
// finish (the carry).  In the window's inflated bytes R[0, L) the record chain starts at a known entry e (0, or the end of the BAM header in
// the first window):
//
//   k_mark         one thread per offset, a warp per 32 offsets: bit p of the candidate mask = R[p..] passes the strict record test
//                  (cand_kind); offsets whose test runs past L are candidates too (a record the window cannot finish)
//   (scan)         popcounts of the mask words -> every candidate's index
//   k_compact      the candidates' offsets, ascending
//   k_link         J_0 = the candidate at next = p + 4 + block_size (binary search), END when next == L, BREAK when next is no candidate,
//                  itself for a record the window cannot finish
//   k_jump         J_{k+1} = J_k o J_k (pointer jumping, ceil(log2 n) levels)
//   k_mark_path    top-down over the levels: the nodes reachable from the entry in < 2^K hops, i.e. the true chain.  A false candidate
//                  whose next lands on a true record is never marked: marks only move forward from the entry
//   (scan)         the chain's complete records, in file order
//   k_rows         one warp per record: tid, beg, end (htslib's bam_endpos: the CIGAR's reference span, 1 for an unmapped read or a zero
//                  span), the virtual offset after it, mapped
//   k_check        v0 = the previous record's v1; sort order against the previous record (also across windows); BAI's 2^29 limit
//
// and, once every window is through, the tables over all rows:
//
//   k_ref_stats    per reference: first v0, last v1, mapped / unmapped counts, the length of the linear index
//   k_chunks       bins (reg2bin at the index geometry), chunk heads (a new (tid, bin) run), linear index (atomicMin of v0 per window)
//   k_lin_fill     an empty linear-index window takes the next window's value (htslib update_loff)
//   (radix sort)   chunks by (tid, bin), stable; unique bins, each bin's parent, CSI loffset
//   k_bin_span / k_bin_lift   level by level from the leaves: a bin whose chunks span < 0x10000 compressed bytes moves them to its parent
//   (radix sort)   chunks by (final bin, file order); k_merge_heads: chunks starting in the block where the previous one ends are merged
#pragma once
#include "common.cuh"
#include "prims.cuh"
#include "ingest_core.h"

namespace bamidx {

using ingest::ld32u; using ingest::ld16u; using ingest::warp_sum;

constexpr uint32_t END_NODE = 0, BREAK_NODE = 1;       // sentinels are nodes n + END_NODE, n + BREAK_NODE
constexpr int CAND_NONE = 0, CAND_COMPLETE = 1, CAND_OPEN = 2;

// one record of the index input; v0 / v1 = virtual offsets of its first byte and of the byte after it
struct Row { unsigned long long v0, v1; long long end; int tid, beg; unsigned mapped, _pad; };
// window geometry: the global offset of R[0], and the members whose inflated bytes follow the carry
// blk_end[k] = global inflated end of member k, first_beg = global inflated start of member 0, coff_end = the file offset after the last member
struct Window { unsigned long long base, first_beg, coff_end; const unsigned long long* blk_end; const unsigned long long* blk_coff; unsigned nb; };
// first failure of a window or of the tables: code << 56 | record index (an atomicMin, so the lowest record wins)
constexpr unsigned long long BAD_NONE = ~0ull;
enum : unsigned { BAD_ORDER = 1, BAD_TID_AFTER_UNPLACED = 2, BAD_TID_BACK = 3, BAD_RANGE = 4 };

__device__ __forceinline__ int cand_kind(const uint8_t* R, unsigned long long L, unsigned long long p, int n_ref, const long long* clen) {
    if (p + 36 > L) return CAND_OPEN;
    const uint32_t bs = ld32u(R, p);
    const int ref = (int)ld32u(R, p + 4), pos = (int)ld32u(R, p + 8);
    const uint32_t l_rn = R[p + 12], n_cig = ld16u(R, p + 16);
    const int l_seq = (int)ld32u(R, p + 20);
    if (bs < 32u || ref < -1 || ref >= n_ref || l_rn < 1u || l_seq < 0 || pos < -1) return CAND_NONE;
    if (ref >= 0 && (long long)pos > clen[ref]) return CAND_NONE;
    if (32ull + l_rn + 4ull * n_cig + (unsigned long long)((l_seq + 1) / 2) + (unsigned long long)l_seq > bs) return CAND_NONE;
    if (p + 36 + l_rn > L) return CAND_OPEN;
    if (R[p + 36 + l_rn - 1] != 0) return CAND_NONE;
    return p + 4 + bs > L ? CAND_OPEN : CAND_COMPLETE;
}

__global__ void k_mark(const uint8_t* __restrict__ R, unsigned long long L, unsigned long long e, int n_ref, const long long* __restrict__ clen,
                       uint32_t* __restrict__ mask, uint32_t* __restrict__ cnt, unsigned long long n_words) {
    for (unsigned long long w = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5; w < n_words; w += (gridDim.x * (unsigned long long)blockDim.x) >> 5) {
        const unsigned long long p = 32ull * w + lane_id();
        const bool c = p >= e && p < L && cand_kind(R, L, p, n_ref, clen) != CAND_NONE;
        const uint32_t m = __ballot_sync(FULL, c);
        if (lane_id() == 0) { mask[w] = m; cnt[w] = __popc(m); }
    }
}

__global__ void k_compact(const uint32_t* __restrict__ mask, const uint32_t* __restrict__ base, unsigned long long n_words, uint32_t* __restrict__ cand) {
    for (unsigned long long w = (blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x) >> 5; w < n_words; w += (gridDim.x * (unsigned long long)blockDim.x) >> 5) {
        const uint32_t m = mask[w];
        if (m >> lane_id() & 1u) cand[base[w] + __popc(m & lanemask_lt())] = (uint32_t)(32ull * w + lane_id());
    }
}

__global__ void k_link(const uint8_t* __restrict__ R, unsigned long long L, int n_ref, const long long* __restrict__ clen, const uint32_t* __restrict__ cand, uint32_t n,
                       uint32_t* __restrict__ J0) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n + 2; i += gridDim.x * blockDim.x) {
        if (i >= n) { J0[i] = i; continue; }
        const unsigned long long p = cand[i];
        if (cand_kind(R, L, p, n_ref, clen) == CAND_OPEN) { J0[i] = i; continue; }
        const unsigned long long s = p + 4 + ld32u(R, p);
        if (s == L) { J0[i] = n + END_NODE; continue; }
        uint32_t lo = i + 1, hi = n;                              // next > p: search above i
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (cand[mid] < s) lo = mid + 1; else hi = mid; }
        J0[i] = lo < n && cand[lo] == s ? lo : n + BREAK_NODE;
    }
}

__global__ void k_jump(const uint32_t* __restrict__ Jk, uint32_t* __restrict__ Jn, uint32_t n2) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x) Jn[i] = Jk[Jk[i]];
}

// marks only ever spread along J from a marked node, so every mark is on the entry's chain; a mark set during the launch and read again by
// it moves 2^k further along the same chain, which is still the chain
__global__ void k_mark_path(const uint32_t* __restrict__ Jk, uint32_t n2, uint8_t* mark) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += gridDim.x * blockDim.x)
        if (mark[i]) mark[Jk[i]] = 1;
}

// complete chain records -> 1 (the scan gives their row index); the open record the chain ends in, and the failing node, to `out`
// out[0] = offset of the open record (or ~0), out[1] = index of the node whose next is no candidate (or ~0)
__global__ void k_path_records(const uint8_t* __restrict__ mark, const uint32_t* __restrict__ J0, uint32_t n, uint32_t* __restrict__ is_rec,
                               const uint32_t* __restrict__ cand, unsigned long long* out) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const bool on = mark[i] != 0;
        is_rec[i] = on && J0[i] != i;
        if (on && J0[i] == i) atomicMin(&out[0], (unsigned long long)cand[i]);
        if (on && J0[i] == n + BREAK_NODE) atomicMin(&out[1], (unsigned long long)i);
    }
}

__device__ __forceinline__ unsigned long long voff(const Window& W, unsigned long long u) {
    unsigned lo = 0, hi = W.nb;                                    // first member whose inflated end is >= u
    while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (W.blk_end[mid] < u) lo = mid + 1; else hi = mid; }
    if (lo < W.nb && W.blk_end[lo] > u) {
        const unsigned long long beg = lo ? W.blk_end[lo - 1] : W.first_beg;
        return W.blk_coff[lo] << 16 | (u - beg);
    }
    // u is the end of member lo: htslib's bgzf_tell moves on to the next member, offset 0
    return (lo + 1 < W.nb ? W.blk_coff[lo + 1] : W.coff_end) << 16;
}

// one warp per chain record: its row without v0, and its offset in the window
__global__ void __launch_bounds__(256) k_rows(const uint8_t* __restrict__ R, const uint32_t* __restrict__ cand, const uint32_t* __restrict__ is_rec,
                                              const uint32_t* __restrict__ rec_idx, uint32_t n, Window W, Row* __restrict__ rows, uint32_t* __restrict__ roff) {
    const int lane = lane_id();
    for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += (gridDim.x * blockDim.x) >> 5) {
        if (!is_rec[i]) continue;
        const unsigned long long p = cand[i];
        const uint32_t bs = ld32u(R, p), l_rn = R[p + 12], n_cig = ld16u(R, p + 16), flag = ld16u(R, p + 18);
        const int tid = (int)ld32u(R, p + 4), pos = (int)ld32u(R, p + 8);
        long long span = 0;
        if (!(flag & 4u)) {
            const unsigned long long c0 = p + 36 + l_rn;
            for (uint32_t k = lane; k < n_cig; k += 32) {
                const uint32_t op = ld32u(R, c0 + 4ull * k);
                const uint32_t code = op & 15u;
                if (code == 0 || code == 2 || code == 3 || code == 7 || code == 8) span += op >> 4;
            }
            span = warp_sum<32>(span);
        }
        if (lane == 0) {
            Row r; r.tid = tid; r.beg = pos; r.end = (long long)pos + (span > 0 ? span : 1); r.mapped = (flag & 4u) ? 0u : 1u; r._pad = 0; r.v0 = 0;
            r.v1 = voff(W, W.base + p + 4 + bs);
            rows[rec_idx[i]] = r; roff[rec_idx[i]] = (uint32_t)p;
        }
    }
}

// v0 and the order checks; prev = the last row of the previous window (tid -2 before the first record)
__global__ void k_check(Row* __restrict__ rows, uint32_t n_rows, unsigned long long v_entry, int prev_tid, int prev_beg, long long max_end, unsigned long long row_base,
                        unsigned long long* __restrict__ bad) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_rows; i += gridDim.x * blockDim.x) {
        Row& r = rows[i];
        r.v0 = i ? rows[i - 1].v1 : v_entry;
        const int pt = i ? rows[i - 1].tid : prev_tid, pb = i ? rows[i - 1].beg : prev_beg;
        unsigned code = 0;
        if (pt == -1 && r.tid != -1) code = BAD_TID_AFTER_UNPLACED;
        else if (r.tid >= 0 && pt > r.tid) code = BAD_TID_BACK;
        else if (r.tid >= 0 && pt == r.tid && pb > r.beg) code = BAD_ORDER;
        else if (r.tid >= 0 && r.end > max_end) code = BAD_RANGE;
        if (code) atomicMin(bad, (unsigned long long)code << 56 | (row_base + i));
    }
}

// ---------------------------------------------------------------- tables
struct Geo { int min_shift, depth; };
__device__ __forceinline__ int bin_first(int l) { return ((1 << (3 * l)) - 1) / 7; }
__device__ __forceinline__ int bin_level(int b) { int l = 0; while (b) { b = (b - 1) >> 3; ++l; } return l; }
__device__ __forceinline__ int reg2bin(long long beg, long long end, Geo g) {          // htslib hts_reg2bin
    int s = g.min_shift, t = bin_first(g.depth);
    --end;
    for (int l = g.depth; l > 0; --l, s += 3, t -= 1 << (3 * l)) if (beg >> s == end >> s) return (int)(t + (beg >> s));
    return 0;
}
__device__ __forceinline__ long long clamp_beg(const Row& r) { return r.beg < 0 ? 0 : r.beg; }
__device__ __forceinline__ long long clamp_end(const Row& r) { return r.end <= 0 ? 1 : r.end; }

// per reference: [0] first v0, [1] last v1, [2] mapped, [3] unmapped, [4] linear-index windows.  Placed rows only (n_placed).
__global__ void k_ref_stats(const Row* __restrict__ rows, uint32_t n_placed, Geo g, unsigned long long* __restrict__ ref) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_placed; i += gridDim.x * blockDim.x) {
        const Row r = rows[i]; unsigned long long* s = ref + 5ull * r.tid;
        atomicMin(&s[0], r.v0); atomicMax(&s[1], r.v1); atomicAdd(&s[r.mapped ? 2 : 3], 1ull);
        atomicMax(&s[4], (unsigned long long)(((clamp_end(r) - 1) >> g.min_shift) + 1));
    }
}

// bins, chunk heads (1 where a new (tid, bin) run starts) and the linear index (lin must start all-ones)
__global__ void k_chunks(const Row* __restrict__ rows, uint32_t n_placed, Geo g, uint32_t n_bins, uint32_t* __restrict__ head, uint64_t* __restrict__ key,
                         const unsigned long long* __restrict__ lin_off, unsigned long long* __restrict__ lin) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_placed; i += gridDim.x * blockDim.x) {
        const Row r = rows[i];
        const long long b = clamp_beg(r), e = clamp_end(r);
        const uint64_t k = (uint64_t)r.tid * n_bins + (uint64_t)reg2bin(b, e, g);
        key[i] = k;
        head[i] = 1;
        if (i) { const Row q = rows[i - 1]; head[i] = (uint64_t)q.tid * n_bins + (uint64_t)reg2bin(clamp_beg(q), clamp_end(q), g) != k; }
        unsigned long long* L = lin + lin_off[r.tid];
        for (long long w = b >> g.min_shift; w <= (e - 1) >> g.min_shift; ++w) atomicMin(&L[w], r.v0);
    }
}

// one block per reference: an unset window (all-ones) takes the next window's value, as htslib's update_loff fills it (the last window is
// always set).  That is a suffix minimum, scanned from the end in tiles of 256 windows.
__global__ void __launch_bounds__(256) k_lin_fill(unsigned long long* __restrict__ lin, const unsigned long long* __restrict__ lin_off, int n_ref) {
    __shared__ unsigned long long wmin[8];
    const int t = blockIdx.x; if (t >= n_ref) return;
    unsigned long long* L = lin + lin_off[t];
    const unsigned long long n = lin_off[t + 1] - lin_off[t];
    unsigned long long carry = ~0ull;
    for (unsigned long long b = 0; b < n; b += 256) {
        const unsigned long long r = b + threadIdx.x, j = n - 1 - r;          // r counts from the last window
        unsigned long long v = r < n ? L[j] : ~0ull;
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long x = __shfl_up_sync(FULL, v, o); if (lane_id() >= o) v = v < x ? v : x; }
        if (lane_id() == 31) wmin[threadIdx.x >> 5] = v;
        __syncthreads();
        unsigned long long pre = carry;
        for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) pre = pre < wmin[w] ? pre : wmin[w];
        v = v < pre ? v : pre;
        if (r < n) L[j] = v;
        unsigned long long tot = carry;
        for (int w = 0; w < 8; ++w) tot = tot < wmin[w] ? tot : wmin[w];
        __syncthreads();
        carry = tot;
    }
}

// chunk c = the run of rows head_idx[c] .. head_idx[c + 1] - 1: its u / v and key, in file order
__global__ void k_chunk_rows(const Row* __restrict__ rows, const uint32_t* __restrict__ head, const uint32_t* __restrict__ cidx, const uint64_t* __restrict__ rkey, uint32_t n_placed,
                             unsigned long long* __restrict__ cu, unsigned long long* __restrict__ cv, uint64_t* __restrict__ ckey, uint32_t* __restrict__ cval) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_placed; i += gridDim.x * blockDim.x) {
        const uint32_t c = cidx[i] + head[i] - 1;
        if (head[i]) { cu[c] = rows[i].v0; ckey[c] = rkey[i]; cval[c] = c; }
        if (i + 1 == n_placed || head[i + 1]) cv[c] = rows[i].v1;
    }
}

// over the chunks sorted by (tid, bin): 1 where a new bin starts
__global__ void k_key_heads(const uint64_t* __restrict__ skey, uint32_t n, uint32_t* __restrict__ h) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) h[s] = s == 0 || skey[s] != skey[s - 1];
}

// unique bins: their key; the chunk's bin index (by original chunk index); each bin's parent index (-1: no such bin) and CSI loffset
__global__ void k_unique_bins(const uint64_t* __restrict__ skey, const uint32_t* __restrict__ sval, const uint32_t* __restrict__ h, const uint32_t* __restrict__ hidx, uint32_t n,
                              uint64_t* __restrict__ ukey, uint32_t* __restrict__ cur) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        const uint32_t b = hidx[s] + h[s] - 1;
        if (h[s]) ukey[b] = skey[s];
        cur[sval[s]] = b;
    }
}
__global__ void k_bin_info(const uint64_t* __restrict__ ukey, uint32_t n_ub, uint32_t n_bins, Geo g, const unsigned long long* __restrict__ lin_off, const unsigned long long* __restrict__ lin,
                           int* __restrict__ parent, int* __restrict__ level, unsigned long long* __restrict__ loff) {
    for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < n_ub; b += gridDim.x * blockDim.x) {
        const uint64_t tid = ukey[b] / n_bins; const int bin = (int)(ukey[b] % n_bins);
        const int l = bin_level(bin);
        level[b] = l;
        int pidx = -1;
        if (l > 0) {
            const uint64_t pk = tid * n_bins + (uint64_t)((bin - 1) >> 3);
            uint32_t lo = 0, hi = b;
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (ukey[mid] < pk) lo = mid + 1; else hi = mid; }
            if (lo < b && ukey[lo] == pk) pidx = (int)lo;
        }
        parent[b] = pidx;
        const unsigned long long bot = (unsigned long long)(bin - bin_first(l)) << (3 * (g.depth - l));
        const unsigned long long n_intv = lin_off[tid + 1] - lin_off[tid];
        loff[b] = bot < n_intv ? lin[lin_off[tid] + bot] : 0ull;
    }
}

// htslib compress_binning at one level: a bin's span is (its last chunk's v >> 16) - (its first chunk's u >> 16)
__global__ void k_bin_span(const uint32_t* __restrict__ cur, const int* __restrict__ level, const unsigned long long* __restrict__ cu, const unsigned long long* __restrict__ cv,
                           uint32_t n_chunk, int l, unsigned long long* __restrict__ bmin, unsigned long long* __restrict__ bmax) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_chunk; c += gridDim.x * blockDim.x) {
        const uint32_t b = cur[c]; if (level[b] != l) continue;
        atomicMin(&bmin[b], cu[c] >> 16); atomicMax(&bmax[b], cv[c] >> 16);
    }
}
__global__ void k_bin_lift(uint32_t* __restrict__ cur, const int* __restrict__ level, const int* __restrict__ parent, uint32_t n_chunk, int l,
                           const unsigned long long* __restrict__ bmin, const unsigned long long* __restrict__ bmax) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_chunk; c += gridDim.x * blockDim.x) {
        const uint32_t b = cur[c]; if (level[b] != l) continue;
        if (bmax[b] - bmin[b] < 0x10000ull && parent[b] >= 0) cur[c] = (uint32_t)parent[b];
    }
}
__global__ void k_cur_keys(const uint32_t* __restrict__ cur, uint32_t n, uint64_t* __restrict__ k, uint32_t* __restrict__ v) {
    for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n; c += gridDim.x * blockDim.x) { k[c] = cur[c]; v[c] = c; }
}
// over the chunks sorted by (bin, file order): a merged chunk starts at a new bin or where the previous chunk ends in an earlier block
__global__ void k_merge_heads(const uint64_t* __restrict__ sb, const uint32_t* __restrict__ sc, const unsigned long long* __restrict__ cu, const unsigned long long* __restrict__ cv,
                              uint32_t n, uint32_t* __restrict__ h) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x)
        h[s] = s == 0 || sb[s] != sb[s - 1] || (cv[sc[s - 1]] >> 16) < (cu[sc[s]] >> 16);
}
// merged chunks: bin index, u of the first, v of the last
__global__ void k_merge_out(const uint64_t* __restrict__ sb, const uint32_t* __restrict__ sc, const unsigned long long* __restrict__ cu, const unsigned long long* __restrict__ cv,
                            const uint32_t* __restrict__ h, const uint32_t* __restrict__ hidx, uint32_t n, uint32_t* __restrict__ mbin, unsigned long long* __restrict__ mu,
                            unsigned long long* __restrict__ mv) {
    for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < n; s += gridDim.x * blockDim.x) {
        const uint32_t m = hidx[s] + h[s] - 1;
        if (h[s]) { mbin[m] = (uint32_t)sb[s]; mu[m] = cu[sc[s]]; }
        if (s + 1 == n || h[s + 1]) mv[m] = cv[sc[s]];
    }
}

}  // namespace bamidx
