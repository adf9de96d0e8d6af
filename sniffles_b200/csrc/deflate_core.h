// deflate_core.h — BGZF DEFLATE encoder (RFC 1951 / RFC 1952 with the BGZF extra field, SAM spec §4.1): one input block of at most
// 0xff00 bytes -> one gzip member of at most 65536 bytes, as htslib's bgzip cuts its input.  Written for "a group of NT threads with a
// barrier between phases": the CUDA kernel (bgzf_write.cuh) runs every phase with a thread block of DEF_THREADS threads and the warp
// phases with 32 lanes; tests/native/deflate_host.cpp runs the same phases with one thread (NT = 1, NL = 1), so the bytes the device
// writes can be checked on the CPU against zlib.  The output is a pure function of the input bytes:
//   * match candidates: the nearest earlier position with the same 4-byte hash (HASH_BITS) within 32 KiB, chained through the
//     candidate's own candidate up to CHAIN times; a warp computes the nearest one 32 positions at a time (__match_any_sync), so no
//     atomics decide it;
//   * per position, the longest candidate match (the nearest wins a tie), then a greedy parse from 0: a token is a match of >= 4 bytes
//     or a literal;
//   * code lengths from the symbol histograms (Moffat-Katajainen, limited to 15 / 7 bits by the JPEG Annex K.3 count adjustment), with
//     zlib's rule that every tree has at least two codes;
//   * the smallest of a stored, a fixed-Huffman and a dynamic-Huffman block, sized from the histograms before anything is written;
//   * every token's bits at the offset an exclusive scan of the per-token bit counts gives it, OR-ed into the bit buffer (disjoint bits:
//     the order of the ORs does not matter).
#pragma once
#include <stdint.h>
#include "ingest_core.h"        // CrcTables / crc32_group, ld32u, warp helpers, SNFB_HD

namespace deflate {

constexpr uint32_t BLOCK_IN = 0xff00;          // input bytes per BGZF block (htslib's BGZF_BLOCK_SIZE)
constexpr uint32_t MEMBER_MAX = 65536;         // a BGZF member's size limit (BSIZE is 16 bits)
constexpr uint32_t HEADER_BYTES = 18, TRAILER_BYTES = 8;
constexpr uint32_t WINDOW = 32768;
constexpr int HASH_BITS = 15, CHAIN = 8, MIN_MATCH = 4, MAX_MATCH = 258;
constexpr int MAX_THREADS = 512;

struct alignas(16) Shared {
    uint8_t data[BLOCK_IN + 64];                               // the block's bytes; 64 zero bytes behind the last one
    union { uint16_t head[1 << HASH_BITS]; uint8_t len[1 << 16]; } lh;   // hash heads (position + 1) while candidates are found, then match length - 3 per position
    uint32_t bits[MEMBER_MAX / 4];                             // the DEFLATE stream being written
    uint32_t start[(BLOCK_IN + 31) / 32];                      // token starts of the greedy parse
    ingest::CrcTables crc;
    uint32_t lit_freq[288], dist_freq[32], clen_freq[20];
    uint32_t sym[288], work[288];                              // Huffman construction: symbols by frequency, frequencies -> lengths
    uint32_t part[MAX_THREADS];                                // bits per thread slice, then each slice's bit offset
    uint32_t blc[32];                                          // codes per length
    uint16_t lit_code[288], dist_code[32], clen_code[20], rle[320];   // codes bit-reversed for LSB-first output; code-length ops (sym | extra << 5)
    uint8_t lit_len[288], dist_len[32], clen_len[20];
    uint32_t n, crc_val, btype, n_rle, hlit, hdist, hclen, hdr_bits, total_bits, slice;
};

// ---------------------------------------------------------------- helpers (the identity / plain operation on the host)
SNFB_HD uint32_t ctz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)(__ffs((int)x) - 1);
#else
    return (uint32_t)__builtin_ctz(x);
#endif
}
SNFB_HD uint32_t clz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return (uint32_t)__clz((int)x);
#else
    return x ? (uint32_t)__builtin_clz(x) : 32u;
#endif
}
SNFB_HD void add_sh(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicAdd(p, v);
#else
    *p += v;
#endif
}
SNFB_HD void or_sh(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
template <int NL> SNFB_HD uint32_t ballot(bool p) {
#if defined(__CUDA_ARCH__)
    if (NL > 1) return __ballot_sync(0xffffffffu, p);
#endif
    return p ? 1u : 0u;
}
// lanes of the warp holding the same key (only this lane for NL = 1)
template <int NL> SNFB_HD uint32_t match_any(uint32_t key, int lane) {
#if defined(__CUDA_ARCH__)
    if (NL > 1) return __match_any_sync(0xffffffffu, key);
#endif
    (void)key; return 1u << lane;
}
SNFB_HD uint32_t hash4(uint32_t w) { return (w * 0x9E3779B1u) >> (32 - HASH_BITS); }

// length symbol (257..285) and extra bits of a match length 3..258; distance symbol (0..29) and extra bits of 1..32768 (RFC 1951 §3.2.5)
SNFB_HD void len_code(uint32_t len, uint32_t* sym, uint32_t* ebits, uint32_t* eval) {
    const uint32_t l = len - 3u;
    if (l < 8u) { *sym = 257u + l; *ebits = 0; *eval = 0; return; }
    if (l == 255u) { *sym = 285u; *ebits = 0; *eval = 0; return; }
    const uint32_t e = 31u - clz32(l) - 2u;
    *sym = 257u + 4u * e + (l >> e); *ebits = e; *eval = l & ((1u << e) - 1u);
}
SNFB_HD void dist_code(uint32_t dist, uint32_t* sym, uint32_t* ebits, uint32_t* eval) {
    const uint32_t d = dist - 1u;
    if (d < 4u) { *sym = d; *ebits = 0; *eval = 0; return; }
    const uint32_t e = 31u - clz32(d) - 1u;
    *sym = 2u * e + (d >> e); *ebits = e; *eval = d & ((1u << e) - 1u);
}
SNFB_HD uint32_t lit_extra(uint32_t s) { return (s >= 265u && s < 285u) ? (s - 261u) >> 2 : 0u; }
SNFB_HD uint32_t dist_extra(uint32_t s) { return s >= 4u ? (s >> 1) - 1u : 0u; }
SNFB_HD uint32_t fixed_lit_len(uint32_t s) { return s < 144u ? 8u : (s < 256u ? 9u : (s < 280u ? 7u : 8u)); }

SNFB_HD bool is_start(const Shared* S, uint32_t i) { return (S->start[i >> 5] >> (i & 31u)) & 1u; }

// OR nbits (<= 57) of v into the bit buffer at bit offset off
SNFB_HD void put_bits(Shared* S, uint32_t off, uint64_t v, uint32_t nbits) {
    if (!nbits) return;
    const uint32_t w = off >> 5, sh = off & 31u;
    const uint32_t w0 = (uint32_t)(v << sh);
    const uint64_t hi = sh ? (v >> (32u - sh)) : (v >> 32);
    or_sh(&S->bits[w], w0);
    if (sh + nbits > 32u) or_sh(&S->bits[w + 1], (uint32_t)hi);
    if (sh + nbits > 64u) or_sh(&S->bits[w + 2], (uint32_t)(hi >> 32));
}

// ---------------------------------------------------------------- phase 1: stage the block, clear the per-block state
SNFB_HD void stage(Shared* S, const uint8_t* in, uint32_t n, int tid, int nt) {
#if defined(__CUDA_ARCH__)
    // 16-byte loads when `in` is 16-byte aligned (fixed cuts start at multiples of 0xff00); byte loads for a member cut anywhere
    const uint32_t n16 = ((uintptr_t)in & 15u) ? 0u : n >> 4;
    for (uint32_t j = tid; j < n16; j += nt) reinterpret_cast<uint4*>(S->data)[j] = reinterpret_cast<const uint4*>(in)[j];
    for (uint32_t j = 16u * n16 + tid; j < n; j += nt) S->data[j] = in[j];
#else
    memcpy(S->data, in, n);
#endif
    for (uint32_t j = n + tid; j < BLOCK_IN + 64u; j += nt) S->data[j] = 0;
    uint32_t* h = reinterpret_cast<uint32_t*>(S->lh.head);
    for (uint32_t j = tid; j < (1u << HASH_BITS) / 2u; j += nt) h[j] = 0;
    for (uint32_t j = tid; j < MEMBER_MAX / 4u; j += nt) S->bits[j] = 0;
    for (uint32_t j = tid; j < (BLOCK_IN + 31u) / 32u; j += nt) S->start[j] = 0;
    for (uint32_t j = tid; j < 288u; j += nt) S->lit_freq[j] = 0;
    for (uint32_t j = tid; j < 32u; j += nt) S->dist_freq[j] = 0;
    if (tid == 0) S->n = n;
}

// ---------------------------------------------------------------- phase 2: nearest earlier position with the same hash (warp, NL lanes)
// cand[i] = distance to it (0 = none within the window).  Positions go NL at a time: a lane takes the nearest lower lane of its hash
// group, the group's lowest lane the head table (the last position of that hash before the tile), and the group's highest lane
// becomes the new head.
template <int NL>
SNFB_HD void find_candidates(Shared* S, uint16_t* cand, int lane) {
    const uint32_t n = S->n;
    for (uint32_t base = 0; base < n; base += NL) {
        const uint32_t i = base + (uint32_t)lane;
        const bool valid = i + 4u <= n;
        const uint32_t h = valid ? hash4(ingest::ld32u(S->data, i)) : 0u;
        const uint32_t peers = match_any<NL>(valid ? h : (1u << 16) + (uint32_t)lane, lane);
        const uint32_t lower = peers & ((1u << lane) - 1u), higher = peers & ~((2u << lane) - 1u);
        uint32_t c = 0;                                        // candidate position + 1
        if (valid) c = lower ? base + (31u - clz32(lower)) + 1u : S->lh.head[h];
        ingest::warp_sync();                                   // every lane has read the head before the group's last lane replaces it
        if (i < n) cand[i] = (uint16_t)((c && i + 1u - c <= WINDOW) ? i + 1u - c : 0u);
        if (valid && !higher) S->lh.head[h] = (uint16_t)(i + 1u);
        ingest::warp_sync();
    }
}

// ---------------------------------------------------------------- phase 3: longest match per position (every thread)
SNFB_HD uint32_t match_len(const uint8_t* d, uint32_t a, uint32_t b, uint32_t maxl) {
    uint32_t l = 0;
    while (l < maxl) {
        const uint32_t x = ingest::ld32u(d, a + l) ^ ingest::ld32u(d, b + l);
        if (x) { l += ctz32(x) >> 3; break; }
        l += 4u;
    }
    return l < maxl ? l : maxl;
}
// lh.len[i] = match length - 3 (0 = no match of MIN_MATCH or more), dist[i] = its distance.  Reads cand[] of earlier positions.
SNFB_HD void longest_matches(Shared* S, const uint16_t* cand, uint16_t* dist, int tid, int nt) {
    const uint32_t n = S->n;
    for (uint32_t i = tid; i < n; i += nt) {
        uint32_t best = 0, bd = 0;
        if (i + (uint32_t)MIN_MATCH <= n) {
            const uint32_t maxl = n - i < (uint32_t)MAX_MATCH ? n - i : (uint32_t)MAX_MATCH;
            uint32_t c = i, tot = 0;
            for (int k = 0; k < CHAIN; ++k) {
                const uint32_t d = cand[c];
                if (!d || tot + d > WINDOW) break;
                tot += d; c = i - tot;
                const uint32_t l = match_len(S->data, c, i, maxl);
                if (l > best) { best = l; bd = tot; if (l == maxl) break; }
            }
        }
        if (best < (uint32_t)MIN_MATCH) best = bd = 0;
        S->lh.len[i] = (uint8_t)(best ? best - 3u : 0u);
        dist[i] = (uint16_t)bd;
    }
}

// ---------------------------------------------------------------- phase 4: greedy parse from position 0 (warp, NL lanes)
// Positions go NL at a time; inside a tile the walk jumps from the current token start straight to the next position with a match
// (every position between is a literal token), then past the match.
template <int NL>
SNFB_HD void greedy_parse(Shared* S, int lane) {
    const uint32_t n = S->n;
    const uint32_t wmask = NL == 32 ? 0xffffffffu : ((1u << NL) - 1u);
    uint32_t p = 0;
    for (uint32_t base = 0; base < n; base += NL) {
        if (p >= base + NL) continue;                          // inside a match
        const uint32_t i = base + (uint32_t)lane;
        const uint32_t l = i < n ? S->lh.len[i] : 0u;
        const uint32_t mask = ballot<NL>(l != 0u);
        uint32_t r = p - base, words = 0;
        while (r < (uint32_t)NL) {
            const uint32_t mm = mask >> r;
            if (!mm) { words |= (wmask << r) & wmask; break; }
            const uint32_t q = r + ctz32(mm);
            words |= (q >= 31u ? 0xffffffffu : ((2u << q) - 1u)) & ~((1u << r) - 1u) & wmask;
            r = q + ingest::warp_shfl<NL>(l, (int)q) + 3u;
        }
        if (r < (uint32_t)NL) r = NL;
        p = base + r;
        if (lane == 0) {
            if (NL == 32) S->start[base >> 5] = words;
            else if (words & 1u) S->start[base >> 5] |= 1u << (base & 31u);
        }
    }
}

// ---------------------------------------------------------------- phase 5: symbol histograms (every thread)
SNFB_HD void histogram(Shared* S, const uint16_t* dist, int tid, int nt) {
    const uint32_t n = S->n;
    for (uint32_t i = tid; i < n; i += nt) {
        if (!is_start(S, i)) continue;
        const uint32_t l = S->lh.len[i];
        if (l) {
            uint32_t s, e, v;
            len_code(l + 3u, &s, &e, &v); add_sh(&S->lit_freq[s], 1u);
            dist_code(dist[i], &s, &e, &v); add_sh(&S->dist_freq[s], 1u);
        } else add_sh(&S->lit_freq[S->data[i]], 1u);
    }
    if (tid == 0) add_sh(&S->lit_freq[256], 1u);              // end of block
}

// ---------------------------------------------------------------- phase 6: codes and block type (one thread)
// Huffman code lengths of freq[0 .. n) limited to `limit` bits, into len[].  Symbols with a zero count get length 0; when fewer than two
// symbols occur, the lowest unused ones get count 1 (zlib's build_tree), so every tree has two codes and every inflater accepts it.
SNFB_HD void huff_lengths(Shared* S, const uint32_t* freq, int n, int limit, uint8_t* len) {
    uint32_t* sym = S->sym; uint32_t* A = S->work; uint32_t* blc = S->blc;
    int m = 0, nz = 0;
    for (int s = 0; s < n; ++s) nz += freq[s] != 0;
    for (int s = 0; s < n; ++s) {
        uint32_t f = freq[s];
        if (!f && nz < 2) { f = 1; ++nz; }
        len[s] = 0;
        if (!f) continue;
        int j = m++;                                           // insertion sort by (frequency, symbol)
        while (j > 0 && A[j - 1] > f) { A[j] = A[j - 1]; sym[j] = sym[j - 1]; --j; }
        A[j] = f; sym[j] = (uint32_t)s;
    }
    // Moffat & Katajainen, "In-place calculation of minimum-redundancy codes" (1995): A[] ascending -> code lengths in place
    A[0] += A[1];
    int root = 0, leaf = 2;
    for (int next = 1; next < m - 1; ++next) {
        if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = (uint32_t)next; } else A[next] = A[leaf++];
        if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = (uint32_t)next; } else A[next] += A[leaf++];
    }
    A[m - 2] = 0;
    for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1u;
    int avbl = 1, used = 0, dpth = 0, next = m - 1; root = m - 2;
    while (avbl > 0) {
        while (root >= 0 && (int)A[root] == dpth) { ++used; --root; }
        while (avbl > used) { A[next--] = (uint32_t)dpth; --avbl; }
        avbl = 2 * used; ++dpth; used = 0;
    }
    // lengths over the limit: JPEG (ITU T.81) Annex K.3 adjustment of the per-length counts, which keeps the code complete
    for (int l = 0; l < 32; ++l) blc[l] = 0;
    for (int k = 0; k < m; ++k) blc[A[k] < 31u ? A[k] : 31u]++;
    for (int l = 31; l > limit; --l) {
        while (blc[l] > 0) {
            int j = l - 2;
            while (blc[j] == 0) --j;
            blc[l] -= 2; blc[l - 1] += 1; blc[j + 1] += 2; blc[j] -= 1;
        }
    }
    // the most frequent symbols take the shortest codes
    int k = m - 1;
    for (int l = 1; l <= limit; ++l) for (uint32_t c = 0; c < blc[l]; ++c) len[sym[k--]] = (uint8_t)l;
}
// canonical codes (RFC 1951 §3.2.2), bit-reversed
SNFB_HD void canonical_codes(Shared* S, const uint8_t* len, int n, uint16_t* code) {
    uint32_t* blc = S->blc; uint32_t nextc[16];
    for (int l = 0; l < 16; ++l) blc[l] = 0;
    for (int s = 0; s < n; ++s) blc[len[s]]++;
    blc[0] = 0; uint32_t c = 0;
    for (int l = 1; l < 16; ++l) { c = (c + blc[l - 1]) << 1; nextc[l] = c; }
    for (int s = 0; s < n; ++s) code[s] = len[s] ? (uint16_t)ingest::bitrev(nextc[len[s]]++, len[s]) : (uint16_t)0;
}
SNFB_HD uint32_t rle_extra_bits(uint32_t sym) { return sym == 16u ? 2u : (sym == 17u ? 3u : (sym == 18u ? 7u : 0u)); }

SNFB_HD void plan(Shared* S) {
    const uint32_t n = S->n;
    huff_lengths(S, S->lit_freq, 286, 15, S->lit_len);
    huff_lengths(S, S->dist_freq, 30, 15, S->dist_len);
    S->lit_len[286] = S->lit_len[287] = 0; S->dist_len[30] = S->dist_len[31] = 0;
    uint32_t hlit = 286, hdist = 30;
    while (hlit > 257 && !S->lit_len[hlit - 1]) --hlit;
    while (hdist > 1 && !S->dist_len[hdist - 1]) --hdist;
    // code lengths of both trees as one sequence, run-length coded with 16 / 17 / 18 (RFC 1951 §3.2.7)
    for (int s = 0; s < 20; ++s) S->clen_freq[s] = 0;
    uint32_t nr = 0; const uint32_t tot = hlit + hdist;
    for (uint32_t i = 0; i < tot;) {
        const uint32_t v = i < hlit ? S->lit_len[i] : S->dist_len[i - hlit];
        uint32_t run = 1;
        while (i + run < tot && (i + run < hlit ? S->lit_len[i + run] : S->dist_len[i + run - hlit]) == v) ++run;
        i += run;
        if (v == 0) {
            while (run >= 11) { const uint32_t r = run < 138 ? run : 138; S->rle[nr++] = (uint16_t)(18u | ((r - 11u) << 5)); run -= r; }
            if (run >= 3) { S->rle[nr++] = (uint16_t)(17u | ((run - 3u) << 5)); run = 0; }
        } else {
            S->rle[nr++] = (uint16_t)v; --run;
            while (run >= 3) { const uint32_t r = run < 6 ? run : 6; S->rle[nr++] = (uint16_t)(16u | ((r - 3u) << 5)); run -= r; }
        }
        while (run) { S->rle[nr++] = (uint16_t)v; --run; }
    }
    for (uint32_t k = 0; k < nr; ++k) S->clen_freq[S->rle[k] & 31u]++;
    huff_lengths(S, S->clen_freq, 19, 7, S->clen_len);
    uint32_t hclen = 19;
    while (hclen > 4 && !S->clen_len[ingest::clen_order((int)hclen - 1)]) --hclen;
    // sizes from the histograms
    uint64_t dyn = 3 + 14 + 3ull * hclen, fix = 3, extra = 0;
    for (uint32_t k = 0; k < nr; ++k) { const uint32_t s = S->rle[k] & 31u; dyn += S->clen_len[s] + rle_extra_bits(s); }
    const uint32_t hdr_dyn = (uint32_t)dyn;
    for (uint32_t s = 0; s < 286; ++s) { dyn += (uint64_t)S->lit_freq[s] * S->lit_len[s]; fix += (uint64_t)S->lit_freq[s] * fixed_lit_len(s); extra += (uint64_t)S->lit_freq[s] * lit_extra(s); }
    for (uint32_t s = 0; s < 30; ++s) { dyn += (uint64_t)S->dist_freq[s] * S->dist_len[s]; fix += 5ull * S->dist_freq[s]; extra += (uint64_t)S->dist_freq[s] * dist_extra(s); }
    dyn += extra; fix += extra;
    const uint64_t stored_bytes = (uint64_t)n + 5u, dyn_bytes = (dyn + 7) / 8, fix_bytes = (fix + 7) / 8;
    S->n_rle = nr; S->hlit = hlit; S->hdist = hdist; S->hclen = hclen;
    if (stored_bytes <= dyn_bytes && stored_bytes <= fix_bytes) { S->btype = 0; return; }
    if (fix_bytes <= dyn_bytes) {
        S->btype = 1; S->hdr_bits = 3;
        for (uint32_t s = 0; s < 288; ++s) S->lit_len[s] = (uint8_t)fixed_lit_len(s);
        for (uint32_t s = 0; s < 32; ++s) S->dist_len[s] = 5;
    } else {
        S->btype = 2; S->hdr_bits = hdr_dyn;
        canonical_codes(S, S->clen_len, 19, S->clen_code);
    }
    canonical_codes(S, S->lit_len, 288, S->lit_code);
    canonical_codes(S, S->dist_len, 32, S->dist_code);
}

// ---------------------------------------------------------------- phase 7: the bit stream (every thread, then thread 0, then every thread)
// the bits of the token that starts at i: *nbits of them, in v
SNFB_HD uint64_t token_bits(const Shared* S, const uint16_t* dist, uint32_t i, uint32_t* nbits) {
    const uint32_t l = S->lh.len[i];
    if (!l) { const uint32_t b = S->data[i]; *nbits = S->lit_len[b]; return S->lit_code[b]; }
    uint32_t ls, le, lv, ds, de, dv;
    len_code(l + 3u, &ls, &le, &lv); dist_code(dist[i], &ds, &de, &dv);
    const uint32_t l1 = S->lit_len[ls], l2 = S->dist_len[ds];
    uint64_t v = S->lit_code[ls];
    v |= (uint64_t)lv << l1;
    v |= (uint64_t)S->dist_code[ds] << (l1 + le);
    v |= (uint64_t)dv << (l1 + le + l2);
    *nbits = l1 + le + l2 + de;
    return v;
}
// every thread owns a contiguous slice of positions; its bit count
SNFB_HD void count_bits(Shared* S, const uint16_t* dist, int tid, int nt) {
    const uint32_t n = S->n;
    uint32_t sl = (n + (uint32_t)nt - 1u) / (uint32_t)nt;
    sl = (sl + 3u) & ~3u; if (nt > 1 && !((sl >> 2) & 1u)) sl += 4u;      // an odd number of words apart: the slices fall in different banks
    const uint32_t b = (uint32_t)tid * sl < n ? (uint32_t)tid * sl : n, e = b + sl < n ? b + sl : n;
    uint32_t bits = 0, nb;
    for (uint32_t i = b; i < e; ++i) if (is_start(S, i)) { token_bits(S, dist, i, &nb); bits += nb; }
    S->part[tid] = bits;
    if (tid == 0) S->slice = sl;
}
// thread 0: slice offsets, the block header and the end-of-block code
SNFB_HD void write_header(Shared* S, int nt) {
    uint32_t off = S->hdr_bits;
    for (int t = 0; t < nt; ++t) { const uint32_t b = S->part[t]; S->part[t] = off; off += b; }
    put_bits(S, 0, 1u | (S->btype << 1), 3);                 // BFINAL = 1
    if (S->btype == 2) {
        uint32_t o = 3;
        put_bits(S, o, (S->hlit - 257u) | ((S->hdist - 1u) << 5) | ((S->hclen - 4u) << 10), 14); o += 14;
        for (uint32_t k = 0; k < S->hclen; ++k) { put_bits(S, o, S->clen_len[ingest::clen_order((int)k)], 3); o += 3; }
        for (uint32_t k = 0; k < S->n_rle; ++k) {
            const uint32_t s = S->rle[k] & 31u, x = rle_extra_bits(s);
            put_bits(S, o, S->clen_code[s] | ((uint64_t)(S->rle[k] >> 5) << S->clen_len[s]), S->clen_len[s] + x); o += S->clen_len[s] + x;
        }
    }
    put_bits(S, off, S->lit_code[256], S->lit_len[256]);
    S->total_bits = off + S->lit_len[256];
}
SNFB_HD void write_tokens(Shared* S, const uint16_t* dist, int tid) {
    const uint32_t n = S->n, sl = S->slice;
    const uint32_t b = (uint32_t)tid * sl < n ? (uint32_t)tid * sl : n, e = b + sl < n ? b + sl : n;
    uint32_t off = S->part[tid], nb;
    for (uint32_t i = b; i < e; ++i) if (is_start(S, i)) { const uint64_t v = token_bits(S, dist, i, &nb); put_bits(S, off, v, nb); off += nb; }
}

// ---------------------------------------------------------------- phase 8: the gzip member (every thread); returns its size
SNFB_HD uint32_t write_member(const Shared* S, uint8_t* out, int tid, int nt) {
    const uint32_t n = S->n;
    const uint32_t dbytes = S->btype == 0 ? n + 5u : (S->total_bits + 7u) >> 3;
    const uint32_t size = HEADER_BYTES + dbytes + TRAILER_BYTES;
    if (S->btype == 0) {
        for (uint32_t j = tid; j < n; j += nt) out[HEADER_BYTES + 5u + j] = S->data[j];
    } else {
        const uint8_t* src = reinterpret_cast<const uint8_t*>(S->bits);
        for (uint32_t j = tid; j < dbytes; j += nt) out[HEADER_BYTES + j] = src[j];
    }
    if (tid == 0) {
        const uint8_t hdr[16] = { 0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0 };
        for (int k = 0; k < 16; ++k) out[k] = hdr[k];
        out[16] = (uint8_t)((size - 1u) & 255u); out[17] = (uint8_t)((size - 1u) >> 8);
        if (S->btype == 0) {
            out[18] = 1;                                       // BFINAL, stored, then LEN and NLEN
            out[19] = (uint8_t)(n & 255u); out[20] = (uint8_t)(n >> 8); out[21] = (uint8_t)(~n & 255u); out[22] = (uint8_t)((~n >> 8) & 255u);
        }
        uint8_t* t = out + HEADER_BYTES + dbytes;
        for (int k = 0; k < 4; ++k) { t[k] = (uint8_t)(S->crc_val >> (8 * k)); t[4 + k] = (uint8_t)(n >> (8 * k)); }
    }
    return size;
}

}  // namespace deflate
