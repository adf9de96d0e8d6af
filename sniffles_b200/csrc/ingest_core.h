// ingest_core.h — SURVEY §8 (f)3: the per-warp pieces of the device BAM ingest — DEFLATE (RFC 1951) of one BGZF block, BAM record
// decode, BAM CIGAR words -> CIGAR16.  Replaces htslib behind `pysam.AlignmentFile.fetch` (call sites parallel.py:95-98,
// leadprov.py:488) for the fields the path reads (SURVEY §8a A0).
//
// Everything here is written for "a warp that executes the scalar decode redundantly": all NL lanes run the same control flow on
// the same values (bit buffer, positions, symbols live in registers, identical in every lane; table look-ups hit one shared-memory
// address and broadcast), so no lane ever waits for a broadcast, and the parts that ARE data parallel — filling the look-up
// tables, LZ77 match copies, stored blocks, byte copies — are split across the lanes.  With NL = 1 the same code is plain
// sequential C++: tests/native/ingest_host.cpp and crc_host.cpp compile this header with g++ and check it against zlib on the CPU (test
// infrastructure).  The kernels instantiate inflate_stream<16>, crc32_group<16> and c16_convert<32>, the host CIGAR16 conversion (api.cu)
// c16_convert<1>.
#pragma once
#include <stdint.h>
#include "cigar16.h"            // also defines SNFB_HD
#if defined(__CUDACC__)
#define SNFB_HDN __host__ __device__ __noinline__
#else
#include <string.h>
#define SNFB_HDN inline
#endif

namespace ingest {

// ---------------------------------------------------------------- lane helpers (identity for NL = 1)
SNFB_HD void warp_sync() {
#if defined(__CUDA_ARCH__)
    __syncwarp();
#endif
}
template <int NL> SNFB_HD bool warp_any(bool p) {
#if defined(__CUDA_ARCH__)
    if (NL > 1) return __any_sync(0xffffffffu, p);
#endif
    return p;
}
template <int NL> SNFB_HD uint32_t warp_shfl(uint32_t v, int src) {
#if defined(__CUDA_ARCH__)
    if (NL > 1) return __shfl_sync(0xffffffffu, v, src);
#endif
    (void)src; return v;
}
template <int NL> SNFB_HD long long warp_sum(long long v) {
#if defined(__CUDA_ARCH__)
    if (NL > 1) { for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o); }
#endif
    return v;
}
// unaligned little-endian 32-bit load; `base` is 4-byte aligned and the buffer has at least 8 bytes of slack behind its last byte
SNFB_HD uint32_t ld32u(const uint8_t* base, uint64_t off) {
#if defined(__CUDA_ARCH__)
    const uint64_t a = off & ~3ull; const unsigned sh = (unsigned)(off & 3ull) * 8u;
    const uint32_t w0 = *reinterpret_cast<const uint32_t*>(base + a);
    if (sh == 0) return w0;
    const uint32_t w1 = *reinterpret_cast<const uint32_t*>(base + a + 4);
    return __funnelshift_r(w0, w1, sh);
#else
    uint32_t v; memcpy(&v, base + off, 4); return v;
#endif
}
SNFB_HD uint32_t ld16u(const uint8_t* base, uint64_t off) { return (uint32_t)base[off] | ((uint32_t)base[off + 1] << 8); }
SNFB_HD unsigned bitrev(unsigned c, int len) {
#if defined(__CUDA_ARCH__)
    return __brev(c) >> (32 - len);
#else
    unsigned r = 0; for (int i = 0; i < len; ++i) { r = (r << 1) | ((c >> i) & 1u); } return r;
#endif
}

// ---------------------------------------------------------------- Huffman tables of one warp (shared memory)
constexpr int LIT_FAST_BITS = 9, DIST_FAST_BITS = 7;
struct WarpTables {
    uint16_t lit_fast[1 << LIT_FAST_BITS];      // (symbol << 4) | code length for codes of at most 9 bits; 0 = longer code
    uint16_t dist_fast[1 << DIST_FAST_BITS];    // same for distance codes (7 bits); also the code-length code while a dynamic header is read
    uint16_t lit_count[16], dist_count[16];     // codes per length (canonical decode of the long codes, as zlib's puff does)
    uint16_t lit_sym[288], dist_sym[32];        // symbols in canonical order
    uint8_t lens[320];                          // code lengths being read
};

enum { INF_OK = 0, INF_BAD_BLOCK_TYPE = 1, INF_BAD_STORED = 2, INF_BAD_CODE = 3, INF_OVERSUBSCRIBED = 4, INF_BAD_SYMBOL = 5, INF_BAD_DISTANCE = 6, INF_OUTPUT_OVERRUN = 7, INF_INPUT_OVERRUN = 8, INF_LENGTH_MISMATCH = 9,
       INF_CRC_MISMATCH = 10 };

// A decoding group = NL lanes of a warp (NL = 32: the whole warp; NL = 16 / 8: two / four BGZF blocks per warp, each decoded by its own
// lanes with its own tables — the groups share the warp's instruction stream wherever they happen to take the same path, and
// diverge like any threads where they do not).  gmask = the lanes of the group, for __syncwarp.
SNFB_HD void group_sync(unsigned gmask) {
#if defined(__CUDA_ARCH__)
    __syncwarp(gmask);
#else
    (void)gmask;
#endif
}

// canonical Huffman code from code lengths: per-length counts, symbols in code order, and the look-up table for codes of at most
// `fbits` bits (bit-reversed: DEFLATE packs codes starting at the most significant bit into a stream read from the least).
// Returns < 0 when the lengths over-subscribe the code space, otherwise the unused code space (0 = complete).
template <int NL>
SNFB_HD int huff_build(const uint8_t* lens, int n, uint16_t* count, uint16_t* symtab, uint16_t* fast, int fbits, int lane, unsigned gmask) {
    group_sync(gmask);                                 // lens[] was written by lane 0
    if (lane == 0) {
        for (int l = 0; l < 16; ++l) count[l] = 0;
        for (int s = 0; s < n; ++s) count[lens[s]]++;
    }
    for (int j = lane; j < (1 << fbits); j += NL) fast[j] = 0;
    group_sync(gmask);
    int left = 1;
    for (int len = 1; len <= 15; ++len) { left <<= 1; left -= (int)count[len]; if (left < 0) return -1; }
    if (lane == 0) {
        uint16_t offs[16]; offs[1] = 0;
        for (int len = 1; len < 15; ++len) offs[len + 1] = (uint16_t)(offs[len] + count[len]);
        for (int s = 0; s < n; ++s) if (lens[s]) symtab[offs[lens[s]]++] = (uint16_t)s;
    }
    group_sync(gmask);
    unsigned code = 0, idx = 0;
    for (int len = 1; len <= fbits; ++len) {
        const unsigned cnt = count[len];
        for (unsigned k = lane; k < cnt; k += NL) {
            const unsigned s = symtab[idx + k], rev = bitrev(code + k, len);
            for (unsigned j = rev; j < (1u << fbits); j += 1u << len) fast[j] = (uint16_t)((s << 4) | (unsigned)len);
        }
        code = (code + cnt) << 1; idx += cnt;
    }
    group_sync(gmask);
    return left;
}

// a code longer than the look-up table: canonical decode bit by bit (zlib's puff).  Returns symbol | length << 16, or -1 = no such code
SNFB_HDN int huff_decode_slow(uint64_t bb, const uint16_t* count, const uint16_t* symtab) {
    int code = 0, first = 0, index = 0;
    for (int len = 1; len <= 15; ++len) {
        code |= (int)((bb >> (len - 1)) & 1u);
        const int cnt = count[len];
        if (code - cnt < first) return (int)symtab[index + (code - first)] | (len << 16);
        index += cnt; first += cnt; first <<= 1; code <<= 1;
    }
    return -1;
}
// next symbol from the low bits of bb; *nbits = its code length; -1 = no such code
SNFB_HD int huff_decode(uint64_t bb, const uint16_t* fast, int fbits, const uint16_t* count, const uint16_t* symtab, int* nbits) {
    const unsigned e = fast[(unsigned)bb & ((1u << fbits) - 1u)];
    if (e) { *nbits = (int)(e & 15u); return (int)(e >> 4); }
    const int r = huff_decode_slow(bb, count, symtab);
    *nbits = r < 0 ? 0 : r >> 16;
    return r < 0 ? -1 : (r & 0xffff);
}

// order in which a dynamic header stores the code-length code lengths (RFC 1951 §3.2.7), 5 bits each
SNFB_HD int clen_order(int i) {
    const uint64_t lo = 16ull | (17ull << 5) | (18ull << 10) | (0ull << 15) | (8ull << 20) | (7ull << 25) | (9ull << 30) | (6ull << 35) | (10ull << 40) | (5ull << 45) | (11ull << 50) | (4ull << 55);
    const uint64_t hi = 12ull | (3ull << 5) | (13ull << 10) | (2ull << 15) | (14ull << 20) | (1ull << 25) | (15ull << 30);
    return (int)(((i < 12 ? lo >> (5 * i) : hi >> (5 * (i - 12)))) & 31ull);
}

// the i-th 32-bit word of the stream, counted from the 4-byte aligned address at or below its first byte (one aligned load on the device)
SNFB_HD uint32_t stream_word(const uint8_t* base, uint32_t i) {
#if defined(__CUDA_ARCH__)
    return reinterpret_cast<const uint32_t*>(base)[i];
#else
    uint32_t v; memcpy(&v, base + 4ull * i, 4); return v;
#endif
}

// Inflate one raw DEFLATE stream in[ipos .. iend) into out[0 .. out_cap); every lane of the group calls it with the same arguments
// (lane = its index in the group, NL = lanes, gmask = the group's lanes in the warp).  `in` is 4-byte aligned with 16 readable bytes
// behind iend.  Returns INF_*; *out_len = bytes produced.
template <int NL>
SNFB_HD int inflate_stream(const uint8_t* in, uint64_t ipos, uint64_t iend, uint8_t* out, uint32_t out_cap, WarpTables* T, int lane, unsigned gmask, uint32_t* out_len) {
    const uint8_t* base = in + (ipos & ~3ull);                                    // the stream as aligned 32-bit words
    const uint32_t iend_rel = (uint32_t)(ipos & 3ull) + (uint32_t)(iend - ipos);    // its end, in bytes from base
    const uint32_t iw_limit = ((iend_rel + 3u) >> 2) + 2u;                          // words a well-formed stream can touch (8 bytes of look-ahead)
    uint64_t bb = 0; int bc = 0; uint32_t iw = 0, op = 0; int err = INF_OK; bool last = false, ovr = false;
#define SNFB_REFILL() do { if (bc <= 32) { uint32_t w_ = 0; if (iw < iw_limit) w_ = stream_word(base, iw); else ovr = true; bb |= (uint64_t)w_ << bc; ++iw; bc += 32; } } while (0)
#define SNFB_TAKE(n) do { bb >>= (n); bc -= (n); } while (0)
    SNFB_REFILL(); SNFB_TAKE(8 * (int)(ipos & 3ull));
    do {
        group_sync(gmask);                             // nobody still reads the previous block's tables
        if (ovr) break;
        SNFB_REFILL();
        last = (bb & 1u) != 0; const unsigned type = (unsigned)(bb >> 1) & 3u; SNFB_TAKE(3);
        if (type == 0) {                               // stored
            SNFB_TAKE(bc & 7);
            uint32_t rel = 4u * iw - (uint32_t)(bc >> 3);      // first unread byte
            if (rel + 4u > iend_rel) { err = INF_BAD_STORED; break; }
            const uint32_t len = ld16u(base, rel), nlen = ld16u(base, rel + 2); rel += 4;
            if ((len ^ 0xffffu) != nlen || rel + len > iend_rel) { err = INF_BAD_STORED; break; }
            if (op + len > out_cap) { err = INF_OUTPUT_OVERRUN; break; }
            for (uint32_t j = lane; j < len; j += NL) out[op + j] = base[rel + j];
            op += len; rel += len;
            iw = rel >> 2; bb = 0; bc = 0;
            SNFB_REFILL(); SNFB_TAKE(8 * (int)(rel & 3u));
            continue;
        }
        if (type == 3) { err = INF_BAD_BLOCK_TYPE; break; }
        int nlit, ndist;
        if (type == 1) {                               // fixed code
            if (lane == 0) {
                for (int s = 0; s < 144; ++s) T->lens[s] = 8;
                for (int s = 144; s < 256; ++s) T->lens[s] = 9;
                for (int s = 256; s < 280; ++s) T->lens[s] = 7;
                for (int s = 280; s < 288; ++s) T->lens[s] = 8;
                for (int s = 0; s < 30; ++s) T->lens[288 + s] = 5;
            }
            nlit = 288; ndist = 30;
        } else {                                       // dynamic code
            SNFB_REFILL();
            nlit = (int)(bb & 31u) + 257; ndist = (int)((bb >> 5) & 31u) + 1; const int nclen = (int)((bb >> 10) & 15u) + 4; SNFB_TAKE(14);
            if (nlit > 286 || ndist > 30) { err = INF_BAD_CODE; break; }
            if (lane == 0) for (int i = 0; i < 19; ++i) T->lens[i] = 0;
            group_sync(gmask);
            for (int i = 0; i < nclen; ++i) { SNFB_REFILL(); if (lane == 0) T->lens[clen_order(i)] = (uint8_t)(bb & 7u); SNFB_TAKE(3); }
            if (huff_build<NL>(T->lens, 19, T->dist_count, T->dist_sym, T->dist_fast, DIST_FAST_BITS, lane, gmask) != 0) { err = INF_BAD_CODE; break; }   // the code-length code must be complete
            int i = 0, prev = 0;
            while (i < nlit + ndist) {
                SNFB_REFILL();
                int nb; const int sym = huff_decode(bb, T->dist_fast, DIST_FAST_BITS, T->dist_count, T->dist_sym, &nb);
                if (sym < 0) { err = INF_BAD_CODE; break; }
                SNFB_TAKE(nb);
                if (sym < 16) { if (lane == 0) T->lens[i] = (uint8_t)sym; prev = sym; ++i; continue; }
                int rep, val = 0;
                if (sym == 16) { if (i == 0) { err = INF_BAD_CODE; break; } val = prev; rep = 3 + (int)(bb & 3u); SNFB_TAKE(2); }
                else if (sym == 17) { rep = 3 + (int)(bb & 7u); SNFB_TAKE(3); }
                else { rep = 11 + (int)(bb & 127u); SNFB_TAKE(7); }
                if (i + rep > nlit + ndist) { err = INF_BAD_CODE; break; }
                if (lane == 0) for (int k = 0; k < rep; ++k) T->lens[i + k] = (uint8_t)val;
                i += rep; prev = val;
            }
            if (err) break;
            group_sync(gmask);
            if (T->lens[256] == 0) { err = INF_BAD_CODE; break; }      // no end-of-block code
            // the distance lengths follow the literal/length lengths: move them to their own base so both builds read aligned arrays
            if (lane == 0) { uint8_t tmp[32]; for (int k = 0; k < ndist; ++k) tmp[k] = T->lens[nlit + k]; for (int k = 0; k < ndist; ++k) T->lens[288 + k] = tmp[k]; }
        }
        if (huff_build<NL>(T->lens, nlit, T->lit_count, T->lit_sym, T->lit_fast, LIT_FAST_BITS, lane, gmask) < 0) { err = INF_OVERSUBSCRIBED; break; }
        if (huff_build<NL>(T->lens + 288, ndist, T->dist_count, T->dist_sym, T->dist_fast, DIST_FAST_BITS, lane, gmask) < 0) { err = INF_OVERSUBSCRIBED; break; }
        const uint16_t* lit_fast = T->lit_fast;
        for (;;) {
            SNFB_REFILL();
            unsigned e = lit_fast[(unsigned)bb & ((1u << LIT_FAST_BITS) - 1u)];
            int nb, sym;
            if (e) { nb = (int)(e & 15u); sym = (int)(e >> 4); }
            else { const int r_ = huff_decode_slow(bb, T->lit_count, T->lit_sym); if (r_ < 0) { err = INF_BAD_SYMBOL; break; } sym = r_ & 0xffff; nb = r_ >> 16; }
            SNFB_TAKE(nb);
            if (sym < 256) {                           // literal; the bits for a second one are already in the buffer (18 or more)
                if (op >= out_cap) { err = INF_OUTPUT_OVERRUN; break; }
                if (lane == 0) out[op] = (uint8_t)sym;
                ++op;
                e = lit_fast[(unsigned)bb & ((1u << LIT_FAST_BITS) - 1u)];
                if (e - 1u < (256u << 4) - 1u && op < out_cap) { SNFB_TAKE((int)(e & 15u)); if (lane == 0) out[op] = (uint8_t)(e >> 4); ++op; }
                continue;
            }
            if (sym == 256) break;
            // length and distance without a branch per case (RFC 1951 §3.2.5): every check of the match is folded into one test
            const unsigned s2 = (unsigned)sym - 257u;                                  // 0..28 are lengths; 28 = 258 without extra bits
            int x = s2 < 8u ? 0 : (int)(((s2 - 4u) >> 2) & 7u);
            uint32_t len = s2 < 8u ? s2 + 3u : 3u + ((4u + ((s2 - 4u) & 3u)) << x);
            if (s2 >= 28u) { len = 258u; x = 0; }
            len += (unsigned)bb & ((1u << x) - 1u); SNFB_TAKE(x);
            SNFB_REFILL();
            int dsym = huff_decode(bb, T->dist_fast, DIST_FAST_BITS, T->dist_count, T->dist_sym, &nb);
            bool bad = s2 > 28u || (unsigned)dsym > 29u;
            if (bad) dsym = 0;
            SNFB_TAKE(nb);
            const int dx = dsym < 4 ? 0 : (dsym >> 1) - 1;
            const uint32_t dist = (dsym < 4 ? (uint32_t)dsym + 1u : 1u + ((2u + (unsigned)(dsym & 1)) << dx)) + ((unsigned)bb & ((1u << dx) - 1u));
            SNFB_TAKE(dx);
            if (bad || dist > op || op + len > out_cap) { err = bad ? INF_BAD_SYMBOL : (dist > op ? INF_BAD_DISTANCE : INF_OUTPUT_OVERRUN); break; }
            group_sync(gmask);                         // the bytes the match reads were written by other lanes
            const uint8_t* src = out + op - dist; uint8_t* dst = out + op;
            if (dist >= len) { for (uint32_t j = lane; j < len; j += NL) dst[j] = src[j]; }
            else { for (uint32_t j = lane; j < len; j += NL) dst[j] = src[j % dist]; }
            op += len;
            if (ovr) break;
        }
    } while (!last && !err && !ovr);
#undef SNFB_REFILL
#undef SNFB_TAKE
    group_sync(gmask);
    *out_len = op;
    if (!err && (ovr || 4u * iw - (uint32_t)(bc >> 3) > iend_rel)) err = INF_INPUT_OVERRUN;
    return err;
}

// ---------------------------------------------------------------- CRC-32 of an inflated block (the gzip trailer every BGZF block carries)
// zlib's CRC-32: reflected polynomial 0xEDB88320, initial value and final XOR 0xFFFFFFFF.  A DEFLATE stream can be damaged and still
// decode to ISIZE bytes (any byte of a stored block, many bit flips in a Huffman-coded one); the CRC is what catches those, as htslib does.
constexpr uint32_t CRC_POLY = 0xEDB88320u;
struct CrcTables {
    uint32_t t[4][256];         // slice-by-4: t[k][b] = CRC register after byte b followed by k zero bytes
    uint32_t x8pow[32];         // x^(8 * 2^k) mod P: multiplying by it moves a CRC past 2^k bytes
};
SNFB_HD uint32_t crc_byte_step(uint32_t c) { for (int k = 0; k < 8; ++k) c = (c >> 1) ^ (CRC_POLY & (0u - (c & 1u))); return c; }
// fill the tables with threads tid = 0 .. nthreads - 1 (the caller synchronises them before use)
SNFB_HD void crc_tables_fill(CrcTables* C, int tid, int nthreads) {
    for (int i = tid; i < 256; i += nthreads) {
        uint32_t c = crc_byte_step((uint32_t)i); C->t[0][i] = c;
        for (int k = 1; k < 4; ++k) { c = (c >> 8) ^ crc_byte_step(c & 0xffu); C->t[k][i] = c; }
    }
    if (tid == 0) {
        // x^8 squared k times, in the reflected representation (x^0 = 0x80000000); zlib's x2n_table from its entry 3 on
        const uint32_t x8pow[32] = { 0x00800000u, 0x00008000u, 0xedb88320u, 0xb1e6b092u, 0xa06a2517u, 0xed627daeu, 0x88d14467u, 0xd7bbfe6au,
                                     0xec447f11u, 0x8e7ea170u, 0x6427800eu, 0x4d47bae0u, 0x09fe548fu, 0x83852d0fu, 0x30362f1au, 0x7b5a9cc3u,
                                     0x31fec169u, 0x9fec022au, 0x6c8dedc4u, 0x15d6874du, 0x5fde7a4eu, 0xbad90e37u, 0x2e4e5eefu, 0x4eaba214u,
                                     0xa8a472c0u, 0x429a969eu, 0x148d302au, 0xc40ba6d0u, 0xc4e22c3cu, 0x40000000u, 0x20000000u, 0x08000000u };
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
        for (int k = 0; k < 32; ++k) C->x8pow[k] = x8pow[k];
    }
}
// a * b mod P in the reflected representation (zlib's multmodp): at most 32 steps, fewer when a's low-order terms are zero
SNFB_HD uint32_t crc_multmodp(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) { p ^= b; if (!(a & (m - 1u))) break; }
        b = (b >> 1) ^ (CRC_POLY & (0u - (b & 1u)));
    }
    return p;
}
// CRC of A || B from crc(A), crc(B) and len(B) (zlib's crc32_combine): crc(A) times x^(8 len(B)), plus crc(B)
SNFB_HD uint32_t crc32_combine(uint32_t crc_a, uint32_t crc_b, uint32_t len_b, const uint32_t* x8pow) {
    uint32_t xn = 1u << 31;
    for (int k = 0; len_b; ++k, len_b >>= 1) if (len_b & 1u) xn = crc_multmodp(x8pow[k], xn);
    return crc_multmodp(xn, crc_a) ^ crc_b;
}
SNFB_HD uint32_t crc_word_step(uint32_t c, const CrcTables* C) { return C->t[3][c & 0xffu] ^ C->t[2][(c >> 8) & 0xffu] ^ C->t[1][(c >> 16) & 0xffu] ^ C->t[0][c >> 24]; }
SNFB_HD uint32_t ld32a(const uint8_t* p) {            // 4-byte aligned load
#if defined(__CUDA_ARCH__)
    return *reinterpret_cast<const uint32_t*>(p);
#else
    uint32_t v; memcpy(&v, p, 4); return v;
#endif
}
struct U32x4 { uint32_t x, y, z, w; };
SNFB_HD U32x4 ld128a(const uint8_t* p) {             // 16-byte aligned load
#if defined(__CUDA_ARCH__)
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    return { v.x, v.y, v.z, v.w };
#else
    U32x4 v; memcpy(&v, p, 16); return v;
#endif
}
// CRC-32 of p[0 .. n), p at any alignment: bytes up to the first 16-byte boundary, then one 16-byte load per four table steps, then
// words, then bytes
SNFB_HD uint32_t crc32_slice(const uint8_t* p, uint32_t n, const CrcTables* C) {
    uint32_t c = 0xffffffffu, i = 0;
    for (; i < n && ((uintptr_t)(p + i) & 15u); ++i) c = (c >> 8) ^ C->t[0][(c ^ p[i]) & 0xffu];
    for (; i + 16u <= n; i += 16u) {
        const U32x4 v = ld128a(p + i);
        c = crc_word_step(c ^ v.x, C); c = crc_word_step(c ^ v.y, C); c = crc_word_step(c ^ v.z, C); c = crc_word_step(c ^ v.w, C);
    }
    for (; i + 4u <= n; i += 4u) c = crc_word_step(c ^ ld32a(p + i), C);
    for (; i < n; ++i) c = (c >> 8) ^ C->t[0][(c ^ p[i]) & 0xffu];
    return ~c;
}
SNFB_HD uint32_t group_shfl_xor(uint32_t v, int d, unsigned gmask) {
#if defined(__CUDA_ARCH__)
    return __shfl_xor_sync(gmask, v, d);
#else
    (void)d; (void)gmask; return v;
#endif
}
// CRC-32 of out[0 .. n) by the NL lanes of a decoding group; every lane calls it and every lane gets the result.  Each lane takes one
// contiguous slice (whole 256-byte units, so that the lengths joined below have few set bits), and the slices' CRCs are joined in
// log2(NL) butterfly steps: the lower half of each pair is A, the upper half B.
template <int NL>
SNFB_HD uint32_t crc32_group(const uint8_t* out, uint32_t n, const CrcTables* C, int lane, unsigned gmask) {
    group_sync(gmask);                                 // the bytes were written by every lane of the group
    const uint32_t per = ((n + NL - 1) / NL + 255u) & ~255u;
    const uint32_t beg = (uint32_t)lane * per < n ? (uint32_t)lane * per : n, end = n - beg > per ? beg + per : n;
    uint32_t crc = crc32_slice(out + beg, end - beg, C), len = end - beg;
    for (int d = 1; d < NL; d <<= 1) {
        const uint32_t o_crc = group_shfl_xor(crc, d, gmask), o_len = group_shfl_xor(len, d, gmask);
        const bool upper = (lane & d) != 0;
        crc = crc32_combine(upper ? o_crc : crc, upper ? crc : o_crc, upper ? len : o_len, C->x8pow);
        len += o_len;
    }
    return crc;
}

// ---------------------------------------------------------------- BAM records (SAM spec §4.2)
struct RawRec {             // what one alignment record of the inflated stream holds, as offsets into that stream
    uint64_t body;          // first byte after block_size
    uint64_t cig_src;       // CIGAR words the record means: its own, or the CG:B,I array of a >65535-op record (SAM spec §4.2.2)
    uint64_t seq_src, sa_src;
    uint32_t body_len, n_cig, sa_len;
    int32_t ref_id, pos, l_seq, nm, ps;
    uint32_t task;
    uint16_t flag; uint8_t mapq, aux_flags, hp, l_qname;      // l_qname without the NUL
    uint8_t status;         // ST_*
    uint8_t _pad[5];
};
enum { ST_OK = 0, ST_MALFORMED = 1, ST_FILTERED = 2 };
constexpr unsigned AUXF_NM = 1, AUXF_HP = 2, AUXF_PS = 4, AUXF_SA = 8;

SNFB_HD int aux_int(const uint8_t* raw, uint64_t p, unsigned typ, int32_t* v) {      // value of an integer aux field, returns its size (0 = not an integer type)
    switch (typ) {
        case 'c': *v = (int8_t)raw[p]; return 1;
        case 'C': *v = raw[p]; return 1;
        case 's': *v = (int16_t)ld16u(raw, p); return 2;
        case 'S': *v = (int32_t)ld16u(raw, p); return 2;
        case 'i': case 'I': *v = (int32_t)ld32u(raw, p); return 4;
        default: return 0;
    }
}
SNFB_HD int aux_array_elem(unsigned sub) { switch (sub) { case 'c': case 'C': return 1; case 's': case 'S': return 2; case 'i': case 'I': case 'f': return 4; default: return 0; } }

// decode the record whose body is raw[body .. body + bs); fills *o (status ST_OK or ST_MALFORMED)
SNFB_HD void parse_record(const uint8_t* raw, uint64_t body, uint32_t bs, RawRec* o) {
    o->body = body; o->body_len = bs; o->status = ST_MALFORMED; o->aux_flags = 0; o->hp = 0; o->nm = 0; o->ps = 0; o->sa_len = 0; o->sa_src = 0; o->task = 0;
    o->cig_src = o->seq_src = 0; o->n_cig = 0; o->ref_id = -1; o->pos = 0; o->l_seq = 0; o->flag = 0; o->mapq = 0; o->l_qname = 0;
    if (bs < 32) return;
    o->ref_id = (int32_t)ld32u(raw, body); o->pos = (int32_t)ld32u(raw, body + 4);
    const uint32_t l_rn = raw[body + 8]; o->mapq = raw[body + 9];
    uint32_t n_cig = ld16u(raw, body + 12); o->flag = (uint16_t)ld16u(raw, body + 14);
    const int32_t l_seq = (int32_t)ld32u(raw, body + 16); o->l_seq = l_seq;
    if (l_rn == 0 || l_seq < 0) return;
    const uint64_t end = body + bs, q = body + 32, cig = q + l_rn, seq = cig + 4ull * n_cig, aux = seq + (uint64_t)((l_seq + 1) / 2) + (uint64_t)l_seq;
    if (aux > end) return;
    o->l_qname = (uint8_t)(l_rn - 1); o->seq_src = seq; o->cig_src = cig;
    uint64_t cg_off = 0; uint32_t cg_n = 0; bool have_cg = false;
    uint64_t p = aux;
    while (p + 3 <= end) {
        const unsigned t0 = raw[p], t1 = raw[p + 1], typ = raw[p + 2]; p += 3;
        int32_t v = 0; const int isz = aux_int(raw, p, typ, &v);
        if (isz) {
            if (p + isz > end) return;
            if (t0 == 'N' && t1 == 'M') { o->nm = v; o->aux_flags |= AUXF_NM; }
            else if (t0 == 'H' && t1 == 'P') { o->hp = (uint8_t)(v & 255); o->aux_flags |= AUXF_HP; }
            else if (t0 == 'P' && t1 == 'S') { o->ps = v; o->aux_flags |= AUXF_PS; }
            p += isz;
        } else if (typ == 'A') { p += 1; }
        else if (typ == 'f') { p += 4; }
        else if (typ == 'Z' || typ == 'H') {
            uint64_t e = p; while (e < end && raw[e]) ++e;
            if (e >= end) return;
            if (t0 == 'S' && t1 == 'A' && typ == 'Z') { o->sa_src = p; o->sa_len = (uint32_t)(e - p); o->aux_flags |= AUXF_SA; }
            p = e + 1;
        } else if (typ == 'B') {
            if (p + 5 > end) return;
            const unsigned sub = raw[p]; const uint32_t cnt = ld32u(raw, p + 1); const int esz = aux_array_elem(sub);
            if (!esz || p + 5 + (uint64_t)esz * cnt > end) return;
            if (t0 == 'C' && t1 == 'G' && sub == 'I') { cg_off = p + 5; cg_n = cnt; have_cg = true; }
            p += 5 + (uint64_t)esz * cnt;
        } else return;
    }
    if (n_cig == 2) {
        const uint32_t op0 = ld32u(raw, cig), op1 = ld32u(raw, cig + 4);
        if ((op0 & 15u) == 4u && (op0 >> 4) == (uint32_t)l_seq && (op1 & 15u) == 3u) {
            if (have_cg) { o->cig_src = cg_off; n_cig = cg_n; }
            else if (l_seq > 0) return;                 // placeholder CIGAR without its CG tag
        }
    }
    o->n_cig = n_cig; o->status = ST_OK;
}

// ---------------------------------------------------------------- BAM CIGAR words -> CIGAR16 (cigar16.h)
// The one CIGAR16 encoder: the ingest kernels run it with 32 lanes, snfb_pack_cigar16 and snfb_load_records with one.
// Convert the n BAM CIGAR words at raw[src ..] ; out == nullptr only counts.  Returns the number of 16-bit words written (pads
// inside the record included, not rounded up); *reflen = reference bases the CIGAR covers; *bad set when an op code is unknown.
template <int NL>
SNFB_HD uint32_t c16_convert(const uint8_t* raw, uint64_t src, uint32_t n, uint16_t* out, uint32_t evt_min, int lane, long long* reflen, int* bad) {
    uint32_t k = 0; long long ref = 0; bool bad_op = false;
    for (uint32_t base = 0; base < n; base += NL) {
        const uint32_t i = base + lane; const bool valid = i < n;
        const uint32_t w = valid ? ld32u(raw, src + 4ull * i) : 0u; const uint32_t len = w >> 4; const unsigned code = w & 15u;
        if (valid && code > 8u) bad_op = true;
        const unsigned cls = c16_op_class(code > 8u ? 6u : code);
        const int g = valid ? c16_op_words(len) : 0;
        if (valid && (cls & 2u)) ref += len;            // class bit 1: the op advances the reference (M, D, N)
        const uint16_t w0 = c16_base_word(cls, len, evt_min);
        const uint32_t cnt = n - base < (uint32_t)NL ? n - base : (uint32_t)NL;
        if (!warp_any<NL>(g > 1)) {                     // 32 short ops: one word each, no group can straddle
            if (valid && out) out[k + lane] = w0;
            k += cnt;
        } else {
            for (uint32_t j = 0; j < cnt; ++j) {
                const int gj = (int)warp_shfl<NL>((uint32_t)g, (int)j);
                if ((k & 7u) + (uint32_t)gj > 8u) { const uint32_t k8 = (k + 7u) & ~7u; if (out && lane == 0) for (uint32_t z = k; z < k8; ++z) out[z] = 0; k = k8; }
                if ((uint32_t)lane == j && out) {
                    out[k] = w0;
                    if (g >= 2) out[k + 1] = c16_ext_word(len, 1);
                    if (g >= 3) out[k + 2] = c16_ext_word(len, 2);
                }
                k += (uint32_t)gj;
            }
        }
    }
    *reflen = warp_sum<NL>(ref);
    if (warp_any<NL>(bad_op)) *bad = 1;
    return k;
}

}  // namespace ingest
