// consensus.cuh — stage C: INS ALT sequences.
//   postprocessing.annotate_sv INS branch (best read selection)        postprocessing.py:33-66
//   consensus.novel_from_reads (k-mer anchored pile-up polish, k = 6)  consensus.py:280-394
// k_plan picks the best read per candidate and sizes the work; k_prep unpacks the best read and builds its anchor
// table; k_align aligns one (candidate, supporting read) pair per warp; k_vote takes the column vote per 4096-column tile.
#pragma once
#include "common.cuh"

namespace consensus {

constexpr int THREADS = 128;
constexpr int TAB = 2048;                  // > 4 x the at most ~500 strided k-mers of the best read
constexpr uint8_t DASH = 0xff;
// strided k-mer hits of one read are bounded by (L + 6) / skip + 1 (skip = 3 + L / 500): < 512 for every L, < 384 for L <= HEAVY_L.
// The light items run with the smaller per-warp hit arrays, i.e. with more warps per SM (they are latency bound).
constexpr int MAXHIT = 512, MAXHIT_LIGHT = 384; constexpr uint32_t HEAVY_L = 3000;

// The five work queues are written in candidate order, each candidate's entries at the exclusive scan of what the candidates before it
// put there, so the entries of candidates [c_lo, c_hi) are one range of every queue.  Stage C runs in slices of candidates cut to about
// equal scratch (rows x length, i.e. work): the kernels of a slice take only its ranges, and its ALT bytes [alt_lo, alt_hi) are final
// when its k_vote ends, so they can go to the host while the next slice runs.
enum { Q_BIG, Q_SMALL, Q_HEAVY, Q_LIGHT, Q_TILE, NQ };      // prep queues (candidates), align queues (items), vote queue (tiles)
constexpr int MAX_SLICES = 8, DEFAULT_SLICES = 2;
struct Slice { uint32_t c_lo, c_hi; uint32_t lo[NQ], hi[NQ]; unsigned long long alt_lo, alt_hi; };
struct Work {
    unsigned long long n[NQ];                 // queue lengths (the scans' totals; may exceed the capacities: the run is redone)
    uint32_t pos[MAX_SLICES][4];              // per slice: next prep candidate, heavy item, light item, vote tile
    Slice slice[MAX_SLICES];
};

struct C {
    const snfb_cand* cand; snfb_cand* cand_rw; const snfb_lead* cand_leads;
    const uint32_t* out_plo; const uint32_t* out_pn;     // per candidate lead: the run of `ord` entries (merge_inner parts) it was folded from
    const uint32_t* ord; const snfb_lead* kleads;         // kept-lead indices in merge_inner order, the kept leads
    const snfb_rec* rec; const uint8_t* seq;
    const uint32_t* arena_off;       // seq on demand: per kept lead, 16-byte unit offset of its bytes in `seq` (which then is the compact arena); nullptr = full arena
    uint32_t* plan_best; uint32_t* plan_nother; uint32_t* plan_otot; uint32_t* alt_len; uint32_t* scr_len; uint32_t* alt_off; uint32_t* scr_off;   // scr in units of 16 bytes
    uint8_t* alt; uint8_t* scr; unsigned long long alt_cap, scr_cap16, cand_cap;
    uint32_t* work_big; uint32_t* work_small; Work* work;
    uint32_t* q_cnt; uint32_t* q_off;     // per queue (Q_*) one column of cand_cap + 1 entries: what each candidate puts in the queue, its scanned position
    // item pipeline: one (candidate, supporting read) pair per warp, one (candidate, column tile) per block
    struct Item { uint32_t cand; uint32_t k; uint32_t row; uint32_t rd_off; };
    Item* items_big; Item* items_small; uint2* tiles; unsigned long long item_cap, tile_cap;
    DevCounters* ctr; snfb_config cfg;
};

__device__ __forceinline__ uint8_t seq_code(const uint8_t* sq, long long q) { const uint8_t v = sq[q >> 1]; return (q & 1) ? (v & 15) : (v >> 4); }
// bytes of a read's 4-bit copy in scratch (the seq arena's packing, from nibble 0): whole 8-byte words
__device__ __forceinline__ uint32_t packed_bytes(uint32_t len) { return ((len + 15u) & ~15u) / 2u; }

// choose the best read, size the outputs
__global__ void k_plan(C c) {
    const unsigned long long nc = c.ctr->n_cand < c.cand_cap ? c.ctr->n_cand : c.cand_cap;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nc; i += (unsigned long long)gridDim.x * blockDim.x) {
        uint32_t al = 0, sl = 0, heavy_n = 0, light_n = 0, tiles = 0; bool big = false;
        if (c.cand[i].svtype == SNFB_INS && !c.cfg.symbolic) {
            const snfb_cand* cd = &c.cand[i]; long nm = 0, bi = -1; long long bd = 0; long long tot = 0, bpk = 0;
            for (int k = 0; k < cd->lead_n; ++k) { const snfb_lead* l = &c.cand_leads[cd->lead_off + k]; if (!(l->flags & SNFB_LF_HAS_SEQ)) continue;
                // abs(len(seq) - svlen) + abs(ref_start - pos) * 1.5, compared exactly in halves
                long long a = (long long)l->seq_len - cd->svlen; if (a < 0) a = -a; long long p = (long long)l->ref_start - cd->pos; if (p < 0) p = -p;
                const long long d = 2 * a + 3 * p; if (nm == 0 || d < bd) { bd = d; bi = k; } ++nm;
                const long long pk = c.out_pn[cd->lead_off + k] != 1 ? packed_bytes((uint32_t)l->seq_len) : 0; tot += pk; if (bi == k) bpk = pk; }
            if (nm > 0) {
                const uint32_t L = (uint32_t)c.cand_leads[cd->lead_off + bi].seq_len; al = L;
                const bool cons = (nm - 1 >= c.cfg.consensus_min_reads) && !c.cfg.no_consensus;
                c.plan_best[i] = (uint32_t)bi; c.plan_nother[i] = cons ? (uint32_t)(nm - 1) : 0u; c.plan_otot[i] = (uint32_t)(tot - bpk);
                // scratch: best codes | best read packed | the merged other reads packed (a slot of packed_bytes(len) each; a read of one
                // piece is read from the seq arena) | one row of align4(L) per other read | accept flags | anchor table; 16-byte units
                const unsigned long long bytes = cons ? (unsigned long long)((L + 7u) & ~7u) + packed_bytes(L) + (unsigned long long)(tot - bpk) + 8 + (unsigned long long)(nm - 1) * ((L + 3u) & ~3u) + (unsigned long long)(nm - 1) * 16 + 64 + 16 + TAB * 8 : (unsigned long long)L + 24;
                sl = (uint32_t)((bytes + 15) / 16);
                c.cand_rw[i].alt_len = (int)L;
                // prep queue: the heavy tail (long insertions with many reads) is scheduled first; one align item per supporting read
                // (heavy rows first) and one vote item per 4096-column tile
                big = (unsigned long long)L * (unsigned long long)nm > 60000ull;
                if (cons) { const bool heavy = L > HEAVY_L; heavy_n = heavy ? (uint32_t)(nm - 1) : 0u; light_n = heavy ? 0u : (uint32_t)(nm - 1); tiles = (L + 4095u) / 4096u; }
            }
        }
        c.alt_len[i] = al; c.scr_len[i] = sl;
        const size_t col = c.cand_cap + 1;
        c.q_cnt[Q_BIG * col + i] = sl && big; c.q_cnt[Q_SMALL * col + i] = sl && !big; c.q_cnt[Q_HEAVY * col + i] = heavy_n; c.q_cnt[Q_LIGHT * col + i] = light_n; c.q_cnt[Q_TILE * col + i] = tiles;
    }
}

// the candidate records are final once the ALT offsets are known (stage C only fills the ALT bytes); every queue entry goes to its
// scanned position
__global__ void k_plan_finish(C c) {
    const unsigned long long nc = c.ctr->n_cand < c.cand_cap ? c.ctr->n_cand : c.cand_cap; const size_t col = c.cand_cap + 1;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nc; i += (unsigned long long)gridDim.x * blockDim.x) {
        if (!c.scr_len[i]) continue;
        c.cand_rw[i].alt_off = (int)c.alt_off[i];
        if (c.q_cnt[Q_BIG * col + i]) c.work_big[c.q_off[Q_BIG * col + i]] = (uint32_t)i; else c.work_small[c.q_off[Q_SMALL * col + i]] = (uint32_t)i;
        const uint32_t nh = c.q_cnt[Q_HEAVY * col + i], no = nh + c.q_cnt[Q_LIGHT * col + i];
        C::Item* dst = nh ? c.items_big : c.items_small; const uint32_t base = c.q_off[(nh ? Q_HEAVY : Q_LIGHT) * col + i];
        const snfb_cand* cd = &c.cand[i]; const uint32_t bi = c.plan_best[i];
        uint32_t row = 0, ro = 0;
        for (int k = 0; no && k < cd->lead_n; ++k) { const snfb_lead* l = &c.cand_leads[cd->lead_off + k]; if (!(l->flags & SNFB_LF_HAS_SEQ) || (uint32_t)k == bi) continue;
            if ((unsigned long long)base + row < c.item_cap) { C::Item it; it.cand = (uint32_t)i; it.k = (uint32_t)k; it.row = row; it.rd_off = ro; dst[base + row] = it; }
            ++row; if (c.out_pn[cd->lead_off + k] != 1) ro += packed_bytes((uint32_t)l->seq_len); }
        const uint32_t nt = c.q_cnt[Q_TILE * col + i], tb = c.q_off[Q_TILE * col + i];
        for (uint32_t t = 0; t < nt; ++t) if ((unsigned long long)tb + t < c.tile_cap) c.tiles[tb + t] = make_uint2((uint32_t)i, t);
    }
}

// the slices: thread s cuts at the first candidate whose scratch starts at or after s / k of the total, and reads every queue's and
// the ALT arena's position there (the totals past the last candidate).  Slices may be empty.
__global__ void k_plan_slices(C c, int k) {
    const int s = threadIdx.x; if (s >= k) return;
    const unsigned long long nc = c.ctr->n_cand < c.cand_cap ? c.ctr->n_cand : c.cand_cap; const size_t col = c.cand_cap + 1;
    const unsigned long long tot = c.ctr->n_seq_bytes;
    auto cut = [&](int j) -> uint32_t {
        if (j <= 0) return 0; if (j >= k) return (uint32_t)nc;
        const unsigned long long want = (tot * (unsigned long long)j + k - 1) / (unsigned long long)k;
        uint32_t lo = 0, hi = (uint32_t)nc;
        while (lo < hi) { const uint32_t m = (lo + hi) / 2; if (c.scr_off[m] < want) lo = m + 1; else hi = m; }
        return lo;
    };
    Slice sl; sl.c_lo = cut(s); sl.c_hi = cut(s + 1);
    for (int q = 0; q < NQ; ++q) { sl.lo[q] = sl.c_lo < nc ? c.q_off[q * col + sl.c_lo] : (uint32_t)c.work->n[q]; sl.hi[q] = sl.c_hi < nc ? c.q_off[q * col + sl.c_hi] : (uint32_t)c.work->n[q]; }
    sl.alt_lo = sl.c_lo < nc ? c.alt_off[sl.c_lo] : c.ctr->n_alt_bytes; sl.alt_hi = sl.c_hi < nc ? c.alt_off[sl.c_hi] : c.ctr->n_alt_bytes;
    c.work->slice[s] = sl;
}

__device__ __forceinline__ uint32_t nib_swap(uint32_t w) { return ((w & 0x0f0f0f0fu) << 4) | ((w >> 4) & 0x0f0f0f0fu); }
__device__ __forceinline__ uint32_t spread4(uint32_t x) { const uint32_t t = (x | (x << 8)) & 0x00ff00ffu; return (t | (t << 4)) & 0x0f0f0f0fu; }
// A 4-bit string: base q is nibble o + q from the aligned word w on (o < 8; high nibble first in each byte, as in the seq arena).
// get8 returns bases [q, q + 8), q >= 0, with base q + t in bits 4t..4t+3: two aligned words (the second only when the first n bases
// reach into it, so no byte past base q + n - 1's word is read), nibbles swapped into little-endian order, one funnel shift to the
// first base.  Plain loads: k_align reads a merged read's copy that the same kernel wrote.  get8<false> reads a string whose words
// already hold base q in nibble q (the best read's copy), without the swap.
struct Nib {
    const uint32_t* w; int o;
    __device__ static __forceinline__ Nib at(const uint8_t* p, long long q) {
        const uintptr_t A = (uintptr_t)(p + (q >> 1));
        Nib r; r.w = reinterpret_cast<const uint32_t*>(A & ~(uintptr_t)3); r.o = (int)((A & 3) << 1) | (int)(q & 1); return r;
    }
    template <bool SWAP = true> __device__ __forceinline__ uint32_t get8(int q, int n) const {
        const int b = o + q; const uint32_t* x = w + (b >> 3); const int qn = b & 7;
        const uint32_t lo = SWAP ? nib_swap(x[0]) : x[0], hi = qn + n > 8 ? (SWAP ? nib_swap(x[1]) : x[1]) : 0u;
        return __funnelshift_r(lo, hi, 4 * qn);
    }
    // bases [r, r + m) (m <= 8) of the string's first n bases at bits 4t; bases outside [0, n) read as 0
    __device__ __forceinline__ uint32_t take(int r, int m, int n) const {
        const int a = r < 0 ? 0 : r, e = r + m < n ? r + m : n;
        if (e <= a) return 0u;
        const int k = e - a; uint32_t x = get8(a, k);
        if (k < 8) x &= (1u << (4 * k)) - 1u;
        return x << (4 * (a - r));
    }
};
__device__ __forceinline__ uint2 unpack8(const uint8_t* __restrict__ sq, long long q, int n) {
    const uint32_t x = Nib::at(sq, q).get8(0, n);
    return make_uint2(spread4(x & 0xffffu), spread4(x >> 16));
}
// unpack `len` bases starting at nibble `off` of sq into dst (one code per byte); `tid`/`nthr` = cooperating threads.
// A thread takes 8 consecutive bases per step (unpack8: get8, two spreads) and stores them as one 8-byte word.
__device__ __forceinline__ void unpack_span(const uint8_t* __restrict__ sq, long long off, int len, uint8_t* __restrict__ dst, int tid, int nthr) {
    const int full = ((uintptr_t)dst & 7) == 0 ? (len & ~7) : 0;          // whole 8-base groups go out as aligned 8-byte stores, eight loads in flight
    int jb = tid * 8;
    for (; jb + 7 * nthr * 8 < full; jb += 8 * nthr * 8) {
        uint2 v[8];
        #pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = unpack8(sq, off + jb + u * nthr * 8, 8);
        #pragma unroll
        for (int u = 0; u < 8; ++u) *reinterpret_cast<uint2*>(dst + jb + u * nthr * 8) = v[u];
    }
    for (; jb < full; jb += nthr * 8) *reinterpret_cast<uint2*>(dst + jb) = unpack8(sq, off + jb, 8);
    for (; jb < len; jb += nthr * 8) {
        const int n = min(8, len - jb); const uint2 v = unpack8(sq, off + jb, n);
        for (int t = 0; t < n; ++t) dst[jb + t] = (uint8_t)(((t < 4 ? v.x : v.y) >> (8 * (t & 3))) & 15u);
    }
}
// the bases of kept lead `slot` in the seq arena (the full arena, or with seq on demand the compact one)
__device__ __forceinline__ Nib lead_bases(const C& c, uint32_t slot) {
    const snfb_lead* l = &c.kleads[slot];
    return c.arena_off ? Nib::at(c.seq + (size_t)c.arena_off[slot] * 16, l->seq_off & 1) : Nib::at(c.seq + c.rec[l->rec].seq_off, l->seq_off);
}
// unpack the (possibly merged) sequence of candidate lead `cl_index` as 4-bit codes, one byte per base, by `nthr` cooperating threads
__device__ inline void unpack_lead(const C& c, uint32_t cl_index, uint8_t* dst, int tid, int nthr) {
    const uint32_t plo = c.out_plo[cl_index], pn = c.out_pn[cl_index];
    long long o = 0;
    for (uint32_t p = 0; p < pn; ++p) {
        const uint32_t slot = c.ord[plo + p]; const snfb_lead* l = &c.kleads[slot];
        const uint8_t* sq = c.arena_off ? c.seq + (size_t)c.arena_off[slot] * 16 : c.seq + c.rec[l->rec].seq_off;
        unpack_span(sq, c.arena_off ? (l->seq_off & 1) : l->seq_off, l->seq_len, dst + o, tid, nthr);
        o += l->seq_len;
    }
}
// pack the (possibly merged) sequence of candidate lead `cl_index`, `len` bases, as one 4-bit string from nibble 0 of the 4-byte
// aligned dst (packed_bytes(len) bytes, the tail of the last word 0), by `nthr` cooperating threads; in the seq arena's order
// (`arena_order`, high nibble first) or with base q in nibble q of the little-endian words.  A thread writes whole words; a word
// gathers 8 bases from the part(s) it overlaps, which it finds by walking the parts forward with its words.
__device__ inline void pack_lead(const C& c, uint32_t cl_index, long len, uint32_t* dst, int tid, int nthr, bool arena_order) {
    const uint32_t plo = c.out_plo[cl_index], pn = c.out_pn[cl_index];
    const long nw = (long)(packed_bytes((uint32_t)len) / 4);
    uint32_t p = 0; int o = 0, n = 0; Nib b{};
    if (pn) { const uint32_t slot = c.ord[plo]; b = lead_bases(c, slot); n = c.kleads[slot].seq_len; }
    for (long w = tid; w < nw; w += nthr) {
        const int q = 8 * (int)w; uint32_t x = 0;
        if (pn) {
            while (o + n <= q && p + 1 < pn) { o += n; ++p; const uint32_t slot = c.ord[plo + p]; b = lead_bases(c, slot); n = c.kleads[slot].seq_len; }
            x = b.take(q - o, 8, n);
            int o2 = o + n;
            for (uint32_t p2 = p + 1; p2 < pn && o2 < q + 8; ++p2) {      // a word that straddles parts
                const uint32_t slot = c.ord[plo + p2]; const int n2 = c.kleads[slot].seq_len;
                x |= lead_bases(c, slot).take(q - o2, 8, n2); o2 += n2;
            }
        }
        dst[w] = arena_order ? nib_swap(x) : x;
    }
}
// the bases of candidate lead `cl_index` as k_align reads them: straight from the seq arena when it is one piece, else from its packed
// copy at `copy` (which the caller fills with pack_lead first)
__device__ __forceinline__ Nib lead_reader(const C& c, uint32_t cl_index, const uint8_t* copy) {
    if (c.out_pn[cl_index] == 1) return lead_bases(c, c.ord[c.out_plo[cl_index]]);
    Nib r; r.w = reinterpret_cast<const uint32_t*>(copy); r.o = 0; return r;
}

__device__ __forceinline__ uint32_t kmer6(const uint8_t* s) { return (uint32_t)s[0] | ((uint32_t)s[1] << 4) | ((uint32_t)s[2] << 8) | ((uint32_t)s[3] << 12) | ((uint32_t)s[4] << 16) | ((uint32_t)s[5] << 20); }
// the same from an unaligned pointer with aligned 32-bit loads (reads at most 3 bytes past s + 5)
__device__ __forceinline__ uint32_t kmer6_u(const uint8_t* s) {
    const uintptr_t A = (uintptr_t)s; const uint32_t* w = reinterpret_cast<const uint32_t*>(A & ~(uintptr_t)3); const uint32_t sh = (uint32_t)(A & 3) * 8;
    const uint32_t l0 = w[0], l1 = w[1], l2 = sh > 16 ? w[2] : 0u;
    const uint32_t x0 = __funnelshift_r(l0, l1, sh), x1 = __funnelshift_r(l1, l2, sh);
    uint32_t t = x0 & 0x0f0f0f0fu; t = (t | (t >> 4)) & 0x00ff00ffu; t = (t | (t >> 8)) & 0xffffu;
    return t | ((x1 & 15u) << 16) | (((x1 >> 8) & 15u) << 20);
}
// kmer6 of the bases [q, q + 6) of a 4-bit string: they are already in kmer6's order
__device__ __forceinline__ uint32_t kmer6_n(const Nib& s, int q) { return s.get8(q, 6) & 0xffffffu; }
__device__ __forceinline__ uint32_t kslot(uint32_t key) { return (key * 2654435761u) >> 21; }    // top 11 bits

// seq on demand: the base slices stage C will read, as (source byte offset in the host seq arena, bytes, destination unit)
struct SeqReq { unsigned long long src; uint32_t nbytes; uint32_t dst16; };
__global__ void k_seq_requests(C c, SeqReq* req, unsigned long long req_cap, uint32_t* arena_off_rw, unsigned long long* n_req, unsigned long long* n_units) {
    const unsigned long long nc = c.ctr->n_cand < c.cand_cap ? c.ctr->n_cand : c.cand_cap;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < nc; i += (unsigned long long)gridDim.x * blockDim.x) {
        if (c.scr_len[i] == 0) continue;
        const snfb_cand* cd = &c.cand[i]; const bool cons = c.plan_nother[i] > 0;
        for (int k = 0; k < cd->lead_n; ++k) {
            const snfb_lead* cl = &c.cand_leads[cd->lead_off + k];
            if (!(cl->flags & SNFB_LF_HAS_SEQ) || (!cons && (uint32_t)k != c.plan_best[i])) continue;
            const uint32_t plo = c.out_plo[cd->lead_off + k], pn = c.out_pn[cd->lead_off + k];
            for (uint32_t p = 0; p < pn; ++p) {
                const uint32_t slot = c.ord[plo + p]; const snfb_lead* l = &c.kleads[slot];
                const unsigned long long b0 = (unsigned long long)l->seq_off >> 1, b1 = ((unsigned long long)l->seq_off + l->seq_len + 1) >> 1;
                const uint32_t nb = (uint32_t)(b1 - b0) + 1;                                  // +1: unpack_span may touch one byte past the last base
                const unsigned long long u = atomicAdd(n_units, (unsigned long long)((nb + 15) / 16));
                const unsigned long long r = atomicAdd(n_req, 1ULL);
                arena_off_rw[slot] = (uint32_t)u;
                if (r < req_cap) { req[r].src = c.rec[l->rec].seq_off + b0; req[r].nbytes = nb; req[r].dst16 = (uint32_t)u; }
            }
        }
    }
}



// ================================================================================================
// k_prep (block per candidate: unpack the best read and pack a nibble-aligned 4-bit copy of it, build its anchor table in global
// scratch, or copy the best read to ALT when there is no consensus) -> k_align (one warp per (candidate, read)
// item from a heavy-first queue: no block barriers, the heaviest candidate's reads spread over the whole GPU)
// -> k_vote (one block per (candidate, 4096-column tile)).
// ================================================================================================
// ---- the row's dashes, four bytes per step where the row is word aligned
__device__ __forceinline__ void fill_dash(uint8_t* dst, long n) {
    long q = 0;
    while (q < n && ((uintptr_t)(dst + q) & 3)) dst[q++] = DASH;
    for (; q + 4 <= n; q += 4) *reinterpret_cast<uint32_t*>(dst + q) = 0xffffffffu;
    for (; q < n; ++q) dst[q] = DASH;
}

// how many of the bases [0, n) of a + ia and b + ib are equal: 8 bases per 32-bit XOR, at any nibble offset on either side (b is the
// best read's copy, in base order); the 8-base words of [0, n) are dealt round robin to the G lanes of a group, the caller adds the
// lanes up
template <int G>
__device__ __forceinline__ int group_match(const Nib& a, long ia, const Nib& b, long ib, long n, int sub) {
    int mt = 0;
    for (long q = 8L * sub; q < n; q += 8L * G) {
        const int k = n - q < 8 ? (int)(n - q) : 8;
        uint32_t x = a.get8((int)(ia + q), k) ^ b.get8<false>((int)(ib + q), k);
        x |= x >> 1; x |= x >> 2;                                       // bit 4t: base t differs
        uint32_t eq = ~x & 0x11111111u;
        if (k < 8) eq &= (1u << (4 * k)) - 1u;
        mt += __popc(eq);
    }
    return mt;
}
template <int G> __device__ __forceinline__ int group_sum(int v) {
    #pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
// ---- cooperating groups of k_align: one warp (light items) or the whole block (heavy items).  `tid` order = element order.
struct WarpGrp {
    static constexpr int NTHR = 32; int tid;
    __device__ __forceinline__ void sync() const { __syncwarp(); }
    // exclusive prefix sum over the group in tid order; tot = group total
    __device__ __forceinline__ int excl(int v, int& tot) const {
        int inc = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(FULL, inc, o); if (tid >= o) inc += t; }
        tot = __shfl_sync(FULL, inc, 31); return inc - v;
    }
    // max over the threads before this one (-1 when none); tot = group max
    __device__ __forceinline__ int exclmax(int v, int& tot) const {
        int inc = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(FULL, inc, o); if (tid >= o) inc = max(inc, t); }
        tot = __shfl_sync(FULL, inc, 31); int e = __shfl_up_sync(FULL, inc, 1); if (tid == 0) e = -1; return e;
    }
    __device__ __forceinline__ long sum(long v) const { return (long)__reduce_add_sync(FULL, (unsigned)v); }
};
template <int WARPS>
struct BlockGrp {
    static constexpr int NTHR = WARPS * 32; int tid; int* red;          // red: 2 * WARPS ints of shared memory
    __device__ __forceinline__ void sync() const { __syncthreads(); }
    __device__ __forceinline__ int excl(int v, int& tot) const {
        const int lane = tid & 31, w = tid >> 5; int inc = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) red[w] = inc;
        __syncthreads();
        int base = 0, all = 0;
        #pragma unroll
        for (int k = 0; k < WARPS; ++k) { const int t = red[k]; if (k < w) base += t; all += t; }
        __syncthreads();
        tot = all; return base + inc - v;
    }
    __device__ __forceinline__ int exclmax(int v, int& tot) const {
        const int lane = tid & 31, w = tid >> 5; int inc = v;
        #pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(FULL, inc, o); if (lane >= o) inc = max(inc, t); }
        int e = __shfl_up_sync(FULL, inc, 1); if (lane == 0) e = -1;
        if (lane == 31) red[w] = inc;
        __syncthreads();
        int all = -1;
        #pragma unroll
        for (int k = 0; k < WARPS; ++k) { const int t = red[k]; if (k < w) e = max(e, t); all = max(all, t); }
        __syncthreads();
        tot = all; return e;
    }
    __device__ __forceinline__ long sum(long v) const {
        const int lane = tid & 31, w = tid >> 5; const int sv = (int)__reduce_add_sync(FULL, (unsigned)v);
        if (lane == 0) red[w] = sv;
        __syncthreads();
        int all = 0;
        #pragma unroll
        for (int k = 0; k < WARPS; ++k) all += red[k];
        __syncthreads();
        return (long)all;
    }
};

// (3a) of k_align with G lanes per segment (1: short segments, a lane walks its own; 4: long segments, 32 bases per group step); `tid` of
// `nthr` cooperating threads (whole warps)
template <int G>
__device__ __forceinline__ long segments_pass(const int* hi, const int* hj, int* hcl, int na, long c0, long j0, long L, const Nib& rd, const Nib& best, int tid, int nthr) {
    const int PER = nthr / G; const int grp = tid / G, sub = tid % G; long span = 0;
    for (int mb = 1; mb < na; mb += PER) {
        const int m = mb + grp; const bool v = m < na;
        long li = 0, lj = 0, i = 0, j = 0; if (v) { li = hi[m - 1]; lj = hj[m - 1]; i = hi[m]; j = hj[m]; }
        long cs = c0 + lj - j0; if (cs > L) cs = L;
        const long d = j - lj; long fwd_j = d; if (cs + fwd_j > L) fwd_j = L - cs;
        const bool el = v && i - li == fwd_j && fwd_j > 0;
        long nc = 0; if (el) { nc = L - 1 - li; if (nc > d) nc = d; if (nc < 0) nc = 0; }      // positions past the end of the best read never match
        const int mt = group_sum<G>(group_match<G>(rd, lj + 1, best, li + 1, nc, sub));
        // column identity of the copied bases.  Without drift (cs == li, nothing clamped) it is the same sum shifted by one
        // position, and both end positions are anchor k-mer bases that match by construction: reuse mt
        int st = -1; bool second = false;
        if (el) { if (sub == 0) span += d; if (__ddiv_rn((double)mt, (double)d) >= 0.5) { if (cs == li && fwd_j == d && nc == d) st = mt; else second = true; } }
        const int m2 = group_sum<G>(group_match<G>(rd, lj, best, cs, second ? fwd_j : 0, sub));
        if (second) st = m2;
        if (v && sub == 0) hcl[m] = st;
    }
    return span;
}

// scratch layout of one consensus candidate: best[align8(L)] | best packed in base order [packed_bytes(L)] | merged other reads packed [otot] |
// rows[no][Ls] (Ls = align4(L)) | accept[no] | ... | table
struct Layout { uint8_t* best; uint8_t* best4; uint8_t* oth; uint8_t* rows; uint8_t* acc; uint32_t Ls; };
__device__ __forceinline__ Layout cand_layout(const C& c, uint32_t ci, uint32_t L, uint32_t no) {
    Layout y; y.best = c.scr + (size_t)c.scr_off[ci] * 16; y.best4 = y.best + ((L + 7u) & ~7u); y.oth = y.best4 + packed_bytes(L);
    y.rows = reinterpret_cast<uint8_t*>(((uintptr_t)(y.oth + c.plan_otot[ci]) + 3) & ~(uintptr_t)3); y.Ls = (L + 3u) & ~3u; y.acc = y.rows + (size_t)no * y.Ls;
    return y;
}
__device__ __forceinline__ uint8_t* cand_table(const C& c, uint32_t ci, uint32_t** keys, int** pos) {
    uint8_t* scr = c.scr + (size_t)c.scr_off[ci] * 16;
    uint8_t* end = scr + (size_t)c.scr_len[ci] * 16;
    *keys = reinterpret_cast<uint32_t*>(end - TAB * 8); *pos = reinterpret_cast<int*>(end - TAB * 4);
    return scr;
}

// the kernels of stage C take slice `s` of every queue
__global__ void __launch_bounds__(128) k_prep(C c, int s) {
    __shared__ uint32_t s_cand;
    static const char CODE[17] = "=ACMGRSVTWYHKDBN";
    const Slice& sl = c.work->slice[s];
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) { const uint32_t q = atomicAdd(&c.work->pos[s][0], 1u); const uint32_t nb = sl.hi[Q_BIG] - sl.lo[Q_BIG], ns = sl.hi[Q_SMALL] - sl.lo[Q_SMALL];
            s_cand = q < nb ? c.work_big[sl.lo[Q_BIG] + q] : (q < nb + ns ? c.work_small[sl.lo[Q_SMALL] + q - nb] : 0xffffffffu); }
        __syncthreads();
        const uint32_t ci = s_cand; if (ci == 0xffffffffu) break;
        const uint32_t L = c.alt_len[ci];
        if ((unsigned long long)c.alt_off[ci] + L > c.alt_cap || (unsigned long long)c.scr_off[ci] + c.scr_len[ci] > c.scr_cap16) { if (threadIdx.x == 0) atomicAdd(&c.ctr->scratch_overflow, 1ULL); continue; }
        const snfb_cand cd = c.cand[ci];
        uint32_t* tk; int* tp; uint8_t* best = cand_table(c, ci, &tk, &tp);
        unpack_lead(c, cd.lead_off + c.plan_best[ci], best, threadIdx.x, blockDim.x);
        const uint32_t no = c.plan_nother[ci];
        if (no == 0 || L == 0) { __syncthreads(); uint8_t* out = c.alt + c.alt_off[ci]; for (uint32_t h = threadIdx.x; h < L; h += blockDim.x) out[h] = (uint8_t)CODE[best[h]]; continue; }
        pack_lead(c, cd.lead_off + c.plan_best[ci], L, reinterpret_cast<uint32_t*>(best + ((L + 7u) & ~7u)), threadIdx.x, blockDim.x, false);
        for (int i = threadIdx.x; i < TAB; i += blockDim.x) { tk[i] = 0xffffffffu; tp[i] = -1; }
        __syncthreads();
        const long skip = c.cfg.consensus_kmer_skip_base + (long)__dmul_rn((double)L, c.cfg.consensus_kmer_skip_seqlen_mult);
        for (long i = (long)threadIdx.x * skip; i < (long)L - 6; i += (long)blockDim.x * skip) {
            const uint32_t key = kmer6_u(best + i); uint32_t s = kslot(key);
            for (;;) { const uint32_t old = atomicCAS(&tk[s], 0xffffffffu, key); if (old == 0xffffffffu || old == key) break; s = (s + 1) & (TAB - 1); }
            if (atomicCAS(&tp[s], -1, (int)i) != -1) tp[s] = -2;
        }
    }
}

// one (candidate, supporting read) item by the cooperating group g; hi / hj / hcl / run_st / run_len hold `cap` ints each
template <typename G>
__device__ __forceinline__ void align_item(const C& c, const C::Item it, const G g, int* hi, int* hj, int* hcl, int* run_st, int* run_len, int cap) {
    const int tid = g.tid; constexpr int NT = G::NTHR; const int klen = 6;
    const uint32_t ci = it.cand; const uint32_t L = c.alt_len[ci];
    if ((unsigned long long)c.scr_off[ci] + c.scr_len[ci] > c.scr_cap16) return;
    const snfb_cand* cd = &c.cand[ci];
    uint32_t* t_key; int* t_pos; cand_table(c, ci, &t_key, &t_pos);
    const uint32_t no = c.plan_nother[ci];
    const Layout y = cand_layout(c, ci, L, no);
    uint8_t* acc = y.acc; const Nib best = Nib::at(y.best4, 0);
    const snfb_lead* l = &c.cand_leads[cd->lead_off + it.k];
    const long Lo = l->seq_len; uint8_t* row = y.rows + (size_t)it.row * y.Ls;
    const long skip = c.cfg.consensus_kmer_skip_base + (long)__dmul_rn((double)L, c.cfg.consensus_kmer_skip_seqlen_mult);
    // the read in 4-bit form: from the seq arena, or, merged from several pieces, from the one packed copy it gets here first
    const Nib rd = lead_reader(c, cd->lead_off + it.k, y.oth + it.rd_off);
    if (c.out_pn[cd->lead_off + it.k] != 1) { pack_lead(c, cd->lead_off + it.k, Lo, reinterpret_cast<uint32_t*>(y.oth + it.rd_off), tid, NT, true); g.sync(); }
    // (1) anchor hits in j order (table lives in global scratch, L2 resident); four k-mers per thread in flight
    int nh = 0;
    const long nk = Lo - klen > 0 ? (Lo - klen + skip - 1) / skip : 0;
    for (long kb = 0; kb < nk; kb += 4 * NT) {
        uint32_t key[4], sl[4], tk[4]; int ai[4];
        #pragma unroll
        for (int u = 0; u < 4; ++u) { const long kk = kb + u * NT + tid; key[u] = kk < nk ? kmer6_n(rd, (int)(kk * skip)) : 0u; sl[u] = kslot(key[u]); }
        #pragma unroll
        for (int u = 0; u < 4; ++u) tk[u] = kb + u * NT + tid < nk ? t_key[sl[u]] : 0xffffffffu;
        #pragma unroll
        for (int u = 0; u < 4; ++u) while (tk[u] != 0xffffffffu && tk[u] != key[u]) { sl[u] = (sl[u] + 1) & (TAB - 1); tk[u] = t_key[sl[u]]; }
        #pragma unroll
        for (int u = 0; u < 4; ++u) ai[u] = tk[u] != 0xffffffffu ? t_pos[sl[u]] : -1;
        #pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (kb + (long)u * NT >= nk) break;
            const long j = (kb + u * NT + tid) * skip;
            if (ai[u] >= 0) { long d = ai[u] - j; if (d < 0) d = -d; if (d > klen) ai[u] = -1; }
            int tot; const int off = g.excl(ai[u] >= 0 ? 1 : 0, tot);
            if (ai[u] >= 0) { const int p = nh + off; if (p < cap) { hi[p] = ai[u]; hj[p] = (int)j; } }
            nh += tot;
        }
    }
    if (nh > cap) nh = cap;
    g.sync();
    // (2) anchor automaton (consensus.py:306-338) in closed form: a hit is accepted iff its i exceeds every earlier hit's i
    //     (the accepted hits are the left-to-right maxima), and len(conseq) before accepted hit m is
    //     min(L, c0 + j[m-1] - j[0]) because every step appends min(j step, room left).  Compacted in place.
    int na = 0, pm = -1;
    for (int hb = 0; hb < nh; hb += NT) {
        const int h = hb + tid; const int vi = h < nh ? hi[h] : -1, vj = h < nh ? hj[h] : 0;
        int tmax; const int exc = max(g.exclmax(vi, tmax), pm);
        const bool accp = h < nh && vi > exc;
        int tot; const int off = g.excl(accp ? 1 : 0, tot);
        g.sync();
        if (accp) { hi[na + off] = vi; hj[na + off] = vj; }
        na += tot; pm = max(pm, tmax);
        g.sync();
    }
    const long j0 = na ? hj[0] : 0, c0 = (na && j0 > 0) ? hi[0] : 0;
    // (3a) agreement with the best read along the diagonal decides copy / dash; a copied segment also gets its column identity
    //      (the bases it shares with the best read at the columns it lands on)
    long span = skip > 12 ? segments_pass<4>(hi, hj, hcl, na, c0, j0, (long)L, rd, best, tid, NT) : segments_pass<1>(hi, hj, hcl, na, c0, j0, (long)L, rd, best, tid, NT);
    span = g.sum(span);
    g.sync();
    // (3b) dash-free runs (= chains of copied segments) survive only with identity > 0.5 and more than 5 matches
    //      (consensus.py:343-360); decided on the segment list before anything is written.  A non-empty dashed segment
    //      ends a run; run ids are prefix counts of those, the per-run sums are accumulated in shared memory.
    {
        int* hr = hi;                                   // the anchor i positions are no longer needed
        for (int m = tid; m < na; m += NT) { run_st[m] = 0; run_len[m] = 0; }
        g.sync();
        int run_base = 0;
        for (int mb = 1; mb < na; mb += NT) {
            const int m = mb + tid; int st = -1; long len = 0;
            if (m < na) { const long lj = hj[m - 1]; long cs = c0 + lj - j0; if (cs > (long)L) cs = (long)L; len = hj[m] - lj; if (cs + len > (long)L) len = (long)L - cs; st = hcl[m]; }
            int tot; const int rid = run_base + g.excl((m < na && st < 0 && len > 0) ? 1 : 0, tot);
            g.sync();
            if (m < na) { hr[m] = rid; if (st >= 0) { atomicAdd(&run_st[rid], st); atomicAdd(&run_len[rid], (int)len); } }
            run_base += tot;
        }
        g.sync();
        for (int m = 1 + tid; m < na; m += NT) {
            if (hcl[m] < 0) continue;
            const int r = hr[m], ident = run_st[r];
            if (!(__ddiv_rn((double)ident, (double)run_len[r]) > 0.5 && ident > 5)) hcl[m] = -1;
        }
        g.sync();
    }
    // (3c) the row: every copied segment lands at row[cs + t] = rd[lj + t] with cs - lj = c0 - j0 for all of them, so the row is
    //      one shifted copy of the read between the first and the last anchor (eight bases unpacked per thread step, two words),
    //      dashes outside, and the rejected segments dashed afterwards
    {
        long cl = 0; if (na) { cl = c0 + hj[na - 1] - j0; if (cl > (long)L) cl = (long)L; }
        for (long X = 8L * tid; X < (long)L; X += 8L * NT) {
            unsigned long long v = ~0ull;
            if (X + 8 > c0 && X < cl) {
                const int q = (int)(X + j0 - c0);                                        // below 0 only where X < c0
                const uint32_t x = q >= 0 && q + 8 <= (int)Lo ? rd.get8(q, 8) : rd.take(q, 8, (int)Lo);
                v = (unsigned long long)spread4(x & 0xffffu) | ((unsigned long long)spread4(x >> 16) << 32);
                if (X < c0) v |= (1ull << (8 * (c0 - X))) - 1ull;                         // bytes before c0
                if (X + 8 > cl) v |= ~((1ull << (8 * (cl - X))) - 1ull);                    // bytes from cl on
            }
            *reinterpret_cast<uint32_t*>(row + X) = (uint32_t)v;                           // rows are 4-byte aligned, align4(L) long
            if (X + 4 < (long)L) *reinterpret_cast<uint32_t*>(row + X + 4) = (uint32_t)(v >> 32);
        }
        g.sync();
        for (int m = 1 + tid; m < na; m += NT) {
            if (hcl[m] >= 0) continue;
            const long lj = hj[m - 1]; long cs = c0 + lj - j0; if (cs > (long)L) cs = (long)L;
            long len = hj[m] - lj; if (cs + len > (long)L) len = (long)L - cs;
            if (len > 0) fill_dash(row + cs, len);
        }
    }
    if (tid == 0) acc[it.row] = __ddiv_rn((double)span, (double)L) > 0.2;
    g.sync();
}

// Heavy items (long insertions) first, the whole block on one item (the longest insertion's reads are the tail of the step);
// then the light items, one per warp.  Per-warp hit arrays of MAXHIT_LIGHT entries; a block item uses all of them as one array.
constexpr int ALIGN_WARPS = 4;
__global__ void __launch_bounds__(ALIGN_WARPS * 32, 7) k_align(C c, int s) {
    __shared__ int sm[5][ALIGN_WARPS * MAXHIT_LIGHT]; __shared__ int s_red[2 * ALIGN_WARPS]; __shared__ uint32_t s_q;
    static_assert(ALIGN_WARPS * MAXHIT_LIGHT >= MAXHIT, "a block item needs MAXHIT entries");
    const int lane = lane_id(), warp = threadIdx.x >> 5;
    const Slice& sl = c.work->slice[s];
    const uint32_t b0 = sl.lo[Q_HEAVY], nb = (uint32_t)min((unsigned long long)sl.hi[Q_HEAVY], c.item_cap), s0 = sl.lo[Q_LIGHT], ns = (uint32_t)min((unsigned long long)sl.hi[Q_LIGHT], c.item_cap);
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) s_q = b0 + atomicAdd(&c.work->pos[s][1], 1u);
        __syncthreads();
        const uint32_t q = s_q; if (q >= nb) break;
        BlockGrp<ALIGN_WARPS> g; g.tid = threadIdx.x; g.red = s_red;
        align_item(c, c.items_big[q], g, sm[0], sm[1], sm[2], sm[3], sm[4], ALIGN_WARPS * MAXHIT_LIGHT);
    }
    __syncthreads();
    for (;;) {
        uint32_t q = 0; if (lane == 0) q = s0 + atomicAdd(&c.work->pos[s][2], 1u);
        q = __shfl_sync(FULL, q, 0);
        if (q >= ns) break;
        WarpGrp g; g.tid = lane; const int o = warp * MAXHIT_LIGHT;
        align_item(c, c.items_small[q], g, sm[0] + o, sm[1] + o, sm[2] + o, sm[3] + o, sm[4] + o, MAXHIT_LIGHT);
    }
}

// column vote (consensus.py:365-380), one block per (candidate, 4096-column tile); every thread takes four adjacent columns
// (rows are 4-byte aligned with a stride of align4(L)), eight rows in flight
constexpr int VOTE_LIST = 256;
// sixteen 16-bit counters (one per base code) in four registers; the selects keep them out of local memory
__device__ __forceinline__ void vote_add(unsigned long long (&cnt)[4], uint32_t code) {
    const unsigned long long inc = 1ull << (16 * (code & 3u)); const uint32_t sel = (code >> 2) & 3u;
    #pragma unroll
    for (int k = 0; k < 4; ++k) cnt[k] += sel == (uint32_t)k ? inc : 0ull;
}
constexpr int VOTE_THREADS = 64;      // most candidates are a few hundred columns: small blocks, many of them
__global__ void __launch_bounds__(VOTE_THREADS) k_vote(C c, int s) {
    __shared__ uint2 s_tile; __shared__ int s_nacc, s_nlist; __shared__ uint16_t s_rows[VOTE_LIST];
    static const char CODE[17] = "=ACMGRSVTWYHKDBN";
    const Slice& sl = c.work->slice[s];
    for (;;) {
        __syncthreads();
        if (threadIdx.x == 0) { const uint32_t q = sl.lo[Q_TILE] + atomicAdd(&c.work->pos[s][3], 1u); s_tile = q < sl.hi[Q_TILE] && q < c.tile_cap ? c.tiles[q] : make_uint2(0xffffffffu, 0); }
        __syncthreads();
        const uint32_t ci = s_tile.x; if (ci == 0xffffffffu) break;
        const uint32_t L = c.alt_len[ci], no = c.plan_nother[ci];
        if ((unsigned long long)c.alt_off[ci] + L > c.alt_cap || (unsigned long long)c.scr_off[ci] + c.scr_len[ci] > c.scr_cap16) continue;
        const Layout y = cand_layout(c, ci, L, no);
        const uint8_t* best = y.best; const uint8_t* rows = y.rows; const uint8_t* acc = y.acc; const uint32_t Ls = y.Ls;
        if (threadIdx.x < 32) {                         // the accepted rows, in order (the first VOTE_LIST rows go through the list)
            int cnt = 0, extra = 0; const uint32_t lim = no < (uint32_t)VOTE_LIST ? no : (uint32_t)VOTE_LIST;
            for (uint32_t r0 = 0; r0 < lim; r0 += 32) { const uint32_t r = r0 + threadIdx.x; const bool a = r < lim && acc[r]; const unsigned bm = __ballot_sync(FULL, a);
                if (a) s_rows[cnt + __popc(bm & lanemask_lt())] = (uint16_t)r; cnt += __popc(bm); }
            for (uint32_t r = lim + threadIdx.x; r < no; r += 32) extra += acc[r] ? 1 : 0;
            extra = (int)__reduce_add_sync(FULL, (unsigned)extra);
            if (threadIdx.x == 0) { s_nlist = cnt; s_nacc = cnt + extra; }
        }
        __syncthreads();
        const double maxal = (double)(1 + s_nacc); const int nlist = s_nlist;
        uint8_t* out = c.alt + c.alt_off[ci];
        const uint32_t h_end = min(L, (s_tile.y + 1u) * 4096u);
        for (uint32_t h = s_tile.y * 4096u + threadIdx.x * 4u; h < h_end; h += blockDim.x * 4u) {
            const uint32_t bw = *reinterpret_cast<const uint32_t*>(best + h);
            // fast path: the four columns of a word are counted byte-parallel.  A, C, G, T are the one-hot codes 1, 2, 4, 8, so bit k
            // of a byte is that base's vote; dashes (0xff) are cleared first; anything else (ambiguity codes, '=') shows up as a byte
            // with two bits set or as a column whose votes and dashes do not add up to the rows, and sends the word down the exact path
            if (nlist == s_nacc && nlist < 255) {
                uint32_t cA = 0, cC = 0, cG = 0, cT = 0, cD = 0, multi = 0;
                for (int r0 = 0; r0 < nlist; r0 += 8) {
                    uint32_t cv[8];
                    #pragma unroll
                    for (int u = 0; u < 8; ++u) cv[u] = r0 + u < nlist ? *reinterpret_cast<const uint32_t*>(rows + (size_t)s_rows[r0 + u] * Ls + h) : 0xffffffffu;
                    #pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const uint32_t hb = cv[u] & 0x80808080u, d1 = hb >> 7, t = cv[u] & ~(hb | (hb - d1));
                        cD += d1; multi |= ((t | 0x10101010u) - 0x01010101u) & t;
                        cA += t & 0x01010101u; cC += (t >> 1) & 0x01010101u; cG += (t >> 2) & 0x01010101u; cT += (t >> 3) & 0x01010101u;
                    }
                }
                // padding rows of the last group of eight counted as dashes
                const uint32_t padded = (uint32_t)((nlist + 7) & ~7);
                const uint32_t tot = cA + cC + cG + cT + cD;                      // per byte: rows accounted for (<= 255 + 7 would overflow: bounded by padded <= 256 only when nlist <= 248)
                const bool best_ok = (((bw | 0x10101010u) - 0x01010101u) & bw) == 0 && ((bw - 0x01010101u) & ~bw & 0x80808080u) == 0;
                if (multi == 0 && best_ok && padded <= 248 && tot == padded * 0x01010101u) {
                    #pragma unroll
                    for (int b2 = 0; b2 < 4; ++b2) {
                        if (h + b2 >= h_end) break;
                        const uint32_t bc = (bw >> (8 * b2)) & 255u; uint32_t res = bc;
                        const int nal = (int)padded - (int)((cD >> (8 * b2)) & 255u);
                        if (!(nal < 2 || __ddiv_rn((double)nal, maxal) < 0.25)) {
                            int v4[4] = { (int)((cA >> (8 * b2)) & 255u), (int)((cC >> (8 * b2)) & 255u), (int)((cG >> (8 * b2)) & 255u), (int)((cT >> (8 * b2)) & 255u) };
                            int t0 = -1, t1 = -1, c0 = 0, nd = 0;
                            #pragma unroll
                            for (int k = 0; k < 4; ++k) { const int v = v4[k] + ((bc >> k) & 1u); if (!v) continue; ++nd; if (v > t0) { t1 = t0; t0 = v; c0 = 1 << k; } else if (v > t1) t1 = v; }
                            if (nd > 1 && t0 - t1 >= 3) res = (uint32_t)c0;
                        }
                        out[h + b2] = (uint8_t)CODE[res];
                    }
                    continue;
                }
            }
            unsigned long long cnt[4][4]; int nal[4];
            #pragma unroll
            for (int b2 = 0; b2 < 4; ++b2) { nal[b2] = 0; cnt[b2][0] = cnt[b2][1] = cnt[b2][2] = cnt[b2][3] = 0; }
            for (int r0 = 0; r0 < nlist; r0 += 8) {
                uint32_t cv[8];
                #pragma unroll
                for (int u = 0; u < 8; ++u) cv[u] = r0 + u < nlist ? *reinterpret_cast<const uint32_t*>(rows + (size_t)s_rows[r0 + u] * Ls + h) : 0xffffffffu;
                #pragma unroll
                for (int u = 0; u < 8; ++u) {
                    #pragma unroll
                    for (int b2 = 0; b2 < 4; ++b2) { const uint32_t cc = (cv[u] >> (8 * b2)) & 255u; if (cc != DASH) { vote_add(cnt[b2], cc); ++nal[b2]; } }
                }
            }
            for (uint32_t r = VOTE_LIST; r < no; ++r) if (acc[r]) {          // more reads than the list holds: never with the default bins
                const uint32_t v = *reinterpret_cast<const uint32_t*>(rows + (size_t)r * Ls + h);
                #pragma unroll
                for (int b2 = 0; b2 < 4; ++b2) { const uint32_t cc = (v >> (8 * b2)) & 255u; if (cc != DASH) { vote_add(cnt[b2], cc); ++nal[b2]; } }
            }
            #pragma unroll
            for (int b2 = 0; b2 < 4; ++b2) {
                if (h + b2 >= h_end) break;
                const uint32_t bc = (bw >> (8 * b2)) & 255u; uint32_t res = bc;
                if (!(nal[b2] < 2 || __ddiv_rn((double)nal[b2], maxal) < 0.25)) {
                    vote_add(cnt[b2], bc);
                    int t0 = -1, t1 = -1, c0 = 0, nd = 0;
                    #pragma unroll
                    for (int code = 0; code < 16; ++code) { const int v = (int)((cnt[b2][code >> 2] >> (16 * (code & 3))) & 0xffff); if (!v) continue; ++nd; if (v > t0) { t1 = t0; t0 = v; c0 = code; } else if (v > t1) t1 = v; }
                    if (nd > 1 && t0 - t1 >= 3) res = (uint32_t)c0;
                }
                out[h + b2] = (uint8_t)CODE[res];
            }
        }
    }
}

}  // namespace consensus
