// reference.cuh — the reference FASTA on the device (--reference): line unwrapping by the .fai geometry, the runs of 'N' that
// LeadProvider._mask_N_coverage zeroes (leadprov.py:420-443), and the REF / anchor gathers of VCF.write_call (vcf.py:299-342).
#pragma once
#include "common.cuh"
#include "prims.cuh"

namespace refseq {

// one contig of the raw (inflated) FASTA bytes and of the unwrapped genome; out_off is a multiple of 16
struct Contig { unsigned long long raw_off, len, out_off; uint32_t linebases, linewidth; };
// one tile of output bases of a contig
struct Tile { uint32_t contig, _pad; unsigned long long start; };
// geometry violations: their count, and the lowest (contig << 40 | line) among them
struct Bad { unsigned long long n, first; };

constexpr int UNW_THREADS = 256;
constexpr int UNW_TILE = 16384;                 // output bases per block
constexpr int UNW_SMEM = 40960;                 // staged source bytes; a wider line geometry reads the source from global memory

__device__ __forceinline__ unsigned long long raw_pos(const Contig& c, unsigned long long p) { return c.raw_off + (p / c.linebases) * c.linewidth + p % c.linebases; }
__device__ __forceinline__ void flag_bad(Bad* bad, uint32_t contig, unsigned long long line) {
    atomicAdd(&bad->n, 1ull); atomicMin(&bad->first, ((unsigned long long)contig << 40) | line);
}

// output base p of a contig = raw byte offset + (p / linebases) * linewidth + p % linebases.  The block stages the source span of its
// tile in shared memory with 16-byte loads, then every thread writes 16 output bytes with one store.  Every line followed by more
// sequence must end in "\n" (linewidth = linebases + 1) or "\r\n" (+ 2), and no base may be a line break: a violation means the
// .fai does not describe the file.  The bytes are copied as they are (case, IUPAC codes), as pysam's fetch returns them.
__global__ void __launch_bounds__(UNW_THREADS) k_ref_unwrap(const uint8_t* __restrict__ raw, const Contig* __restrict__ ctg, const Tile* __restrict__ tiles, unsigned n_tiles,
                                                           uint8_t* __restrict__ out, Bad* bad) {
    __shared__ __align__(16) uint8_t stage[UNW_SMEM];
    for (unsigned t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const Tile tl = tiles[t]; const Contig c = ctg[tl.contig];
        const unsigned long long p0 = tl.start, p1 = min(tl.start + (unsigned long long)UNW_TILE, c.len);
        const unsigned long long lb = c.linebases, lw = c.linewidth;
        // source span of the tile, with the terminator of its last line
        const unsigned long long s0 = raw_pos(c, p0), s1 = raw_pos(c, p1 - 1) + 1 + (lw - lb);
        const unsigned long long a0 = s0 & ~15ull, a1 = (s1 + 15) & ~15ull;
        const bool staged = a1 - a0 <= (unsigned long long)UNW_SMEM;
        __syncthreads();                                                   // the previous tile's readers are done with `stage`
        if (staged)
            for (unsigned long long i = threadIdx.x; i < (a1 - a0) >> 4; i += UNW_THREADS) reinterpret_cast<uint4*>(stage)[i] = reinterpret_cast<const uint4*>(raw + a0)[i];
        __syncthreads();
        auto src = [&](unsigned long long s) -> uint8_t { return staged ? stage[s - a0] : raw[s]; };
        bool nl = false;
        for (unsigned long long q = p0 + 16ull * threadIdx.x; q < p1; q += 16ull * UNW_THREADS) {
            unsigned long long line = q / lb, col = q % lb, s = c.raw_off + line * lw + col;
            const int n = (int)min(16ull, p1 - q);
            uint8_t v[16];
            #pragma unroll
            for (int k = 0; k < 16; ++k) {
                if (k < n) { v[k] = src(s); nl = nl || v[k] == '\n' || v[k] == '\r'; } else v[k] = 0;
                if (++col == lb) { col = 0; s += lw - lb + 1; } else ++s;
            }
            uint8_t* dst = out + c.out_off + q;
            if (n == 16) { uint4 w; memcpy(&w, v, 16); *reinterpret_cast<uint4*>(dst) = w; }
            else for (int k = 0; k < n; ++k) dst[k] = v[k];
        }
        if (nl) flag_bad(bad, tl.contig, ~0ull >> 24);       // a line break inside the bases: the .fai length or offset is wrong; the line is found below
        // terminators of the lines whose last base lies in this tile and that more sequence follows
        for (unsigned long long k = p0 / lb + threadIdx.x; (k + 1) * lb - 1 < p1; k += UNW_THREADS) {
            if ((k + 1) * lb - 1 < p0 || (k + 1) * lb >= c.len) continue;
            const unsigned long long e = c.raw_off + k * lw + lb;
            const bool ok = lw == lb + 1 ? src(e) == '\n' : (src(e) == '\r' && src(e + 1) == '\n');
            if (!ok) flag_bad(bad, tl.contig, k);
        }
        if (nl) {      // name the first line of this tile that holds a line break among its bases
            for (unsigned long long k = p0 / lb + threadIdx.x; k * lb < p1; k += UNW_THREADS) {
                const unsigned long long b0 = max(k * lb, p0), b1 = min((k + 1) * lb, p1);
                for (unsigned long long p = b0; p < b1; ++p) { const uint8_t x = src(c.raw_off + k * lw + (p - k * lb)); if (x == '\n' || x == '\r') { atomicMin(&bad->first, ((unsigned long long)tl.contig << 40) | k); break; } }
            }
        }
    }
}

// ---- runs of 'N' (0x4E only: leadprov.py:439 compares with 78, so 'n' is not masked) ----
constexpr int NR_THREADS = 256;
constexpr int NR_TILE = 65536;                  // bases per tile (a tile never crosses a contig); every thread owns NR_PER consecutive bases
constexpr int NR_PER = NR_TILE / NR_THREADS;

// the run events among bases [b0, b0 + NR_PER) of a contig, in position order: on(p, true) where a run starts at p, on(p, false) where a
// run whose last base lies in the range ends (exclusive end p).  A run that crosses a tile or a thread boundary is one start and one end;
// runs never cross contigs, so the k-th start of the genome and its k-th end belong to the same run.
template <class F> __device__ __forceinline__ void nr_events(const uint8_t* __restrict__ g, const Contig& c, unsigned long long b0, F on) {
    if (b0 >= c.len) return;
    const unsigned long long b1 = min(b0 + (unsigned long long)NR_PER, c.len);
    const uint8_t* base = g + c.out_off;
    bool prev = b0 > 0 && base[b0 - 1] == 'N';
    const bool after = b1 < c.len && base[b1] == 'N';
    const uint4* w = reinterpret_cast<const uint4*>(base + b0);
    for (int j = 0; j < NR_PER / 16 && b0 + 16ull * j < b1; ++j) {
        const uint4 x = w[j]; uint8_t v[16]; memcpy(v, &x, 16);
        #pragma unroll
        for (int k = 0; k < 16; ++k) {
            const unsigned long long p = b0 + 16ull * j + k;
            if (p >= b1) break;
            const bool in = v[k] == 'N';
            if (in && !prev) on(p, true);
            if (!in && prev && p > b0) on(p, false);
            prev = in;
        }
    }
    if (prev && !after) on(b1, false);
}

// count pass: starts and ends per tile
__global__ void __launch_bounds__(NR_THREADS) k_ref_nruns_count(const uint8_t* __restrict__ g, const Contig* __restrict__ ctg, const Tile* __restrict__ tiles,
                                                                uint32_t* __restrict__ n_start, uint32_t* __restrict__ n_end) {
    const Tile tl = tiles[blockIdx.x]; const Contig c = ctg[tl.contig];
    uint32_t s = 0, e = 0;
    nr_events(g, c, tl.start + (unsigned long long)threadIdx.x * NR_PER, [&](unsigned long long, bool st) { if (st) ++s; else ++e; });
    uint32_t ts, te;
    prims::block_excl_scan(s, &ts); prims::block_excl_scan(e, &te);
    if (threadIdx.x == 0) { n_start[blockIdx.x] = ts; n_end[blockIdx.x] = te; }
}
// write pass: with the exclusive scans of the tile counts, every start and every end has its index; runs[2 i] = start, runs[2 i + 1] = end
__global__ void __launch_bounds__(NR_THREADS) k_ref_nruns_write(const uint8_t* __restrict__ g, const Contig* __restrict__ ctg, const Tile* __restrict__ tiles,
                                                                const uint32_t* __restrict__ off_start, const uint32_t* __restrict__ off_end, int32_t* __restrict__ runs) {
    const Tile tl = tiles[blockIdx.x]; const Contig c = ctg[tl.contig];
    const unsigned long long b0 = tl.start + (unsigned long long)threadIdx.x * NR_PER;
    uint32_t s = 0, e = 0;
    nr_events(g, c, b0, [&](unsigned long long, bool st) { if (st) ++s; else ++e; });
    uint32_t ts, te;
    uint32_t is = prims::block_excl_scan(s, &ts) + off_start[blockIdx.x], ie = prims::block_excl_scan(e, &te) + off_end[blockIdx.x];
    nr_events(g, c, b0, [&](unsigned long long p, bool st) { if (st) runs[2ull * is++] = (int32_t)p; else runs[2ull * ie++ + 1] = (int32_t)p; });
}

// ---- gathers: one warp per query, the lanes copy consecutive bytes ----
struct Query { unsigned long long src, len, dst; };
__global__ void k_ref_gather(const uint8_t* __restrict__ g, const Query* __restrict__ q, unsigned long long n, uint8_t* __restrict__ out) {
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    for (unsigned long long i = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += nw) {
        const Query x = q[i];
        for (unsigned long long k = lane_id(); k < x.len; k += 32) out[x.dst + k] = g[x.src + k];
    }
}

}  // namespace refseq
