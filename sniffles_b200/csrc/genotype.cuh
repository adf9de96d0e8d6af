// genotype.cuh — force calling of given SVs (GenotypeTask.execute, parallel.py:300-369): every target is matched against the
// resident candidates of its task and gets the three coverage probes of postprocessing.coverage.  Runs after stage B on the same
// context and reads only what the run left (candidates, per-record arrays); it writes nothing the run reads.
#pragma once
#include "common.cuh"
#include "cluster.cuh"

namespace genotype {

constexpr int BINSIZE = 5000, BINEDGE = 500;          // parallel.py:307-308
constexpr int BIN_BITS = 20, TYPE_BITS = 3;           // |pos / 5000| < 2^19 for int32 positions
constexpr int KEY_BITS = BIN_BITS + TYPE_BITS;        // + the task bits above them

// candidate bin key (task, svtype, bin); SINGLE_* get svtype field 7, which no target asks for
__device__ __forceinline__ uint64_t bin_key(uint64_t task, int svtype, long long bin) {
    return (task << KEY_BITS) | ((uint64_t)svtype << BIN_BITS) | (uint64_t)(bin + (1ll << (BIN_BITS - 1)));
}

__global__ void k_cand_keys(const snfb_cand* __restrict__ cand, unsigned long long n, uint64_t* __restrict__ key, uint32_t* __restrict__ val) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const snfb_cand& c = cand[i];
        const int ty = c.svtype == SNFB_SINGLE_LEFT || c.svtype == SNFB_SINGLE_RIGHT ? 7 : c.svtype;
        key[i] = bin_key((uint64_t)c.task, ty, c.pos / BINSIZE); val[i] = (uint32_t)i;      // int(cand.pos / binsize), C truncation
    }
}

struct P {
    cluster::B b;                                     // the run's bound arrays: candidates, records, tasks
    const uint64_t* key; const uint32_t* val; unsigned long long n_cand;     // candidate keys sorted, candidate index per key
    unsigned long long n;                             // targets, ordered by task then input order
    const int32_t* task; const int32_t* svtype; const int32_t* pos; const int32_t* svlen; const int32_t* bnd_is_first; const int32_t* mate_contig;
    const int64_t* prev;                              // previous non-BND target of the same task, -1 none (filled on the host)
    int combine_match, combine_match_max, cluster_merge_bnd;
    long long* match; int32_t* cov_start; int32_t* cov_center; int32_t* cov_end; int32_t* bnd_no_prev;
};

__device__ __forceinline__ unsigned long long lower_bound(const uint64_t* k, unsigned long long n, uint64_t x) {
    unsigned long long a = 0, z = n;
    while (a < z) { const unsigned long long m = a + ((z - a) >> 1); if (k[m] < x) a = m + 1; else z = m; }
    return a;
}

// one warp per target: the nearest candidate of the target's bins (distance, then emission order), then the coverage probes
__global__ void k_genotype(P g) {
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const auto at = [&](long long j) { return cluster::CovSv{ g.task[j], g.svtype[j], g.pos[j], g.svlen[j], g.bnd_is_first[j] }; };
    const auto prev = [&](long long j) { return (long long)g.prev[j]; };
    for (unsigned long long i = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < g.n; i += nw) {
        const int t = g.task[i], st = g.svtype[i]; const long long pos = g.pos[i], tlen = g.svlen[i] < 0 ? -(long long)g.svlen[i] : g.svlen[i];
        const int mate = g.mate_contig[i];
        unsigned long long best = ~0ull;              // (dist << 32) | candidate index
        if (st >= SNFB_INS && st <= SNFB_BND) {
            const long long bin = pos / BINSIZE, m = ((pos % BINSIZE) + BINSIZE) % BINSIZE;      // int(pos / binsize); Python's floor modulo
            const long long bins[2] = { bin, m < BINEDGE ? bin - 1 : (m > BINSIZE - BINEDGE ? bin + 1 : bin) };
            for (int k = 0; k < (bins[1] != bin ? 2 : 1); ++k) {
                const uint64_t key = bin_key((uint64_t)t, st, bins[k]);
                const unsigned long long lo = lower_bound(g.key, g.n_cand, key), hi = lower_bound(g.key, g.n_cand, key + 1);
                for (unsigned long long j = lo + lane_id(); j < hi; j += 32) {
                    const uint32_t ci = g.val[j]; const snfb_cand& c = g.b.cand[ci];
                    const long long dpos = pos > c.pos ? pos - c.pos : c.pos - pos;
                    long long dist; bool ok;
                    if (st == SNFB_BND) { dist = dpos; ok = dist <= g.cluster_merge_bnd && mate >= 0 && c.bnd_mate_contig == mate; }
                    else {
                        const long long clen = c.svlen < 0 ? -(long long)c.svlen : c.svlen;
                        dist = dpos + (tlen > clen ? tlen - clen : clen - tlen);
                        const long long minlen = tlen < clen ? tlen : clen;
                        // dist <= combine_match * math.sqrt(minlen): both operations correctly rounded, no contraction, as in CPython
                        ok = minlen > 0 && (double)dist <= __dmul_rn((double)g.combine_match, __dsqrt_rn((double)minlen)) && dist <= g.combine_match_max;
                    }
                    if (ok) { const unsigned long long v = ((unsigned long long)dist << 32) | ci; if (v < best) best = v; }
                }
            }
            #pragma unroll
            for (int o = 16; o; o >>= 1) { const unsigned long long x = __shfl_xor_sync(FULL, best, o); if (x < best) best = x; }
        }
        long long p[5];
        const bool has_end = cluster::cov_probes((long long)i, at, prev, (long long)g.b.cfg.coverage_binsize, (long long)g.b.cfg.coverage_binsize * g.b.cfg.coverage_updown_bins, p);
        int v[3] = { 0, 0, 0 };
        for (int k = 0; k < 3; ++k) cluster::cov_at_warp(g.b, t, p[k + 1], &v[k]);
        if (lane_id() == 0) {
            g.match[i] = best == ~0ull ? -1ll : (long long)(best & 0xffffffffull);
            g.cov_start[i] = v[0]; g.cov_center[i] = v[1]; g.cov_end[i] = v[2]; g.bnd_no_prev[i] = has_end ? 0 : 1;
        }
    }
}

}  // namespace genotype
