// rnames.cuh — the names of every candidate's supporting reads (--output-rnames; sv.py:520-525, 555): the candidate's sorted distinct
// qname hashes, which stage B leaves next to its leads, resolved to the query name bytes of the record block still resident on the
// context.  Runs after stage B and writes nothing the run reads.
#pragma once
#include "common.cuh"

namespace rnames {

struct P {
    const snfb_cand* cand; unsigned long long n_cand;
    const snfb_lead* leads;                           // the run's cand_leads: a candidate owns [lead_off, lead_off + lead_n + long_n)
    const uint64_t* hash; const uint32_t* rn_off; unsigned long long n_names;      // per candidate its names hash[rn_off[c] .. rn_off[c + 1])
    const snfb_rec* rec; const uint8_t* var;          // the record block: a name is var[var_off .. + l_qname)
    uint32_t* first;                                  // per name: the index in leads[] of the candidate's first lead with its hash
    uint32_t* len;                                    // per name: its length in bytes (0 when no lead carries the hash)
    uint64_t* src;                                    // per name: its var offset
    uint32_t* off;                                    // per name: its offset in text (exclusive scan of len)
    unsigned long long* ctr;                          // [0] text bytes (64-bit: the u32 offsets must not wrap), [1] leads whose name differs
                                                      // from the one kept for their hash (a 64-bit hash collision), [2] names no lead carries
    uint8_t* text;
};

__device__ __forceinline__ unsigned long long name_end(const P& p, unsigned long long c) { return c + 1 < p.n_cand ? p.rn_off[c + 1] : p.n_names; }

// one warp per candidate: every lead finds its hash in the candidate's sorted list (binary search) and the smallest lead index per name
// wins (the first match in lead order); then each name takes its record's name, and every lead checks its own bytes against that name
__global__ void __launch_bounds__(128) k_resolve(P p) {
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const int lane = lane_id();
    for (unsigned long long c = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < p.n_cand; c += nw) {
        const snfb_cand cd = p.cand[c];
        const uint32_t lo = p.rn_off[c], hi = (uint32_t)name_end(p, c);
        const uint32_t l0 = (uint32_t)cd.lead_off, nl = (uint32_t)(cd.lead_n + cd.long_n);
        for (uint32_t j = lo + lane; j < hi; j += 32) p.first[j] = 0xffffffffu;
        __syncwarp();
        for (uint32_t i = lane; i < nl; i += 32) {
            const uint64_t h = p.leads[l0 + i].qname_hash;
            uint32_t a = lo, z = hi;
            while (a < z) { const uint32_t m = a + ((z - a) >> 1); if (p.hash[m] < h) a = m + 1; else z = m; }
            if (a < hi && p.hash[a] == h) atomicMin(&p.first[a], l0 + i);
        }
        __syncwarp();
        unsigned long long missing = 0, bytes = 0;
        for (uint32_t j = lo + lane; j < hi; j += 32) {
            const uint32_t f = p.first[j];
            if (f == 0xffffffffu) { p.len[j] = 0; p.src[j] = 0; ++missing; continue; }
            const snfb_rec& r = p.rec[p.leads[f].rec];
            p.len[j] = r.l_qname; p.src[j] = r.var_off; bytes += r.l_qname;
        }
        __syncwarp();
        unsigned long long differ = 0;
        for (uint32_t i = lane; i < nl; i += 32) {
            const snfb_lead& l = p.leads[l0 + i];
            uint32_t a = lo, z = hi;
            while (a < z) { const uint32_t m = a + ((z - a) >> 1); if (p.hash[m] < l.qname_hash) a = m + 1; else z = m; }
            if (!(a < hi && p.hash[a] == l.qname_hash) || p.first[a] == l0 + i) continue;
            const snfb_rec& r = p.rec[l.rec];
            const uint32_t n = p.len[a];
            bool same = r.l_qname == n;
            for (uint32_t k = 0; same && k < n; ++k) same = p.var[r.var_off + k] == p.var[p.src[a] + k];
            differ += !same;
        }
        #pragma unroll
        for (int o = 16; o; o >>= 1) { missing += __shfl_xor_sync(FULL, missing, o); differ += __shfl_xor_sync(FULL, differ, o); bytes += __shfl_xor_sync(FULL, bytes, o); }
        if (lane == 0 && bytes) atomicAdd(&p.ctr[0], bytes);
        if (lane == 0 && differ) atomicAdd(&p.ctr[1], differ);
        if (lane == 0 && missing) atomicAdd(&p.ctr[2], missing);
    }
}

// one warp per name: its bytes from the record block to text[off[j] ..), coalesced on both sides
__global__ void __launch_bounds__(256) k_copy(P p) {
    const unsigned long long nw = ((unsigned long long)gridDim.x * blockDim.x) >> 5;
    const int lane = lane_id();
    for (unsigned long long j = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < p.n_names; j += nw) {
        const uint32_t n = p.len[j]; const uint8_t* s = p.var + p.src[j]; uint8_t* d = p.text + p.off[j];
        for (uint32_t k = lane; k < n; k += 32) d[k] = s[k];
    }
}

}  // namespace rnames
