// bgzf_write.cuh — BGZF compression on the device (snfb_deflate_bgzf): the encoder of deflate_core.h with a thread block per BGZF block.
//
//   k_deflate   one thread block (DEF_THREADS) per member of the table moff (member k = in[moff[k], moff[k + 1]), at most 0xff00 bytes;
//               snfb_deflate_bgzf passes fixed 0xff00 cuts, snfb_sort_bam htslib's record-aware ones), grid-stride over the members with one resident block per SM
//               (the block's bytes, match lengths and bit buffer take ~217 KB of shared memory).  Warp 0 finds the hash candidates
//               while warp 1 computes the CRC-32 (crc32_group<32>); every thread computes match lengths; warp 0 parses; every thread
//               counts symbols, thread 0 builds the codes and picks the block type; every thread writes its slice's tokens; the member
//               goes to a 64 KiB slot.  cand[] / dist[] (2 x 0xff00 u16 per resident block) live in global memory.
//   (scan)      member sizes -> offsets in the packed output (prims::exclusive_scan)
//   k_pack      one thread block per member: slot -> packed output
#pragma once
#include "common.cuh"
#include "deflate_core.h"

namespace bgzfw {

constexpr int DEF_THREADS = 512;
static_assert(DEF_THREADS <= deflate::MAX_THREADS, "one bit count per thread");
constexpr size_t DEF_SMEM_BYTES = sizeof(deflate::Shared);
static_assert(DEF_SMEM_BYTES <= 227 * 1024, "k_deflate's shared memory must fit one thread block per SM on sm_90");

__global__ void __launch_bounds__(DEF_THREADS, 1) k_deflate(const uint8_t* __restrict__ in, const unsigned long long* __restrict__ moff, unsigned nb, uint16_t* __restrict__ scratch,
                                                             uint8_t* __restrict__ slots, uint32_t* __restrict__ sizes) {
    extern __shared__ __align__(16) uint8_t deflate_smem[];
    deflate::Shared* S = reinterpret_cast<deflate::Shared*>(deflate_smem);
    const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
    ingest::crc_tables_fill(&S->crc, tid, DEF_THREADS);
    uint16_t* cand = scratch + 2ull * deflate::BLOCK_IN * blockIdx.x;
    uint16_t* dist = cand + deflate::BLOCK_IN;
    for (unsigned k = blockIdx.x; k < nb; k += gridDim.x) {
        const unsigned long long off = moff[k];
        const uint32_t n = (uint32_t)(moff[k + 1] - off);
        __syncthreads();                                       // the previous block is written out
        deflate::stage(S, in + off, n, tid, DEF_THREADS);
        __syncthreads();
        if (w == 0) deflate::find_candidates<32>(S, cand, lane);
        else if (w == 1) { const uint32_t c = ingest::crc32_group<32>(S->data, n, &S->crc, lane, 0xffffffffu); if (lane == 0) S->crc_val = c; }
        __syncthreads();
        deflate::longest_matches(S, cand, dist, tid, DEF_THREADS);
        __syncthreads();
        if (w == 0) deflate::greedy_parse<32>(S, lane);
        __syncthreads();
        deflate::histogram(S, dist, tid, DEF_THREADS);
        __syncthreads();
        if (tid == 0) deflate::plan(S);
        __syncthreads();
        if (S->btype != 0) {
            deflate::count_bits(S, dist, tid, DEF_THREADS);
            __syncthreads();
            if (tid == 0) deflate::write_header(S, DEF_THREADS);
            __syncthreads();
            deflate::write_tokens(S, dist, tid);
            __syncthreads();
        }
        const uint32_t size = deflate::write_member(S, slots + (unsigned long long)k * deflate::MEMBER_MAX, tid, DEF_THREADS);
        if (tid == 0) sizes[k] = size;
    }
}

__global__ void __launch_bounds__(256) k_pack(const uint8_t* __restrict__ slots, const uint32_t* __restrict__ sizes, const uint32_t* __restrict__ offs, unsigned nb, uint8_t* __restrict__ out) {
    for (unsigned k = blockIdx.x; k < nb; k += gridDim.x) {
        const uint8_t* src = slots + (unsigned long long)k * deflate::MEMBER_MAX; uint8_t* dst = out + offs[k];
        const uint32_t n = sizes[k];
        for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) dst[j] = src[j];
    }
}

}  // namespace bgzfw
