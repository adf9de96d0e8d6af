// ingest.cuh — SURVEY §8 (f)3: compressed BAM bytes -> the packed record block of include/snfb.h, on the device.
// Replaces the host decode behind `bam.fetch(contig, start, end)` (parallel.py:95-98, leadprov.py:488): only the BGZF bytes cross
// PCIe; inflate, record decode, filtering to the task's region, the CG long-CIGAR escape and the CIGAR16 packing run here.
//
//   k_inflate      16 lanes per BGZF block (ingest_core.h inflate_stream<16>): the Huffman tables of a block in
//                  shared memory, the scalar decode executed redundantly by the block's lanes, match copies / table fills / stored blocks split
//                  across them; the two blocks of a warp share its instruction stream wherever they run the same path; then the same
//                  lanes check the block's CRC-32 (crc32_group<16>)
//   k_walk         one thread per span (a record-aligned range of the inflated stream, cut at the BAI's linear-index anchors):
//                  follows the block_size chain, first to count, then to write the record offsets
//   k_parse        one thread per raw record: fixed fields, aux walk (NM, HP, PS, SA, CG), task filter on contig and end
//   k_rec_sizes    one warp per raw record: CIGAR16 word count + reference span (finishes the region-overlap filter)
//   (four scans)   new record index / CIGAR16 groups / var and seq arenas in 16-byte units
//   k_pack         one warp per kept record: snfb_rec, names + SA text, 4-bit bases, CIGAR16 words
#pragma once
#include "common.cuh"
#include "prims.cuh"
#include "ingest_core.h"

namespace ingest {

// DEFLATE payload in the compressed buffer, its inflated size and CRC-32 (the block's gzip trailer), where it lands
struct BgzfBlock { unsigned long long in_off; unsigned in_len; unsigned isize; unsigned long long out_off; unsigned crc; unsigned _pad; };
struct Span { unsigned long long ubeg, uend; unsigned task; unsigned region; };                                   // record-aligned range of the inflated stream owned by one task (and region)
// first_bad_inv = ~(block << 8 | INF_* code) of the lowest failing block: an atomicMax of the complement, so the zeroed counters need no
// other initial value and the block reported does not depend on which group failed first
struct IngestCounters { unsigned long long bad_blocks, first_bad_inv, bad_chain, malformed, bad_cigar, n_raw, n_keep, n_groups, n_var, n_seq16; };

constexpr int INF_WARPS = 8;
// lanes per BGZF block: two blocks per warp (their decodes share the warp's instruction stream where they run the same path — a
// literal-heavy stream mostly does — and diverge where they do not)
constexpr int INF_LANES = 16;
// the CRC tables once per thread block, then one WarpTables per block being decoded.  41,088 B: launch_inflate still sizes its grid for 5 thread blocks per SM
constexpr size_t INF_SMEM_BYTES = sizeof(CrcTables) + sizeof(WarpTables) * INF_WARPS * (32 / INF_LANES);
static_assert(INF_SMEM_BYTES <= 48 * 1024, "k_inflate's tables must fit the default dynamic shared memory limit (48 KB)");

// every block is decoded, checked against its ISIZE, then against its CRC-32
__global__ void __launch_bounds__(INF_WARPS * 32) k_inflate(const uint8_t* __restrict__ comp, const BgzfBlock* __restrict__ blocks, unsigned n_blocks, uint8_t* __restrict__ raw, IngestCounters* ctr) {
    extern __shared__ __align__(16) uint8_t inflate_smem[];
    constexpr int GPW = 32 / INF_LANES;                       // groups per warp
    CrcTables* crc_tab = reinterpret_cast<CrcTables*>(inflate_smem);
    WarpTables* tables = reinterpret_cast<WarpTables*>(inflate_smem + sizeof(CrcTables));
    crc_tables_fill(crc_tab, threadIdx.x, blockDim.x);
    __syncthreads();
    const int w = threadIdx.x >> 5, g = (threadIdx.x & 31) / INF_LANES, lane = (threadIdx.x & 31) % INF_LANES;
    const unsigned gmask = ((1u << INF_LANES) - 1u) << (g * INF_LANES);
    WarpTables* T = tables + (w * GPW + g);
    const unsigned stride = gridDim.x * INF_WARPS * GPW;
    for (unsigned b = (blockIdx.x * INF_WARPS + w) * GPW + g; b < n_blocks; b += stride) {
        const BgzfBlock B = blocks[b];
        uint32_t produced = 0;
        int rc = inflate_stream<INF_LANES>(comp, B.in_off, B.in_off + B.in_len, raw + B.out_off, B.isize, T, lane, gmask, &produced);
        if (rc == INF_OK && produced != B.isize) rc = INF_LENGTH_MISMATCH;
        if (rc == INF_OK && crc32_group<INF_LANES>(raw + B.out_off, B.isize, crc_tab, lane, gmask) != B.crc) rc = INF_CRC_MISMATCH;
        if (rc != INF_OK && lane == 0) { atomicAdd(&ctr->bad_blocks, 1ULL); atomicMax(&ctr->first_bad_inv, ~(((unsigned long long)b << 8) | (unsigned)rc)); }
    }
}

// the fetch window of a raw record: its region with a region table (snfb_set_regions), else its task's
__device__ __forceinline__ int2 fetch_window(const snfb_task* task, const snfb_region* region, unsigned t, const uint32_t* raw_region, unsigned i) {
    if (region) { const snfb_region g = region[raw_region[i]]; return make_int2(g.start, g.end); }
    return make_int2(task[t].start, task[t].end);
}

// mode 0: span_cnt[s] = records in the span; mode 1: rec_body[base[s] + k] / rec_bs / rec_task, and the span's region
__global__ void k_walk(const uint8_t* __restrict__ raw, unsigned long long raw_len, const Span* __restrict__ spans, unsigned n_spans, int mode,
                       uint32_t* __restrict__ span_cnt, const uint32_t* __restrict__ span_base, RawRec* __restrict__ recs, uint32_t* __restrict__ raw_region, unsigned long long rec_cap, IngestCounters* ctr) {
    const unsigned s = blockIdx.x * blockDim.x + threadIdx.x; if (s >= n_spans) return;
    const Span sp = spans[s];
    unsigned long long off = sp.ubeg; uint32_t n = 0; const uint32_t base = mode ? span_base[s] : 0u;
    while (off + 4 <= sp.uend && off + 4 <= raw_len) {
        const uint32_t bs = ld32u(raw, off);
        if (bs < 32u || off + 4ull + bs > raw_len) { if (!mode) atomicAdd(&ctr->bad_chain, 1ULL); break; }
        if (mode && (unsigned long long)base + n < rec_cap) { RawRec& r = recs[base + n]; r.body = off + 4; r.body_len = bs; r.task = sp.task; raw_region[base + n] = sp.region; }
        ++n; off += 4ull + bs;
    }
    if (!mode) { if (off != sp.uend && off + 4 <= raw_len) atomicAdd(&ctr->bad_chain, 1ULL); span_cnt[s] = n; }      // a span must end on a record boundary
}

__global__ void k_parse(const uint8_t* __restrict__ raw, RawRec* __restrict__ recs, const uint32_t* __restrict__ raw_region, unsigned n_raw, const snfb_task* __restrict__ task,
                        const snfb_region* __restrict__ region, IngestCounters* ctr) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x; if (i >= n_raw) return;
    const unsigned long long body = recs[i].body; const uint32_t bs = recs[i].body_len; const unsigned t = recs[i].task;
    RawRec r; parse_record(raw, body, bs, &r); r.task = t;
    if (r.status == ST_MALFORMED) atomicAdd(&ctr->malformed, 1ULL);
    else {
        const snfb_task k = task[t];
        if (r.ref_id != k.contig || r.pos >= fetch_window(task, region, t, raw_region, i).y) r.status = ST_FILTERED;      // bam.fetch(contig, start, end): the overlap test on the start side needs the CIGAR (k_rec_sizes)
    }
    recs[i] = r;
}

// warp per raw record
__global__ void __launch_bounds__(256) k_rec_sizes(const uint8_t* __restrict__ raw, RawRec* __restrict__ recs, const uint32_t* __restrict__ raw_region, unsigned n_raw, const snfb_task* __restrict__ task,
                                                   const snfb_region* __restrict__ region, uint32_t evt_min,
                                                   uint32_t* __restrict__ keep, uint32_t* __restrict__ groups, uint32_t* __restrict__ var16, uint32_t* __restrict__ seq16, IngestCounters* ctr) {
    const int lane = threadIdx.x & 31;
    for (unsigned i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_raw; i += (gridDim.x * blockDim.x) >> 5) {
        const RawRec r = recs[i];
        uint32_t kp = 0, g = 0, vb = 0, sq = 0;
        if (r.status == ST_OK) {
            long long reflen = 0; int bad = 0;
            const uint32_t words = c16_convert<32>(raw, r.cig_src, r.n_cig, nullptr, evt_min, lane, &reflen, &bad);
            if (bad) { if (lane == 0) { atomicAdd(&ctr->bad_cigar, 1ULL); recs[i].status = ST_MALFORMED; } }
            else if ((long long)r.pos + (reflen > 1 ? reflen : 1) > (long long)fetch_window(task, region, r.task, raw_region, i).x) {
                kp = 1; g = (words + 7u) >> 3; vb = ((uint32_t)r.l_qname + r.sa_len + 15u) >> 4; sq = ((uint32_t)((r.l_seq + 1) / 2) + 15u) >> 4;
            } else if (lane == 0) recs[i].status = ST_FILTERED;
        }
        if (lane == 0) { keep[i] = kp; groups[i] = g; var16[i] = vb; seq16[i] = sq; }
    }
}

// warp per raw record; the four scans gave every kept record its index and its arena offsets
__global__ void __launch_bounds__(256) k_pack(const uint8_t* __restrict__ raw, const RawRec* __restrict__ recs, const uint32_t* __restrict__ raw_region, unsigned n_raw, uint32_t evt_min,
                                              const uint32_t* __restrict__ keep, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ grp_off, const uint32_t* __restrict__ groups,
                                              const uint32_t* __restrict__ var_off16, const uint32_t* __restrict__ seq_off16,
                                              snfb_rec* __restrict__ out_rec, uint16_t* __restrict__ out_cigar, uint8_t* __restrict__ out_var, uint8_t* __restrict__ out_seq) {
    const int lane = threadIdx.x & 31;
    for (unsigned i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_raw; i += (gridDim.x * blockDim.x) >> 5) {
        if (!keep[i]) continue;
        const RawRec r = recs[i];
        const unsigned long long co = 8ull * grp_off[i], vo = 16ull * var_off16[i], so = 16ull * seq_off16[i];
        uint16_t* cg = out_cigar + co;
        long long reflen; int bad = 0;
        const uint32_t words = c16_convert<32>(raw, r.cig_src, r.n_cig, cg, evt_min, lane, &reflen, &bad);
        for (uint32_t k = words + lane; k < 8u * groups[i]; k += 32) cg[k] = 0;           // pad the record to whole 16-byte groups
        const uint8_t* q = raw + r.body + 32;
        for (uint32_t j = lane; j < r.l_qname; j += 32) out_var[vo + j] = q[j];
        for (uint32_t j = lane; j < r.sa_len; j += 32) out_var[vo + r.l_qname + j] = raw[r.sa_src + j];
        const uint32_t nb = (uint32_t)((r.l_seq + 1) / 2);
        uint32_t* dst = reinterpret_cast<uint32_t*>(out_seq + so);                         // 16-byte aligned
        for (uint32_t j = 4u * lane; j < nb; j += 128u) {
            uint32_t v = ld32u(raw, r.seq_src + j);
            if (j + 4u > nb) v &= 0xffffffffu >> (8u * (j + 4u - nb));
            dst[j >> 2] = v;
        }
        if (lane == 0) {
            snfb_rec o; memset(&o, 0, sizeof(o));
            o.task = (int32_t)r.task; o.pos = r.pos; o.flag = r.flag; o.mapq = r.mapq; o.aux_flags = r.aux_flags; o.hp = r.hp; o.l_qname = r.l_qname; o.nm = r.nm; o.ps = r.ps;
            o.n_cigar = words; o.l_seq = r.l_seq; o.sa_len = r.sa_len; o.cigar_off = co; o.seq_off = so; o.var_off = vo; o.region = raw_region[i];
            out_rec[idx[i]] = o;
        }
    }
}

}  // namespace ingest
