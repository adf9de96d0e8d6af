// api.cu — C ABI of libsnfb200.so (include/snfb.h): context, memory, stage drivers.
// The product path has no CPU implementation: every stage below launches CUDA kernels.
//
// Run model.  Every buffer of the pipeline has a capacity kept in the context.  A run enqueues stage A -> B -> C on the
// context's stream WITHOUT host synchronisation: sizes live in device counters, kernels are launched for the capacities
// and bound their loops and stores by the device-side counts.  The host looks at the counters twice: once on the copy
// stream after stage B (while the consensus kernels run) to size the device -> host copies, and once at the end.  If a
// capacity was too small (first run on a context, or a block unlike the previous one) the run is repeated with
// capacities that fit — the counters always report what was needed.
#include <algorithm>
#include <chrono>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <dlfcn.h>
#include <omp.h>

#include "common.cuh"
#include "prims.cuh"
#include "extract.cuh"
#include "cluster.cuh"
#include "consensus.cuh"
#include "poa.cuh"
#include "combine.cuh"
#include "population.cuh"
#include "ingest.cuh"
#include "bgzf_write.cuh"
#include "genotype.cuh"
#include "rnames.cuh"
#include "reference.cuh"
#include "bam_index.cuh"
#include "bam_sort.cuh"

// one owning allocation of device memory, or of pinned host memory when Pinned; freed by the destructor
template <bool Pinned> struct Buf {
    void* p = nullptr; size_t cap = 0;
    Buf() = default;
    Buf(const Buf&) = delete; Buf& operator=(const Buf&) = delete;
    ~Buf() { release(); }
    // grows only; the old allocation is freed before the new one is made, so the peak holds one of them
    int ensure(size_t bytes) {
        if (bytes <= cap) return 0;
        release();
        size_t want = bytes + bytes / 8 + 256;
        if ((Pinned ? cudaMallocHost(&p, want) : cudaMalloc(&p, want)) != cudaSuccess) { p = nullptr; cudaGetLastError(); return 1; }
        cap = want; return 0;
    }
    template <class T> T* as() { return reinterpret_cast<T*>(p); }
    void reset() { release(); }      // gives the memory back (a transient buffer)
private:
    void release() { if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); } p = nullptr; cap = 0; }
};
using DevBuf = Buf<false>;
using HostBuf = Buf<true>;
// one allocation carved into 256-byte aligned arrays: a measuring pass, then an assigning pass over the same list
struct Carver {
    uint8_t* base = nullptr; size_t off = 0;
    template <class T> T* take(size_t n) { const size_t o = off; off += (n * sizeof(T) + 255) & ~(size_t)255; return base ? reinterpret_cast<T*>(base + o) : nullptr; }
};
// runs the layout lay(Carver&) to measure, grows buf to fit, runs it again over buf to assign the pointers; nonzero when out of memory
template <bool Pinned, class Lay> static int carve(Buf<Pinned>& buf, Lay&& lay) {
    Carver m; lay(m);
    if (buf.ensure(m.off + 256)) return 1;
    Carver a; a.base = buf.template as<uint8_t>(); lay(a);
    return 0;
}

constexpr int MAX_TIMINGS = 64;

// ---- NCCL, resolved at run time (the library links no collective library: a process that never gathers needs none) ----
struct Id128 { char b[128]; };      // ncclUniqueId is passed by value: 128 bytes
struct NcclApi {
    void* h = nullptr; bool tried = false;
    int (*GetUniqueId)(void*) = nullptr; int (*CommInitRank)(void**, int, Id128, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr; int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr; const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl;
static bool nccl_load(std::string* err) {
    if (g_nccl.tried) { if (!g_nccl.AllGather && err) *err = "NCCL is not available in this process"; return g_nccl.AllGather != nullptr; }
    g_nccl.tried = true;
    // a process that already carries NCCL (torch) must use that copy: two NCCL instances do not share bootstrap state
    void* h = dlopen(nullptr, RTLD_NOW | RTLD_GLOBAL);
    if (!h || !dlsym(h, "ncclAllGather")) { h = nullptr; const char* names[] = { "libnccl.so.2", "libnccl.so" }; for (const char* n : names) { h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (h) break; } }
    if (!h) { if (err) *err = "libnccl.so.2 not found"; return false; }
    g_nccl.h = h;
    g_nccl.GetUniqueId = (int (*)(void*))dlsym(h, "ncclGetUniqueId");
    g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(h, "ncclCommInitRank");
    g_nccl.CommDestroy = (int (*)(void*))dlsym(h, "ncclCommDestroy");
    g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(h, "ncclAllGather");
    g_nccl.GetErrorString = (const char* (*)(int))dlsym(h, "ncclGetErrorString");
    if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.CommDestroy || !g_nccl.AllGather) { g_nccl.AllGather = nullptr; if (err) *err = "NCCL symbols missing"; return false; }
    return true;
}

struct Caps { unsigned long long lead = 0, cand = 0, cand_lead = 0, rn = 0, alt = 0, scr16 = 0, item = 0, tile = 0, req = 0, req16 = 0; };

struct snfb_ctx {
    int device = 0; cudaStream_t st = nullptr, st_copy = nullptr, st_side = nullptr; cudaEvent_t ev_b = nullptr, ev_mid = nullptr, ev_fork = nullptr, ev_join = nullptr; std::string err;
    // stage C slices: each one's k_align / k_vote has ended
    cudaEvent_t ev_aligned[consensus::MAX_SLICES] = {}, ev_slice[consensus::MAX_SLICES] = {}; int n_slices = consensus::DEFAULT_SLICES;
    snfb_config cfg{}; bool have_cfg = false;
    // records
    bool loaded = false, on_device = false, seq_on_demand = false; const uint8_t* h_seq = nullptr; uint32_t evt_min = 0;     // E-bit threshold of the loaded CIGAR16 arena
    uint64_t n_rec = 0, n_cigar = 0, n_var = 0, n_seq = 0; uint32_t n_task = 0, n_contig = 0, n_tr = 0, n_mask = 0;
    const snfb_rec* d_rec = nullptr; const uint16_t* d_cigar = nullptr; const uint8_t* d_var = nullptr; const uint8_t* d_seq = nullptr;
    DevBuf b_rec, b_cigar, b_var, b_seq, b_task, b_contig, b_tr, b_trp, b_mask, b_mask_off, b_mask_task;
    HostBuf h_c16, h_rec16;        // BAM32 host input converted to CIGAR16 before the upload
    DevBuf b_comp, b_raw, b_ing, b_ing_span, b_ing_work; HostBuf h_ing; uint64_t ing_sizes[8] = {0, 0, 0, 0, 0, 0, 0, 0}; bool from_bam = false;      // device BAM ingest: BGZF bytes, inflated stream, counters / block table, span tables, per-raw-record work arrays
    DevBuf b_zin, b_zslot, b_zout, b_zwork;          // BGZF compression: input bytes, 64 KiB member slots, packed members, sizes / offsets / candidate scratch
    DevBuf b_gt;                                     // force calling: candidate bin keys, sort scratch, targets and their results
    DevBuf b_rn, b_rn_text; HostBuf h_rn_meta, h_rn_text;     // read names: per-name scratch and counters, the text; counters + offsets, text on the host
    // population table (snfb_population_load): sorted keys and columns, the ALT arena; b_popq: one batch of queries and their results
    DevBuf b_pop, b_popq; population::P pop{}; bool have_pop = false;
    DevBuf b_ref, b_ref_work; std::vector<refseq::Contig> ref_ctg; bool have_ref = false;     // the unwrapped reference genome; tables / counters / N-run scratch
    HostBuf h_ref_runs, h_ref_coff, h_ref_out; uint64_t ref_n_runs = 0;                       // N runs and per-contig offsets; gather staging
    // BAM index (snfb_index_bam): per-window candidate masks, chain nodes, the carried record; all rows; the table work; the tables on the host
    DevBuf b_ix_mask, b_ix_node, b_ix_carry, b_ix_rows, b_ix_tab;
    std::vector<uint64_t> ix_ref, ix_lin_off, ix_lin, ix_bin_key, ix_bin_loff, ix_chunk_u, ix_chunk_v; std::vector<uint32_t> ix_chunk_bin;
    // BAM sort (snfb_sort_bam): per-record keys, lengths, offsets and their sort; one window's keys; bucket and window tables; a bucket's bytes
    DevBuf b_st_rec, b_st_win, b_st_lay, b_st_bkt;
    std::vector<snfb_task> tasks;
    // region table (snfb_set_regions): host copy, device copy followed by each task's last region index; cov_view: some task's regions
    // are not increasing and disjoint, so stage A builds the coordinate-ordered (pos, end, flags) the coverage readers search
    std::vector<snfb_region> regions, next_regions; DevBuf b_region; uint32_t n_region = 0; bool cov_view = false;
    // capacities and the three arenas carved by them
    Caps cap; bool force_no_cuts = false;
    DevBuf b_ctr, arena_r, arena_l, arena_c;            // counters; per-record arrays; per-lead arrays (stages A + B); stage C
    // per-record (arena_r)
    int32_t* rec_pos; int32_t* rec_end; uint8_t* rec_flags; double* rec_nm; uint32_t* rec_nlead; uint32_t* rec_lead_off; uint32_t* sa_list; extract::RecScan* scanrec; extract::RecClip* clip; int32_t* rec_big;
    uint32_t* task_first; uint32_t* task_last; uint32_t* task_reads; unsigned long long* task_cov; int32_t* task_span; double* task_nm; double* nm_part; unsigned* nm_cnt; extract::Seg* sa_seg; uint32_t* scan_tmp_r;
    // the coordinate-ordered copy of (rec_pos, rec_end, rec_flags) and its sort scratch (one element each unless cov_view)
    int32_t* v_pos; int32_t* v_end; uint8_t* v_flags; uint64_t* v_k0; uint64_t* v_k1; uint32_t* v_v0; uint32_t* v_v1; uint32_t* v_hist; uint32_t* v_scan; unsigned long long* v_n;
    // per-lead (arena_l): stage A leads + the whole of stage B
    snfb_lead* leads; extract::Event* ev_buf; snfb_lead* sorted_leads; uint32_t* radix_hist;
    cluster::B B{};
    // stage C (arena_c)
    consensus::C Cc{}; consensus::SeqReq* seq_req; uint32_t* arena_off; uint8_t* seq_arena; uint32_t* q_scan_tmp;
    HostBuf h_seq_req, h_seq_arena; uint64_t seq_h2d_bytes = 0;
    bool stage_a_done = false, stage_b_done = false, stage_c_done = false;
    // host staging
    HostBuf h_ctr_buf; DevCounters* h_mid = nullptr; DevCounters* h_fin = nullptr; consensus::Work* h_work = nullptr;      // h_work[0] read with h_mid, h_work[1] with h_fin
    HostBuf h_leads, h_task_reads, h_task_nm, h_rec_nm, h_cand, h_cand_leads, h_rnames, h_rn_off, h_task_cov, h_task_cov_raw, h_alt, h_cov_bins;
    // gather
    void* comm = nullptr; int rank = 0, nranks = 1; DevBuf b_gsend, b_grecv; HostBuf h_gather, h_gather_out; unsigned long long gather_cap = 0;     // h_gather: layout words, header table, rank_n_cand; h_gather_out: the merged arrays
    // timings
    cudaEvent_t ev[MAX_TIMINGS + 1]; const char* ev_name[MAX_TIMINGS + 1]; uint64_t ev_bytes[MAX_TIMINGS + 1]; int n_ev = 0; int n_ev_load = 0; uint64_t launches = 0; uint64_t reruns = 0;
};

// the shortest I / D / S the configured path looks at: SV signatures of minsvlen_screen, indels above 10 for the NM correction (leadprov.py:198-224)
static uint32_t evt_need(const snfb_ctx* ctx) {
    if (!ctx->have_cfg) return SNFB_CIGAR16_EVT_MIN;
    int t = ctx->cfg.minsvlen_screen < 1 ? 1 : ctx->cfg.minsvlen_screen;
    if ((ctx->cfg.qc_nm_measure || ctx->cfg.phase) && t > 11) t = 11;
    return (uint32_t)(t < (int)SNFB_CIGAR16_EVT_MIN ? t : (int)SNFB_CIGAR16_EVT_MIN);
}
static void ctx_fail(snfb_ctx* ctx, const char* what, const char* msg) { ctx->err = std::string(what) + ": " + msg; }
static int fail(snfb_ctx* ctx, const std::string& m) { ctx->err = m; return 1; }

// timing marks: every call records an event on the ctx stream; a named mark opens an interval that the
// next mark (named or not) closes, so host-side gaps between stages are never attributed to a kernel
static void mark(snfb_ctx* ctx, const char* name, uint64_t bytes = 0) {
    if (ctx->n_ev >= MAX_TIMINGS) return;
    cudaEventRecord(ctx->ev[ctx->n_ev], ctx->st);
    ctx->ev_name[ctx->n_ev] = name; ctx->ev_bytes[ctx->n_ev] = bytes; ++ctx->n_ev;
}
static int grid_for(unsigned long long n, int threads) { unsigned long long g = (n + threads - 1) / threads; if (g < 1) g = 1; if (g > (uint64_t)NUM_SMS * 32) g = (uint64_t)NUM_SMS * 32; return (int)g; }
static int bits_for(uint32_t n) { int b = 0; while ((1ull << b) < n) ++b; return b; }

__global__ void k_gather_leads(const snfb_lead* __restrict__ leads, const uint32_t* __restrict__ sval, snfb_lead* __restrict__ out, const unsigned long long* n_ptr, unsigned long long cap) {
    const unsigned long long n = *n_ptr < cap ? *n_ptr : cap;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) out[i] = leads[sval[i]];
}
// sort keys of the coordinate-ordered record view: (task, pos) with the sign of pos flipped so that unsigned order is numeric order
__global__ void k_view_keys(const snfb_rec* __restrict__ rec, const int32_t* __restrict__ rec_pos, unsigned long long n, uint64_t* __restrict__ key, uint32_t* __restrict__ val, unsigned long long* n_out) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        key[i] = ((uint64_t)(uint32_t)__ldg(&rec[i].task) << 32) | (uint64_t)((uint32_t)rec_pos[i] ^ 0x80000000u); val[i] = (uint32_t)i;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) *n_out = n;
}
__global__ void k_view_gather(const uint32_t* __restrict__ ord, unsigned long long n, const int32_t* __restrict__ pos, const int32_t* __restrict__ end, const uint8_t* __restrict__ flags,
                              int32_t* __restrict__ v_pos, int32_t* __restrict__ v_end, uint8_t* __restrict__ v_flags) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const uint32_t j = ord[i]; v_pos[i] = pos[j]; v_end[i] = end[j]; v_flags[i] = flags[j];
    }
}
// mean coverage per bin of `binsize` bases over the whole contig (snf.py:248-267): sum over the bin's positions of the per-base
// depth / binsize, from the per-record (start, end) arrays: one thread per record adds its overlap with every bin it touches
__global__ void k_cov_bins(const int32_t* __restrict__ rec_pos, const int32_t* __restrict__ rec_end, const uint8_t* __restrict__ rec_flags, uint32_t lo, uint32_t hi,
                           int binsize, long long contig_len, long long nbins, unsigned long long* __restrict__ acc) {
    for (unsigned long long i = lo + blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < hi; i += (unsigned long long)gridDim.x * blockDim.x) {
        if (!(rec_flags[i] & extract::RF_PASS)) continue;
        long long a = rec_pos[i], e = rec_end[i]; if (a < 0) a = 0; if (e > contig_len) e = contig_len;      // numpy slice clipping (leadprov.py:510)
        if (e <= a) continue;
        for (long long bb = a / binsize; bb <= (e - 1) / binsize && bb < nbins; ++bb) {
            const long long s0 = bb * binsize, s1 = s0 + binsize;
            const long long o0 = a > s0 ? a : s0, o1 = e < s1 ? e : s1;
            if (o1 > o0) atomicAdd(&acc[bb], (unsigned long long)(o1 - o0));
        }
    }
}


// ------------------------------------------------------------------------------------------------ all-gather of the candidate buffers
// slot of one rank: [GatherHdr][cand][alt][rnames][rn_off][cand_leads], every section 16-byte aligned
struct GatherHdr { unsigned long long n_cand, n_alt, n_rn, n_leads, need_bytes, overflow, pad0, pad1; };
__host__ __device__ inline void gather_offsets(const GatherHdr& h, unsigned long long off[6]) {
    auto al = [](unsigned long long x) { return (x + 15ull) & ~15ull; };
    off[0] = sizeof(GatherHdr); off[1] = al(off[0] + h.n_cand * sizeof(snfb_cand)); off[2] = al(off[1] + h.n_alt); off[3] = al(off[2] + 8 * h.n_rn);
    off[4] = al(off[3] + 4 * h.n_cand); off[5] = al(off[4] + h.n_leads * sizeof(snfb_lead));
}
__device__ inline void copy16(uint8_t* dst, const uint8_t* src, unsigned long long nbytes) {      // both 16-byte aligned, whole grid cooperates
    const unsigned long long n16 = (nbytes + 15) >> 4;
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n16; i += (unsigned long long)gridDim.x * blockDim.x)
        reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
}
__global__ void k_gather_pack(const DevCounters* ctr, const snfb_cand* cand, const uint8_t* alt, const uint64_t* rnames, const uint32_t* rn_off, const snfb_lead* leads, int with_leads,
                              uint8_t* slot, unsigned long long cap) {
    GatherHdr h; h.n_cand = ctr->n_cand; h.n_alt = ctr->n_alt_bytes; h.n_rn = ctr->n_rnames; h.n_leads = with_leads ? ctr->n_cand_leads : 0ull; h.pad0 = h.pad1 = 0;
    unsigned long long off[6]; gather_offsets(h, off);
    h.need_bytes = off[5]; h.overflow = off[5] > cap ? 1ull : 0ull;
    if (blockIdx.x == 0 && threadIdx.x == 0) *reinterpret_cast<GatherHdr*>(slot) = h;
    if (h.overflow) return;
    copy16(slot + off[0], reinterpret_cast<const uint8_t*>(cand), h.n_cand * sizeof(snfb_cand));
    copy16(slot + off[1], alt, h.n_alt);
    copy16(slot + off[2], reinterpret_cast<const uint8_t*>(rnames), 8 * h.n_rn);
    copy16(slot + off[3], reinterpret_cast<const uint8_t*>(rn_off), 4 * h.n_cand);
    if (with_leads) copy16(slot + off[4], reinterpret_cast<const uint8_t*>(leads), h.n_leads * sizeof(snfb_lead));
}
// gathered slots -> merged arrays with the offsets of every rank rebased; merged layout: [nranks headers][cand][alt][rnames][rn_off (+1)][leads]
__global__ void k_gather_merge(const uint8_t* recv, unsigned long long cap, int nranks, int with_leads, uint8_t* out, unsigned long long out_cap, unsigned long long* out_layout /* [8] */) {
    GatherHdr tot{}; bool ovf = false;
    for (int r = 0; r < nranks; ++r) { const GatherHdr* h = reinterpret_cast<const GatherHdr*>(recv + (size_t)r * cap); tot.n_cand += h->n_cand; tot.n_alt += h->n_alt; tot.n_rn += h->n_rn; tot.n_leads += h->n_leads; ovf = ovf || h->overflow; }
    auto al = [](unsigned long long x) { return (x + 255ull) & ~255ull; };
    const unsigned long long o_hdr = 0, o_cand = al((unsigned long long)nranks * sizeof(GatherHdr)), o_alt = al(o_cand + tot.n_cand * sizeof(snfb_cand)), o_rn = al(o_alt + tot.n_alt), o_ro = al(o_rn + 8 * tot.n_rn),
                             o_leads = al(o_ro + 4 * (tot.n_cand + 1)), o_end = al(o_leads + tot.n_leads * sizeof(snfb_lead));
    const bool fits = !ovf && o_end <= out_cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) { out_layout[0] = o_cand; out_layout[1] = o_alt; out_layout[2] = o_rn; out_layout[3] = o_ro; out_layout[4] = o_leads; out_layout[5] = o_end; out_layout[6] = fits ? 0 : 1; out_layout[7] = tot.n_cand; }
    if (!fits) return;
    const unsigned long long tid = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x, nthr = (unsigned long long)gridDim.x * blockDim.x;
    unsigned long long b_cand = 0, b_alt = 0, b_rn = 0, b_leads = 0;
    for (int r = 0; r < nranks; ++r) {
        const uint8_t* slot = recv + (size_t)r * cap; const GatherHdr h = *reinterpret_cast<const GatherHdr*>(slot);
        unsigned long long off[6]; gather_offsets(h, off);
        if (tid == 0) reinterpret_cast<GatherHdr*>(out + o_hdr)[r] = h;
        const snfb_cand* sc = reinterpret_cast<const snfb_cand*>(slot + off[0]); snfb_cand* dc = reinterpret_cast<snfb_cand*>(out + o_cand) + b_cand;
        for (unsigned long long i = tid; i < h.n_cand; i += nthr) { snfb_cand c = sc[i]; if (c.alt_off >= 0) c.alt_off += (int)b_alt; if (with_leads) { c.lead_off += (int)b_leads; c.long_off += (int)b_leads; } dc[i] = c; }
        for (unsigned long long i = tid; i < h.n_alt; i += nthr) (out + o_alt + b_alt)[i] = (slot + off[1])[i];
        const uint64_t* sr = reinterpret_cast<const uint64_t*>(slot + off[2]); uint64_t* dr = reinterpret_cast<uint64_t*>(out + o_rn) + b_rn;
        for (unsigned long long i = tid; i < h.n_rn; i += nthr) dr[i] = sr[i];
        const uint32_t* so = reinterpret_cast<const uint32_t*>(slot + off[3]); uint32_t* dof = reinterpret_cast<uint32_t*>(out + o_ro) + b_cand;
        for (unsigned long long i = tid; i < h.n_cand; i += nthr) dof[i] = so[i] + (uint32_t)b_rn;
        if (with_leads) { const uint4* sl = reinterpret_cast<const uint4*>(slot + off[4]); uint4* dl = reinterpret_cast<uint4*>(out + o_leads) + 4 * b_leads; for (unsigned long long i = tid; i < 4 * h.n_leads; i += nthr) dl[i] = sl[i]; }
        b_cand += h.n_cand; b_alt += h.n_alt; b_rn += h.n_rn; b_leads += h.n_leads;
    }
    if (tid == 0) reinterpret_cast<uint32_t*>(out + o_ro)[tot.n_cand] = (uint32_t)tot.n_rn;
}

// the DEFLATE kernel over nb BGZF blocks: as many blocks per SM as the tables' shared memory allows (at most 8)
static void launch_inflate(snfb_ctx* ctx, const ingest::BgzfBlock* d_blk, unsigned nb, ingest::IngestCounters* d_ctr) {
    const size_t smem = ingest::INF_SMEM_BYTES;
    const unsigned per_block = ingest::INF_WARPS * (32 / ingest::INF_LANES);
    const unsigned resident = (unsigned)std::max<size_t>(1, std::min<size_t>(8, (220 * 1024) / (smem + 1024)));
    const unsigned grid = std::min<unsigned>((nb + per_block - 1) / per_block, (unsigned)NUM_SMS * resident);
    launch(ctx->launches, ingest::k_inflate, grid, ingest::INF_WARPS * 32, smem, ctx->st, ctx->b_comp.as<uint8_t>(), d_blk, nb, ctx->b_raw.as<uint8_t>(), d_ctr);
}

extern "C" {

int snfb_version(void) { return SNFB_ABI_VERSION; }
size_t snfb_sizeof(int which) {
    switch (which) { case 0: return sizeof(snfb_rec); case 1: return sizeof(snfb_task); case 2: return sizeof(snfb_contig); case 3: return sizeof(snfb_records);
                     case 4: return sizeof(snfb_config); case 5: return sizeof(snfb_lead); case 6: return sizeof(snfb_cand); case 7: return sizeof(snfb_gather_view);
                     case 8: return sizeof(snfb_gt_in); case 9: return sizeof(snfb_gt_out);
                     case 10: return sizeof(snfb_ref_contig); case 11: return sizeof(snfb_ref_input); case 12: return sizeof(snfb_ref_query); case 13: return sizeof(snfb_region);
                     case 14: return sizeof(snfb_combine_plan_in); case 15: return sizeof(snfb_combine_plan_out);
                     case 16: return sizeof(snfb_pop_table); case 17: return sizeof(snfb_pop_query); case 18: return sizeof(snfb_rnames_view);
                     case 19: return sizeof(snfb_sort_input); case 20: return sizeof(snfb_sort_view); default: return 0; }
}

uint64_t snfb_hash_name(const char* s, size_t n) {
    uint64_t h = 0xcbf29ce484222325ull; for (size_t i = 0; i < n; ++i) { h ^= (uint8_t)s[i]; h *= 0x100000001b3ull; } return h;
}

int snfb_ctx_create(int device, snfb_ctx** out) {
    if (!out) return 1;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) return 2;   // no CPU fallback
    if (cudaSetDevice(device) != cudaSuccess) return 3;
    snfb_ctx* ctx = new snfb_ctx();
    ctx->device = device;
    if (cudaStreamCreateWithFlags(&ctx->st, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->st_copy, cudaStreamNonBlocking) != cudaSuccess
        || cudaStreamCreateWithFlags(&ctx->st_side, cudaStreamNonBlocking) != cudaSuccess) { delete ctx; return 4; }
    cudaEventCreateWithFlags(&ctx->ev_b, cudaEventDisableTiming); cudaEventCreateWithFlags(&ctx->ev_mid, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming); cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming);
    for (int i = 0; i < consensus::MAX_SLICES; ++i) { cudaEventCreateWithFlags(&ctx->ev_aligned[i], cudaEventDisableTiming); cudaEventCreateWithFlags(&ctx->ev_slice[i], cudaEventDisableTiming); }
    for (int i = 0; i <= MAX_TIMINGS; ++i) cudaEventCreate(&ctx->ev[i]);
    const size_t ctr_bytes = 2 * sizeof(DevCounters) + 2 * sizeof(consensus::Work);
    if (ctx->h_ctr_buf.ensure(ctr_bytes) || ctx->b_ctr.ensure(sizeof(DevCounters) + 64)) { delete ctx; return 5; }
    ctx->h_mid = ctx->h_ctr_buf.as<DevCounters>(); ctx->h_fin = ctx->h_mid + 1; ctx->h_work = reinterpret_cast<consensus::Work*>(ctx->h_fin + 1);
    memset(ctx->h_ctr_buf.p, 0, ctr_bytes);
    cudaFuncSetAttribute(cluster::k_cluster_warp<cluster::SMALL_CAP, cluster::CWS_WARPS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cluster::CwCfg<cluster::SMALL_CAP, cluster::CWS_WARPS>::smem);
    cudaFuncSetAttribute(cluster::k_cluster_warp<cluster::WARP_CAP, cluster::CWM_WARPS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cluster::CwCfg<cluster::WARP_CAP, cluster::CWM_WARPS>::smem);
    cudaFuncSetAttribute(cluster::k_cluster_block, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cluster::CB_SMEM);
    cudaFuncSetAttribute(bgzfw::k_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bgzfw::DEF_SMEM_BYTES);
    *out = ctx; return 0;
}

void snfb_ctx_destroy(snfb_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->st); cudaStreamSynchronize(ctx->st_copy); cudaStreamSynchronize(ctx->st_side);
    if (ctx->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->comm);
    for (int i = 0; i <= MAX_TIMINGS; ++i) cudaEventDestroy(ctx->ev[i]);
    cudaEventDestroy(ctx->ev_b); cudaEventDestroy(ctx->ev_mid); cudaEventDestroy(ctx->ev_fork); cudaEventDestroy(ctx->ev_join);
    for (int i = 0; i < consensus::MAX_SLICES; ++i) { cudaEventDestroy(ctx->ev_aligned[i]); cudaEventDestroy(ctx->ev_slice[i]); }
    cudaStreamDestroy(ctx->st_side); cudaStreamDestroy(ctx->st_copy); cudaStreamDestroy(ctx->st);
    delete ctx;      // frees every buffer
}

const char* snfb_last_error(snfb_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

int snfb_set_config(snfb_ctx* ctx, const snfb_config* cfg) {
    if (!ctx || !cfg) return 1;
    ctx->force_no_cuts = false;      // a new configuration decides again where chains of bins may be cut
    if (cfg->consensus_kmer_len != 6) return fail(ctx, "consensus_kmer_len must be 6 (the reference fixes it, config.py:550)");
    if (cfg->cluster_binsize <= 0 || cfg->cluster_resplit_binsize <= 0 || cfg->coverage_binsize <= 0) return fail(ctx, "bin sizes must be positive");
    ctx->cfg = *cfg; ctx->have_cfg = true; ctx->stage_a_done = ctx->stage_b_done = ctx->stage_c_done = false; return 0;
}

// ---- BAM CIGAR words -> CIGAR16 on the host: the ingest encoder run with one lane.  The only place the 32-bit form is read. ----
// pass 1: off[i] = first word of record i in the 16-bit arena (every record starts a 16-byte group); false when an op code is unknown
static bool c16_offsets(const snfb_rec* rec_in, uint64_t n_rec, const uint32_t* cigar32, std::vector<uint64_t>& off) {
    off.assign(n_rec + 1, 0);
    const uint8_t* raw = reinterpret_cast<const uint8_t*>(cigar32);
    bool bad = false;
    #pragma omp parallel for schedule(static) reduction(|| : bad)
    for (long long i = 0; i < (long long)n_rec; ++i) {
        long long ref; int b = 0;
        const uint32_t w = ingest::c16_convert<1>(raw, 4ull * rec_in[i].cigar_off, rec_in[i].n_cigar, nullptr, 0, 0, &ref, &b);
        bad = bad || b; off[i + 1] = (w + 7) & ~7ull;
    }
    if (bad) return false;
    for (uint64_t i = 0; i < n_rec; ++i) off[i + 1] += off[i];
    return true;
}
// pass 2: the words and the rewritten records
static void c16_fill(const snfb_rec* rec_in, uint64_t n_rec, const uint32_t* cigar32, const std::vector<uint64_t>& off, snfb_rec* rec_out, uint16_t* out16, uint32_t evt_min) {
    const uint8_t* raw = reinterpret_cast<const uint8_t*>(cigar32);
    #pragma omp parallel for schedule(static)
    for (long long i = 0; i < (long long)n_rec; ++i) {
        uint16_t* dst = out16 + off[i]; const uint64_t span = off[i + 1] - off[i];
        long long ref; int bad = 0;      // c16_offsets has rejected a block with an unknown op
        const uint64_t k = ingest::c16_convert<1>(raw, 4ull * rec_in[i].cigar_off, rec_in[i].n_cigar, dst, evt_min, 0, &ref, &bad);
        if (k < span) memset(dst + k, 0, 2 * (span - k));
        snfb_rec r = rec_in[i]; r.n_cigar = (uint32_t)k; r.cigar_off = off[i];
        rec_out[i] = r;
    }
    memset(out16 + off[n_rec], 0, 16);                            // one zero group of slack after the last record
}
uint64_t snfb_pack_cigar16(const snfb_rec* rec_in, uint64_t n_rec, const uint32_t* cigar32, snfb_rec* rec_out, uint16_t* out16, uint64_t out_cap, uint32_t evt_min) {
    if (n_rec && (!rec_in || !cigar32)) return UINT64_MAX;
    if (evt_min == 0) evt_min = SNFB_CIGAR16_EVT_MIN;
    std::vector<uint64_t> off;
    if (!c16_offsets(rec_in, n_rec, cigar32, off)) return UINT64_MAX;
    const uint64_t total = off[n_rec] + 8;
    if (!out16) return total;
    if (!rec_out || out_cap < total) return UINT64_MAX;
    c16_fill(rec_in, n_rec, cigar32, off, rec_out, out16, evt_min);
    return total;
}

// host-side checks of the small tables of a block
static int check_tables(snfb_ctx* ctx, const snfb_records* R) {
    for (uint32_t t = 0; t < R->n_task; ++t) {
        const snfb_task& k = R->task[t];
        if (k.tr_n < 0 || k.tr_off < 0 || (uint64_t)k.tr_off + (uint64_t)k.tr_n > R->n_tr) return fail(ctx, "task table: tandem-repeat range outside tr[]");
        if (R->n_contig && (k.contig < 0 || (uint32_t)k.contig >= R->n_contig)) return fail(ctx, "task table: contig index out of range");
        if (k.contig_len < 0 || k.start > k.end) return fail(ctx, "task table: bad region");
        if ((long long)k.contig_len >= ((long long)1 << 26) * (long long)(ctx->have_cfg ? ctx->cfg.cluster_binsize : 100)) return fail(ctx, "contig too long for the bin field of the sort key (contig_len / cluster_binsize must stay below 2^26)");
    }
    if (ctx->n_region) {
        for (uint32_t g = 0; g < ctx->n_region; ++g) {
            const snfb_region& r = ctx->regions[g];
            const std::string who = "region " + std::to_string(g) + " (task " + std::to_string(r.task) + ")";
            if (r.task < 0 || (uint32_t)r.task >= R->n_task) return fail(ctx, "region table: " + who + ": task index out of range");
            if (g && r.task < ctx->regions[g - 1].task) return fail(ctx, "region table: " + who + ": regions must be grouped by task in task order");
            if (r.start < 0 || r.start > r.end) return fail(ctx, "region table: " + who + ": start < 0 or start > end");
        }
    }
    if (R->n_mask && R->mask && R->mask_task_off) {
        for (uint32_t t = 0; t < R->n_task; ++t) if (R->mask_task_off[t] > R->mask_task_off[t + 1] || R->mask_task_off[t + 1] > R->n_mask) return fail(ctx, "mask_task_off must be non-decreasing and end at n_mask");
        // the probes binary-search a task's runs and the contig mean subtracts each run once: they must be sorted and disjoint
        for (uint32_t t = 0; t < R->n_task; ++t)
            for (uint32_t m = R->mask_task_off[t]; m < R->mask_task_off[t + 1]; ++m) {
                const uint32_t k = m - R->mask_task_off[t];
                if (R->mask[2 * m] > R->mask[2 * m + 1]) return fail(ctx, "N mask of task " + std::to_string(t) + ": run " + std::to_string(k) + " has start > end");
                if (k && R->mask[2 * m] < R->mask[2 * m - 1]) return fail(ctx, "N mask of task " + std::to_string(t) + ": run " + std::to_string(k) + " starts before run " + std::to_string(k - 1) + " ends (runs must be sorted and disjoint)");
            }
    }
    return 0;
}
// task / contig / tandem-repeat / N-mask tables -> device
static int upload_tables(snfb_ctx* ctx, const snfb_records* R) {
    ctx->tasks.assign(R->task, R->task + R->n_task);
    if (ctx->b_task.ensure(sizeof(snfb_task) * R->n_task) || ctx->b_contig.ensure(sizeof(snfb_contig) * (R->n_contig + 1)) || ctx->b_tr.ensure(8 * ((size_t)R->n_tr + 1)) || ctx->b_trp.ensure(4 * ((size_t)R->n_tr + 1)))
        return fail(ctx, "out of device memory for the task tables");
    CUDA_TRY(cudaMemcpyAsync(ctx->b_task.p, R->task, sizeof(snfb_task) * R->n_task, cudaMemcpyHostToDevice, ctx->st));
    if (R->n_contig) CUDA_TRY(cudaMemcpyAsync(ctx->b_contig.p, R->contig, sizeof(snfb_contig) * R->n_contig, cudaMemcpyHostToDevice, ctx->st));
    if (R->n_tr) {
        // running maximum of the interval ends per task: makes the reference's forward-only scan (cluster.py:240-246) a binary search
        std::vector<int32_t> pm(R->n_tr);
        for (uint32_t t = 0; t < R->n_task; ++t) { int32_t m = INT32_MIN; for (int k = 0; k < R->task[t].tr_n; ++k) { const int idx = R->task[t].tr_off + k; if (R->tr[2 * idx + 1] > m) m = R->tr[2 * idx + 1]; pm[idx] = m; } }
        CUDA_TRY(cudaMemcpyAsync(ctx->b_tr.p, R->tr, 8 * (size_t)R->n_tr, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaMemcpyAsync(ctx->b_trp.p, pm.data(), 4 * (size_t)R->n_tr, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaStreamSynchronize(ctx->st));     // pm is a stack-owned staging vector
    }
    ctx->cov_view = false;
    if (ctx->n_region) {
        // the table, then per task the index of its last region (-1: none).  Block order is coordinate order inside a task only when it
        // has one region: a later region's fetch also returns the reads that start before it and overlap it, even when the regions are
        // sorted and disjoint
        std::vector<int32_t> last(R->n_task, -1);
        for (uint32_t g = 0; g < ctx->n_region; ++g) {
            const snfb_region& r = ctx->regions[g];
            if (last[r.task] >= 0) ctx->cov_view = true;
            last[r.task] = (int32_t)g;
        }
        if (ctx->b_region.ensure(sizeof(snfb_region) * ctx->n_region + 4 * (size_t)R->n_task)) return fail(ctx, "out of device memory (region table)");
        CUDA_TRY(cudaMemcpyAsync(ctx->b_region.p, ctx->regions.data(), sizeof(snfb_region) * ctx->n_region, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaMemcpyAsync(ctx->b_region.as<uint8_t>() + sizeof(snfb_region) * ctx->n_region, last.data(), 4 * (size_t)R->n_task, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaStreamSynchronize(ctx->st));     // last is a stack-owned staging vector
    }
    ctx->n_mask = (R->mask && R->mask_task_off) ? R->n_mask : 0;
    if (ctx->n_mask) {
        std::vector<uint32_t> mt(ctx->n_mask);
        for (uint32_t t = 0; t < R->n_task; ++t) for (uint32_t m = R->mask_task_off[t]; m < R->mask_task_off[t + 1] && m < ctx->n_mask; ++m) mt[m] = t;
        if (ctx->b_mask.ensure(8 * (size_t)ctx->n_mask) || ctx->b_mask_off.ensure(4 * ((size_t)R->n_task + 1)) || ctx->b_mask_task.ensure(4 * (size_t)ctx->n_mask)) return fail(ctx, "out of device memory (N mask)");
        CUDA_TRY(cudaMemcpyAsync(ctx->b_mask.p, R->mask, 8 * (size_t)ctx->n_mask, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaMemcpyAsync(ctx->b_mask_off.p, R->mask_task_off, 4 * ((size_t)R->n_task + 1), cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaMemcpyAsync(ctx->b_mask_task.p, mt.data(), 4 * (size_t)ctx->n_mask, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaStreamSynchronize(ctx->st));
    }
    return 0;
}

int snfb_set_regions(snfb_ctx* ctx, const snfb_region* regions, uint32_t n) {
    if (!ctx || (n && !regions)) return 1;
    ctx->next_regions.assign(regions, regions + n);
    return 0;
}
// a load takes the table snfb_set_regions left for it, or none
static void take_regions(snfb_ctx* ctx) { ctx->regions.swap(ctx->next_regions); ctx->next_regions.clear(); ctx->n_region = (uint32_t)ctx->regions.size(); }
static const snfb_region* dev_regions(snfb_ctx* ctx) { return ctx->n_region ? ctx->b_region.as<snfb_region>() : nullptr; }
static const int32_t* dev_last_region(snfb_ctx* ctx) { return ctx->n_region ? reinterpret_cast<const int32_t*>(ctx->b_region.as<uint8_t>() + sizeof(snfb_region) * ctx->n_region) : nullptr; }

int snfb_load_records(snfb_ctx* ctx, const snfb_records* R) {
    if (!ctx || !R) return 1;
    cudaSetDevice(ctx->device);
    ctx->loaded = false; ctx->stage_a_done = ctx->stage_b_done = ctx->stage_c_done = false; ctx->force_no_cuts = false;
    take_regions(ctx);
    if (R->n_task == 0 || R->n_task > 65535) return fail(ctx, "n_task must be in 1..65535");
    if (R->n_rec >= (1ull << 28)) return fail(ctx, "too many records in one block (2^28)");
    if (!R->task || (R->n_rec && (!R->rec || !R->cigar))) return fail(ctx, "null table in the record block");
    if (check_tables(ctx, R)) return 1;
    if (ctx->n_region && R->on_device != SNFB_MEM_DEVICE)           // device-resident records are checked by k_rec_index (bad_records)
        for (uint64_t i = 0; i < R->n_rec; ++i) {
            const uint32_t g = R->rec[i].region;
            if (g >= ctx->n_region || ctx->regions[g].task != R->rec[i].task)
                return fail(ctx, "record " + std::to_string(i) + " (task " + std::to_string(R->rec[i].task) + "): region " + std::to_string(g) + " is not a region of its task");
        }
    ctx->n_rec = R->n_rec; ctx->n_cigar = R->n_cigar; ctx->n_var = R->n_var; ctx->n_seq = R->n_seq;
    ctx->n_task = R->n_task; ctx->n_contig = R->n_contig; ctx->n_tr = R->n_tr; ctx->on_device = R->on_device == SNFB_MEM_DEVICE; ctx->seq_on_demand = R->on_device == SNFB_MEM_HOST_SEQ_ON_DEMAND; ctx->h_seq = ctx->seq_on_demand ? R->seq : nullptr;
    ctx->n_ev = 0;
    const snfb_rec* src_rec = R->rec; const uint16_t* src_cigar = reinterpret_cast<const uint16_t*>(R->cigar); uint64_t n_words = R->n_cigar;
    if (R->cigar_fmt == SNFB_CIGAR_BAM32) {
        if (R->on_device == SNFB_MEM_DEVICE) return fail(ctx, "device-resident records must carry CIGAR16 (convert with snfb_pack_cigar16)");
        for (uint64_t i = 0; i < R->n_rec; ++i) if (R->rec[i].cigar_off + (uint64_t)R->rec[i].n_cigar > R->n_cigar) return fail(ctx, "a record's CIGAR lies outside the cigar arena");
        // host conversion: the kernels only read CIGAR16 (two passes over the BAM words: offsets, then the words)
        std::vector<uint64_t> off;
        if (!c16_offsets(R->rec, R->n_rec, reinterpret_cast<const uint32_t*>(R->cigar), off)) return fail(ctx, "a CIGAR holds an operation the path does not know");
        const uint64_t need = off[R->n_rec] + 8;
        if (ctx->h_c16.ensure(2 * need + 16) || ctx->h_rec16.ensure(sizeof(snfb_rec) * (R->n_rec + 1))) return fail(ctx, "out of pinned memory for the CIGAR16 conversion");
        c16_fill(R->rec, R->n_rec, reinterpret_cast<const uint32_t*>(R->cigar), off, ctx->h_rec16.as<snfb_rec>(), ctx->h_c16.as<uint16_t>(), evt_need(ctx));
        src_rec = ctx->h_rec16.as<snfb_rec>(); src_cigar = ctx->h_c16.as<uint16_t>(); n_words = need;
        ctx->evt_min = evt_need(ctx);
    } else if (R->cigar_fmt != SNFB_CIGAR_16) return fail(ctx, "unknown cigar_fmt");
    else ctx->evt_min = R->cigar_evt_min ? R->cigar_evt_min : SNFB_CIGAR16_EVT_MIN;
    if (n_words & 7) return fail(ctx, "a CIGAR16 arena must be padded to a multiple of 8 words");
    ctx->n_cigar = n_words;
    mark(ctx, "h2d_records", sizeof(snfb_rec) * R->n_rec + 2 * n_words + R->n_var + (R->on_device == SNFB_MEM_HOST_SEQ_ON_DEMAND ? 0 : R->n_seq));
    if (ctx->on_device) {
        ctx->d_rec = R->rec; ctx->d_cigar = src_cigar; ctx->d_var = R->var; ctx->d_seq = R->seq;     // caller keeps them alive
    } else {
        if (ctx->b_rec.ensure(sizeof(snfb_rec) * (R->n_rec + 1)) || ctx->b_cigar.ensure(2 * (n_words + 16)) || ctx->b_var.ensure(R->n_var + 16) || (!ctx->seq_on_demand && ctx->b_seq.ensure(R->n_seq + 16)))
            return fail(ctx, "out of device memory for the record block");
        CUDA_TRY(cudaMemcpyAsync(ctx->b_rec.p, src_rec, sizeof(snfb_rec) * R->n_rec, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaMemcpyAsync(ctx->b_cigar.p, src_cigar, 2 * n_words, cudaMemcpyHostToDevice, ctx->st));
        CUDA_TRY(cudaMemcpyAsync(ctx->b_var.p, R->var, R->n_var, cudaMemcpyHostToDevice, ctx->st));
        if (!ctx->seq_on_demand) CUDA_TRY(cudaMemcpyAsync(ctx->b_seq.p, R->seq, R->n_seq, cudaMemcpyHostToDevice, ctx->st));
        ctx->d_rec = ctx->b_rec.as<snfb_rec>(); ctx->d_cigar = ctx->b_cigar.as<uint16_t>(); ctx->d_var = ctx->b_var.as<uint8_t>(); ctx->d_seq = ctx->b_seq.as<uint8_t>();
    }
    if (upload_tables(ctx, R)) return 1;
    mark(ctx, nullptr);
    ctx->n_ev_load = ctx->n_ev;
    ctx->loaded = true; return 0;
}


// ---- device BAM ingest (SURVEY §8 (f)3) ----
namespace {
// device time: events around each phase of work the host hands the stream; the host's file reading between phases is not counted
struct PhaseTimer {
    cudaEvent_t a = nullptr, b = nullptr; double ms = 0;
    PhaseTimer() { cudaEventCreate(&a); cudaEventCreate(&b); }
    ~PhaseTimer() { cudaEventDestroy(a); cudaEventDestroy(b); }
    void begin(cudaStream_t st) { cudaEventRecord(a, st); }
    void end(cudaStream_t st) { cudaEventRecord(b, st); cudaEventSynchronize(b); float x = 0; cudaEventElapsedTime(&x, a, b); ms += x; }
};
// the BGZF member at z[o, n) (SAM spec §4.1): bad = 0 and its total size, XLEN, ISIZE and CRC32, or the first rule it breaks (BGZF_*);
// cut: the rule could not be checked because z ends inside the member
enum { BGZF_GZIP = 1, BGZF_XLEN, BGZF_BSIZE, BGZF_ISIZE };
struct BgzfMember { int bad = 0; bool cut = false; uint32_t size = 0, xlen = 0, isize = 0, crc = 0; };
BgzfMember bgzf_member(const uint8_t* z, uint64_t n, uint64_t o) {
    BgzfMember m;
    auto broken = [&](int rule, bool cut) { m.bad = rule; m.cut = cut; return m; };
    if (o + 18 > n) return broken(BGZF_GZIP, true);
    if (z[o] != 0x1f || z[o + 1] != 0x8b || z[o + 2] != 8 || !(z[o + 3] & 4)) return broken(BGZF_GZIP, false);      // gzip, DEFLATE, FEXTRA
    m.xlen = z[o + 10] | (z[o + 11] << 8);
    const uint64_t xend = o + 12 + m.xlen;
    if (xend > n) return broken(BGZF_XLEN, true);
    for (uint64_t e = o + 12; e + 4 <= xend; e += 4 + (z[e + 2] | (z[e + 3] << 8)))
        if (z[e] == 66 && z[e + 1] == 67 && (z[e + 2] | (z[e + 3] << 8)) == 2 && e + 6 <= xend) m.size = (z[e + 4] | (z[e + 5] << 8)) + 1u;
    if (!m.size || m.size < 12 + m.xlen + 8) return broken(BGZF_BSIZE, false);
    if (o + m.size > n) return broken(BGZF_BSIZE, true);
    memcpy(&m.crc, z + o + m.size - 8, 4); memcpy(&m.isize, z + o + m.size - 4, 4);
    if (m.isize > 65536u) return broken(BGZF_ISIZE, false);
    return m;
}
// whole BGZF members at the start of a host buffer: their k_inflate table, each one's start in the buffer, their total size and inflated
// size; d_ctr: the counters inflate_members launched k_inflate with
struct BgzfMembers {
    std::vector<ingest::BgzfBlock> blk; std::vector<uint64_t> cstart; uint64_t n = 0, raw_len = 0; ingest::IngestCounters* d_ctr = nullptr;
    void add(const BgzfMember& m) {
        blk.push_back(ingest::BgzfBlock{ n + 12 + m.xlen, m.size - 12 - m.xlen - 8, m.isize, raw_len, m.crc, 0 });
        cstart.push_back(n); n += m.size; raw_len += m.isize;
    }
};
}  // namespace

// the members of z[0, n), which must be whole BGZF members
static int walk_bgzf(snfb_ctx* ctx, const uint8_t* z, uint64_t n, BgzfMembers& w) {
    static const char* const why[] = { "", "not a BGZF block (gzip member with an extra field expected)", "truncated BGZF header",
                                       "BGZF block without a BC field or truncated", "BGZF block claims more than 64 KiB of data" };
    while (w.n < n) {
        const BgzfMember m = bgzf_member(z, n, w.n);
        if (m.bad) return fail(ctx, why[m.bad]);
        w.add(m);
    }
    if (w.raw_len >= (1ull << 36)) return fail(ctx, "more than 64 GiB of inflated BAM in one ingest call: split the task list");
    return 0;
}

// how one inflate_members call is timed and what it reports when a buffer cannot grow.  Timing opens once the buffers have grown: tm's
// phase and `mark` (with mark_bytes) where the uploads start, launch_mark where k_inflate starts.
struct InflateCall {
    PhaseTimer* tm = nullptr; const char* mark = nullptr; uint64_t mark_bytes = 0; const char* launch_mark = nullptr;
    std::string oom = "out of device memory for the BGZF bytes / the inflated stream", oom_tables = "out of device memory (ingest tables)";
};
// Enqueues on ctx->st, with no host synchronisation: the members z[0, w.n) to b_comp, their table (out_off added to every block's output
// offset) and the zeroed counters w.d_ctr to b_ing, and k_inflate of them into b_raw[out_off, out_off + w.raw_len); both buffers get 64
// zero bytes of pad.
static int inflate_members(snfb_ctx* ctx, const uint8_t* z, BgzfMembers& w, uint64_t out_off, const InflateCall& call) {
    const uint64_t raw_end = out_off + w.raw_len; const size_t nb = w.blk.size();
    if (ctx->b_comp.ensure(w.n + 64) || ctx->b_raw.ensure(raw_end + 64)) return fail(ctx, call.oom);
    ingest::BgzfBlock* d_blk = nullptr;
    if (carve(ctx->b_ing, [&](Carver& c) { w.d_ctr = c.take<ingest::IngestCounters>(1); d_blk = c.take<ingest::BgzfBlock>(nb + 1); })) return fail(ctx, call.oom_tables);
    cudaStream_t st = ctx->st;
    if (call.tm) call.tm->begin(st);
    if (call.mark) mark(ctx, call.mark, call.mark_bytes);
    CUDA_TRY(cudaMemcpyAsync(ctx->b_comp.p, z, w.n, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(ctx->b_comp.as<uint8_t>() + w.n, 0, 64, st));
    CUDA_TRY(cudaMemsetAsync(ctx->b_raw.as<uint8_t>() + raw_end, 0, 64, st));
    CUDA_TRY(cudaMemsetAsync(w.d_ctr, 0, sizeof(ingest::IngestCounters), st));
    std::vector<ingest::BgzfBlock> moved;
    if (out_off) { moved = w.blk; for (auto& b : moved) b.out_off += out_off; }
    CUDA_TRY(cudaMemcpyAsync(d_blk, (out_off ? moved : w.blk).data(), sizeof(ingest::BgzfBlock) * nb, cudaMemcpyHostToDevice, st));
    if (call.launch_mark) mark(ctx, call.launch_mark, w.n + w.raw_len);
    if (nb) launch_inflate(ctx, d_blk, (unsigned)nb, w.d_ctr);
    return 0;
}

// the lowest failing block of a k_inflate launch and its INF_* code
struct BadBlock { uint64_t block; unsigned code; bool crc() const { return code == ingest::INF_CRC_MISMATCH; } };
static BadBlock first_bad(const ingest::IngestCounters& hc) { const unsigned long long f = ~hc.first_bad_inv; return BadBlock{ f >> 8, (unsigned)(f & 255u) }; }
// the error of a k_inflate launch over a caller's buffer: the count of failed blocks, the lowest one and its byte in the buffer
static int inflate_failed(snfb_ctx* ctx, const ingest::IngestCounters& hc, const BgzfMembers& w) {
    const BadBlock x = first_bad(hc);
    return fail(ctx, "inflate: " + std::to_string(hc.bad_blocks) + " BGZF block(s) failed to decode (first: block " + std::to_string(x.block) + ", code " + std::to_string(x.code)
                     + (x.crc() ? ", CRC32 mismatch" : "") + ", at byte " + std::to_string(w.cstart[x.block]) + " of the buffer)");
}
// the error of a k_inflate launch over members read from file offset file_off: the lowest failing block's file offset
static int inflate_failed_in_file(snfb_ctx* ctx, const ingest::IngestCounters& hc, const BgzfMembers& w, uint64_t file_off) {
    const BadBlock x = first_bad(hc);
    return fail(ctx, "BGZF block at file offset " + std::to_string(file_off + w.cstart[x.block]) + (x.crc() ? ": CRC32 mismatch" : ": failed to inflate (code " + std::to_string(x.code) + ")"));
}

int snfb_inflate_bgzf(snfb_ctx* ctx, const uint8_t* bgzf, uint64_t n_bytes, uint8_t* out, uint64_t out_cap, uint64_t* out_len) {
    if (!ctx || !bgzf || !out_len) return 1;
    cudaSetDevice(ctx->device);
    ctx->n_ev = 0;
    BgzfMembers w;
    if (walk_bgzf(ctx, bgzf, n_bytes, w) || inflate_members(ctx, bgzf, w, 0, InflateCall{ nullptr, "h2d_bgzf", n_bytes, "inflate" })) return 1;
    const uint64_t raw_len = w.raw_len;
    *out_len = raw_len;
    mark(ctx, nullptr);
    ingest::IngestCounters hc;
    CUDA_TRY(cudaMemcpyAsync(&hc, w.d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, ctx->st));
    CUDA_TRY(cudaStreamSynchronize(ctx->st));
    if (hc.bad_blocks) return inflate_failed(ctx, hc, w);
    if (out) {
        if (out_cap < raw_len) return fail(ctx, "snfb_inflate_bgzf: output buffer too small");
        CUDA_TRY(cudaMemcpy(out, ctx->b_raw.p, raw_len, cudaMemcpyDeviceToHost));
    }
    return 0;
}

}  // extern "C"

// BGZF members of device bytes: member k = d_in[moff[k], moff[k + 1]) (at most 0xff00 bytes, nb <= 65535) compressed by k_deflate into
// ctx->b_zout, packed in member order; *n_out = their total size, h_offs[k] = member k's offset in b_zout.  Enqueued on ctx->st; the
// caller synchronises before it reads h_offs / *n_out.
static int deflate_members(snfb_ctx* ctx, const uint8_t* d_in, const std::vector<unsigned long long>& moff, unsigned long long* n_out, std::vector<uint32_t>& h_offs) {
    const uint64_t nb = moff.size() - 1;
    const unsigned grid = (unsigned)std::min<uint64_t>(nb, (uint64_t)NUM_SMS);
    uint32_t *sizes = nullptr, *offs = nullptr, *tmp = nullptr; unsigned long long *total = nullptr, *d_moff = nullptr; uint16_t* scratch = nullptr;
    auto lay = [&](Carver& c) { sizes = c.take<uint32_t>(nb + 1); offs = c.take<uint32_t>(nb + 1); tmp = c.take<uint32_t>(prims::scan_tmp_elems(nb));
                                total = c.take<unsigned long long>(1); scratch = c.take<uint16_t>(2ull * deflate::BLOCK_IN * grid); d_moff = c.take<unsigned long long>(nb + 1); };
    if (ctx->b_zslot.ensure(nb * deflate::MEMBER_MAX) || ctx->b_zout.ensure(nb * deflate::MEMBER_MAX) || carve(ctx->b_zwork, lay))
        return fail(ctx, "out of device memory (BGZF compression)");
    cudaStream_t st = ctx->st;
    CUDA_TRY(cudaMemcpyAsync(d_moff, moff.data(), 8 * (nb + 1), cudaMemcpyHostToDevice, st));
    launch(ctx->launches, bgzfw::k_deflate, grid, bgzfw::DEF_THREADS, bgzfw::DEF_SMEM_BYTES, st, d_in, (const unsigned long long*)d_moff, (unsigned)nb, scratch,
           ctx->b_zslot.as<uint8_t>(), sizes);
    prims::exclusive_scan(ctx->launches, sizes, offs, tmp, nullptr, nb, total, st);
    launch(ctx->launches, bgzfw::k_pack, (unsigned)std::min<uint64_t>(nb, (uint64_t)NUM_SMS * 16), 256, 0, st, ctx->b_zslot.as<const uint8_t>(), sizes, offs, (unsigned)nb, ctx->b_zout.as<uint8_t>());
    h_offs.resize(nb);
    CUDA_TRY(cudaMemcpyAsync(n_out, total, sizeof(*n_out), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(h_offs.data(), offs, 4 * nb, cudaMemcpyDeviceToHost, st));
    return 0;
}

extern "C" {

int snfb_deflate_bgzf(snfb_ctx* ctx, const uint8_t* in, uint64_t n_in, uint8_t* out, uint64_t out_cap, uint64_t* out_len, uint64_t* coffset) {
    if (!ctx || !out_len || (n_in && (!in || !out))) return 1;
    cudaSetDevice(ctx->device);
    const uint64_t nb = (n_in + deflate::BLOCK_IN - 1) / deflate::BLOCK_IN;
    if (nb > 65535) return fail(ctx, "snfb_deflate_bgzf: more than 65535 BGZF blocks (~4 GiB) in one call: split the input");
    if (out_cap < nb * deflate::MEMBER_MAX) return fail(ctx, "snfb_deflate_bgzf: out_cap must be at least ceil(n_in / 0xff00) * 65536");
    ctx->n_ev = 0;
    *out_len = 0;
    if (nb == 0) return 0;
    if (ctx->b_zin.ensure(n_in + 64)) return fail(ctx, "out of device memory (BGZF compression)");
    std::vector<unsigned long long> moff(nb + 1);                   // fixed cuts: 0xff00 bytes per member, the rest in the last
    for (uint64_t k = 0; k < nb; ++k) moff[k] = k * deflate::BLOCK_IN;
    moff[nb] = n_in;
    cudaStream_t st = ctx->st;
    mark(ctx, "h2d_deflate", n_in);
    CUDA_TRY(cudaMemcpyAsync(ctx->b_zin.p, in, n_in, cudaMemcpyHostToDevice, st));
    mark(ctx, "deflate", n_in);
    unsigned long long n_out = 0;
    std::vector<uint32_t> h_offs;
    if (deflate_members(ctx, ctx->b_zin.as<const uint8_t>(), moff, &n_out, h_offs)) return 1;
    mark(ctx, "d2h_deflate", 0);
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaMemcpyAsync(out, ctx->b_zout.p, n_out, cudaMemcpyDeviceToHost, st));
    mark(ctx, nullptr);
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    if (coffset) for (uint64_t k = 0; k < nb; ++k) coffset[k] = h_offs[k];
    *out_len = n_out;
    return 0;
}

int snfb_load_bam(snfb_ctx* ctx, const snfb_bam_input* in) {
    if (!ctx || !in) return 1;
    cudaSetDevice(ctx->device);
    ctx->loaded = false; ctx->from_bam = false; ctx->stage_a_done = ctx->stage_b_done = ctx->stage_c_done = false; ctx->force_no_cuts = false;
    take_regions(ctx);
    if (in->n_task == 0 || in->n_task > 65535) return fail(ctx, "n_task must be in 1..65535");
    if (!in->task || (in->n_bytes && !in->bgzf) || (in->n_span && !in->span)) return fail(ctx, "null table in the BAM input");
    snfb_records T; memset(&T, 0, sizeof(T));
    T.n_task = in->n_task; T.n_contig = in->n_contig; T.n_tr = in->n_tr; T.n_mask = in->n_mask; T.task = in->task; T.contig = in->contig; T.tr = in->tr; T.mask = in->mask; T.mask_task_off = in->mask_task_off;
    if (check_tables(ctx, &T)) return 1;
    ctx->n_ev = 0;
    BgzfMembers w;
    if (walk_bgzf(ctx, in->bgzf, in->n_bytes, w)) return 1;
    const size_t nb = w.blk.size(); const uint64_t ns = in->n_span, raw_len = w.raw_len;
    mark(ctx, "h2d_bgzf", in->n_bytes);
    // spans: virtual offsets -> offsets in the inflated stream
    std::vector<ingest::Span> spans(ns);
    for (uint64_t i = 0; i < ns; ++i) {
        const snfb_bam_span& sp = in->span[i];
        if (sp.task >= in->n_task) return fail(ctx, "span: task index out of range");
        auto resolve = [&](uint64_t c, uint32_t u, uint64_t* out) -> bool {
            if (c == in->n_bytes) { *out = raw_len; return u == 0; }
            auto it = std::lower_bound(w.cstart.begin(), w.cstart.end(), c);
            if (it == w.cstart.end() || *it != c) return false;
            const ingest::BgzfBlock& b = w.blk[(size_t)(it - w.cstart.begin())];
            if (u > b.isize) return false;
            *out = b.out_off + u; return true;
        };
        uint64_t ub = 0, ue = 0;
        if (!resolve(sp.cbeg, sp.ubeg, &ub) || !resolve(sp.cend, sp.uend, &ue) || ue < ub) return fail(ctx, "span: a virtual offset does not name a BGZF block of the buffer");
        const uint32_t rg = ctx->n_region ? sp.region : 0u;
        if (ctx->n_region && (rg >= ctx->n_region || (uint32_t)ctx->regions[rg].task != sp.task))
            return fail(ctx, "span " + std::to_string(i) + " (task " + std::to_string(sp.task) + "): region " + std::to_string(rg) + " is not a region of its task");
        if (i && spans[i - 1].task > sp.task) return fail(ctx, "spans must be listed task by task");
        if (i && spans[i - 1].task == sp.task && spans[i - 1].region > rg) return fail(ctx, "spans of a task must be listed region by region");
        if (i && spans[i - 1].task == sp.task && spans[i - 1].region == rg && spans[i - 1].uend > ub) return fail(ctx, "spans of a region must be in file order and must not overlap");
        spans[i].ubeg = ub; spans[i].uend = ue; spans[i].task = sp.task; spans[i].region = rg;
    }
    if (upload_tables(ctx, &T)) return 1;
    ingest::Span* d_span = nullptr; uint32_t* span_cnt = nullptr; uint32_t* span_base = nullptr; uint32_t* scan_tmp0 = nullptr;
    if (carve(ctx->b_ing_span, [&](Carver& c) { d_span = c.take<ingest::Span>(ns + 1); span_cnt = c.take<uint32_t>(ns + 1); span_base = c.take<uint32_t>(ns + 1);
                                                scan_tmp0 = c.take<uint32_t>(prims::scan_tmp_elems(ns + 1) + 16); }))
        return fail(ctx, "out of device memory (ingest tables)");
    cudaStream_t st = ctx->st;
    if (ns) CUDA_TRY(cudaMemcpyAsync(d_span, spans.data(), sizeof(ingest::Span) * ns, cudaMemcpyHostToDevice, st));
    if (inflate_members(ctx, in->bgzf, w, 0, InflateCall{ nullptr, nullptr, 0, "inflate" })) return 1;
    ingest::IngestCounters* d_ctr = w.d_ctr; const uint8_t* raw = ctx->b_raw.as<uint8_t>();
    mark(ctx, "walk_records", 0);
    if (ns) {
        launch(ctx->launches, ingest::k_walk, (unsigned)((ns + 127) / 128), 128, 0, st, raw, raw_len, d_span, (unsigned)ns, 0, span_cnt, nullptr, nullptr, nullptr, 0, d_ctr);
        prims::exclusive_scan(ctx->launches, span_cnt, span_base, scan_tmp0, nullptr, ns, &d_ctr->n_raw, st);
    }
    if (ctx->h_ing.ensure(2 * sizeof(ingest::IngestCounters))) return fail(ctx, "out of pinned memory");
    ingest::IngestCounters* hc = ctx->h_ing.as<ingest::IngestCounters>();
    CUDA_TRY(cudaMemcpyAsync(hc, d_ctr, sizeof(*hc), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (hc->bad_blocks) return inflate_failed(ctx, *hc, w);
    if (hc->bad_chain) return fail(ctx, "BAM record chain broken in " + std::to_string(hc->bad_chain) + " span(s): a span does not start or end on a record boundary, or the data is truncated");
    const uint64_t n_raw = hc->n_raw;
    if (n_raw >= (1ull << 28)) return fail(ctx, "too many records in one block (2^28)");
    // per-raw-record work arrays
    ingest::RawRec* recs = nullptr; uint32_t *raw_region = nullptr, *keep = nullptr, *idx = nullptr, *groups = nullptr, *grp_off = nullptr, *var16 = nullptr, *var_off = nullptr, *seq16 = nullptr, *seq_off = nullptr, *scan_tmp = nullptr;
    if (carve(ctx->b_ing_work, [&](Carver& c) { recs = c.take<ingest::RawRec>(n_raw + 1); raw_region = c.take<uint32_t>(n_raw + 1); keep = c.take<uint32_t>(n_raw + 1); idx = c.take<uint32_t>(n_raw + 1); groups = c.take<uint32_t>(n_raw + 1); grp_off = c.take<uint32_t>(n_raw + 1);
                                                var16 = c.take<uint32_t>(n_raw + 1); var_off = c.take<uint32_t>(n_raw + 1); seq16 = c.take<uint32_t>(n_raw + 1); seq_off = c.take<uint32_t>(n_raw + 1); scan_tmp = c.take<uint32_t>(prims::scan_tmp_elems(n_raw + 1) + 16); }))
        return fail(ctx, "out of device memory (ingest work arrays)");
    const uint32_t evt = evt_need(ctx);
    uint64_t n_rec = 0, n_groups = 0, n_var16 = 0, n_seq16 = 0;
    if (n_raw) {
        const unsigned warp_grid = (unsigned)std::min<uint64_t>((n_raw + 7) / 8, (uint64_t)NUM_SMS * 16);
        launch(ctx->launches, ingest::k_walk, (unsigned)((ns + 127) / 128), 128, 0, st, raw, raw_len, d_span, (unsigned)ns, 1, span_cnt, span_base, recs, raw_region, n_raw, d_ctr);
        mark(ctx, "parse_records", 0);
        launch(ctx->launches, ingest::k_parse, (unsigned)((n_raw + 127) / 128), 128, 0, st, raw, recs, raw_region, (unsigned)n_raw, ctx->b_task.as<snfb_task>(), dev_regions(ctx), d_ctr);
        mark(ctx, "record_sizes", 0);
        launch(ctx->launches, ingest::k_rec_sizes, warp_grid, 256, 0, st, raw, recs, raw_region, (unsigned)n_raw, ctx->b_task.as<snfb_task>(), dev_regions(ctx), evt, keep, groups, var16, seq16, d_ctr);
        prims::exclusive_scan(ctx->launches, keep, idx, scan_tmp, nullptr, n_raw, &d_ctr->n_keep, st);
        prims::exclusive_scan(ctx->launches, groups, grp_off, scan_tmp, nullptr, n_raw, &d_ctr->n_groups, st);
        prims::exclusive_scan(ctx->launches, var16, var_off, scan_tmp, nullptr, n_raw, &d_ctr->n_var, st);
        prims::exclusive_scan(ctx->launches, seq16, seq_off, scan_tmp, nullptr, n_raw, &d_ctr->n_seq16, st);
        CUDA_TRY(cudaMemcpyAsync(hc, d_ctr, sizeof(*hc), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (hc->malformed || hc->bad_cigar) return fail(ctx, std::to_string(hc->malformed) + " malformed BAM record(s), " + std::to_string(hc->bad_cigar) + " with a CIGAR operation the path does not know");
        n_rec = hc->n_keep; n_groups = hc->n_groups; n_var16 = hc->n_var; n_seq16 = hc->n_seq16;
    }
    const uint64_t n_words = 8 * n_groups + 8;               // one zero group of slack after the last record (as snfb_pack_cigar16)
    if (ctx->b_rec.ensure(sizeof(snfb_rec) * (n_rec + 1)) || ctx->b_cigar.ensure(2 * (n_words + 16)) || ctx->b_var.ensure(16 * n_var16 + 16) || ctx->b_seq.ensure(16 * n_seq16 + 16))
        return fail(ctx, "out of device memory for the record block");
    mark(ctx, "pack_records", sizeof(snfb_rec) * n_rec + 2 * n_words + 16 * n_var16 + 16 * n_seq16);
    CUDA_TRY(cudaMemsetAsync(ctx->b_cigar.as<uint16_t>() + 8 * n_groups, 0, 2 * 24, st));
    if (n_raw) {
        const unsigned warp_grid = (unsigned)std::min<uint64_t>((n_raw + 7) / 8, (uint64_t)NUM_SMS * 16);
        launch(ctx->launches, ingest::k_pack, warp_grid, 256, 0, st, raw, recs, raw_region, (unsigned)n_raw, evt, keep, idx, grp_off, groups, var_off, seq_off, ctx->b_rec.as<snfb_rec>(), ctx->b_cigar.as<uint16_t>(), ctx->b_var.as<uint8_t>(), ctx->b_seq.as<uint8_t>());
    }
    mark(ctx, nullptr);
    ctx->n_ev_load = ctx->n_ev;
    ctx->n_rec = n_rec; ctx->n_cigar = n_words; ctx->n_var = 16 * n_var16; ctx->n_seq = 16 * n_seq16; ctx->n_task = in->n_task; ctx->n_contig = in->n_contig; ctx->n_tr = in->n_tr;
    ctx->on_device = false; ctx->seq_on_demand = false; ctx->h_seq = nullptr; ctx->evt_min = evt;
    ctx->d_rec = ctx->b_rec.as<snfb_rec>(); ctx->d_cigar = ctx->b_cigar.as<uint16_t>(); ctx->d_var = ctx->b_var.as<uint8_t>(); ctx->d_seq = ctx->b_seq.as<uint8_t>();
    ctx->ing_sizes[0] = n_rec; ctx->ing_sizes[1] = n_words; ctx->ing_sizes[2] = 16 * n_var16; ctx->ing_sizes[3] = 16 * n_seq16; ctx->ing_sizes[4] = n_raw; ctx->ing_sizes[5] = nb; ctx->ing_sizes[6] = raw_len; ctx->ing_sizes[7] = in->n_bytes;
    CUDA_TRY(cudaStreamSynchronize(st));
    ctx->loaded = true; ctx->from_bam = true; return 0;
}

int snfb_ingest_sizes(snfb_ctx* ctx, uint64_t out[8]) {
    if (!ctx || !out || !ctx->from_bam) return 1;
    for (int i = 0; i < 8; ++i) out[i] = ctx->ing_sizes[i];
    return 0;
}
int snfb_ingest_fetch(snfb_ctx* ctx, snfb_rec* rec, uint16_t* cigar16, uint8_t* var, uint8_t* seq) {
    if (!ctx || !ctx->from_bam || !ctx->loaded) return ctx ? fail(ctx, "snfb_ingest_fetch: no block built by snfb_load_bam") : 1;
    cudaSetDevice(ctx->device);
    if (rec && ctx->n_rec) CUDA_TRY(cudaMemcpy(rec, ctx->d_rec, sizeof(snfb_rec) * ctx->n_rec, cudaMemcpyDeviceToHost));
    if (cigar16 && ctx->n_cigar) CUDA_TRY(cudaMemcpy(cigar16, ctx->d_cigar, 2 * ctx->n_cigar, cudaMemcpyDeviceToHost));
    if (var && ctx->n_var) CUDA_TRY(cudaMemcpy(var, ctx->d_var, ctx->n_var, cudaMemcpyDeviceToHost));
    if (seq && ctx->n_seq) CUDA_TRY(cudaMemcpy(seq, ctx->d_seq, ctx->n_seq, cudaMemcpyDeviceToHost));
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ arenas
static void carve_r(snfb_ctx* ctx, Carver& c) {
    const size_t n = ctx->n_rec + 1, nt = ctx->n_task;
    ctx->rec_pos = c.take<int32_t>(n); ctx->rec_end = c.take<int32_t>(n); ctx->rec_flags = c.take<uint8_t>(n); ctx->rec_nm = c.take<double>(n); ctx->rec_nlead = c.take<uint32_t>(n); ctx->rec_lead_off = c.take<uint32_t>(n);
    ctx->sa_list = c.take<uint32_t>(n); ctx->scanrec = c.take<extract::RecScan>(n); ctx->clip = c.take<extract::RecClip>(n); ctx->rec_big = c.take<int32_t>(n);
    ctx->task_first = c.take<uint32_t>(nt); ctx->task_last = c.take<uint32_t>(nt); ctx->task_reads = c.take<uint32_t>(nt); ctx->task_cov = c.take<unsigned long long>(nt); ctx->task_span = c.take<int32_t>(nt); ctx->task_nm = c.take<double>(nt);
    const size_t cpt = (ctx->n_rec + extract::NM_CHUNK - 1) / extract::NM_CHUNK + 1;
    ctx->nm_part = c.take<double>(cpt * nt + 1); ctx->nm_cnt = c.take<unsigned>(cpt * nt + 1);
    ctx->sa_seg = c.take<extract::Seg>((size_t)extract::MAXSEG * extract::SA_THREADS * extract::SA_BLOCKS);
    ctx->scan_tmp_r = c.take<uint32_t>(prims::scan_tmp_elems(n) + 16);
    const size_t nv = ctx->cov_view ? n : 1;
    ctx->v_pos = c.take<int32_t>(nv); ctx->v_end = c.take<int32_t>(nv); ctx->v_flags = c.take<uint8_t>(nv);
    ctx->v_k0 = c.take<uint64_t>(nv); ctx->v_k1 = c.take<uint64_t>(nv); ctx->v_v0 = c.take<uint32_t>(nv); ctx->v_v1 = c.take<uint32_t>(nv);
    ctx->v_hist = c.take<uint32_t>(prims::radix_hist_elems(nv) + 16); ctx->v_scan = c.take<uint32_t>(prims::scan_tmp_elems(std::max<size_t>(nv, prims::radix_hist_elems(nv))) + 16);
    ctx->v_n = c.take<unsigned long long>(1);
}
static void carve_l(snfb_ctx* ctx, Carver& c) {
    const size_t n = (size_t)ctx->cap.lead + 8; cluster::B& b = ctx->B;
    ctx->leads = c.take<snfb_lead>(n); ctx->ev_buf = c.take<extract::Event>(n); ctx->sorted_leads = c.take<snfb_lead>(n);
    b.key0 = c.take<uint64_t>(n); b.val0 = c.take<uint32_t>(n); b.key1 = c.take<uint64_t>(n); b.val1 = c.take<uint32_t>(n); b.flag = c.take<uint32_t>(n); b.scan = c.take<uint32_t>(n);
    b.scan_tmp = c.take<uint32_t>(prims::scan_tmp_elems(std::max<unsigned long long>(n, prims::radix_hist_elems(n))) + 16);
    ctx->radix_hist = c.take<uint32_t>(prims::radix_hist_elems(n) + 16);
    b.bin_start = c.take<uint32_t>(n); b.bin_nl = c.take<uint32_t>(n); b.bin_nlong = c.take<uint32_t>(n); b.bin_kept = c.take<uint32_t>(n); b.bin_hap = c.take<uint32_t>(3 * n);
    b.kl_off = c.take<uint32_t>(n); b.kll_off = c.take<uint32_t>(n); b.kb_idx = c.take<uint32_t>(n); b.kl = c.take<uint32_t>(n); b.kll = c.take<uint32_t>(n); b.kleads = c.take<snfb_lead>(n); b.klleads = c.take<snfb_lead>(n);
    b.kb_bin = c.take<uint32_t>(n); b.kb_lead_off = c.take<uint32_t>(n); b.kb_lead_n = c.take<uint32_t>(n); b.kb_long_off = c.take<uint32_t>(n); b.kb_long_n = c.take<uint32_t>(n); b.kb_seed = c.take<int32_t>(n); b.kb_chain = c.take<uint32_t>(n); b.kb_repeat = c.take<uint8_t>(n);
    b.seg_start = c.take<uint32_t>(n); b.c_next = c.take<uint32_t>(n); b.c_last = c.take<uint32_t>(n); b.c_sd = c.take<double>(n); b.c_mean = c.take<double>(n); b.c_rep = c.take<uint8_t>(n);
    b.seg_sd_last = c.take<double>(n); b.seg_maxsd_first = c.take<double>(n); b.cl_first = c.take<uint32_t>(n); b.cl_last = c.take<uint32_t>(n); b.cl_rep = c.take<uint8_t>(n); b.big_list = c.take<uint32_t>(n); b.mid_list = c.take<uint32_t>(n);
    b.g_khi = c.take<uint64_t>(n); b.g_klo = c.take<uint64_t>(n); b.g_u32 = c.take<uint32_t>((size_t)cluster::coop::NU32 * n);
    b.ord = c.take<uint32_t>(n); b.st_leads = c.take<snfb_lead>(n); b.st_plo = c.take<uint32_t>(n); b.st_pn = c.take<uint32_t>(n); b.st_rn = c.take<uint64_t>(n); b.cand_tmp = c.take<snfb_cand>(n); b.sub_valid = c.take<uint8_t>(n);
    b.cl_nsub = c.take<uint32_t>(n); b.cl_nvalid = c.take<uint32_t>(n); b.cl_nlead = c.take<uint32_t>(n); b.cl_nrn = c.take<uint32_t>(n); b.cl_cand_base = c.take<uint32_t>(n); b.cl_lead_base = c.take<uint32_t>(n); b.cl_rn_base = c.take<uint32_t>(n);
    ctx->arena_off = c.take<uint32_t>(n);
}
static void carve_c(snfb_ctx* ctx, Carver& c) {
    const Caps& k = ctx->cap; cluster::B& b = ctx->B; consensus::C& cc = ctx->Cc;
    b.cand = c.take<snfb_cand>(k.cand + 1); b.cand_leads = c.take<snfb_lead>(k.cand_lead + 1); b.out_plo = c.take<uint32_t>(k.cand_lead + 1); b.out_pn = c.take<uint32_t>(k.cand_lead + 1);
    b.rnames = c.take<uint64_t>(k.rn + 1); b.rn_off_out = c.take<uint32_t>(k.cand + 2);
    cc.plan_best = c.take<uint32_t>(k.cand + 1); cc.plan_nother = c.take<uint32_t>(k.cand + 1); cc.plan_otot = c.take<uint32_t>(k.cand + 1); cc.alt_len = c.take<uint32_t>(k.cand + 1); cc.scr_len = c.take<uint32_t>(k.cand + 1);
    cc.alt_off = c.take<uint32_t>(k.cand + 1); cc.scr_off = c.take<uint32_t>(k.cand + 1); cc.work_big = c.take<uint32_t>(k.cand + 1); cc.work_small = c.take<uint32_t>(k.cand + 1); cc.work = c.take<consensus::Work>(1);
    cc.q_cnt = c.take<uint32_t>(consensus::NQ * (k.cand + 1)); cc.q_off = c.take<uint32_t>(consensus::NQ * (k.cand + 1)); ctx->q_scan_tmp = c.take<uint32_t>(consensus::NQ * prims::scan_tmp_elems(k.cand));
    cc.items_big = c.take<consensus::C::Item>(k.item + 1); cc.items_small = c.take<consensus::C::Item>(k.item + 1); cc.tiles = c.take<uint2>(k.tile + 1);
    cc.alt = c.take<uint8_t>(k.alt + 64); cc.scr = c.take<uint8_t>(k.scr16 * 16 + 64);
    ctx->seq_req = c.take<consensus::SeqReq>(k.req + 1); ctx->seq_arena = c.take<uint8_t>(k.req16 * 16 + 64);
}
// carved on every attempt: an arena is reallocated only when it must grow, so unchanged capacities give the same pointers
static int ensure_arenas(snfb_ctx* ctx) {
    if (carve(ctx->arena_r, [&](Carver& c) { carve_r(ctx, c); })) return fail(ctx, "out of device memory (per-record arrays)");
    if (carve(ctx->arena_l, [&](Carver& c) { carve_l(ctx, c); })) return fail(ctx, "out of device memory (per-lead arrays)");
    if (carve(ctx->arena_c, [&](Carver& c) { carve_c(ctx, c); })) return fail(ctx, "out of device memory (candidate / consensus arrays)");
    return 0;
}

// ------------------------------------------------------------------------------------------------ stage drivers (no host synchronisation inside)
static void bind_inputs(snfb_ctx* ctx) {
    cluster::B& b = ctx->B;
    b.leads = ctx->leads; b.rec = ctx->d_rec; b.task = ctx->b_task.as<snfb_task>(); b.contig = ctx->b_contig.as<snfb_contig>();
    b.tr = ctx->n_tr ? ctx->b_tr.as<int32_t>() : nullptr; b.tr_pmax = ctx->b_trp.as<int32_t>();
    // the coverage readers binary-search these: block order, or the coordinate-ordered copy stage A builds when block order is not
    b.rec_pos = ctx->cov_view ? ctx->v_pos : ctx->rec_pos; b.rec_end = ctx->cov_view ? ctx->v_end : ctx->rec_end; b.rec_flags = ctx->cov_view ? ctx->v_flags : ctx->rec_flags; b.rec_nm = ctx->rec_nm; b.rec_nlead = ctx->rec_nlead; b.rec_lead_off = ctx->rec_lead_off;
    b.task_first = ctx->task_first; b.task_last = ctx->task_last; b.task_maxspan = ctx->task_span;
    b.mask = ctx->n_mask ? ctx->b_mask.as<int32_t>() : nullptr; b.mask_task_off = ctx->n_mask ? ctx->b_mask_off.as<uint32_t>() : nullptr;
    b.n_task = ctx->n_task; b.n_bound = ctx->cap.lead; b.ctr = ctx->b_ctr.as<DevCounters>(); b.cfg = ctx->cfg;
    b.cut_gap = ctx->force_no_cuts ? INT_MAX : cluster::break_gap(ctx->cfg);
    b.cand_cap = ctx->cap.cand; b.cand_lead_cap = ctx->cap.cand_lead; b.rn_cap = ctx->cap.rn;
    consensus::C& c = ctx->Cc;
    c.cand = b.cand; c.cand_rw = b.cand; c.cand_leads = b.cand_leads; c.out_plo = b.out_plo; c.out_pn = b.out_pn; c.ord = b.ord; c.kleads = b.kleads; c.rec = ctx->d_rec; c.seq = ctx->d_seq; c.arena_off = nullptr;
    c.cand_cap = ctx->cap.cand; c.ctr = b.ctr; c.cfg = ctx->cfg; c.item_cap = ctx->cap.item; c.tile_cap = ctx->cap.tile; c.alt_cap = ctx->cap.alt; c.scr_cap16 = ctx->cap.scr16;
}

// stage A plus the bin sort: everything LeadProvider.build_leadtab leaves behind
static int enqueue_stage_a(snfb_ctx* ctx) {
    const uint64_t nrec = ctx->n_rec; const uint32_t nt = ctx->n_task; const snfb_config& cf = ctx->cfg; cluster::B& b = ctx->B;
    DevCounters* ctr = b.ctr; cudaStream_t st = ctx->st;
    CUDA_TRY(cudaMemsetAsync(ctr, 0, sizeof(DevCounters), st));
    CUDA_TRY(cudaMemsetAsync(ctx->task_first, 0, 4 * nt, st)); CUDA_TRY(cudaMemsetAsync(ctx->task_last, 0, 4 * nt, st));
    CUDA_TRY(cudaMemsetAsync(ctx->task_reads, 0, 4 * nt, st)); CUDA_TRY(cudaMemsetAsync(ctx->task_cov, 0, 8 * nt, st)); CUDA_TRY(cudaMemsetAsync(ctx->task_span, 0, 4 * nt, st));
    CUDA_TRY(cudaMemsetAsync(ctx->task_nm, 0, 8 * nt, st));
    extract::WalkParams S{};
    S.scan = ctx->scanrec; S.n_rec = (uint32_t)nrec; S.cigar = ctx->d_cigar; S.task = b.task;
    S.rec_end = ctx->rec_end; S.rec_nlead = ctx->rec_nlead; S.rec_big = ctx->rec_big; S.rec = ctx->d_rec; S.region = dev_regions(ctx);
    S.ev = ctx->ev_buf; S.ev_cap = ctx->cap.lead; S.n_ev = &ctr->n_ev; S.ctr = ctr; S.minsv = cf.minsvlen_screen;
    if (evt_need(ctx) < ctx->evt_min) {
        // the block's E bits were set for longer events than this configuration looks at: lower the threshold in place
        if (ctx->on_device) return fail(ctx, "the device-resident CIGAR16 arena was packed with a larger event length than the configuration needs: repack with snfb_pack_cigar16(evt_min)");
        launch(ctx->launches, extract::k_reflag, NUM_SMS * 8, 256, 0, st, const_cast<uint16_t*>(ctx->d_cigar), ctx->n_cigar, evt_need(ctx));
        ctx->evt_min = evt_need(ctx);
    }
    mark(ctx, "k_rec_index");
    if (nrec) {
        extract::IndexParams I{};
        I.rec = ctx->d_rec; I.cigar = ctx->d_cigar; I.task = b.task; I.n_rec = (uint32_t)nrec; I.n_task = nt; I.rec_pos = ctx->rec_pos; I.task_first = ctx->task_first; I.task_last = ctx->task_last;
        I.scan = ctx->scanrec; I.clip = ctx->clip; I.rec_end = ctx->rec_end; I.rec_flags = ctx->rec_flags; I.rec_nm = ctx->rec_nm; I.rec_nlead = ctx->rec_nlead; I.ctr = ctr;
        I.mapq_min = cf.mapq; I.alen_min = cf.min_alignment_length; I.excl = cf.exclude_flags; I.want_nm = (cf.qc_nm_measure || cf.phase) ? 1 : 0;
        I.n_cigar = ctx->n_cigar; I.n_var = ctx->n_var; I.n_seq = ctx->n_seq; I.check_seq = ctx->seq_on_demand ? 0 : 1;
        I.sa_list = ctx->sa_list; I.n_sa = &ctr->n_sa; I.region = dev_regions(ctx); I.last_region = dev_last_region(ctx); I.n_region = ctx->n_region;
        launch(ctx->launches, extract::k_rec_index, (unsigned)((nrec + 255) / 256), 256, 0, st, I);
        // the CIGAR walk: bytes = the CIGAR16 arena (bench.py counts the passing records' groups)
        mark(ctx, "k_scan", 2 * ctx->n_cigar);
        if (nrec >= extract::WALK_WIDE_MIN) launch(ctx->launches, extract::k_cigar_walk<32>, extract::WALK_BLOCKS, extract::WALK_THREADS, 0, st, S);
        else launch(ctx->launches, extract::k_cigar_walk<1>, extract::WALK_BLOCKS, extract::WALK_THREADS, 0, st, S);
        mark(ctx, "k_rec_post");
        extract::PostParams Q{};
        Q.scan = I.scan; Q.clip = I.clip; Q.task = b.task; Q.n_rec = (uint32_t)nrec; Q.rec_end = ctx->rec_end; Q.rec_big = ctx->rec_big; Q.rec_nm = ctx->rec_nm;
        Q.task_reads = ctx->task_reads; Q.task_cov_bp = ctx->task_cov; Q.task_maxspan = ctx->task_span;
        launch(ctx->launches, extract::k_rec_post, (unsigned)((nrec + 255) / 256), 256, 0, st, Q);
        mark(ctx, "k_emit");
        extract::EmitParams E{};
        E.rec = ctx->d_rec; E.clip = ctx->clip; E.var = ctx->d_var; E.ev = S.ev; E.n_ev = S.n_ev; E.ev_cap = ctx->cap.lead;
        E.leads = ctx->leads; E.ctr = ctr; E.maxlen = cf.dev_seq_cache_maxlen; E.detect_large_ins = cf.detect_large_ins; E.longinslen = (double)cf.long_ins_length / 2.0;
        launch(ctx->launches, extract::k_emit, NUM_SMS * 16, 128, 0, st, E);
        mark(ctx, "k_sa");
        extract::SaParams A{};
        A.rec = ctx->d_rec; A.clip = ctx->clip; A.var = ctx->d_var; A.task = b.task; A.contig = b.contig; A.n_contig = ctx->n_contig;
        A.sa_list = ctx->sa_list; A.n_sa = &ctr->n_sa; A.rec_end = ctx->rec_end; A.rec_nlead = ctx->rec_nlead; A.leads = E.leads; A.lead_cap = ctx->cap.lead; A.ctr = ctr; A.cfg = cf; A.seg_scratch = ctx->sa_seg; A.region = dev_regions(ctx);
        launch(ctx->launches, extract::k_sa, extract::SA_BLOCKS, extract::SA_THREADS, 0, st, A);
        mark(ctx, "k_task_nm");
        const int cpt = (int)((nrec + extract::NM_CHUNK - 1) / extract::NM_CHUNK);
        launch(ctx->launches, extract::k_nm_partial, dim3(cpt, nt), 256, 0, st, ctx->rec_flags, ctx->rec_nm, ctx->task_first, ctx->task_last, ctx->nm_part, ctx->nm_cnt);
        launch(ctx->launches, extract::k_task_nm, nt, 256, 0, st, ctx->task_first, ctx->task_last, ctx->nm_part, ctx->nm_cnt, cpt, ctx->task_nm);
        if (ctx->cov_view) {
            // records grouped by region are out of coordinate order inside a task: a stable sort of (task, pos) gives the order the
            // coverage readers binary-search (duplicates of a read stay adjacent, each counted)
            mark(ctx, "cov_order");
            launch(ctx->launches, k_view_keys, grid_for(nrec, 256), 256, 0, st, ctx->d_rec, ctx->rec_pos, (unsigned long long)nrec, ctx->v_k0, ctx->v_v0, ctx->v_n);
            prims::RadixTemp vt{ ctx->v_hist, ctx->v_scan };
            bool vfirst = true;
            prims::radix_sort(ctx->launches, ctx->v_k0, ctx->v_v0, ctx->v_k1, ctx->v_v1, vt, ctx->v_n, nrec, 32 + bits_for(nt), &vfirst, st);
            launch(ctx->launches, k_view_gather, grid_for(nrec, 256), 256, 0, st, vfirst ? ctx->v_v0 : ctx->v_v1, (unsigned long long)nrec, ctx->rec_pos, ctx->rec_end, ctx->rec_flags, ctx->v_pos, ctx->v_end, ctx->v_flags);
        }
    }
    mark(ctx, "scan_rec_leads");
    prims::exclusive_scan(ctx->launches, ctx->rec_nlead, ctx->rec_lead_off, ctx->scan_tmp_r, nullptr, nrec, &ctr->n_leads, st);
    const unsigned long long nb = b.n_bound; const int g = grid_for(nb, 256);
    mark(ctx, "sort_leads");
    launch(ctx->launches, cluster::k_scatter_keys, g, 256, 0, st, b);
    prims::RadixTemp rt{ ctx->radix_hist, b.scan_tmp };
    bool first = true;
    prims::radix_sort(ctx->launches, b.key0, b.val0, b.key1, b.val1, rt, &ctr->n_leads, nb, cluster::TASK_SHIFT + bits_for(ctx->n_task), &first, st);
    b.skey = first ? b.key0 : b.key1; b.sval = first ? b.val0 : b.val1;
    mark(ctx, "bins");
    launch(ctx->launches, cluster::k_bin_heads, g, 256, 0, st, b);
    prims::exclusive_scan(ctx->launches, b.flag, b.scan, b.scan_tmp, &ctr->n_leads, nb, &ctr->n_bins, st);
    launch(ctx->launches, cluster::k_bin_build, g, 256, 0, st, b);
    launch(ctx->launches, cluster::k_bin_stats, g, 256, 0, st, b);
    mark(ctx, nullptr);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

static int enqueue_stage_b(snfb_ctx* ctx) {
    cluster::B& b = ctx->B; DevCounters* ctr = b.ctr; cudaStream_t st = ctx->st;
    const unsigned long long nb = b.n_bound; const int g = grid_for(nb, 128);
    mark(ctx, "kept_bins");
    prims::exclusive_scan(ctx->launches, b.bin_nl, b.kl_off, b.scan_tmp, &ctr->n_bins, nb, &ctr->n_kl, st);
    prims::exclusive_scan(ctx->launches, b.bin_nlong, b.kll_off, b.scan_tmp, &ctr->n_bins, nb, &ctr->n_kll, st);
    prims::exclusive_scan(ctx->launches, b.bin_kept, b.kb_idx, b.scan_tmp, &ctr->n_bins, nb, &ctr->n_kbins, st);
    launch(ctx->launches, cluster::k_kbin_build, g, 128, 0, st, b);
    launch(ctx->launches, cluster::k_gather_kept, grid_for(nb, 256), 256, 0, st, b);
    mark(ctx, "merge_chains");
    launch(ctx->launches, cluster::k_seg_heads, g, 128, 0, st, b);
    prims::exclusive_scan(ctx->launches, b.flag, b.scan, b.scan_tmp, &ctr->n_kbins, nb, &ctr->n_segs, st);
    launch(ctx->launches, cluster::k_seg_build, g, 128, 0, st, b);
    launch(ctx->launches, cluster::k_merge, g, 128, 0, st, b);
    launch(ctx->launches, cluster::k_verify_cuts, g, 128, 0, st, b);
    prims::exclusive_scan(ctx->launches, b.flag, b.scan, b.scan_tmp, &ctr->n_kbins, nb, &ctr->n_clusters, st);
    launch(ctx->launches, cluster::k_cluster_build, g, 128, 0, st, b);
    mark(ctx, "cluster_call");
    // clusters too large for one warp's shared memory go to a block each, next to the warp-per-cluster kernel
    CUDA_TRY(cudaEventRecord(ctx->ev_fork, st)); CUDA_TRY(cudaStreamWaitEvent(ctx->st_side, ctx->ev_fork, 0));
    launch(ctx->launches, cluster::k_cluster_block, NUM_SMS, cluster::CB_THREADS, cluster::CB_SMEM, ctx->st_side, b);
    launch(ctx->launches, cluster::k_cluster_warp<cluster::WARP_CAP, cluster::CWM_WARPS, true>, NUM_SMS * 2, cluster::CWM_WARPS * 32, cluster::CwCfg<cluster::WARP_CAP, cluster::CWM_WARPS>::smem, ctx->st_side, b);
    CUDA_TRY(cudaEventRecord(ctx->ev_join, ctx->st_side));
    launch(ctx->launches, cluster::k_cluster_warp<cluster::SMALL_CAP, cluster::CWS_WARPS, false>, NUM_SMS * 4, cluster::CWS_WARPS * 32, cluster::CwCfg<cluster::SMALL_CAP, cluster::CWS_WARPS>::smem, st, b);
    CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_join, 0));
    mark(ctx, "emit_cands");
    prims::exclusive_scan(ctx->launches, b.cl_nvalid, b.cl_cand_base, b.scan_tmp, &ctr->n_clusters, nb, &ctr->n_cand, st);
    prims::exclusive_scan(ctx->launches, b.cl_nlead, b.cl_lead_base, b.scan_tmp, &ctr->n_clusters, nb, &ctr->n_cand_leads, st);
    prims::exclusive_scan(ctx->launches, b.cl_nrn, b.cl_rn_base, b.scan_tmp, &ctr->n_clusters, nb, &ctr->n_rnames, st);
    launch(ctx->launches, cluster::k_emit_cands, NUM_SMS * 8, 128, 0, st, b);
    mark(ctx, "coverage");
    if (ctx->n_mask) launch(ctx->launches, cluster::k_mask_bp, grid_for((unsigned long long)ctx->n_mask * 32, 128), 128, 0, st, b, ctx->b_mask_task.as<uint32_t>(), ctx->n_mask, ctx->task_cov);
    launch(ctx->launches, cluster::k_coverage, NUM_SMS * 32, 128, 0, st, b);
    // consensus plan: best read per INS candidate, sizes and offsets of the ALT bytes and of the scratch; the candidate records are final after this
    consensus::C& c = ctx->Cc;
    CUDA_TRY(cudaMemsetAsync(c.work, 0, sizeof(consensus::Work), st));
    mark(ctx, "consensus_plan");
    launch(ctx->launches, consensus::k_plan, grid_for(ctx->cap.cand, 128), 128, 0, st, c);
    prims::exclusive_scan(ctx->launches, c.alt_len, c.alt_off, b.scan_tmp, &ctr->n_cand, ctx->cap.cand, &ctr->n_alt_bytes, st);
    prims::exclusive_scan(ctx->launches, c.scr_len, c.scr_off, b.scan_tmp, &ctr->n_cand, ctx->cap.cand, &ctr->n_seq_bytes, st);
    prims::exclusive_scan_cols(ctx->launches, c.q_cnt, c.q_off, ctx->cap.cand + 1, consensus::NQ, ctx->q_scan_tmp, &ctr->n_cand, ctx->cap.cand, c.work->n, st);
    launch(ctx->launches, consensus::k_plan_finish, grid_for(ctx->cap.cand, 128), 128, 0, st, c);
    launch(ctx->launches, consensus::k_plan_slices, 1, 32, 0, st, c, ctx->n_slices);
    mark(ctx, nullptr);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// the consensus kernels; with the seq arena on the host ("seq on demand") the base slices are requested, gathered and uploaded first
static int enqueue_stage_c(snfb_ctx* ctx) {
    cluster::B& b = ctx->B; consensus::C& c = ctx->Cc; DevCounters* ctr = b.ctr; cudaStream_t st = ctx->st;
    c.seq = ctx->d_seq; c.arena_off = nullptr; ctx->seq_h2d_bytes = 0;
    if (ctx->seq_on_demand) {
        // the device lists the base slices it will read, the host gathers exactly those bytes from its arena into pinned staging,
        // one H2D copy brings them in (PCIe bytes ~ algorithmic bytes instead of the whole arena).  This path needs the host in the loop.
        mark(ctx, "seq_requests");
        launch(ctx->launches, consensus::k_seq_requests, grid_for(ctx->cap.cand, 128), 128, 0, st, c, ctx->seq_req, ctx->cap.req, ctx->arena_off, &ctr->n_req, &ctr->n_req_units);
        mark(ctx, nullptr);
        CUDA_TRY(cudaMemcpyAsync(ctx->h_fin, ctr, sizeof(DevCounters), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        const unsigned long long nreq = ctx->h_fin->n_req, nunits = ctx->h_fin->n_req_units;
        // slices that do not fit the arena are not gathered and their offsets point past it: the kernels would read outside the arena.
        // caps_fit sees the counts at the end of the run and redoes it with a larger arena, so stage C is left out of this attempt.
        if (nreq > ctx->cap.req || nunits > ctx->cap.req16) return 0;
        if (nreq) {
            if (ctx->h_seq_req.ensure(sizeof(consensus::SeqReq) * (nreq + 1)) || ctx->h_seq_arena.ensure(nunits * 16 + 64)) return fail(ctx, "out of pinned memory (seq arena)");
            CUDA_TRY(cudaMemcpyAsync(ctx->h_seq_req.p, ctx->seq_req, sizeof(consensus::SeqReq) * nreq, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            const consensus::SeqReq* rq = ctx->h_seq_req.as<consensus::SeqReq>(); uint8_t* dst = ctx->h_seq_arena.as<uint8_t>(); const uint8_t* src = ctx->h_seq; const uint64_t nseq = ctx->n_seq;
            #pragma omp parallel for schedule(static, 256)
            for (long long i = 0; i < (long long)nreq; ++i) {
                unsigned long long s0 = rq[i].src; unsigned long long nbytes = rq[i].nbytes; if (s0 > nseq) s0 = nseq; if (s0 + nbytes > nseq) nbytes = nseq - s0;
                memcpy(dst + (size_t)rq[i].dst16 * 16, src + s0, (size_t)nbytes);
            }
            mark(ctx, "h2d_seq_slices", nunits * 16);
            CUDA_TRY(cudaMemcpyAsync(ctx->seq_arena, ctx->h_seq_arena.p, nunits * 16, cudaMemcpyHostToDevice, st));
            mark(ctx, nullptr);
            ctx->seq_h2d_bytes = nunits * 16;
        }
        c.seq = ctx->seq_arena; c.arena_off = ctx->arena_off;
    }
    // Slice by slice, the slices alternating between the main and the side stream.  The slices share no candidate, scratch or ALT byte, so
    // a slice's k_prep and k_align only wait for the previous slice's k_align: they fill the SMs while it votes, and the slices still end
    // in order.  The event after a slice's vote lets the copy stream take its ALT bytes while the next slice runs.  The marks are on the
    // main stream: together they span the whole stage (the interval of a vote there runs until the next slice on the main stream starts,
    // or until the side stream has finished).
    CUDA_TRY(cudaEventRecord(ctx->ev_fork, st)); CUDA_TRY(cudaStreamWaitEvent(ctx->st_side, ctx->ev_fork, 0));
    for (int s = 0; s < ctx->n_slices; ++s) {
        cudaStream_t ss = (s & 1) ? ctx->st_side : st; const bool on_main = ss == st;
        if (s) CUDA_TRY(cudaStreamWaitEvent(ss, ctx->ev_aligned[s - 1], 0));
        if (on_main) mark(ctx, "consensus");
        launch(ctx->launches, consensus::k_prep, NUM_SMS * 8, 128, 0, ss, c, s);
        if (on_main) mark(ctx, "consensus_align");
        launch(ctx->launches, consensus::k_align, NUM_SMS * 7, consensus::ALIGN_WARPS * 32, 0, ss, c, s);
        CUDA_TRY(cudaEventRecord(ctx->ev_aligned[s], ss));
        if (on_main) mark(ctx, "consensus_vote");
        launch(ctx->launches, consensus::k_vote, NUM_SMS * 16, consensus::VOTE_THREADS, 0, ss, c, s);
        CUDA_TRY(cudaEventRecord(ctx->ev_slice[s], ss));
    }
    CUDA_TRY(cudaEventRecord(ctx->ev_join, ctx->st_side)); CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_join, 0));
    mark(ctx, nullptr);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// ------------------------------------------------------------------------------------------------ capacities
static void initial_caps(snfb_ctx* ctx) {
    Caps& k = ctx->cap;
    const unsigned long long nrec = ctx->n_rec;
    // slack for the slots the allocators retire as holes: k_cigar_walk's warps and (a quarter of) k_sa's threads
    const unsigned long long lead = std::max<unsigned long long>(1ull << 16, nrec) + (unsigned long long)extract::WALK_BLOCKS * (extract::WALK_THREADS / 32) * extract::WALK_SLOTS
                                    + (unsigned long long)extract::SA_BLOCKS * extract::SA_THREADS * extract::SLOT_CHUNK / 4;
    if (k.lead < lead) k.lead = lead;
    if (k.cand < k.lead / 8 + 1024) k.cand = k.lead / 8 + 1024;
    if (k.cand_lead < k.lead / 2 + 1024) k.cand_lead = k.lead / 2 + 1024;
    if (k.rn < k.lead / 2 + 1024) k.rn = k.lead / 2 + 1024;
    if (k.alt < (4ull << 20)) k.alt = 4ull << 20;
    if (k.scr16 < (2ull << 20)) k.scr16 = 2ull << 20;
    if (k.item < k.cand_lead / 2 + 1024) k.item = k.cand_lead / 2 + 1024;
    if (k.tile < k.cand + 4096) k.tile = k.cand + 4096;
    if (ctx->seq_on_demand) { if (k.req < k.cand_lead / 2 + 1024) k.req = k.cand_lead / 2 + 1024; if (k.req16 < (1ull << 20)) k.req16 = 1ull << 20; }
    else { if (k.req < 16) k.req = 16; if (k.req16 < 16) k.req16 = 16; }
}
static unsigned long long grown(unsigned long long need) { return need + need / 4 + 1024; }
// does everything the counters report fit the capacities the run used?  If not, raise them (what was needed + 25 %).
static bool caps_fit(snfb_ctx* ctx, const DevCounters& c, const consensus::Work& work, int upto) {
    Caps& k = ctx->cap; bool ok = true;
    const unsigned long long need_lead = std::max(c.n_slots, c.n_leads);
    if (need_lead > k.lead || c.lead_overflow) { k.lead = std::max(grown(need_lead), k.lead + k.lead / 2); ok = false; }
    if (upto >= 2) {
        if (c.n_cand > k.cand) { k.cand = grown(c.n_cand); ok = false; }
        if (c.n_cand_leads > k.cand_lead) { k.cand_lead = grown(c.n_cand_leads); ok = false; }
        if (c.n_rnames > k.rn) { k.rn = grown(c.n_rnames); ok = false; }
        if (c.n_alt_bytes > k.alt) { k.alt = grown(c.n_alt_bytes); ok = false; }
        if (c.n_seq_bytes > k.scr16) { k.scr16 = grown(c.n_seq_bytes); ok = false; }
        const unsigned long long items = std::max(work.n[consensus::Q_HEAVY], work.n[consensus::Q_LIGHT]);
        if (items > k.item) { k.item = grown(items); ok = false; }
        if (work.n[consensus::Q_TILE] > k.tile) { k.tile = grown(work.n[consensus::Q_TILE]); ok = false; }
    }
    if (upto >= 3) {
        if (c.n_req > k.req) { k.req = grown(c.n_req); ok = false; }
        if (c.n_req_units > k.req16) { k.req16 = grown(c.n_req_units); ok = false; }
        if (ok && c.scratch_overflow) { ok = false; k.alt = grown(k.alt); k.scr16 = grown(k.scr16); }      // should not happen: every capacity above fit
    } else if (ok && c.scratch_overflow) { ok = false; k.cand_lead = grown(k.cand_lead); k.rn = grown(k.rn); }
    return ok;
}

// ------------------------------------------------------------------------------------------------ views
static int fill_lead_view(snfb_ctx* ctx, snfb_lead_view* out) {
    const DevCounters& c = *ctx->h_fin; const unsigned long long nl = c.n_leads; const uint32_t nt = ctx->n_task;
    if (ctx->h_leads.ensure(sizeof(snfb_lead) * (nl + 1)) || ctx->h_task_reads.ensure(4 * nt) || ctx->h_task_nm.ensure(8 * nt) || ctx->h_rec_nm.ensure(8 * (ctx->n_rec + 1)))
        return fail(ctx, "out of memory for the lead view");
    if (nl) {
        launch(ctx->launches, k_gather_leads, grid_for(nl, 256), 256, 0, ctx->st, ctx->leads, ctx->B.sval, ctx->sorted_leads, &ctx->B.ctr->n_leads, ctx->cap.lead);
        CUDA_TRY(cudaMemcpyAsync(ctx->h_leads.p, ctx->sorted_leads, sizeof(snfb_lead) * nl, cudaMemcpyDeviceToHost, ctx->st));
    }
    CUDA_TRY(cudaMemcpyAsync(ctx->h_task_reads.p, ctx->task_reads, 4 * nt, cudaMemcpyDeviceToHost, ctx->st));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_task_nm.p, ctx->task_nm, 8 * nt, cudaMemcpyDeviceToHost, ctx->st));
    if (ctx->n_rec) CUDA_TRY(cudaMemcpyAsync(ctx->h_rec_nm.p, ctx->rec_nm, 8 * ctx->n_rec, cudaMemcpyDeviceToHost, ctx->st));
    CUDA_TRY(cudaStreamSynchronize(ctx->st));
    out->n_leads = nl; out->leads = ctx->h_leads.as<snfb_lead>();
    out->task_read_count = ctx->h_task_reads.as<uint32_t>(); out->task_mean_nm = ctx->h_task_nm.as<double>(); out->rec_nm = ctx->h_rec_nm.as<double>();
    uint64_t np = 0; for (uint32_t t = 0; t < nt; ++t) np += out->task_read_count[t];
    out->n_pass = np; out->soft_errors = c.soft_errors;
    return 0;
}
// device -> host copies of the candidate view on `stream`, sized by the counters `c`
static int enqueue_cand_copies(snfb_ctx* ctx, const DevCounters& c, cudaStream_t stream) {
    cluster::B& b = ctx->B; const uint32_t nt = ctx->n_task;
    if (ctx->h_cand.ensure(sizeof(snfb_cand) * (c.n_cand + 1)) || ctx->h_cand_leads.ensure(sizeof(snfb_lead) * (c.n_cand_leads + 1)) || ctx->h_rnames.ensure(8 * (c.n_rnames + 1)) || ctx->h_rn_off.ensure(4 * (c.n_cand + 2))
        || ctx->h_task_cov.ensure(8 * nt) || ctx->h_task_cov_raw.ensure(8 * nt)) return fail(ctx, "out of pinned memory for the candidate view");
    if (c.n_cand) { CUDA_TRY(cudaMemcpyAsync(ctx->h_cand.p, b.cand, sizeof(snfb_cand) * c.n_cand, cudaMemcpyDeviceToHost, stream)); CUDA_TRY(cudaMemcpyAsync(ctx->h_rn_off.p, b.rn_off_out, 4 * c.n_cand, cudaMemcpyDeviceToHost, stream)); }
    if (c.n_cand_leads) CUDA_TRY(cudaMemcpyAsync(ctx->h_cand_leads.p, b.cand_leads, sizeof(snfb_lead) * c.n_cand_leads, cudaMemcpyDeviceToHost, stream));
    if (c.n_rnames) CUDA_TRY(cudaMemcpyAsync(ctx->h_rnames.p, b.rnames, 8 * c.n_rnames, cudaMemcpyDeviceToHost, stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_task_cov_raw.p, ctx->task_cov, 8 * nt, cudaMemcpyDeviceToHost, stream));
    return 0;
}
static void finish_cand_view(snfb_ctx* ctx, const DevCounters& c, snfb_cand_view* out) {
    const uint32_t nt = ctx->n_task;
    ctx->h_rn_off.as<uint32_t>()[c.n_cand] = (uint32_t)c.n_rnames;
    // coverage_average_total: integer base-pair sum / contig length, one rounding (postprocessing.py:130)
    double* cm = ctx->h_task_cov.as<double>(); const unsigned long long* cov = ctx->h_task_cov_raw.as<unsigned long long>();
    for (uint32_t t = 0; t < nt; ++t) cm[t] = ctx->tasks[t].contig_len > 0 ? (double)cov[t] / (double)ctx->tasks[t].contig_len : 0.0;
    out->n_cand = c.n_cand; out->cand = ctx->h_cand.as<snfb_cand>(); out->n_cand_leads = c.n_cand_leads; out->cand_leads = ctx->h_cand_leads.as<snfb_lead>();
    out->rnames = ctx->h_rnames.as<uint64_t>(); out->rnames_off = ctx->h_rn_off.as<uint32_t>(); out->task_coverage_mean = cm; out->unverified_breaks = c.unverified_breaks;
}

// ------------------------------------------------------------------------------------------------ the run loop
// the message of the first counter that fails the run whatever the capacities, or nullptr
static const char* fatal_counter(const DevCounters& c) {
    if (c.bad_records) return "the record block is malformed: a record points outside its task table or arenas";
    if (c.unsorted) return "records are not coordinate sorted inside a task";
    if (c.ordinal_overflow) return "a read carries more than 65535 SV signatures (16-bit lead ordinal)";
    return nullptr;
}
// every copy and kernel of the context has ended: before buffers they use may be reallocated, and before an error return
static void drain(snfb_ctx* ctx) { cudaStreamSynchronize(ctx->st); cudaStreamSynchronize(ctx->st_side); cudaStreamSynchronize(ctx->st_copy); }
static int run_attempts(snfb_ctx* ctx, int upto, snfb_cand_view* cands, snfb_seq_view* seqs) {
    for (int attempt = 0; ; ++attempt) {
        if (attempt == 6) return fail(ctx, "buffer capacities did not converge");
        if (ensure_arenas(ctx)) return 1;
        bind_inputs(ctx);
        ctx->n_ev = ctx->n_ev_load;
        cudaStream_t st = ctx->st; DevCounters* ctr = ctx->B.ctr;
        if (enqueue_stage_a(ctx)) return 1;
        bool mid = false;
        if (upto >= 2) {
            if (enqueue_stage_b(ctx)) return 1;
            // the host reads the counters and the slice table on the copy stream while the consensus kernels run
            CUDA_TRY(cudaEventRecord(ctx->ev_b, st)); CUDA_TRY(cudaStreamWaitEvent(ctx->st_copy, ctx->ev_b, 0));
            CUDA_TRY(cudaMemcpyAsync(ctx->h_mid, ctr, sizeof(DevCounters), cudaMemcpyDeviceToHost, ctx->st_copy));
            CUDA_TRY(cudaMemcpyAsync(&ctx->h_work[0], ctx->Cc.work, sizeof(consensus::Work), cudaMemcpyDeviceToHost, ctx->st_copy));
            CUDA_TRY(cudaEventRecord(ctx->ev_mid, ctx->st_copy));
            mid = true;
        }
        if (upto >= 3 && !ctx->seq_on_demand) { if (enqueue_stage_c(ctx)) return 1; }
        if (mid) {
            CUDA_TRY(cudaEventSynchronize(ctx->ev_mid));
            if (const char* m = fatal_counter(*ctx->h_mid)) return fail(ctx, m);
            if (!caps_fit(ctx, *ctx->h_mid, ctx->h_work[0], 2)) { drain(ctx); ++ctx->reruns; continue; }
            if (ctx->h_mid->unverified_breaks && !ctx->force_no_cuts) { drain(ctx); ctx->force_no_cuts = true; ++ctx->reruns; continue; }   // a chain cut was wrong: redo with whole chains
            if (cands) { if (enqueue_cand_copies(ctx, *ctx->h_mid, ctx->st_copy)) return 1; }
            if (upto >= 3 && ctx->seq_on_demand) { if (enqueue_stage_c(ctx)) return 1; }
        }
        if (upto >= 3 && seqs) {
            // each slice's ALT bytes, behind the candidate copies, as soon as its vote has ended
            const unsigned long long na = ctx->h_mid->n_alt_bytes;
            if (ctx->h_alt.ensure(na + 16)) return fail(ctx, "out of pinned memory for the ALT arena");
            for (int s = 0; s < ctx->n_slices; ++s) {
                const consensus::Slice& sl = ctx->h_work[0].slice[s];
                if (sl.alt_hi <= sl.alt_lo) continue;
                CUDA_TRY(cudaStreamWaitEvent(ctx->st_copy, ctx->ev_slice[s], 0));
                CUDA_TRY(cudaMemcpyAsync(ctx->h_alt.as<uint8_t>() + sl.alt_lo, ctx->Cc.alt + sl.alt_lo, sl.alt_hi - sl.alt_lo, cudaMemcpyDeviceToHost, ctx->st_copy));
            }
        }
        CUDA_TRY(cudaMemcpyAsync(ctx->h_fin, ctr, sizeof(DevCounters), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(&ctx->h_work[1], ctx->Cc.work, sizeof(consensus::Work), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        CUDA_TRY(cudaStreamSynchronize(ctx->st_copy));
        CUDA_TRY(cudaGetLastError());
        if (const char* m = fatal_counter(*ctx->h_fin)) return fail(ctx, m);
        if (!caps_fit(ctx, *ctx->h_fin, ctx->h_work[upto >= 2 ? 1 : 0], upto)) { ++ctx->reruns; continue; }
        return 0;
    }
}
// upto: 1 = stage A (+ sort and bins), 2 = + stage B and the consensus plan, 3 = + consensus.
static int run_pipeline(snfb_ctx* ctx, int upto, snfb_lead_view* leads, snfb_cand_view* cands, snfb_seq_view* seqs) {
    if (!ctx->loaded) return fail(ctx, "no records loaded");
    if (!ctx->have_cfg) return fail(ctx, "snfb_set_config was not called");
    cudaSetDevice(ctx->device);
    for (uint32_t t = 0; t < ctx->n_task; ++t) if ((long long)ctx->tasks[t].contig_len / ctx->cfg.cluster_binsize >= (1ll << 26)) return fail(ctx, "contig_len / cluster_binsize must stay below 2^26 (bin field of the sort key)");
    initial_caps(ctx);
    ctx->stage_a_done = ctx->stage_b_done = ctx->stage_c_done = false;
    if (run_attempts(ctx, upto, cands, seqs)) { drain(ctx); return 1; }
    ctx->stage_a_done = true; ctx->stage_b_done = upto >= 2; ctx->stage_c_done = upto >= 3;
    if (leads) { memset(leads, 0, sizeof *leads); if (fill_lead_view(ctx, leads)) return 1; }
    if (cands) { memset(cands, 0, sizeof *cands); finish_cand_view(ctx, *ctx->h_fin, cands); }
    if (seqs) { memset(seqs, 0, sizeof *seqs); seqs->n_alt_bytes = ctx->h_fin->n_alt_bytes; seqs->alt = ctx->h_alt.as<uint8_t>(); }
    return 0;
}

extern "C" {

int snfb_extract_leads(snfb_ctx* ctx, snfb_lead_view* out) {
    if (!ctx) return 1;
    return run_pipeline(ctx, 1, out, nullptr, nullptr);
}
int snfb_cluster_call(snfb_ctx* ctx, snfb_cand_view* out) {
    if (!ctx) return 1;
    if (!ctx->stage_a_done) return fail(ctx, "snfb_extract_leads must run first");
    return run_pipeline(ctx, 2, nullptr, out, nullptr);
}
int snfb_consensus(snfb_ctx* ctx, snfb_seq_view* out) {
    if (!ctx) return 1;
    if (!ctx->stage_b_done) return fail(ctx, "snfb_cluster_call must run first");
    snfb_seq_view tmp; return run_pipeline(ctx, 3, nullptr, nullptr, out ? out : &tmp);
}
int snfb_run(snfb_ctx* ctx, snfb_lead_view* leads, snfb_cand_view* cands, snfb_seq_view* seqs) {
    if (!ctx) return 1;
    snfb_seq_view tmp; return run_pipeline(ctx, 3, leads, cands, seqs ? seqs : &tmp);
}

int snfb_last_timings(snfb_ctx* ctx, const char** names, float* ms, uint64_t* bytes, int cap) {
    if (!ctx) return 0;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->st);
    int n = 0;
    for (int i = 0; i + 1 < ctx->n_ev && n < cap; ++i) {
        if (!ctx->ev_name[i]) continue;
        float t = 0; if (cudaEventElapsedTime(&t, ctx->ev[i], ctx->ev[i + 1]) != cudaSuccess) t = -1.f;
        names[n] = ctx->ev_name[i]; ms[n] = t; if (bytes) bytes[n] = ctx->ev_bytes[i]; ++n;
    }
    if (ctx->n_ev - ctx->n_ev_load >= 2 && n < cap) {   // first stage mark .. last mark: device time of the run
        float t = 0; if (cudaEventElapsedTime(&t, ctx->ev[ctx->n_ev_load], ctx->ev[ctx->n_ev - 1]) != cudaSuccess) t = -1.f;
        names[n] = "total"; ms[n] = t; if (bytes) bytes[n] = 0; ++n;
    }
    return n;
}

int snfb_device_candidates(snfb_ctx* ctx, void** dptr, uint64_t* n_cand) {
    if (!ctx || !ctx->stage_b_done) return 1;
    if (dptr) *dptr = ctx->B.cand; if (n_cand) *n_cand = ctx->h_fin->n_cand; return 0;
}
int snfb_device_alt(snfb_ctx* ctx, void** dptr, uint64_t* n_bytes) {
    if (!ctx || !ctx->stage_c_done) return 1;
    if (dptr) *dptr = ctx->Cc.alt; if (n_bytes) *n_bytes = ctx->h_fin->n_alt_bytes; return 0;
}
uint64_t snfb_launch_count(snfb_ctx* ctx) { return ctx ? ctx->launches : 0; }
double snfb_selftest_sqrt_frac(uint64_t p_hi, uint64_t p_lo, uint64_t q, int slow) { const u128 P = ((u128)p_hi << 64) | p_lo; return slow ? sqrt_frac_rn_slow(P, q) : sqrt_frac_rn(P, q); }
uint64_t snfb_rerun_count(snfb_ctx* ctx) { return ctx ? ctx->reruns : 0; }
int snfb_set_consensus_slices(snfb_ctx* ctx, int k) {
    if (!ctx) return 1;
    if (k < 1 || k > consensus::MAX_SLICES) return fail(ctx, "snfb_set_consensus_slices: k must be 1 to 8");
    ctx->n_slices = k; return 0;
}
int snfb_pin_host(void* p, size_t bytes) { return cudaHostRegister(p, bytes, cudaHostRegisterDefault) == cudaSuccess ? 0 : 1; }
int snfb_unpin_host(void* p) { return cudaHostUnregister(p) == cudaSuccess ? 0 : 1; }

int snfb_nccl_unique_id(void* out128) {
    std::string e; if (!out128 || !nccl_load(&e)) return 1;
    Id128 id; memset(&id, 0, sizeof id);
    if (g_nccl.GetUniqueId(&id) != 0) return 2;
    memcpy(out128, &id, 128); return 0;
}
int snfb_comm_init(snfb_ctx* ctx, const void* unique_id128, int rank, int nranks) {
    if (!ctx || !unique_id128 || nranks < 1 || rank < 0 || rank >= nranks) return 1;
    std::string e; if (!nccl_load(&e)) return fail(ctx, "NCCL: " + e);
    cudaSetDevice(ctx->device);
    if (ctx->comm) { g_nccl.CommDestroy(ctx->comm); ctx->comm = nullptr; }
    Id128 id; memcpy(&id, unique_id128, 128);
    const int rc = g_nccl.CommInitRank(&ctx->comm, nranks, id, rank);
    if (rc != 0) { ctx->comm = nullptr; return fail(ctx, std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "error")); }
    ctx->rank = rank; ctx->nranks = nranks; ctx->gather_cap = 0; return 0;
}
int snfb_allgather_candidates(snfb_ctx* ctx, uint32_t flags, snfb_gather_view* out) {
    if (!ctx || !out) return 1;
    if (!ctx->stage_c_done) return fail(ctx, "snfb_run must run first");
    if (ctx->nranks > 1 && !ctx->comm) return fail(ctx, "snfb_comm_init was not called");
    cudaSetDevice(ctx->device);
    const int nr = ctx->nranks, with_leads = (flags & SNFB_GATHER_LEADS) ? 1 : 0; cudaStream_t st = ctx->st; cluster::B& b = ctx->B;
    memset(out, 0, sizeof *out);
    unsigned long long* h_layout = nullptr; GatherHdr* h_hdr = nullptr; uint64_t* rank_n = nullptr;      // k_gather_merge's [8] layout words, the header table, rank_n_cand
    if (carve(ctx->h_gather, [&](Carver& c) { h_layout = c.take<unsigned long long>(8); h_hdr = c.take<GatherHdr>(nr); rank_n = c.take<uint64_t>(nr); })) return fail(ctx, "out of pinned memory (gather)");
    for (int attempt = 0; attempt < 4; ++attempt) {
        if (ctx->gather_cap == 0) {
            // first call: the slot size every rank uses is agreed through a small all-gather of what each rank needs
            const DevCounters& c = *ctx->h_fin; GatherHdr h{}; h.n_cand = c.n_cand; h.n_alt = c.n_alt_bytes; h.n_rn = c.n_rnames; h.n_leads = with_leads ? c.n_cand_leads : 0;
            unsigned long long off[6]; gather_offsets(h, off);
            unsigned long long mx = off[5];
            if (nr > 1) {
                if (ctx->b_gsend.ensure(256) || ctx->b_grecv.ensure(8 * (size_t)nr + 256)) return fail(ctx, "out of device memory (gather)");
                CUDA_TRY(cudaMemcpyAsync(ctx->b_gsend.p, &off[5], 8, cudaMemcpyHostToDevice, st));
                if (g_nccl.AllGather(ctx->b_gsend.p, ctx->b_grecv.p, 8, 0 /* ncclChar */, ctx->comm, st) != 0) return fail(ctx, "ncclAllGather (sizes) failed");
                std::vector<unsigned long long> all(nr);
                CUDA_TRY(cudaMemcpyAsync(all.data(), ctx->b_grecv.p, 8 * (size_t)nr, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
                for (int r = 0; r < nr; ++r) mx = std::max(mx, all[r]);
            }
            ctx->gather_cap = (grown(mx) + 255ull) & ~255ull;
        }
        const unsigned long long cap = ctx->gather_cap, out_cap = (unsigned long long)nr * cap + 4096ull * 8;
        uint8_t* recv = nullptr; uint8_t* merged = nullptr; unsigned long long* d_layout = nullptr;
        if (ctx->b_gsend.ensure(cap + 256) || carve(ctx->b_grecv, [&](Carver& c) { recv = c.take<uint8_t>((size_t)nr * cap); merged = c.take<uint8_t>(out_cap); d_layout = c.take<unsigned long long>(8); }))
            return fail(ctx, "out of device memory (gather)");
        mark(ctx, "allgather");
        launch(ctx->launches, k_gather_pack, NUM_SMS * 4, 256, 0, st, b.ctr, b.cand, ctx->Cc.alt, b.rnames, b.rn_off_out, b.cand_leads, with_leads, nr > 1 ? ctx->b_gsend.as<uint8_t>() : recv, cap);
        if (nr > 1 && g_nccl.AllGather(ctx->b_gsend.p, recv, cap, 0 /* ncclChar */, ctx->comm, st) != 0) return fail(ctx, "ncclAllGather failed");
        launch(ctx->launches, k_gather_merge, NUM_SMS * 4, 256, 0, st, recv, cap, nr, with_leads, merged, out_cap, d_layout);
        mark(ctx, nullptr);
        CUDA_TRY(cudaMemcpyAsync(h_layout, d_layout, 64, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(h_hdr, recv, sizeof(GatherHdr), cudaMemcpyDeviceToHost, st));     // slot 0's header; the rest below
        for (int r = 1; r < nr; ++r) CUDA_TRY(cudaMemcpyAsync(h_hdr + r, recv + (size_t)r * cap, sizeof(GatherHdr), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        unsigned long long mx = 0; for (int r = 0; r < nr; ++r) mx = std::max(mx, h_hdr[r].need_bytes);
        if (h_layout[6]) { ctx->gather_cap = (grown(mx) + 255ull) & ~255ull; ++ctx->reruns; continue; }          // every rank sees the same table: the same new slot size everywhere
        // next call: a slot size every rank derives from the same table
        if (grown(mx) > cap) ctx->gather_cap = (grown(mx) + 255ull) & ~255ull;
        GatherHdr tot{}; for (int r = 0; r < nr; ++r) { tot.n_cand += h_hdr[r].n_cand; tot.n_alt += h_hdr[r].n_alt; tot.n_rn += h_hdr[r].n_rn; tot.n_leads += h_hdr[r].n_leads; }
        for (int r = 0; r < nr; ++r) rank_n[r] = h_hdr[r].n_cand;
        out->n_cand = tot.n_cand; out->n_alt_bytes = tot.n_alt; out->n_rnames = tot.n_rn; out->n_cand_leads = tot.n_leads; out->rank_n_cand = rank_n;
        out->dev_buffer = merged; out->dev_bytes_per_rank = cap;
        if (!(flags & SNFB_GATHER_DEVICE_ONLY)) {
            const unsigned long long total = h_layout[5];
            if (ctx->h_gather_out.ensure(total)) return fail(ctx, "out of pinned memory (gather result)");
            uint8_t* hm = ctx->h_gather_out.as<uint8_t>();
            CUDA_TRY(cudaMemcpyAsync(hm, merged, total, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
            out->cand = reinterpret_cast<const snfb_cand*>(hm + h_layout[0]); out->alt = hm + h_layout[1]; out->rnames = reinterpret_cast<const uint64_t*>(hm + h_layout[2]);
            out->rnames_off = reinterpret_cast<const uint32_t*>(hm + h_layout[3]); out->cand_leads = with_leads ? reinterpret_cast<const snfb_lead*>(hm + h_layout[4]) : nullptr;
        }
        return 0;
    }
    return fail(ctx, "gather buffer sizes did not converge");
}

// partial-order-alignment jobs (LocalAsm, local_asm.py:254-304): host buffers in, host buffers out; a block per job
int snfb_poa(snfb_ctx* ctx, const snfb_poa_job* jobs, uint32_t n_jobs, const uint8_t* seqs, uint64_t n_seq_bytes, const int32_t* offs, uint64_t n_offs, uint8_t* out, uint64_t out_bytes, int32_t* out_len) {
    if (!ctx || (n_jobs && (!jobs || !seqs || !offs || !out || !out_len))) return ctx ? fail(ctx, "snfb_poa: null argument") : 1;
    if (n_jobs == 0) return 0;
    cudaSetDevice(ctx->device);
    // scratch: the largest job decides the per-block size; as many blocks as a third of the free memory allows
    size_t smax = 0;
    for (uint32_t k = 0; k < n_jobs; ++k) {
        const snfb_poa_job& j = jobs[k];
        if ((uint64_t)j.offs_off + j.n_seq + 1 > n_offs) return fail(ctx, "snfb_poa: offsets outside offs[]");
        const int32_t* o = offs + j.offs_off; int total = 0, maxl = 0;
        for (uint32_t i = 0; i < j.n_seq; ++i) { const int l = o[i + 1] - o[i]; if (l < 0) return fail(ctx, "snfb_poa: decreasing offsets"); total += l; if (l > maxl) maxl = l; }
        if (j.seq_off + (uint64_t)(j.n_seq ? o[j.n_seq] : 0) > n_seq_bytes) return fail(ctx, "snfb_poa: sequences outside seqs[]");
        if (j.out_off + (uint64_t)j.out_cap * (j.mode == 1 ? 2 : 1) > out_bytes) return fail(ctx, "snfb_poa: output outside out[]");
        if (j.mode == 1 && j.n_seq != 2) return fail(ctx, "snfb_poa: the MSA mode takes exactly two sequences");
        const int bw = 2 * j.band + 1 < maxl ? 2 * j.band + 1 : (maxl > 0 ? maxl : 1);
        smax = std::max(smax, poa::scratch_bytes(total, maxl, bw));
    }
    size_t free_b = 0, total_b = 0; cudaMemGetInfo(&free_b, &total_b);
    size_t nblk = std::min<size_t>(n_jobs, NUM_SMS * 2);
    while (nblk > 1 && nblk * smax > free_b / 3) --nblk;
    if (smax > free_b / 2) return fail(ctx, "snfb_poa: a job needs more scratch than the device has free");
    DevBuf d_jobs, d_seqs, d_offs, d_out, d_len, d_scr, d_ctr;
    if (d_jobs.ensure(sizeof(snfb_poa_job) * n_jobs) || d_seqs.ensure(n_seq_bytes + 16) || d_offs.ensure(4 * n_offs + 16) || d_out.ensure(out_bytes + 16) || d_len.ensure(4 * (size_t)n_jobs) || d_scr.ensure(nblk * smax) || d_ctr.ensure(64))
        return fail(ctx, "snfb_poa: out of device memory");
    cudaStream_t st = ctx->st;
    CUDA_TRY(cudaMemcpyAsync(d_jobs.p, jobs, sizeof(snfb_poa_job) * n_jobs, cudaMemcpyHostToDevice, st)); CUDA_TRY(cudaMemcpyAsync(d_seqs.p, seqs, n_seq_bytes, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(d_offs.p, offs, 4 * n_offs, cudaMemcpyHostToDevice, st)); CUDA_TRY(cudaMemsetAsync(d_ctr.p, 0, 64, st)); CUDA_TRY(cudaMemsetAsync(d_out.p, 0, out_bytes, st));
    poa::Params P{}; P.jobs = d_jobs.as<poa::Job>(); P.n_jobs = n_jobs; P.seqs = d_seqs.as<uint8_t>(); P.offs = d_offs.as<int>(); P.out = d_out.as<uint8_t>(); P.out_len = d_len.as<int>();
    P.scratch = d_scr.as<uint8_t>(); P.scratch_per_block = smax; P.next_job = d_ctr.as<unsigned>();
    mark(ctx, "poa");
    launch(ctx->launches, poa::k_poa, (unsigned)nblk, poa::THREADS, 0, st, P);
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(out, d_out.p, out_bytes, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaMemcpyAsync(out_len, d_len.p, 4 * (size_t)n_jobs, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_poa: ") + cudaGetErrorString(e));
    return 0;
}

// k_combine over a plan whose inputs P already holds in device memory: carves the group state and the outputs, launches, copies the four
// outputs to the host and synchronises
static int combine_run_groups(snfb_ctx* ctx, const snfb_combine_in* in, combine::P& P, uint32_t n_chain, uint32_t n_chunk, size_t n, bool use_alt, uint32_t max_alt,
                              DevBuf& b_state, DevBuf& b_out, const snfb_combine_out* out, const char* who) {
    const size_t S = in->n_samples, W = (S + 31) / 32;
    const unsigned blocks = (unsigned)std::min<size_t>((n_chain + 3) / 4, NUM_SMS * 4);
    auto lay_state = [&](Carver& c) {
        P.g_pos = c.take<double>(n); P.g_len = c.take<double>(n); P.g_mate = c.take<double>(n); P.g_n = c.take<uint32_t>(n); P.g_mc = c.take<int32_t>(n); P.g_incl = c.take<uint32_t>(n * W); P.act = c.take<uint32_t>(n);
        P.next_chain = c.take<unsigned int>(4); P.g_first = c.take<uint32_t>(n); P.ex_stamp = c.take<uint32_t>(n); if (use_alt) P.hs = c.take<int8_t>((size_t)blocks * 4 * max_alt + 16);
    };
    auto lay_out = [&](Carver& c) { P.cand_group = c.take<uint32_t>(n); P.emit_chunk = c.take<int32_t>(n); P.emit_ord = c.take<uint32_t>(n); P.cov_non = c.take<int32_t>(n * S); };
    if (carve(b_state, lay_state) || carve(b_out, lay_out)) return fail(ctx, std::string(who) + ": out of device memory");
    P.n_chain = n_chain; P.n_chunk = n_chunk; P.n_cand = (uint32_t)n; P.n_samples = in->n_samples; P.words = (uint32_t)W;
    P.bins_per_block = in->bins_per_block; P.cov_binsize = in->cov_binsize;
    P.combine_match = in->combine_match; P.combine_match_max = in->combine_match_max; P.cluster_merge_bnd = in->cluster_merge_bnd; P.separate_intra = in->combine_separate_intra; P.overlap_abs = in->combine_overlap_abs;
    P.pctseq = use_alt ? in->combine_pctseq : 0.0; P.max_alt = max_alt;
    cudaStream_t st = ctx->st;
    CUDA_TRY(cudaMemsetAsync(P.next_chain, 0, 16, st));
    mark(ctx, "combine_groups");
    launch(ctx->launches, combine::k_combine, blocks, 128, 0, st, P);
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(out->cand_group, P.cand_group, 4 * n, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaMemcpyAsync(out->emit_chunk, P.emit_chunk, 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->emit_ord, P.emit_ord, 4 * n, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaMemcpyAsync(out->cov_non, P.cov_non, 4 * n * S, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string(who) + ": " + cudaGetErrorString(e));
    return 0;
}

// multi-sample combine: every (task, svtype) chain of the plan by one warp (combine.cuh); host buffers in, host buffers out
int snfb_combine_groups(snfb_ctx* ctx, const snfb_combine_in* in, snfb_combine_out* out) {
    if (!ctx || !in || !out) return ctx ? fail(ctx, "snfb_combine_groups: null argument") : 1;
    if (in->n_cand == 0 || in->n_chain == 0) return 0;
    if (!in->chains || !in->chunks || !in->pos || !in->svlen || !in->sample || !out->cand_group || !out->emit_chunk || !out->emit_ord || !out->cov_non)
        return fail(ctx, "snfb_combine_groups: null array");
    if (in->n_samples == 0 || in->bins_per_block <= 0 || in->cov_binsize <= 0) return fail(ctx, "snfb_combine_groups: bad sample count / coverage geometry");
    // the plan must tile [0, n_cand) and [0, n_chunk): chains in order, chunks of a chain consecutive
    { uint64_t c = 0, k = 0;
      for (uint32_t i = 0; i < in->n_chain; ++i) { const snfb_combine_chain& ch = in->chains[i];
          if (ch.cand_off != c || ch.chunk_off != k || ch.n_chunk == 0) return fail(ctx, "snfb_combine_groups: chains do not tile the candidates / chunks");
          uint64_t cc = c;
          for (uint32_t j = 0; j < ch.n_chunk; ++j) { if (k + j >= in->n_chunk) return fail(ctx, "snfb_combine_groups: chunk index out of range"); const snfb_combine_chunk& ck = in->chunks[k + j];
              if ((uint64_t)ck.cand_off != cc || ck.n_cand <= 0 || ck.cov_block < -1 || ck.cov_block >= (int64_t)in->n_cov_block) return fail(ctx, "snfb_combine_groups: bad chunk"); cc += ck.n_cand; }
          if (cc != c + ch.n_cand) return fail(ctx, "snfb_combine_groups: chunk sizes do not add up to the chain");
          if (ch.is_bnd && (!in->mate_contig || !in->mate_pos)) return fail(ctx, "snfb_combine_groups: BND chain without mate arrays");
          c += ch.n_cand; k += ch.n_chunk; }
      if (c != in->n_cand || k != in->n_chunk) return fail(ctx, "snfb_combine_groups: plan does not cover n_cand / n_chunk");
      for (uint32_t i = 0; i < in->n_cand; ++i) if (in->sample[i] >= in->n_samples) return fail(ctx, "snfb_combine_groups: sample index out of range"); }
    cudaSetDevice(ctx->device);
    const size_t n = in->n_cand, S = in->n_samples, ncov = (size_t)in->n_cov_block * S * in->bins_per_block;
    const bool use_alt = in->combine_pctseq != 0.0 && in->alt && in->alt_off && in->alt_len;
    uint32_t max_alt = 16;
    if (use_alt) for (uint32_t i = 0; i < in->n_cand; ++i) { if (in->alt_off[i] + in->alt_len[i] > in->n_alt_bytes) return fail(ctx, "snfb_combine_groups: ALT outside alt[]"); max_alt = std::max(max_alt, in->alt_len[i]); }
    max_alt = (max_alt + 15u) & ~15u;
    // inputs in one buffer, group state in one, outputs in one
    DevBuf b_in, b_state, b_out;
    combine::P P{};
    auto lay_in = [&](Carver& c) {
        P.chains = c.take<snfb_combine_chain>(in->n_chain); P.chunks = c.take<snfb_combine_chunk>(in->n_chunk); P.pos = c.take<int32_t>(n); P.svlen = c.take<int32_t>(n); P.sample = c.take<uint32_t>(n);
        P.mate_contig = c.take<int32_t>(n); P.mate_pos = c.take<int32_t>(n); P.block_start = c.take<long long>(in->n_cov_block + 1); P.cov = c.take<int32_t>(ncov + 1);
        if (use_alt) { P.alt = c.take<uint8_t>(in->n_alt_bytes + 16); P.alt_off = c.take<unsigned long long>(n); P.alt_len = c.take<uint32_t>(n); }
    };
    if (carve(b_in, lay_in)) return fail(ctx, "snfb_combine_groups: out of device memory");
    cudaStream_t st = ctx->st;
    auto up = [&](const void* dst, const void* src, size_t bytes) { if (bytes && src) CUDA_TRY(cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, st)); return 0; };
    if (up(P.chains, in->chains, sizeof(snfb_combine_chain) * in->n_chain) || up(P.chunks, in->chunks, sizeof(snfb_combine_chunk) * in->n_chunk)
        || up(P.pos, in->pos, 4 * n) || up(P.svlen, in->svlen, 4 * n) || up(P.sample, in->sample, 4 * n) || up(P.mate_contig, in->mate_contig, 4 * n) || up(P.mate_pos, in->mate_pos, 4 * n)
        || up(P.block_start, in->block_start, 8 * (size_t)in->n_cov_block) || up(P.cov, in->cov, 4 * ncov)) return 1;
    if (use_alt && (up(P.alt, in->alt, in->n_alt_bytes) || up(P.alt_off, in->alt_off, 8 * n) || up(P.alt_len, in->alt_len, 4 * n))) return 1;
    return combine_run_groups(ctx, in, P, in->n_chain, in->n_chunk, in->n_cand, use_alt, max_alt, b_state, b_out, out, "snfb_combine_groups");
}

// the chunk plan on the device (combine.cuh k_plan_*), then the grouping over the tables it left in device memory
int snfb_combine_plan(snfb_ctx* ctx, const snfb_combine_plan_in* in, snfb_combine_plan_out* out) {
    if (!ctx || !in || !out) return ctx ? fail(ctx, "snfb_combine_plan: null argument") : 1;
    const snfb_combine_in& g = in->group;
    const uint32_t nf = in->n_flat;
    out->n_cand = out->n_chain = out->n_chunk = 0;
    if (nf == 0) return 0;
    if (!in->task || !in->row || !in->svtype || !in->support || !g.pos || !g.svlen || !g.sample || !g.mate_contig || !g.mate_pos || !out->perm || !out->chains || !out->chunks
        || !out->group.cand_group || !out->group.emit_chunk || !out->group.emit_ord || !out->group.cov_non) return fail(ctx, "snfb_combine_plan: null array");
    if (g.n_samples == 0 || g.bins_per_block <= 0 || g.cov_binsize <= 0) return fail(ctx, "snfb_combine_plan: bad sample count / coverage geometry");
    if (in->n_task == 0 || in->n_task > (1u << 24) || in->bin_min_size <= 0 || in->bin_max_candidates <= 0) return fail(ctx, "snfb_combine_plan: bad task count / bin sizes");
    for (uint32_t i = 0; i < nf; ++i)
        if (in->task[i] >= in->n_task || in->row[i] >= g.n_cov_block || in->svtype[i] < 0 || in->svtype[i] > 4 || g.sample[i] >= g.n_samples)
            return fail(ctx, "snfb_combine_plan: candidate " + std::to_string(i) + " has a task, row, svtype or sample out of range");
    const size_t S = g.n_samples, ncov = (size_t)g.n_cov_block * S * g.bins_per_block;
    const bool use_alt = g.combine_pctseq != 0.0 && g.alt && g.alt_off && g.alt_len;
    uint32_t max_alt = 16;
    if (use_alt) for (uint32_t i = 0; i < nf; ++i) { if (g.alt_off[i] + g.alt_len[i] > g.n_alt_bytes) return fail(ctx, "snfb_combine_plan: ALT outside alt[]"); max_alt = std::max(max_alt, g.alt_len[i]); }
    max_alt = (max_alt + 15u) & ~15u;
    cudaSetDevice(ctx->device);
    cudaStream_t st = ctx->st;
    ctx->n_ev = 0;
    // flat columns, the sort and plan scratch, then the slot-ordered columns and the tables k_combine reads
    DevBuf b_in, b_plan, b_state, b_out;
    const uint32_t *f_task, *f_row, *f_sample; const int32_t *f_svtype, *f_support, *f_pos, *f_svlen, *f_mc, *f_mp; const unsigned long long* f_alt_off = nullptr; const uint32_t* f_alt_len = nullptr;
    uint64_t *k0, *k1; uint32_t *v0, *v1, *keep, *at, *seg_head, *seg_id, *chain_head, *chain_id, *seg_start, *seg_nchunk, *chunk_off, *chunk_of, *scan_tmp; unsigned long long* tot;
    prims::RadixTemp rt{};
    combine::P P{};
    auto lay_in = [&](Carver& c) {
        f_task = c.take<uint32_t>(nf); f_row = c.take<uint32_t>(nf); f_svtype = c.take<int32_t>(nf); f_support = c.take<int32_t>(nf); f_pos = c.take<int32_t>(nf); f_svlen = c.take<int32_t>(nf);
        f_sample = c.take<uint32_t>(nf); f_mc = c.take<int32_t>(nf); f_mp = c.take<int32_t>(nf); P.block_start = c.take<long long>(g.n_cov_block + 1); P.cov = c.take<int32_t>(ncov + 1);
        if (use_alt) { P.alt = c.take<uint8_t>(g.n_alt_bytes + 16); f_alt_off = c.take<unsigned long long>(nf); f_alt_len = c.take<uint32_t>(nf); }
    };
    auto lay_plan = [&](Carver& c) {
        k0 = c.take<uint64_t>(nf); k1 = c.take<uint64_t>(nf); v0 = c.take<uint32_t>(nf); v1 = c.take<uint32_t>(nf); keep = c.take<uint32_t>(nf); at = c.take<uint32_t>(nf);
        seg_head = c.take<uint32_t>(nf); seg_id = c.take<uint32_t>(nf); chain_head = c.take<uint32_t>(nf); chain_id = c.take<uint32_t>(nf); seg_start = c.take<uint32_t>(nf);
        seg_nchunk = c.take<uint32_t>(nf); chunk_off = c.take<uint32_t>(nf); chunk_of = c.take<uint32_t>(nf); tot = c.take<unsigned long long>(4);
        scan_tmp = c.take<uint32_t>(prims::scan_tmp_elems(std::max<unsigned long long>(nf, prims::radix_hist_elems(nf))));
        rt.hist = c.take<uint32_t>(prims::radix_hist_elems(nf)); rt.scan_tmp = scan_tmp;
        P.chains = c.take<snfb_combine_chain>(nf); P.chunks = c.take<snfb_combine_chunk>(nf);
        P.pos = c.take<int32_t>(nf); P.svlen = c.take<int32_t>(nf); P.sample = c.take<uint32_t>(nf); P.mate_contig = c.take<int32_t>(nf); P.mate_pos = c.take<int32_t>(nf);
        if (use_alt) { P.alt_off = c.take<unsigned long long>(nf); P.alt_len = c.take<uint32_t>(nf); }
    };
    if (carve(b_in, lay_in) || carve(b_plan, lay_plan)) return fail(ctx, "snfb_combine_plan: out of device memory");
    auto up = [&](const void* dst, const void* src, size_t bytes) { if (bytes && src) CUDA_TRY(cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, st)); return 0; };
    if (up(f_task, in->task, 4 * (size_t)nf) || up(f_row, in->row, 4 * (size_t)nf) || up(f_svtype, in->svtype, 4 * (size_t)nf) || up(f_support, in->support, 4 * (size_t)nf)
        || up(f_pos, g.pos, 4 * (size_t)nf) || up(f_svlen, g.svlen, 4 * (size_t)nf) || up(f_sample, g.sample, 4 * (size_t)nf) || up(f_mc, g.mate_contig, 4 * (size_t)nf) || up(f_mp, g.mate_pos, 4 * (size_t)nf)
        || up(P.block_start, g.block_start, 8 * (size_t)g.n_cov_block) || up(P.cov, g.cov, 4 * ncov)) return 1;
    if (use_alt && (up(P.alt, g.alt, g.n_alt_bytes) || up(f_alt_off, g.alt_off, 8 * (size_t)nf) || up(f_alt_len, g.alt_len, 4 * (size_t)nf))) return 1;
    // three counts come back to the host (kept candidates, segments and chains, chunks): they size the launches that follow
    uint64_t h_tot[4];
    auto counts = [&]() -> int { CUDA_TRY(cudaMemcpyAsync(h_tot, tot, 32, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st)); return 0; };
    auto sort = [&](int bits, uint64_t*& k, uint32_t*& v) {
        uint64_t* ka = k; uint32_t* va = v; uint64_t* kb = k == k0 ? k1 : k0; uint32_t* vb = v == v0 ? v1 : v0; bool in_first = true;
        prims::radix_sort(ctx->launches, ka, va, kb, vb, rt, tot, nf, bits, &in_first, st);
        if (!in_first) { k = kb; v = vb; }
    };
    mark(ctx, "combine_plan");
    CUDA_TRY(cudaMemsetAsync(tot, 0, 32, st));
    launch(ctx->launches, combine::k_plan_keep, grid_for(nf, 256), 256, 0, st, f_support, nf, in->support_threshold, keep);
    prims::exclusive_scan(ctx->launches, keep, at, scan_tmp, nullptr, nf, tot, st);
    launch(ctx->launches, combine::k_plan_compact, grid_for(nf, 256), 256, 0, st, keep, at, nf, f_pos, in->bin_min_size, k0, v0);
    if (counts()) return 1;
    const uint32_t n = (uint32_t)h_tot[0];
    if (n == 0) { mark(ctx, nullptr); return 0; }
    uint64_t* K = k0; uint32_t* V = v0;
    sort(32, K, V);                                                                   // by bin ...
    launch(ctx->launches, combine::k_plan_segkey, grid_for(n, 256), 256, 0, st, V, n, f_task, f_svtype, f_row, K);
    sort(35 + bits_for(in->n_task), K, V);                                            // ... then stably by (task, svtype, block)
    launch(ctx->launches, combine::k_plan_heads, grid_for(n, 256), 256, 0, st, K, n, seg_head, chain_head);
    prims::exclusive_scan(ctx->launches, seg_head, seg_id, scan_tmp, nullptr, n, tot + 1, st);
    prims::exclusive_scan(ctx->launches, chain_head, chain_id, scan_tmp, nullptr, n, tot + 2, st);
    launch(ctx->launches, combine::k_plan_seg_start, grid_for(n, 256), 256, 0, st, seg_head, seg_id, n, seg_start);
    if (counts()) return 1;
    const uint32_t n_seg = (uint32_t)h_tot[1], n_chain = (uint32_t)h_tot[2];
    launch(ctx->launches, combine::k_plan_cut, grid_for(n_seg, 128), 128, 0, st, seg_start, n_seg, n, V, f_pos, K, in->bin_min_size, in->bin_max_candidates, in->exhaustive,
           seg_nchunk, (const uint32_t*)nullptr, (snfb_combine_chunk*)nullptr, (uint32_t*)nullptr);
    prims::exclusive_scan(ctx->launches, seg_nchunk, chunk_off, scan_tmp, nullptr, n_seg, tot + 3, st);
    launch(ctx->launches, combine::k_plan_cut, grid_for(n_seg, 128), 128, 0, st, seg_start, n_seg, n, V, f_pos, K, in->bin_min_size, in->bin_max_candidates, in->exhaustive,
           seg_nchunk, (const uint32_t*)chunk_off, const_cast<snfb_combine_chunk*>(P.chunks), chunk_of);
    launch(ctx->launches, combine::k_plan_chains, grid_for(n, 256), 256, 0, st, chain_head, chain_id, K, chunk_of, n, const_cast<snfb_combine_chain*>(P.chains));
    if (counts()) return 1;
    const uint32_t n_chunk = (uint32_t)h_tot[3];
    launch(ctx->launches, combine::k_plan_chain_len, grid_for(n_chain, 256), 256, 0, st, const_cast<snfb_combine_chain*>(P.chains), n_chain, n, n_chunk);
    launch(ctx->launches, combine::k_plan_supkey, grid_for(n, 256), 256, 0, st, V, chunk_of, n, f_support, K);
    sort(32 + bits_for(n_chunk), K, V);                                               // support, descending, inside each chunk
    launch(ctx->launches, combine::k_plan_gather, grid_for(n, 256), 256, 0, st, V, n, f_pos, f_svlen, f_sample, f_mc, f_mp, f_alt_off, f_alt_len,
           const_cast<int32_t*>(P.pos), const_cast<int32_t*>(P.svlen), const_cast<uint32_t*>(P.sample), const_cast<int32_t*>(P.mate_contig), const_cast<int32_t*>(P.mate_pos),
           const_cast<unsigned long long*>(P.alt_off), const_cast<uint32_t*>(P.alt_len));
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(out->perm, V, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->chains, P.chains, sizeof(snfb_combine_chain) * n_chain, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(out->chunks, P.chunks, sizeof(snfb_combine_chunk) * n_chunk, cudaMemcpyDeviceToHost, st));
    if (combine_run_groups(ctx, &g, P, n_chain, n_chunk, n, use_alt, max_alt, b_state, b_out, &out->group, "snfb_combine_plan")) return 1;
    out->n_cand = n; out->n_chain = n_chain; out->n_chunk = n_chunk;
    return 0;
}

// the population table (PopulationSNF.get_all_blocks, snfp.py:139-140): keyed on the device, sorted stably, kept on the context
int snfb_population_load(snfb_ctx* ctx, const snfb_pop_table* in) {
    if (!ctx || !in) return ctx ? fail(ctx, "snfb_population_load: null argument") : 1;
    const uint32_t n = in->n;
    if (n && (!in->contig || !in->block || !in->svtype || !in->pos || !in->svlen || !in->alt_off || !in->alt_len || (in->n_alt_bytes && !in->alt)))
        return fail(ctx, "snfb_population_load: null array");
    int32_t max_contig = -1; uint32_t max_alt = 16;
    for (uint32_t i = 0; i < n; ++i) {
        if (in->contig[i] < -1 || in->contig[i] >= (1 << 24) - 1 || in->svtype[i] < 0 || in->svtype[i] > 4)
            return fail(ctx, "snfb_population_load: variant " + std::to_string(i) + " has a contig or svtype out of range");
        if (in->alt_off[i] + in->alt_len[i] > in->n_alt_bytes) return fail(ctx, "snfb_population_load: ALT outside alt[]");
        max_contig = std::max(max_contig, in->contig[i]); max_alt = std::max(max_alt, in->alt_len[i]);
    }
    cudaSetDevice(ctx->device);
    cudaStream_t st = ctx->st;
    ctx->have_pop = false; ctx->n_ev = 0;
    population::P& P = ctx->pop;
    P = population::P{};
    int32_t *f_contig, *f_block, *f_svtype, *f_pos, *f_svlen; unsigned long long* f_alt_off; uint32_t* f_alt_len; unsigned long long* d_n;
    uint64_t *k0, *k1; uint32_t *v0, *v1; prims::RadixTemp rt{};
    auto lay = [&](Carver& c) {
        f_contig = c.take<int32_t>(n + 1); f_block = c.take<int32_t>(n + 1); f_svtype = c.take<int32_t>(n + 1); f_pos = c.take<int32_t>(n + 1); f_svlen = c.take<int32_t>(n + 1);
        f_alt_off = c.take<unsigned long long>(n + 1); f_alt_len = c.take<uint32_t>(n + 1); d_n = c.take<unsigned long long>(2);
        k0 = c.take<uint64_t>(n + 1); k1 = c.take<uint64_t>(n + 1); v0 = c.take<uint32_t>(n + 1); v1 = c.take<uint32_t>(n + 1);
        rt.hist = c.take<uint32_t>(prims::radix_hist_elems(n)); rt.scan_tmp = c.take<uint32_t>(prims::scan_tmp_elems(prims::radix_hist_elems(n)) + 16);
        P.pos = c.take<int32_t>(n + 1); P.svlen = c.take<int32_t>(n + 1); P.alt_off = c.take<unsigned long long>(n + 1); P.alt_len = c.take<uint32_t>(n + 1);
        P.alt = c.take<uint8_t>(in->n_alt_bytes + 16);
    };
    if (carve(ctx->b_pop, lay)) return fail(ctx, "snfb_population_load: out of device memory");
    auto up = [&](const void* dst, const void* src, size_t bytes) { if (bytes && src) CUDA_TRY(cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, st)); return 0; };
    const unsigned long long nn = n;
    if (up(f_contig, in->contig, 4 * (size_t)n) || up(f_block, in->block, 4 * (size_t)n) || up(f_svtype, in->svtype, 4 * (size_t)n) || up(f_pos, in->pos, 4 * (size_t)n)
        || up(f_svlen, in->svlen, 4 * (size_t)n) || up(f_alt_off, in->alt_off, 8 * (size_t)n) || up(f_alt_len, in->alt_len, 4 * (size_t)n)
        || up(P.alt, in->alt, in->n_alt_bytes) || up(d_n, &nn, 8)) return 1;
    const uint32_t absent = (uint32_t)(max_contig + 1);
    mark(ctx, "population_load", 32ull * n + in->n_alt_bytes);
    bool first = true;
    if (n) {
        launch(ctx->launches, population::k_pop_keys, grid_for(n, 256), 256, 0, st, f_contig, f_block, f_svtype, n, absent, k0, v0);
        prims::radix_sort(ctx->launches, k0, v0, k1, v1, rt, d_n, n, 35 + bits_for(absent + 1), &first, st);
        launch(ctx->launches, population::k_pop_gather, grid_for(n, 256), 256, 0, st, first ? v0 : v1, n, f_pos, f_svlen, f_alt_off, f_alt_len,
               const_cast<int32_t*>(P.pos), const_cast<int32_t*>(P.svlen), const_cast<unsigned long long*>(P.alt_off), const_cast<uint32_t*>(P.alt_len));
    }
    mark(ctx, nullptr);
    P.key = first ? k0 : k1; P.idx = first ? v0 : v1; P.n_var = n; P.n_contig = absent; P.max_alt = max_alt;
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_population_load: ") + cudaGetErrorString(e));
    ctx->have_pop = true;
    return 0;
}

// PopulationSNF.get_population_AF (snfp.py:131-155) for one batch of calls: one warp per call (population.cuh)
int snfb_population_match(snfb_ctx* ctx, const snfb_pop_query* in, int32_t* best) {
    if (!ctx || !in || !best) return ctx ? fail(ctx, "snfb_population_match: null argument") : 1;
    if (!ctx->have_pop) return fail(ctx, "snfb_population_match: no population table (snfb_population_load)");
    const uint32_t n = in->n;
    if (n == 0) return 0;
    if (!in->contig || !in->svtype || !in->pos || !in->svlen || !in->alt_off || !in->alt_len || (in->n_alt_bytes && !in->alt)) return fail(ctx, "snfb_population_match: null array");
    if (in->block_size <= 0) return fail(ctx, "snfb_population_match: bad block size");
    uint32_t max_alt = ctx->pop.max_alt;
    for (uint32_t i = 0; i < n; ++i) {
        if (in->svtype[i] < 0 || in->svtype[i] > 4 || in->contig[i] < -1 || in->contig[i] >= (1 << 24) - 1)
            return fail(ctx, "snfb_population_match: query " + std::to_string(i) + " has a contig or svtype out of range");
        if (in->alt_off[i] + in->alt_len[i] > in->n_alt_bytes) return fail(ctx, "snfb_population_match: ALT outside alt[]");
        max_alt = std::max(max_alt, in->alt_len[i]);
    }
    max_alt = (max_alt + 15u) & ~15u;
    cudaSetDevice(ctx->device);
    cudaStream_t st = ctx->st;
    ctx->n_ev = 0;
    population::P P = ctx->pop;
    const unsigned blocks = (unsigned)std::min<uint32_t>((n + 3) / 4, NUM_SMS * 8);
    auto lay = [&](Carver& c) {
        P.q_contig = c.take<int32_t>(n); P.q_svtype = c.take<int32_t>(n); P.q_pos = c.take<int32_t>(n); P.q_svlen = c.take<int32_t>(n);
        P.q_alt_off = c.take<unsigned long long>(n); P.q_alt_len = c.take<uint32_t>(n); P.q_alt = c.take<uint8_t>(in->n_alt_bytes + 16);
        P.best = c.take<int32_t>(n); P.hs = c.take<int8_t>((size_t)blocks * 4 * max_alt + 16);
    };
    if (carve(ctx->b_popq, lay)) return fail(ctx, "snfb_population_match: out of device memory");
    auto up = [&](const void* dst, const void* src, size_t bytes) { if (bytes && src) CUDA_TRY(cudaMemcpyAsync(const_cast<void*>(dst), src, bytes, cudaMemcpyHostToDevice, st)); return 0; };
    if (up(P.q_contig, in->contig, 4 * (size_t)n) || up(P.q_svtype, in->svtype, 4 * (size_t)n) || up(P.q_pos, in->pos, 4 * (size_t)n) || up(P.q_svlen, in->svlen, 4 * (size_t)n)
        || up(P.q_alt_off, in->alt_off, 8 * (size_t)n) || up(P.q_alt_len, in->alt_len, 4 * (size_t)n) || up(P.q_alt, in->alt, in->n_alt_bytes)) return 1;
    P.n_q = n; P.combine_match = in->combine_match; P.combine_match_max = in->combine_match_max; P.block_size = in->block_size; P.pctseq = in->combine_pctseq; P.max_alt = max_alt;
    mark(ctx, "population_match");
    launch(ctx->launches, population::k_pop_match, blocks, 128, 0, st, P);
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(best, P.best, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_population_match: ") + cudaGetErrorString(e));
    return 0;
}

int snfb_selftest_edit_distance(snfb_ctx* ctx, const uint8_t* bytes, uint64_t n_bytes, const uint64_t* a_off, const uint32_t* a_len, const uint64_t* b_off, const uint32_t* b_len, uint32_t n_pairs, int32_t* out) {
    if (!ctx || !bytes || !a_off || !a_len || !b_off || !b_len || !out) return ctx ? fail(ctx, "snfb_selftest_edit_distance: null argument") : 1;
    if (n_pairs == 0) return 0;
    uint32_t max_len = 16;
    for (uint32_t i = 0; i < n_pairs; ++i) { if (a_off[i] + a_len[i] > n_bytes || b_off[i] + b_len[i] > n_bytes) return fail(ctx, "snfb_selftest_edit_distance: string outside bytes[]"); max_len = std::max(max_len, std::max(a_len[i], b_len[i])); }
    max_len = (max_len + 15u) & ~15u;
    cudaSetDevice(ctx->device);
    const unsigned blocks = (unsigned)std::min<uint32_t>((n_pairs + 3) / 4, NUM_SMS * 4);
    DevBuf d_b, d_o, d_hs, d_out;
    if (d_b.ensure(n_bytes + 16) || d_o.ensure((size_t)n_pairs * 24 + 64) || d_hs.ensure((size_t)blocks * 4 * max_len + 16) || d_out.ensure((size_t)n_pairs * 4)) return fail(ctx, "snfb_selftest_edit_distance: out of device memory");
    unsigned long long* ao = d_o.as<unsigned long long>(); unsigned long long* bo = ao + n_pairs; uint32_t* al = reinterpret_cast<uint32_t*>(bo + n_pairs); uint32_t* bl = al + n_pairs;
    cudaStream_t st = ctx->st;
    CUDA_TRY(cudaMemcpyAsync(d_b.p, bytes, n_bytes, cudaMemcpyHostToDevice, st)); CUDA_TRY(cudaMemcpyAsync(ao, a_off, 8 * (size_t)n_pairs, cudaMemcpyHostToDevice, st)); CUDA_TRY(cudaMemcpyAsync(bo, b_off, 8 * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(al, a_len, 4 * (size_t)n_pairs, cudaMemcpyHostToDevice, st)); CUDA_TRY(cudaMemcpyAsync(bl, b_len, 4 * (size_t)n_pairs, cudaMemcpyHostToDevice, st));
    launch(ctx->launches, combine::k_edit_selftest, blocks, 128, 0, st, d_b.as<uint8_t>(), ao, al, bo, bl, n_pairs, d_hs.as<int8_t>(), max_len, d_out.as<int>());
    CUDA_TRY(cudaMemcpyAsync(out, d_out.p, 4 * (size_t)n_pairs, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_selftest_edit_distance: ") + cudaGetErrorString(e));
    return 0;
}

// mean coverage of `binsize`-base bins over one task's region (snf.py:248-267: the 500-bp means the SNF writer stores), N-masked as the
// contig mean is
int snfb_coverage_bins(snfb_ctx* ctx, uint32_t task, int binsize, const double** out, uint64_t* n_bins) {
    if (!ctx || !ctx->stage_a_done) return ctx ? fail(ctx, "snfb_extract_leads must run first") : 1;
    if (task >= ctx->n_task || binsize <= 0 || !out || !n_bins) return fail(ctx, "bad arguments");
    cudaSetDevice(ctx->device);
    const snfb_task& tk = ctx->tasks[task];
    // the reference pads the contig-long coverage vector with zeros to a multiple of the bin size and takes row means (snf.py:255-256)
    const long long L = tk.contig_len; const long long nb = L > 0 ? (L + binsize - 1) / binsize : 0;
    if (ctx->h_cov_bins.ensure(16 * (size_t)(nb + 1))) return fail(ctx, "out of pinned memory (coverage bins)");
    DevBuf acc; if (acc.ensure(8 * (size_t)(nb + 1))) return fail(ctx, "out of device memory (coverage bins)");
    CUDA_TRY(cudaMemsetAsync(acc.p, 0, 8 * (size_t)(nb + 1), ctx->st));
    uint32_t lohi[2], runs[2] = { 0, 0 };
    CUDA_TRY(cudaMemcpyAsync(&lohi[0], ctx->task_first + task, 4, cudaMemcpyDeviceToHost, ctx->st)); CUDA_TRY(cudaMemcpyAsync(&lohi[1], ctx->task_last + task, 4, cudaMemcpyDeviceToHost, ctx->st));
    if (ctx->n_mask) CUDA_TRY(cudaMemcpyAsync(runs, ctx->b_mask_off.as<uint32_t>() + task, 8, cudaMemcpyDeviceToHost, ctx->st));
    CUDA_TRY(cudaStreamSynchronize(ctx->st));
    if (nb && lohi[1] > lohi[0]) {
        launch(ctx->launches, k_cov_bins, grid_for(lohi[1] - lohi[0], 256), 256, 0, ctx->st, ctx->rec_pos, ctx->rec_end, ctx->rec_flags, lohi[0], lohi[1], binsize, L, nb, acc.as<unsigned long long>());
        // the writer averages the N-masked vector (leadprov.py:470, snf.py:258): take the read bases inside the task's runs back out
        if (runs[1] > runs[0]) launch(ctx->launches, cluster::k_mask_bins, grid_for((unsigned long long)(runs[1] - runs[0]) * 32, 128), 128, 0, ctx->st, ctx->B, (int)task, binsize, acc.as<unsigned long long>());
    }
    unsigned long long* raw = reinterpret_cast<unsigned long long*>(ctx->h_cov_bins.as<uint8_t>() + 8 * (size_t)(nb + 1));
    CUDA_TRY(cudaMemcpyAsync(raw, acc.p, 8 * (size_t)nb, cudaMemcpyDeviceToHost, ctx->st));
    CUDA_TRY(cudaStreamSynchronize(ctx->st));
    double* o = ctx->h_cov_bins.as<double>();
    for (long long i = 0; i < nb; ++i) o[i] = (double)raw[i] / (double)binsize;
    *out = o; *n_bins = (uint64_t)nb; return 0;
}

// force calling (GenotypeTask.execute, parallel.py:300-369): targets matched against the resident candidates, plus their coverage probes
int snfb_genotype_targets(snfb_ctx* ctx, const snfb_gt_in* in, snfb_gt_out* out) {
    if (!ctx || !in || !out) return ctx ? fail(ctx, "snfb_genotype_targets: null argument") : 1;
    if (!ctx->stage_b_done) return fail(ctx, "snfb_genotype_targets: snfb_run or snfb_cluster_call must run first");
    const uint64_t n = in->n;
    if (n == 0) return 0;
    if (!in->task || !in->svtype || !in->pos || !in->svlen || !in->bnd_is_first || !in->mate_contig || !out->match || !out->cov_start || !out->cov_center || !out->cov_end || !out->bnd_no_prev)
        return fail(ctx, "snfb_genotype_targets: null array");
    // the leaked `end` of a BND comes from the last non-BND target of its task before it: found here in one pass, so a long run of BNDs
    // costs no walk on the device
    std::vector<int64_t> prev(n);
    int64_t last = -1;
    for (uint64_t i = 0; i < n; ++i) {
        if (in->task[i] < 0 || (uint32_t)in->task[i] >= ctx->n_task) return fail(ctx, "snfb_genotype_targets: target task out of range");
        if (i && in->task[i] < in->task[i - 1]) return fail(ctx, "snfb_genotype_targets: targets are not ordered by task");
        if (in->svtype[i] < -1 || in->svtype[i] > SNFB_BND) return fail(ctx, "snfb_genotype_targets: target svtype must be SNFB_INS .. SNFB_BND or -1");
        if (i && in->task[i] != in->task[i - 1]) last = -1;
        prev[i] = last;
        if (in->svtype[i] != SNFB_BND) last = (int64_t)i;
    }
    cudaSetDevice(ctx->device);
    const unsigned long long nc = ctx->h_fin->n_cand;
    genotype::P G{}; uint64_t* k1 = nullptr; uint32_t* v1 = nullptr; prims::RadixTemp rt{};
    int32_t* t_in = nullptr; uint64_t* k0 = nullptr; uint32_t* v0 = nullptr;
    auto lay = [&](Carver& c) {
        k0 = c.take<uint64_t>(nc + 1); v0 = c.take<uint32_t>(nc + 1); k1 = c.take<uint64_t>(nc + 1); v1 = c.take<uint32_t>(nc + 1);
        rt.hist = c.take<uint32_t>(prims::radix_hist_elems(nc)); rt.scan_tmp = c.take<uint32_t>(prims::scan_tmp_elems(prims::radix_hist_elems(nc)) + 16);
        t_in = c.take<int32_t>(6 * n); G.prev = c.take<int64_t>(n); G.match = c.take<long long>(n); G.cov_start = c.take<int32_t>(4 * n);
    };
    if (carve(ctx->b_gt, lay)) return fail(ctx, "snfb_genotype_targets: out of device memory");
    G.task = t_in; G.svtype = t_in + n; G.pos = t_in + 2 * n; G.svlen = t_in + 3 * n; G.bnd_is_first = t_in + 4 * n; G.mate_contig = t_in + 5 * n;
    G.cov_center = G.cov_start + n; G.cov_end = G.cov_start + 2 * n; G.bnd_no_prev = G.cov_start + 3 * n;
    cudaStream_t st = ctx->st;
    const int32_t* src[6] = { in->task, in->svtype, in->pos, in->svlen, in->bnd_is_first, in->mate_contig };
    for (int k = 0; k < 6; ++k) CUDA_TRY(cudaMemcpyAsync(t_in + (size_t)k * n, src[k], 4 * n, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(const_cast<int64_t*>(G.prev), prev.data(), 8 * n, cudaMemcpyHostToDevice, st));
    ctx->n_ev = 0;
    mark(ctx, "genotype");
    bool first = true;
    if (nc) {
        launch(ctx->launches, genotype::k_cand_keys, grid_for(nc, 256), 256, 0, st, ctx->B.cand, nc, k0, v0);
        prims::radix_sort(ctx->launches, k0, v0, k1, v1, rt, &ctx->B.ctr->n_cand, nc, genotype::KEY_BITS + bits_for(ctx->n_task), &first, st);
    }
    G.b = ctx->B; G.key = first ? k0 : k1; G.val = first ? v0 : v1; G.n_cand = nc; G.n = n;
    G.combine_match = in->combine_match; G.combine_match_max = in->combine_match_max; G.cluster_merge_bnd = ctx->cfg.cluster_merge_bnd;
    launch(ctx->launches, genotype::k_genotype, grid_for(n * 32, 128), 128, 0, st, G);
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(out->match, G.match, 8 * n, cudaMemcpyDeviceToHost, st));
    int32_t* dst[4] = { out->cov_start, out->cov_center, out->cov_end, out->bnd_no_prev };
    for (int k = 0; k < 4; ++k) CUDA_TRY(cudaMemcpyAsync(dst[k], G.cov_start + (size_t)k * n, 4 * n, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_genotype_targets: ") + cudaGetErrorString(e));
    return 0;
}

// read names (--output-rnames): the candidates' hash lists resolved to the resident records' names, gathered into one text
int snfb_read_names(snfb_ctx* ctx, snfb_rnames_view* out) {
    if (!ctx || !out) return ctx ? fail(ctx, "snfb_read_names: null argument") : 1;
    if (!ctx->stage_b_done) return fail(ctx, "snfb_read_names: snfb_run or snfb_cluster_call must run first");
    cudaSetDevice(ctx->device);
    memset(out, 0, sizeof *out);
    const unsigned long long nc = ctx->h_fin->n_cand, nn = ctx->h_fin->n_rnames;
    rnames::P P{}; uint32_t* scan_tmp = nullptr;
    auto lay = [&](Carver& c) {
        P.first = c.take<uint32_t>(nn + 1); P.len = c.take<uint32_t>(nn + 1); P.off = c.take<uint32_t>(nn + 1); P.src = c.take<uint64_t>(nn + 1);
        scan_tmp = c.take<uint32_t>(prims::scan_tmp_elems(nn) + 16); P.ctr = c.take<unsigned long long>(4);
    };
    if (carve(ctx->b_rn, lay)) return fail(ctx, "snfb_read_names: out of device memory");
    if (ctx->h_rn_meta.ensure(32 + 4 * (nn + 1))) return fail(ctx, "snfb_read_names: out of pinned memory");
    unsigned long long* h_ctr = ctx->h_rn_meta.as<unsigned long long>(); uint32_t* h_off = reinterpret_cast<uint32_t*>(h_ctr + 4);
    P.cand = ctx->B.cand; P.n_cand = nc; P.leads = ctx->B.cand_leads; P.hash = ctx->B.rnames; P.rn_off = ctx->B.rn_off_out; P.n_names = nn;
    P.rec = ctx->d_rec; P.var = ctx->d_var;
    cudaStream_t st = ctx->st;
    ctx->n_ev = 0;
    mark(ctx, "rnames_resolve");
    CUDA_TRY(cudaMemsetAsync(P.ctr, 0, 32, st));
    if (nn) {
        launch(ctx->launches, rnames::k_resolve, grid_for(nc * 32, 128), 128, 0, st, P);
        prims::exclusive_scan(ctx->launches, P.len, P.off, scan_tmp, nullptr, nn, nullptr, st);
    }
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(h_ctr, P.ctr, 32, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const unsigned long long n_text = h_ctr[0];
    if (h_ctr[2]) return fail(ctx, "snfb_read_names: " + std::to_string(h_ctr[2]) + " read name hash(es) carried by none of their candidate's leads");
    if (n_text > 0xffffffffull) return fail(ctx, "snfb_read_names: the names of one pass exceed 4 GiB of text (32-bit offsets); use smaller passes");
    if (ctx->b_rn_text.ensure(n_text + 16) || ctx->h_rn_text.ensure(n_text + 16)) return fail(ctx, "snfb_read_names: out of memory for the text");
    P.text = ctx->b_rn_text.as<uint8_t>();
    mark(ctx, "rnames_copy");
    if (nn) launch(ctx->launches, rnames::k_copy, grid_for(nn * 32, 256), 256, 0, st, P);
    mark(ctx, nullptr);
    if (nn) CUDA_TRY(cudaMemcpyAsync(h_off, P.off, 4 * nn, cudaMemcpyDeviceToHost, st));
    if (n_text) CUDA_TRY(cudaMemcpyAsync(ctx->h_rn_text.p, P.text, n_text, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_read_names: ") + cudaGetErrorString(e));
    h_off[nn] = (uint32_t)n_text;
    out->n_names = nn; out->n_text = n_text; out->text = ctx->h_rn_text.as<uint8_t>(); out->off = h_off; out->collisions = h_ctr[1];
    return 0;
}

// ---- the reference FASTA (--reference): raw bytes -> unwrapped genome, its 'N' runs, REF / anchor gathers ----
int snfb_load_reference(snfb_ctx* ctx, const snfb_ref_input* in) {
    if (!ctx || !in) return ctx ? fail(ctx, "snfb_load_reference: null argument") : 1;
    if ((in->n_bytes && !in->bytes) || (in->n_contig && !in->contig)) return fail(ctx, "snfb_load_reference: null table");
    cudaSetDevice(ctx->device);
    ctx->have_ref = false; ctx->ref_n_runs = 0; ctx->n_ev = 0;
    cudaStream_t st = ctx->st;
    uint64_t raw_len = 0;
    if (in->is_bgzf) {      // the ingest's inflate, CRC-checked; the raw stream lives in b_raw until the genome is built
        BgzfMembers w; InflateCall call{ nullptr, "h2d_ref", in->n_bytes, "inflate" };
        call.oom_tables = "out of device memory (reference inflate tables)";
        if (walk_bgzf(ctx, in->bytes, in->n_bytes, w) || inflate_members(ctx, in->bytes, w, 0, call)) return 1;
        raw_len = w.raw_len;
        mark(ctx, nullptr);
        ingest::IngestCounters hc;
        CUDA_TRY(cudaMemcpyAsync(&hc, w.d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (hc.bad_blocks) { ctx->b_raw.reset(); ctx->b_comp.reset(); inflate_failed(ctx, hc, w); ctx->err = "reference " + ctx->err; return 1; }
        ctx->b_comp.reset();
    } else {
        raw_len = in->n_bytes;
        if (ctx->b_raw.ensure(raw_len + 64)) return fail(ctx, "out of device memory for the reference FASTA bytes");
        mark(ctx, "h2d_ref", raw_len);
        CUDA_TRY(cudaMemcpyAsync(ctx->b_raw.p, in->bytes, raw_len, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemsetAsync(ctx->b_raw.as<uint8_t>() + raw_len, 0, 64, st));
    }
    // the .fai geometry: checked on the host, laid out as 16-byte aligned contigs of the genome and cut into tiles
    const uint32_t nc = in->n_contig;
    std::vector<refseq::Contig> ctg(nc); std::vector<refseq::Tile> ut, nt; std::vector<int64_t> first_nt(nc, -1);
    uint64_t total = 0;
    for (uint32_t c = 0; c < nc; ++c) {
        const snfb_ref_contig& k = in->contig[c];
        const std::string who = "snfb_load_reference: contig " + std::to_string(c);
        if (k.length >= (1ull << 31)) { ctx->b_raw.reset(); return fail(ctx, who + " is 2^31 bases or longer"); }
        if (k.length) {
            if (k.linebases == 0) { ctx->b_raw.reset(); return fail(ctx, who + ": LINEBASES is 0"); }
            const bool multi = k.length > k.linebases;
            if (k.linewidth != k.linebases + 1 && k.linewidth != k.linebases + 2 && (multi || k.linewidth != k.linebases)) { ctx->b_raw.reset(); return fail(ctx, who + ": LINEWIDTH must be LINEBASES + 1 or + 2"); }
            const uint64_t last = k.length - 1, end = k.offset + (last / k.linebases) * k.linewidth + last % k.linebases + 1;
            if (end > raw_len || end < k.offset) { ctx->b_raw.reset(); return fail(ctx, who + ": the .fai geometry reaches byte " + std::to_string(end) + " of a " + std::to_string(raw_len) + "-byte file"); }
        }
        total = (total + 15) & ~15ull;
        ctg[c] = refseq::Contig{ k.offset, k.length, total, k.linebases, k.linewidth };
        for (uint64_t p = 0; p < k.length; p += refseq::UNW_TILE) ut.push_back(refseq::Tile{ c, 0, p });
        if (k.length) first_nt[c] = (int64_t)nt.size();
        for (uint64_t p = 0; p < k.length; p += refseq::NR_TILE) nt.push_back(refseq::Tile{ c, 0, p });
        total += k.length;
    }
    if (nt.size() >= (1ull << 31)) { ctx->b_raw.reset(); return fail(ctx, "snfb_load_reference: genome too large"); }
    if (ctx->b_ref.ensure(total + 256)) { ctx->b_raw.reset(); return fail(ctx, "out of device memory for the reference genome"); }
    const size_t nu = ut.size(), nn = nt.size();
    refseq::Contig* d_ctg = nullptr; refseq::Tile* d_ut = nullptr; refseq::Tile* d_nt = nullptr; refseq::Bad* d_bad = nullptr;
    uint32_t *n_s = nullptr, *n_e = nullptr, *o_s = nullptr, *o_e = nullptr, *tmp = nullptr; unsigned long long* tot = nullptr;
    if (carve(ctx->b_ref_work, [&](Carver& c) { d_ctg = c.take<refseq::Contig>(nc + 1); d_ut = c.take<refseq::Tile>(nu + 1); d_nt = c.take<refseq::Tile>(nn + 1); d_bad = c.take<refseq::Bad>(1);
                                                n_s = c.take<uint32_t>(nn + 1); n_e = c.take<uint32_t>(nn + 1); o_s = c.take<uint32_t>(nn + 1); o_e = c.take<uint32_t>(nn + 1);
                                                tmp = c.take<uint32_t>(prims::scan_tmp_elems(nn + 1) + 16); tot = c.take<unsigned long long>(2); }))
        { ctx->b_raw.reset(); return fail(ctx, "out of device memory (reference tables)"); }
    if (nc) CUDA_TRY(cudaMemcpyAsync(d_ctg, ctg.data(), sizeof(refseq::Contig) * nc, cudaMemcpyHostToDevice, st));
    if (nu) CUDA_TRY(cudaMemcpyAsync(d_ut, ut.data(), sizeof(refseq::Tile) * nu, cudaMemcpyHostToDevice, st));
    if (nn) CUDA_TRY(cudaMemcpyAsync(d_nt, nt.data(), sizeof(refseq::Tile) * nn, cudaMemcpyHostToDevice, st));
    const refseq::Bad bad0{ 0ull, ~0ull };
    CUDA_TRY(cudaMemcpyAsync(d_bad, &bad0, sizeof(bad0), cudaMemcpyHostToDevice, st));
    mark(ctx, "ref_unwrap", raw_len + total);
    if (nu) launch(ctx->launches, refseq::k_ref_unwrap, (unsigned)std::min<size_t>(nu, (size_t)NUM_SMS * 8), refseq::UNW_THREADS, 0, st, ctx->b_raw.as<const uint8_t>(), d_ctg, d_ut, (unsigned)nu, ctx->b_ref.as<uint8_t>(), d_bad);
    mark(ctx, "ref_nruns", 2 * total);
    if (nn) {
        launch(ctx->launches, refseq::k_ref_nruns_count, (unsigned)nn, refseq::NR_THREADS, 0, st, ctx->b_ref.as<const uint8_t>(), d_ctg, d_nt, n_s, n_e);
        prims::exclusive_scan(ctx->launches, n_s, o_s, tmp, nullptr, nn, tot, st);
        prims::exclusive_scan(ctx->launches, n_e, o_e, tmp, nullptr, nn, tot + 1, st);
    } else CUDA_TRY(cudaMemsetAsync(tot, 0, 16, st));
    refseq::Bad hb; unsigned long long ht[2];
    CUDA_TRY(cudaMemcpyAsync(&hb, d_bad, sizeof(hb), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(ht, tot, sizeof(ht), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    ctx->b_raw.reset();                                   // only the unwrapped genome stays resident
    if (hb.n) return fail(ctx, "snfb_load_reference: " + std::to_string(hb.n) + " line(s) do not match the .fai geometry (first: contig " + std::to_string(hb.first >> 40)
                               + ", line " + std::to_string(hb.first & ((1ull << 40) - 1)) + "): the index does not describe this file");
    if (ht[0] != ht[1]) return fail(ctx, "snfb_load_reference: N-run starts and ends do not pair up");
    const uint64_t nr = ht[0];
    if (ctx->h_ref_runs.ensure(8 * (nr + 1)) || ctx->h_ref_coff.ensure(8 * ((size_t)nc + 1)) || ctx->h_ref_out.ensure(4 * (nn + 1))) return fail(ctx, "out of pinned memory (reference N runs)");
    DevBuf d_runs;
    if (d_runs.ensure(8 * (nr + 1))) return fail(ctx, "out of device memory (reference N runs)");
    if (nn && nr) launch(ctx->launches, refseq::k_ref_nruns_write, (unsigned)nn, refseq::NR_THREADS, 0, st, ctx->b_ref.as<const uint8_t>(), d_ctg, d_nt, o_s, o_e, d_runs.as<int32_t>());
    mark(ctx, nullptr);
    if (nr) CUDA_TRY(cudaMemcpyAsync(ctx->h_ref_runs.p, d_runs.p, 8 * nr, cudaMemcpyDeviceToHost, st));
    uint32_t* h_os = ctx->h_ref_out.as<uint32_t>();
    if (nn) CUDA_TRY(cudaMemcpyAsync(h_os, o_s, 4 * nn, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    uint64_t* coff = ctx->h_ref_coff.as<uint64_t>();
    coff[nc] = nr;
    for (int64_t c = (int64_t)nc - 1; c >= 0; --c) coff[c] = first_nt[c] >= 0 ? h_os[first_nt[c]] : coff[c + 1];
    ctx->ref_ctg = std::move(ctg); ctx->ref_n_runs = nr; ctx->have_ref = true;
    return 0;
}

int snfb_reference_runs(snfb_ctx* ctx, const int32_t** runs, const uint64_t** contig_off, uint64_t* n_runs) {
    if (!ctx || !runs || !contig_off || !n_runs) return ctx ? fail(ctx, "snfb_reference_runs: null argument") : 1;
    if (!ctx->have_ref) return fail(ctx, "snfb_reference_runs: no reference is loaded (snfb_load_reference)");
    *runs = ctx->h_ref_runs.as<int32_t>(); *contig_off = ctx->h_ref_coff.as<uint64_t>(); *n_runs = ctx->ref_n_runs;
    return 0;
}

int snfb_fetch_reference(snfb_ctx* ctx, const snfb_ref_query* q, uint64_t n, uint8_t* out, uint64_t out_cap) {
    if (!ctx || (n && (!q || !out))) return ctx ? fail(ctx, "snfb_fetch_reference: null argument") : 1;
    if (!ctx->have_ref) return fail(ctx, "snfb_fetch_reference: no reference is loaded (snfb_load_reference)");
    std::vector<refseq::Query> hq(n); uint64_t span = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const snfb_ref_query& x = q[i];
        if (x.contig >= ctx->ref_ctg.size()) return fail(ctx, "snfb_fetch_reference: query " + std::to_string(i) + ": contig index out of range");
        const refseq::Contig& c = ctx->ref_ctg[x.contig];
        if (x.start > c.len || x.length > c.len - x.start) return fail(ctx, "snfb_fetch_reference: query " + std::to_string(i) + " reaches past the end of contig " + std::to_string(x.contig));
        if (x.out_off > out_cap || x.length > out_cap - x.out_off) return fail(ctx, "snfb_fetch_reference: query " + std::to_string(i) + " does not fit out_cap");
        hq[i] = refseq::Query{ c.out_off + x.start, x.length, x.out_off };
        span = std::max<uint64_t>(span, x.out_off + x.length);
    }
    ctx->n_ev = 0;
    if (n == 0) return 0;
    cudaSetDevice(ctx->device);
    refseq::Query* d_q = nullptr; uint8_t* d_out = nullptr;
    if (carve(ctx->b_ref_work, [&](Carver& c) { d_q = c.take<refseq::Query>(n); d_out = c.take<uint8_t>(span + 16); })) return fail(ctx, "snfb_fetch_reference: out of device memory");
    cudaStream_t st = ctx->st;
    CUDA_TRY(cudaMemcpyAsync(d_q, hq.data(), sizeof(refseq::Query) * n, cudaMemcpyHostToDevice, st));
    mark(ctx, "ref_gather", 2 * span);
    launch(ctx->launches, refseq::k_ref_gather, grid_for(n * 32, 256), 256, 0, st, ctx->b_ref.as<const uint8_t>(), d_q, (unsigned long long)n, d_out);
    mark(ctx, nullptr);
    CUDA_TRY(cudaMemcpyAsync(out, d_out, span, cudaMemcpyDeviceToHost, st));
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, std::string("snfb_fetch_reference: ") + cudaGetErrorString(e));
    return 0;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ BAM index (bam_index.cuh)
namespace {
// one window's members on the host: global inflated end and file offset of each, the inflated start of the first, the file offset after the last
struct IxWin { uint64_t first_beg = 0, coff_end = 0; std::vector<uint64_t> end, coff; };
uint64_t ix_voff(const IxWin& w, uint64_t u) {
    const size_t j = (size_t)(std::lower_bound(w.end.begin(), w.end.end(), u) - w.end.begin());
    if (j < w.end.size() && w.end[j] > u) return w.coff[j] << 16 | (u - (j ? w.end[j - 1] : w.first_beg));
    return (j + 1 < w.end.size() ? w.coff[j + 1] : w.coff_end) << 16;
}
std::string voff_str(uint64_t v) { return std::to_string(v >> 16) + ":" + std::to_string(v & 0xffff); }
}  // namespace

// the name of the record at R[p] of the window on the device
static std::string ix_name(const uint8_t* d_raw, uint64_t p) {
    uint8_t h[36 + 256] = {0};
    if (cudaMemcpy(h, d_raw + p, sizeof(h), cudaMemcpyDeviceToHost) != cudaSuccess) return "?";
    const uint32_t l = h[12];
    return std::string(reinterpret_cast<const char*>(h + 36), l ? strnlen(reinterpret_cast<const char*>(h + 36), l) : 0);
}

namespace {
// one window of the record chain, as stream_windows hands it over: the inflated bytes R[0, L) at global offset base (the carried bytes, then
// the window's members from global offset G), the candidates cand[0, n) of which is_rec marks the n_rows complete chain records (rec_idx:
// their index in the window, in file order); open: the chain ends in a record the window cannot finish (it is carried into the next one);
// v_entry: the virtual offset of the window's first chain record
struct ChainWin {
    uint8_t* R; uint64_t base, L, G, coff_beg; const uint32_t *cand, *is_rec, *rec_idx; uint32_t n; uint64_t n_rows; bool open; uint64_t v_entry;
    const IxWin* W; const unsigned long long *d_end, *d_coff;
};
}  // namespace

// The BAM at `path` streamed through the device in windows of whole BGZF members of at most `win` inflated bytes: each window inflated and
// CRC-checked behind the record the previous one could not finish, its record starts found from the entry by pointer jumping over the
// offsets that pass the strict record test (bam_index.cuh), and on_window(const ChainWin&) called once the chain is resolved (nonzero: stop).
// Failures name the block or the record; `what` prefixes the out-of-memory ones.  *n_windows, *file_bytes: windows read, bytes read.
template <class OnWindow> static int stream_windows(snfb_ctx* ctx, const char* what, const char* path, uint64_t first_record, int n_ref, const long long* d_clen,
                                                    uint64_t win, PhaseTimer& tm, uint64_t* n_windows_out, uint64_t* file_bytes, OnWindow&& on_window) {
    cudaStream_t st = ctx->st;
    const std::string oom = std::string(what) + ": out of device memory";
    FILE* f = fopen(path, "rb");
    if (!f) return fail(ctx, std::string("cannot open ") + path);
    struct Closer { FILE* f; ~Closer() { fclose(f); } } closer{ f };

    std::vector<uint8_t> hb; uint64_t hb_off = 0; bool eof = false;      // read-ahead: file bytes from hb_off
    fseeko(f, 0, SEEK_END); const uint64_t file_size = (uint64_t)ftello(f); fseeko(f, 0, SEEK_SET);
    auto fill = [&](uint64_t target) {                                     // at most the rest of the file, in reads of up to 64 MiB
        target = std::min<uint64_t>(target, file_size - hb_off + 1);
        while (!eof && hb.size() < target) {
            const size_t old = hb.size(), want = (size_t)std::min<uint64_t>(std::max<uint64_t>(target - old, 1 << 20), 64ull << 20);
            hb.resize(old + want);
            const size_t got = fread(hb.data() + old, 1, want, f);
            hb.resize(old + got);
            if (got == 0) eof = true;
        }
    };
    // the entry: global inflated offset of the next record, its virtual offset
    uint64_t G = 0, n_windows = 0;
    uint64_t u_entry = 0, v_entry = first_record; bool entry_known = false;
    uint64_t carry = 0;
    for (;;) {
        fill(std::max<uint64_t>(win, 1 << 17) + 65536 + 64);
        if (hb.empty()) break;
        BgzfMembers M;                                                         // the window's members: hb[0, M.n)
        while (M.n < hb.size()) {
            const BgzfMember m = bgzf_member(hb.data(), hb.size(), M.n);
            if (m.bad && !m.cut) return fail(ctx, "not a BGZF block at file offset " + std::to_string(hb_off + M.n) + ": not a BGZF-compressed BAM file");
            if (m.cut) {
                if (eof) return fail(ctx, "truncated BGZF block at file offset " + std::to_string(hb_off + M.n) + ": the file is truncated");
                if (M.blk.size()) break;
                fill(hb.size() + (1 << 17));
                continue;
            }
            if (M.blk.size() && M.raw_len + m.isize > win) break;
            M.add(m);
        }
        const uint64_t sel = M.n, raw_len = M.raw_len;
        IxWin W; W.first_beg = G; W.coff_end = hb_off + sel;
        for (size_t k = 0; k < M.blk.size(); ++k) { W.end.push_back(G + M.blk[k].out_off + M.blk[k].isize); W.coff.push_back(hb_off + M.cstart[k]); }
        if (!entry_known) {                                                    // the header's end, as a global inflated offset
            const uint64_t c = first_record >> 16, u = first_record & 0xffff;
            auto it = std::find(W.coff.begin(), W.coff.end(), c);
            if (it != W.coff.end()) { const size_t k = (size_t)(it - W.coff.begin()); u_entry = (k ? W.end[k - 1] : G) + u; entry_known = true; }
        }
        const uint64_t base = G - carry, L = carry + raw_len, G_win = G, coff_beg = hb_off;
        // inflate and CRC-check the window behind the carried bytes
        if (inflate_members(ctx, hb.data(), M, carry, InflateCall{ &tm, nullptr, 0, nullptr, oom + " for the window", oom + " (ingest tables)" })) return 1;
        uint8_t* R = ctx->b_raw.as<uint8_t>();
        if (carry) CUDA_TRY(cudaMemcpyAsync(R, ctx->b_ix_carry.p, carry, cudaMemcpyDeviceToDevice, st));
        ingest::IngestCounters hc;
        CUDA_TRY(cudaMemcpyAsync(&hc, M.d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, st));
        tm.end(st);
        CUDA_TRY(cudaStreamSynchronize(st));
        if (hc.bad_blocks) return inflate_failed_in_file(ctx, hc, M, hb_off);
        hb.erase(hb.begin(), hb.begin() + (ptrdiff_t)sel); hb_off += sel;
        G += raw_len; ++n_windows;
        if (!entry_known || u_entry >= base + L) continue;                   // still inside the header
        const uint64_t e = u_entry - base;
        // candidates
        const uint64_t n_words = (L + 31) / 32;
        uint32_t *mask = nullptr, *cnt = nullptr, *wbase = nullptr, *stmp = nullptr; unsigned long long* misc = nullptr; unsigned long long *d_end = nullptr, *d_coff = nullptr;
        if (carve(ctx->b_ix_mask, [&](Carver& c) { mask = c.take<uint32_t>(n_words); cnt = c.take<uint32_t>(n_words); wbase = c.take<uint32_t>(n_words); stmp = c.take<uint32_t>(prims::scan_tmp_elems(n_words) + 16);
                                                   misc = c.take<unsigned long long>(8); d_end = c.take<unsigned long long>(W.end.size()); d_coff = c.take<unsigned long long>(W.coff.size()); }))
            return fail(ctx, oom + " (candidate masks)");
        tm.begin(st);
        CUDA_TRY(cudaMemcpyAsync(d_end, W.end.data(), 8 * W.end.size(), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_coff, W.coff.data(), 8 * W.coff.size(), cudaMemcpyHostToDevice, st));
        mark(ctx, "index_candidates", L);
        launch(ctx->launches, bamidx::k_mark, grid_for(n_words * 32, 256), 256, 0, st, (const uint8_t*)R, (unsigned long long)L, (unsigned long long)e, n_ref, d_clen, mask, cnt, (unsigned long long)n_words);
        prims::exclusive_scan(ctx->launches, cnt, wbase, stmp, nullptr, n_words, &misc[0], st);
        unsigned long long n_cand = 0;
        CUDA_TRY(cudaMemcpyAsync(&n_cand, &misc[0], 8, cudaMemcpyDeviceToHost, st));
        tm.end(st);
        CUDA_TRY(cudaStreamSynchronize(st));
        const uint64_t v_e = e == 0 && carry ? v_entry : ix_voff(W, base + e);
        if (n_cand == 0) return fail(ctx, "the record at virtual offset " + voff_str(v_e) + " is not a valid BAM record");
        const uint32_t n = (uint32_t)n_cand, n2 = n + 2;
        const int K = std::max(1, bits_for(n2));
        uint32_t *cand = nullptr, *J = nullptr, *is_rec = nullptr, *rec_idx = nullptr, *ntmp = nullptr; uint8_t* pmark = nullptr; unsigned long long* res = nullptr;
        if (carve(ctx->b_ix_node, [&](Carver& c) { cand = c.take<uint32_t>(n); J = c.take<uint32_t>((size_t)K * n2); pmark = c.take<uint8_t>(n2); is_rec = c.take<uint32_t>(n + 1); rec_idx = c.take<uint32_t>(n + 1);
                                                   ntmp = c.take<uint32_t>(prims::scan_tmp_elems(n) + 16); res = c.take<unsigned long long>(8); }))
            return fail(ctx, oom + " (" + std::to_string(n) + " candidate record starts)");
        tm.begin(st);
        mark(ctx, "index_chain", 0);
        launch(ctx->launches, bamidx::k_compact, grid_for(n_words * 32, 256), 256, 0, st, (const uint32_t*)mask, (const uint32_t*)wbase, (unsigned long long)n_words, cand);
        launch(ctx->launches, bamidx::k_link, grid_for(n2, 256), 256, 0, st, (const uint8_t*)R, (unsigned long long)L, n_ref, d_clen, (const uint32_t*)cand, n, J);
        for (int k = 0; k + 1 < K; ++k) launch(ctx->launches, bamidx::k_jump, grid_for(n2, 256), 256, 0, st, (const uint32_t*)(J + (size_t)k * n2), J + (size_t)(k + 1) * n2, n2);
        CUDA_TRY(cudaMemsetAsync(pmark, 0, n2, st));
        CUDA_TRY(cudaMemsetAsync(pmark, 1, 1, st));
        for (int k = K - 1; k >= 0; --k) launch(ctx->launches, bamidx::k_mark_path, grid_for(n2, 256), 256, 0, st, (const uint32_t*)(J + (size_t)k * n2), n2, pmark);
        CUDA_TRY(cudaMemsetAsync(res, 0xff, 16, st));
        launch(ctx->launches, bamidx::k_path_records, grid_for(n, 256), 256, 0, st, (const uint8_t*)pmark, (const uint32_t*)J, n, is_rec, (const uint32_t*)cand, res);
        prims::exclusive_scan(ctx->launches, is_rec, rec_idx, ntmp, nullptr, n, &res[2], st);
        unsigned long long hres[3]; uint32_t cand0 = 0; uint8_t end_marked = 0;
        CUDA_TRY(cudaMemcpyAsync(hres, res, 24, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(&cand0, cand, 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(&end_marked, pmark + n + bamidx::END_NODE, 1, cudaMemcpyDeviceToHost, st));
        tm.end(st);
        CUDA_TRY(cudaStreamSynchronize(st));
        if (cand0 != e) return fail(ctx, "the record at virtual offset " + voff_str(v_e) + " is not a valid BAM record");
        if (hres[1] != ~0ull) {
            uint32_t p = 0; CUDA_TRY(cudaMemcpy(&p, cand + hres[1], 4, cudaMemcpyDeviceToHost));
            uint32_t bs = 0; CUDA_TRY(cudaMemcpy(&bs, R + p, 4, cudaMemcpyDeviceToHost));
            const uint64_t vp = p == 0 && carry ? v_entry : ix_voff(W, base + p);
            return fail(ctx, "the record chain breaks after record '" + ix_name(R, p) + "' at virtual offset " + voff_str(vp) + ": the bytes at virtual offset "
                             + voff_str(ix_voff(W, base + p + 4 + bs)) + " are not a BAM record (corrupt or not a BAM file)");
        }
        if (hres[0] == ~0ull && !end_marked) return fail(ctx, std::string(what) + ": the record chain did not resolve");
        const ChainWin cw{ R, base, L, G_win, coff_beg, cand, is_rec, rec_idx, n, hres[2], hres[0] != ~0ull, v_entry, &W, d_end, d_coff };
        if (on_window(cw)) return 1;
        if (hres[2]) v_entry = ix_voff(W, hres[0] != ~0ull ? base + hres[0] : base + L);      // the virtual offset after the last complete record
        mark(ctx, nullptr);
        if (hres[0] != ~0ull) {                        // the chain ends in a record the window cannot finish: carry it into the next one
            const uint64_t o = hres[0];
            carry = L - o;
            if (ctx->b_ix_carry.ensure(carry + 64)) return fail(ctx, oom + " (carried record)");
            CUDA_TRY(cudaMemcpyAsync(ctx->b_ix_carry.p, R + o, carry, cudaMemcpyDeviceToDevice, st));
            u_entry = base + o;
        } else { carry = 0; u_entry = base + L; }
    }
    if (!entry_known && first_record == hb_off << 16) entry_known = true, u_entry = G;      // a header-only file without the EOF member
    if (!entry_known || u_entry != G)
        return fail(ctx, "truncated BAM file: the record at virtual offset " + voff_str(v_entry) + " extends past the end of the data (" + std::to_string(G) + " inflated bytes)");
    CUDA_TRY(cudaStreamSynchronize(st));
    *n_windows_out = n_windows; *file_bytes = hb_off;
    return 0;
}

extern "C" int snfb_index_bam(snfb_ctx* ctx, const snfb_index_input* in, snfb_index_view* out) {
    using bamidx::Row;
    if (!ctx || !in || !out || !in->path || (in->n_ref && !in->contig_len)) return ctx ? fail(ctx, "snfb_index_bam: null argument") : 1;
    if (in->min_shift < 1 || in->depth < 1 || in->min_shift + 3 * in->depth > 40) return fail(ctx, "snfb_index_bam: min_shift + 3 * depth must be in 4..40");
    cudaSetDevice(ctx->device);
    ctx->n_ev = 0;
    const uint64_t win = std::min<uint64_t>(std::max<uint64_t>(in->window_bytes, 1), 1ull << 31);
    const bamidx::Geo geo{ in->min_shift, in->depth };
    const uint32_t n_bins = (uint32_t)(((1ull << (3 * (in->depth + 1))) - 1) / 7);
    const long long max_end = 1ll << (in->min_shift + 3 * in->depth);
    const int n_ref = (int)in->n_ref;
    cudaStream_t st = ctx->st;
    PhaseTimer tm;
    auto t_begin = [&]() { tm.begin(st); };
    auto t_end = [&]() { tm.end(st); };
    long long* d_clen = nullptr;
    if (carve(ctx->b_ix_tab, [&](Carver& c) { d_clen = c.take<long long>(n_ref + 1); })) return fail(ctx, "snfb_index_bam: out of device memory");
    if (n_ref) CUDA_TRY(cudaMemcpyAsync(d_clen, in->contig_len, 8ull * n_ref, cudaMemcpyHostToDevice, st));
    // the previous row's tid / beg for the order check
    int prev_tid = -2, prev_beg = 0;
    std::vector<Row> rows;
    uint64_t n_windows = 0, file_bytes = 0;
    auto on_window = [&](const ChainWin& c) -> int {
        const uint64_t n_rows = c.n_rows;
        if (!n_rows) return 0;
        const uint64_t row_base = rows.size();
        const uint32_t n = c.n;
        uint32_t* roff = nullptr; Row* d_rows = nullptr; unsigned long long* bad_d = nullptr;
        if (carve(ctx->b_ix_rows, [&](Carver& cv) { roff = cv.take<uint32_t>(n + 1); d_rows = cv.take<Row>(n + 1); bad_d = cv.take<unsigned long long>(1); }))
            return fail(ctx, "snfb_index_bam: out of device memory (" + std::to_string(n) + " candidate record starts)");
        t_begin();
        mark(ctx, "index_rows", 0);
        bamidx::Window DW{ c.base, c.W->first_beg, c.W->coff_end, c.d_end, c.d_coff, (unsigned)c.W->end.size() };
        launch(ctx->launches, bamidx::k_rows, grid_for((uint64_t)n * 32, 256), 256, 0, st, (const uint8_t*)c.R, c.cand, c.is_rec, c.rec_idx, n, DW, d_rows, roff);
        CUDA_TRY(cudaMemsetAsync(bad_d, 0xff, 8, st));
        launch(ctx->launches, bamidx::k_check, grid_for(n_rows, 256), 256, 0, st, d_rows, (uint32_t)n_rows, (unsigned long long)c.v_entry, prev_tid, prev_beg, max_end, (unsigned long long)row_base, bad_d);
        rows.resize(row_base + n_rows);
        unsigned long long bad = 0;
        CUDA_TRY(cudaMemcpyAsync(rows.data() + row_base, d_rows, sizeof(Row) * n_rows, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(&bad, bad_d, 8, cudaMemcpyDeviceToHost, st));
        t_end();
        CUDA_TRY(cudaStreamSynchronize(st));
        if (bad != bamidx::BAD_NONE) {
            const uint64_t r = bad & ((1ull << 56) - 1), i = r - row_base; const unsigned code = (unsigned)(bad >> 56);
            uint32_t p = 0; CUDA_TRY(cudaMemcpy(&p, roff + i, 4, cudaMemcpyDeviceToHost));
            const Row& x = rows[r];
            const int pt = r ? rows[r - 1].tid : prev_tid, pb = r ? rows[r - 1].beg : prev_beg;
            std::string why;
            if (code == bamidx::BAD_ORDER) why = "unsorted positions on reference #" + std::to_string(x.tid) + ": " + std::to_string(x.beg + 1) + " after " + std::to_string(pb + 1);
            else if (code == bamidx::BAD_TID_AFTER_UNPLACED) why = "a record on reference #" + std::to_string(x.tid) + " after the unplaced records (reference -1), which must come last";
            else if (code == bamidx::BAD_TID_BACK) why = "reference #" + std::to_string(x.tid) + " after reference #" + std::to_string(pt) + ": the records are not sorted by coordinate";
            else why = "end " + std::to_string(x.end) + " beyond the " + std::to_string(max_end) + " positions the index geometry covers (a BAI covers 2^29: use -c for a CSI index)";
            return fail(ctx, "record '" + ix_name(c.R, p) + "' (record " + std::to_string(r + 1) + " of the file, virtual offset " + voff_str(x.v0) + "): " + why);
        }
        prev_tid = rows.back().tid; prev_beg = rows.back().beg;
        return 0;
    };
    if (stream_windows(ctx, "snfb_index_bam", in->path, in->first_record, n_ref, d_clen, win, tm, &n_windows, &file_bytes, on_window)) return 1;

    // ---- tables over all rows
    const uint64_t n_rec = rows.size();
    uint64_t n_placed = 0;
    while (n_placed < n_rec && rows[n_placed].tid >= 0) ++n_placed;
    if (n_rec >= (1ull << 32)) return fail(ctx, "snfb_index_bam: more than 2^32 records");
    ctx->ix_ref.assign(5ull * n_ref, 0);
    for (int t = 0; t < n_ref; ++t) ctx->ix_ref[5ull * t] = ~0ull;
    uint64_t* d_ref = nullptr; Row* d_all = nullptr;
    if (ctx->b_ix_rows.ensure(sizeof(Row) * (n_placed + 1))) return fail(ctx, "snfb_index_bam: out of device memory (rows)");
    d_all = ctx->b_ix_rows.as<Row>();
    if (carve(ctx->b_ix_tab, [&](Carver& c) { d_clen = c.take<long long>(n_ref + 1); d_ref = c.take<uint64_t>(5ull * n_ref + 1); })) return fail(ctx, "snfb_index_bam: out of device memory");
    t_begin();
    mark(ctx, "index_tables", sizeof(Row) * n_placed);
    if (n_placed) CUDA_TRY(cudaMemcpyAsync(d_all, rows.data(), sizeof(Row) * n_placed, cudaMemcpyHostToDevice, st));
    if (n_ref) CUDA_TRY(cudaMemcpyAsync(d_ref, ctx->ix_ref.data(), 8 * ctx->ix_ref.size(), cudaMemcpyHostToDevice, st));
    if (n_placed) launch(ctx->launches, bamidx::k_ref_stats, grid_for(n_placed, 256), 256, 0, st, (const Row*)d_all, (uint32_t)n_placed, geo, (unsigned long long*)d_ref);
    if (n_ref) CUDA_TRY(cudaMemcpyAsync(ctx->ix_ref.data(), d_ref, 8 * ctx->ix_ref.size(), cudaMemcpyDeviceToHost, st));
    t_end();
    CUDA_TRY(cudaStreamSynchronize(st));
    ctx->ix_lin_off.assign(n_ref + 1, 0);
    for (int t = 0; t < n_ref; ++t) ctx->ix_lin_off[t + 1] = ctx->ix_lin_off[t] + ctx->ix_ref[5ull * t + 4];
    const uint64_t n_lin = ctx->ix_lin_off[n_ref];
    const uint64_t np = n_placed;
    uint64_t *lin_off = nullptr, *lin = nullptr, *rkey = nullptr, *ckey = nullptr, *ckey2 = nullptr, *ukey = nullptr, *cu = nullptr, *cv = nullptr, *bmin = nullptr, *bmax = nullptr, *loff = nullptr, *mu = nullptr, *mv = nullptr, *cnts = nullptr;
    uint32_t *head = nullptr, *cidx = nullptr, *cval = nullptr, *cval2 = nullptr, *h = nullptr, *hidx = nullptr, *cur = nullptr, *mbin = nullptr, *stmp = nullptr, *hist = nullptr; int *parent = nullptr, *level = nullptr;
    const size_t hist_n = prims::radix_hist_elems(np + 1);
    if (carve(ctx->b_ix_tab, [&](Carver& c) {
            lin_off = c.take<uint64_t>(n_ref + 1); lin = c.take<uint64_t>(n_lin + 1); rkey = c.take<uint64_t>(np + 1);
            head = c.take<uint32_t>(np + 1); cidx = c.take<uint32_t>(np + 1); cu = c.take<uint64_t>(np + 1); cv = c.take<uint64_t>(np + 1); ckey = c.take<uint64_t>(np + 1); ckey2 = c.take<uint64_t>(np + 1);
            cval = c.take<uint32_t>(np + 1); cval2 = c.take<uint32_t>(np + 1); h = c.take<uint32_t>(np + 1); hidx = c.take<uint32_t>(np + 1); ukey = c.take<uint64_t>(np + 1); cur = c.take<uint32_t>(np + 1);
            parent = c.take<int>(np + 1); level = c.take<int>(np + 1); loff = c.take<uint64_t>(np + 1); bmin = c.take<uint64_t>(np + 1); bmax = c.take<uint64_t>(np + 1);
            mbin = c.take<uint32_t>(np + 1); mu = c.take<uint64_t>(np + 1); mv = c.take<uint64_t>(np + 1); cnts = c.take<uint64_t>(8);
            hist = c.take<uint32_t>(hist_n); stmp = c.take<uint32_t>(prims::scan_tmp_elems(std::max<uint64_t>(hist_n, np + 1)) + 16); }))
        return fail(ctx, "snfb_index_bam: out of device memory (tables)");
    CUDA_TRY(cudaMemcpyAsync(lin_off, ctx->ix_lin_off.data(), 8 * (n_ref + 1), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(lin, 0xff, 8 * (n_lin + 1), st));
    uint64_t h_n[3] = { 0, 0, 0 };            // chunks, unique bins, merged chunks
    t_begin();
    if (np) {
        const int grid = grid_for(np, 256);
        launch(ctx->launches, bamidx::k_chunks, grid, 256, 0, st, (const Row*)d_all, (uint32_t)np, geo, n_bins, head, rkey, (const unsigned long long*)lin_off, (unsigned long long*)lin);
        prims::exclusive_scan(ctx->launches, head, cidx, stmp, nullptr, np, (unsigned long long*)&cnts[0], st);
        launch(ctx->launches, bamidx::k_chunk_rows, grid, 256, 0, st, (const Row*)d_all, (const uint32_t*)head, (const uint32_t*)cidx, (const uint64_t*)rkey, (uint32_t)np,
               (unsigned long long*)cu, (unsigned long long*)cv, ckey, cval);
        CUDA_TRY(cudaMemcpyAsync(&h_n[0], &cnts[0], 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    if (n_ref) launch(ctx->launches, bamidx::k_lin_fill, n_ref, 256, 0, st, (unsigned long long*)lin, (const unsigned long long*)lin_off, n_ref);
    const uint32_t nc = (uint32_t)h_n[0];
    if (nc) {
        const int grid = grid_for(nc, 256);
        bool in_first = true;
        int key_bits = 1; while (key_bits < 64 && ((uint64_t)n_ref * n_bins) >> key_bits) ++key_bits;
        prims::radix_sort(ctx->launches, ckey, cval, ckey2, cval2, prims::RadixTemp{ hist, stmp }, (const unsigned long long*)&cnts[0], nc, key_bits, &in_first, st);
        const uint64_t* sk = in_first ? ckey : ckey2; const uint32_t* sv = in_first ? cval : cval2;
        launch(ctx->launches, bamidx::k_key_heads, grid, 256, 0, st, sk, nc, h);
        prims::exclusive_scan(ctx->launches, h, hidx, stmp, nullptr, nc, (unsigned long long*)&cnts[1], st);
        launch(ctx->launches, bamidx::k_unique_bins, grid, 256, 0, st, sk, sv, (const uint32_t*)h, (const uint32_t*)hidx, nc, ukey, cur);
        CUDA_TRY(cudaMemcpyAsync(&h_n[1], &cnts[1], 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        const uint32_t nub = (uint32_t)h_n[1];
        launch(ctx->launches, bamidx::k_bin_info, grid_for(nub, 256), 256, 0, st, (const uint64_t*)ukey, nub, n_bins, geo, (const unsigned long long*)lin_off, (const unsigned long long*)lin, parent, level, (unsigned long long*)loff);
        for (int l = in->depth; l >= 1; --l) {
            CUDA_TRY(cudaMemsetAsync(bmin, 0xff, 8ull * nub, st));
            CUDA_TRY(cudaMemsetAsync(bmax, 0, 8ull * nub, st));
            launch(ctx->launches, bamidx::k_bin_span, grid, 256, 0, st, (const uint32_t*)cur, (const int*)level, (const unsigned long long*)cu, (const unsigned long long*)cv, nc, l, (unsigned long long*)bmin, (unsigned long long*)bmax);
            launch(ctx->launches, bamidx::k_bin_lift, grid, 256, 0, st, cur, (const int*)level, (const int*)parent, nc, l, (const unsigned long long*)bmin, (const unsigned long long*)bmax);
        }
        launch(ctx->launches, bamidx::k_cur_keys, grid, 256, 0, st, (const uint32_t*)cur, nc, ckey, cval);
        prims::radix_sort(ctx->launches, ckey, cval, ckey2, cval2, prims::RadixTemp{ hist, stmp }, (const unsigned long long*)&cnts[0], nc, std::max(1, bits_for(nub)), &in_first, st);
        const uint64_t* sb = in_first ? ckey : ckey2; const uint32_t* sc = in_first ? cval : cval2;
        launch(ctx->launches, bamidx::k_merge_heads, grid, 256, 0, st, sb, sc, (const unsigned long long*)cu, (const unsigned long long*)cv, nc, h);
        prims::exclusive_scan(ctx->launches, h, hidx, stmp, nullptr, nc, (unsigned long long*)&cnts[2], st);
        launch(ctx->launches, bamidx::k_merge_out, grid, 256, 0, st, sb, sc, (const unsigned long long*)cu, (const unsigned long long*)cv, (const uint32_t*)h, (const uint32_t*)hidx, nc, mbin,
               (unsigned long long*)mu, (unsigned long long*)mv);
        CUDA_TRY(cudaMemcpyAsync(&h_n[2], &cnts[2], 8, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    mark(ctx, nullptr);
    const uint64_t nub = h_n[1], nm = h_n[2];
    ctx->ix_lin.resize(n_lin + 1); ctx->ix_bin_key.resize(nub + 1); ctx->ix_bin_loff.resize(nub + 1); ctx->ix_chunk_bin.resize(nm + 1); ctx->ix_chunk_u.resize(nm + 1); ctx->ix_chunk_v.resize(nm + 1);
    if (n_lin) CUDA_TRY(cudaMemcpyAsync(ctx->ix_lin.data(), lin, 8 * n_lin, cudaMemcpyDeviceToHost, st));
    if (nub) { CUDA_TRY(cudaMemcpyAsync(ctx->ix_bin_key.data(), ukey, 8 * nub, cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaMemcpyAsync(ctx->ix_bin_loff.data(), loff, 8 * nub, cudaMemcpyDeviceToHost, st)); }
    if (nm) {
        CUDA_TRY(cudaMemcpyAsync(ctx->ix_chunk_bin.data(), mbin, 4 * nm, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(ctx->ix_chunk_u.data(), mu, 8 * nm, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(ctx->ix_chunk_v.data(), mv, 8 * nm, cudaMemcpyDeviceToHost, st));
    }
    t_end();
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    out->ref = ctx->ix_ref.data(); out->lin_off = ctx->ix_lin_off.data(); out->lin = ctx->ix_lin.data();
    out->bin_key = ctx->ix_bin_key.data(); out->bin_loff = ctx->ix_bin_loff.data(); out->chunk_bin = ctx->ix_chunk_bin.data(); out->chunk_beg = ctx->ix_chunk_u.data(); out->chunk_end = ctx->ix_chunk_v.data();
    out->n_bin = nub; out->n_chunk = nm; out->n_no_coor = n_rec - n_placed; out->n_records = n_rec; out->n_windows = n_windows;
    out->device_ms = tm.ms;
    out->device_bytes = ctx->b_comp.cap + ctx->b_raw.cap + ctx->b_ing.cap + ctx->b_ix_mask.cap + ctx->b_ix_node.cap + ctx->b_ix_carry.cap + ctx->b_ix_rows.cap + ctx->b_ix_tab.cap;
    return 0;
}

// ------------------------------------------------------------------------------------------------ BAM sort (bam_sort.cuh)
extern "C" int snfb_sort_bam(snfb_ctx* ctx, const snfb_sort_input* in, snfb_sort_view* out) {
    if (!ctx || !in || !out || !in->path || !in->out_path || !in->header || (in->n_ref && !in->contig_len)) return ctx ? fail(ctx, "snfb_sort_bam: null argument") : 1;
    if (in->header_len < 12) return fail(ctx, "snfb_sort_bam: the output header must hold at least the magic, l_text and n_ref");
    cudaSetDevice(ctx->device);
    ctx->n_ev = 0;
    *out = snfb_sort_view{};
    const uint64_t win = std::min<uint64_t>(std::max<uint64_t>(in->window_bytes, 1), 1ull << 31);
    const uint64_t bucket_cap = std::max<uint64_t>(in->bucket_bytes, 1);
    const uint64_t BS = deflate::BLOCK_IN;
    const int n_ref = (int)in->n_ref;
    cudaStream_t st = ctx->st;
    PhaseTimer t_keys, t_sort, t_layout, t_scatter, t_deflate;
    long long* d_clen = nullptr;
    if (carve(ctx->b_st_lay, [&](Carver& c) { d_clen = c.take<long long>(n_ref + 1); })) return fail(ctx, "snfb_sort_bam: out of device memory");
    if (n_ref) CUDA_TRY(cudaMemcpyAsync(d_clen, in->contig_len, 8ull * n_ref, cudaMemcpyHostToDevice, st));

    // ---- keys pass: per record its key, its length 4 + block_size and its global inflated offset; per window its geometry and the
    // input ordinals of the records with bytes in it (those completed in it, and the one carried out of it)
    struct SWin { uint64_t coff_beg, coff_end, G, raw_len, o0, o1; };
    std::vector<SWin> wins;
    std::vector<uint64_t> h_key, h_src; std::vector<uint32_t> h_len;
    auto on_window = [&](const ChainWin& c) -> int {
        const uint64_t row_base = h_key.size();
        if (row_base + c.n_rows >= (1ull << 32)) return fail(ctx, "snfb_sort_bam: 2^32 records or more (record " + std::to_string(row_base + c.n_rows) + "): more than the sort's 32-bit ordinals hold");
        wins.push_back(SWin{ c.coff_beg, c.W->coff_end, c.G, c.W->end.back() - c.G, row_base, row_base + c.n_rows + (c.open ? 1 : 0) });
        if (!c.n_rows) return 0;
        uint64_t* key = nullptr; uint32_t* len = nullptr; unsigned long long* src = nullptr;
        if (carve(ctx->b_st_win, [&](Carver& cv) { key = cv.take<uint64_t>(c.n_rows); len = cv.take<uint32_t>(c.n_rows); src = cv.take<unsigned long long>(c.n_rows); }))
            return fail(ctx, "snfb_sort_bam: out of device memory (window keys)");
        h_key.resize(row_base + c.n_rows); h_len.resize(row_base + c.n_rows); h_src.resize(row_base + c.n_rows);
        t_keys.begin(st);
        mark(ctx, "sort_keys", 0);
        launch(ctx->launches, bamsort::k_keys, grid_for(c.n, 256), 256, 0, st, (const uint8_t*)c.R, c.cand, c.is_rec, c.rec_idx, c.n, (unsigned long long)c.base, n_ref, key, len, src);
        CUDA_TRY(cudaMemcpyAsync(h_key.data() + row_base, key, 8 * c.n_rows, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(h_len.data() + row_base, len, 4 * c.n_rows, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(h_src.data() + row_base, src, 8 * c.n_rows, cudaMemcpyDeviceToHost, st));
        t_keys.end(st);
        return 0;
    };
    uint64_t n_windows = 0, bytes_in = 0;
    if (stream_windows(ctx, "snfb_sort_bam", in->path, in->first_record, n_ref, d_clen, win, t_keys, &n_windows, &bytes_in, on_window)) return 1;
    const uint64_t n = h_key.size();
    const uint32_t n_win = (uint32_t)wins.size();

    // ---- sort: one stable radix sort of the keys, over only the bits they use; values = input ordinals
    uint64_t *k0 = nullptr, *k1 = nullptr; uint32_t *v0 = nullptr, *v1 = nullptr, *len = nullptr, *hist = nullptr, *stmp = nullptr;
    unsigned long long *src = nullptr, *dest = nullptr, *dsort = nullptr, *cnt = nullptr;
    const size_t hist_n = prims::radix_hist_elems(n + 1);
    if (carve(ctx->b_st_rec, [&](Carver& c) { k0 = c.take<uint64_t>(n + 1); k1 = c.take<uint64_t>(n + 1); v0 = c.take<uint32_t>(n + 1); v1 = c.take<uint32_t>(n + 1);
                                              len = c.take<uint32_t>(n + 1); src = c.take<unsigned long long>(n + 1); dest = c.take<unsigned long long>(n + 1); dsort = c.take<unsigned long long>(n + 1);
                                              cnt = c.take<unsigned long long>(8); hist = c.take<uint32_t>(hist_n); stmp = c.take<uint32_t>(prims::scan_tmp_elems(hist_n) + 16); }))
        return fail(ctx, "snfb_sort_bam: out of device memory (" + std::to_string(n) + " record keys)");
    std::vector<uint32_t> h_slen(n);
    const uint32_t* ord = v0;
    if (n) {
        const unsigned long long hn = n;
        t_sort.begin(st);
        mark(ctx, "sort_radix", 12 * n);
        CUDA_TRY(cudaMemcpyAsync(k0, h_key.data(), 8 * n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(len, h_len.data(), 4 * n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(src, h_src.data(), 8 * n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(cnt, &hn, 8, cudaMemcpyHostToDevice, st));
        launch(ctx->launches, bamsort::k_iota, grid_for(n, 256), 256, 0, st, v0, (unsigned long long)n);
        bool in_first = true;
        prims::radix_sort(ctx->launches, k0, v0, k1, v1, prims::RadixTemp{ hist, stmp }, (const unsigned long long*)cnt, n, 33 + bits_for((uint32_t)n_ref + 1), &in_first, st);
        ord = in_first ? v0 : v1;
        uint32_t* slen = in_first ? v1 : v0;
        t_sort.end(st);
        t_layout.begin(st);
        mark(ctx, "sort_layout", 4 * n);
        launch(ctx->launches, bamsort::k_gather_len, grid_for(n, 256), 256, 0, st, ord, (const uint32_t*)len, (unsigned long long)n, slen);
        CUDA_TRY(cudaMemcpyAsync(h_slen.data(), slen, 4 * n, cudaMemcpyDeviceToHost, st));
        t_layout.end(st);
    }
    std::vector<uint64_t>().swap(h_key); std::vector<uint32_t>().swap(h_len); std::vector<uint64_t>().swap(h_src);

    // ---- layout: htslib's member cuts over the sorted lengths (sequential by definition: one host loop), each record's output offset,
    // then buckets of whole members that start at a record start
    const auto h0 = std::chrono::steady_clock::now();
    const uint64_t H = in->header_len;
    std::vector<uint64_t> mend;                    // member k = output bytes [k ? mend[k - 1] : 0, mend[k])
    std::vector<uint32_t> unit{ 0 };               // members that start at a record start (or at the header)
    std::vector<unsigned long long> h_dsort(n);
    for (uint64_t o = 0; o < H;) { o = std::min(o + BS, H); mend.push_back(o); }
    uint64_t pos = H, cur = 0;
    for (uint64_t s = 0; s < n; ++s) {
        uint64_t r = h_slen[s];
        if (cur && cur + r > BS) { mend.push_back(pos); cur = 0; }
        if (!cur) unit.push_back((uint32_t)mend.size());
        h_dsort[s] = pos;
        while (r) { const uint64_t take = std::min(r, BS - cur); cur += take; pos += take; r -= take; if (cur == BS) { mend.push_back(pos); cur = 0; } }
    }
    if (cur) mend.push_back(pos);
    const uint32_t nm = (uint32_t)mend.size();
    auto mbeg = [&](uint32_t m) -> uint64_t { return m ? mend[m - 1] : 0; };
    std::vector<uint32_t> bm{ 0 };                 // bucket k = members [bm[k], bm[k + 1])
    {
        uint32_t last = 0;
        for (size_t i = 1; i <= unit.size(); ++i) {
            const uint32_t c = i < unit.size() ? unit[i] : nm;
            if (mend[c - 1] - mbeg(bm.back()) > bucket_cap && last > bm.back()) bm.push_back(last);
            last = c;
        }
        bm.push_back(nm);
    }
    const uint32_t n_bkt = (uint32_t)bm.size() - 1;
    std::vector<unsigned long long> h_bkt_beg(n_bkt), h_win_beg(n_win);
    for (uint32_t k = 0; k < n_bkt; ++k) h_bkt_beg[k] = mbeg(bm[k]);
    for (uint32_t w = 0; w < n_win; ++w) h_win_beg[w] = wins[w].G;
    out->ms_layout_host = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - h0).count();
    std::vector<uint32_t> win_lo(n_win, ~0u), win_hi(n_win, 0);
    if (n) {
        unsigned long long *d_bkt = nullptr, *d_win = nullptr; uint32_t *d_lo = nullptr, *d_hi = nullptr;
        if (carve(ctx->b_st_lay, [&](Carver& c) { d_bkt = c.take<unsigned long long>(n_bkt + 1); d_win = c.take<unsigned long long>(n_win + 1); d_lo = c.take<uint32_t>(n_win + 1); d_hi = c.take<uint32_t>(n_win + 1); }))
            return fail(ctx, "snfb_sort_bam: out of device memory (bucket tables)");
        t_layout.begin(st);
        mark(ctx, "sort_place", 8 * n);
        CUDA_TRY(cudaMemcpyAsync(dsort, h_dsort.data(), 8 * n, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_bkt, h_bkt_beg.data(), 8ull * n_bkt, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_win, h_win_beg.data(), 8ull * n_win, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemsetAsync(d_lo, 0xff, 4ull * n_win, st));
        CUDA_TRY(cudaMemsetAsync(d_hi, 0, 4ull * n_win, st));
        launch(ctx->launches, bamsort::k_place, grid_for(n, 256), 256, 0, st, ord, (const unsigned long long*)dsort, (unsigned long long)n, (const unsigned long long*)src,
               (const uint32_t*)len, (const unsigned long long*)d_bkt, n_bkt, (const unsigned long long*)d_win, n_win, dest, d_lo, d_hi);
        CUDA_TRY(cudaMemcpyAsync(win_lo.data(), d_lo, 4ull * n_win, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(win_hi.data(), d_hi, 4ull * n_win, cudaMemcpyDeviceToHost, st));
        t_layout.end(st);
    }
    mark(ctx, nullptr);

    // ---- per bucket: the windows holding its records read again, their records scattered into the bucket, its members compressed
    FILE* fi = fopen(in->path, "rb");
    if (!fi) return fail(ctx, std::string("cannot open ") + in->path);
    struct Closer { FILE* f; ~Closer() { if (f) fclose(f); } } cin{ fi };
    FILE* fo = fopen(in->out_path, "wb");
    if (!fo) return fail(ctx, std::string("cannot create ") + in->out_path);
    Closer cout_{ fo };
    std::vector<uint8_t> hz, hout;
    uint64_t reads = n_windows, bytes_out = 0;
    for (uint32_t k = 0; k < n_bkt; ++k) {
        const uint64_t O0 = mbeg(bm[k]), O1 = mend[bm[k + 1] - 1];
        if (ctx->b_st_bkt.ensure(O1 - O0 + 64)) return fail(ctx, "snfb_sort_bam: out of device memory (a bucket of " + std::to_string(O1 - O0) + " bytes)");
        uint8_t* B = ctx->b_st_bkt.as<uint8_t>();
        if (O0 < H) CUDA_TRY(cudaMemcpyAsync(B, in->header, std::min(H, O1) - O0, cudaMemcpyHostToDevice, st));
        for (uint32_t w = 0; w < n_win; ++w) {
            if (win_lo[w] > k || win_hi[w] < k) continue;
            const SWin& W = wins[w];
            const uint64_t nz = W.coff_end - W.coff_beg;
            hz.resize(nz);
            if (fseeko(fi, (off_t)W.coff_beg, SEEK_SET) != 0 || fread(hz.data(), 1, nz, fi) != nz)
                return fail(ctx, "cannot read the input again at file offset " + std::to_string(W.coff_beg) + ": the file changed while it was sorted");
            BgzfMembers M;
            if (walk_bgzf(ctx, hz.data(), nz, M)) return 1;
            const uint64_t raw_len = M.raw_len;
            if (raw_len != W.raw_len) return fail(ctx, "the input changed while it was sorted (window at file offset " + std::to_string(W.coff_beg) + ")");
            if (inflate_members(ctx, hz.data(), M, 0, InflateCall{ &t_scatter, "sort_scatter", raw_len, nullptr, "snfb_sort_bam: out of device memory for the window",
                                                                   "snfb_sort_bam: out of device memory (ingest tables)" })) return 1;
            if (W.o1 > W.o0)
                launch(ctx->launches, bamsort::k_scatter, grid_for((W.o1 - W.o0) * 32, 256), 256, 0, st, (const uint8_t*)ctx->b_raw.p, (unsigned long long)W.G, (unsigned long long)raw_len,
                       (uint32_t)W.o0, (uint32_t)W.o1, (const unsigned long long*)src, (const uint32_t*)len, (const unsigned long long*)dest, (unsigned long long)O0, (unsigned long long)O1, B);
            ingest::IngestCounters hc;
            CUDA_TRY(cudaMemcpyAsync(&hc, M.d_ctr, sizeof(hc), cudaMemcpyDeviceToHost, st));
            t_scatter.end(st);
            mark(ctx, nullptr);
            if (hc.bad_blocks) return inflate_failed_in_file(ctx, hc, M, W.coff_beg);
            ++reads; bytes_in += nz;
        }
        // the bucket's members, at most 65535 per launch
        for (uint32_t m = bm[k]; m < bm[k + 1];) {
            const uint32_t m2 = std::min<uint32_t>(bm[k + 1], m + 65535u);
            std::vector<unsigned long long> moff(m2 - m + 1);
            for (uint32_t j = m; j <= m2; ++j) moff[j - m] = mbeg(j) - mbeg(m);
            unsigned long long n_z = 0; std::vector<uint32_t> offs;
            t_deflate.begin(st);
            mark(ctx, "sort_deflate", moff.back());
            if (deflate_members(ctx, B + (mbeg(m) - O0), moff, &n_z, offs)) return 1;
            CUDA_TRY(cudaStreamSynchronize(st));
            hout.resize(n_z);
            CUDA_TRY(cudaMemcpyAsync(hout.data(), ctx->b_zout.p, n_z, cudaMemcpyDeviceToHost, st));
            t_deflate.end(st);
            mark(ctx, nullptr);
            if (fwrite(hout.data(), 1, n_z, fo) != n_z) return fail(ctx, std::string("cannot write ") + in->out_path);
            bytes_out += n_z;
            m = m2;
        }
    }
    static const uint8_t eof_member[28] = { 0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 0x42, 0x43, 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0 };
    if (fwrite(eof_member, 1, 28, fo) != 28 || fflush(fo) != 0) return fail(ctx, std::string("cannot write ") + in->out_path);
    bytes_out += 28;
    cout_.f = nullptr;
    if (fclose(fo) != 0) return fail(ctx, std::string("cannot write ") + in->out_path);
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    out->n_records = n; out->n_windows = n_windows; out->n_buckets = n_bkt; out->n_members = nm; out->n_input_reads = reads;
    out->bytes_in = bytes_in; out->bytes_out = bytes_out;
    out->device_bytes = ctx->b_comp.cap + ctx->b_raw.cap + ctx->b_ing.cap + ctx->b_ix_mask.cap + ctx->b_ix_node.cap + ctx->b_ix_carry.cap + ctx->b_st_rec.cap + ctx->b_st_win.cap
                        + ctx->b_st_lay.cap + ctx->b_st_bkt.cap + ctx->b_zslot.cap + ctx->b_zout.cap + ctx->b_zwork.cap;
    out->ms_keys = t_keys.ms; out->ms_sort = t_sort.ms; out->ms_layout = t_layout.ms; out->ms_scatter = t_scatter.ms; out->ms_deflate = t_deflate.ms;
    return 0;
}
