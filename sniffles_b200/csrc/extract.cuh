// extract.cuh — stage A: alignment records -> SV leads.
//
// One warp per alignment record streams the record's CIGAR16 words with 16-byte loads (256 words
// per warp step, coalesced); SV signatures become 64-byte leads in a second, event-driven pass.
// Reference behaviour reproduced (paths relative to /root/reference/src/sniffles/):
//   LeadProvider.iter_region filters / NM / coverage bookkeeping     leadprov.py:474-581
//   get_cigar_indels                                                  leadprov.py:198-224
//   read_iterindels                                                   leadprov.py:583-670
//   Lead.for_bnd + CIGAR_analyze                                      leadprov.py:57-176
//   read_itersplits + sv.classify_splits                              leadprov.py:227-355, sv.py:649-782
//   build_leadtab region filter                                       leadprov.py:464-468
#pragma once
#include "common.cuh"
#include "cigar16.h"

namespace extract {

constexpr int MAXSEG = 40;     // primary + supplementary segments per read held in shared memory

// rec_flags bits
constexpr uint8_t RF_PASS = 1, RF_HAS_NM = 2;   // bits 2..3: hp
constexpr uint8_t RF_NM_MEAN = 16;              // the read's nm enters config.average_regional_nm: it has one and belongs to its task's last region

// the fetch window a record was read for: its region with a region table (snfb_set_regions, leadprov.py:445-470), else its task's
__device__ __forceinline__ int2 rec_window(const snfb_region* region, const snfb_task* task, const snfb_rec* rec, uint32_t i, int t) {
    if (region) { const snfb_region g = region[__ldg(&rec[i].region)]; return make_int2(g.start, g.end); }
    return make_int2(task[t].start, task[t].end);
}

struct Seg {
    int contig, ref_start, ref_end, qry_start, qry_end;
    int meta;                 // bit0 rev, bits 8..15 mapq, bits 16..17 source, bit 20 has_seq
    int nhint;
    int h_type[2], h_start[2], h_len[2], h_none[2];
    int seq_off, seq_len;
};

__device__ __forceinline__ bool op_adds_read(int op) { return (0x193u >> op) & 1u; }   // M I S = X  (0,1,4,7,8)
__device__ __forceinline__ bool op_adds_ref(int op) { return (0x18Du >> op) & 1u; }    // M D N = X  (0,2,3,7,8)
__device__ __forceinline__ bool op_is_event(int op) { return (0x016u >> op) & 1u; }    // I D S      (1,2,4)

__device__ __forceinline__ void store_lead(snfb_lead* dst, const snfb_lead& l) {
    store16(dst, l);
}

// ---- text helpers (lane-serial; SA tags are short in the compact form aligners write) ----
__device__ inline bool parse_int_dev(const uint8_t* s, int n, long long* out) {
    if (n <= 0) return false; long long v = 0; int i = 0; bool neg = false;
    if (s[0] == '-' || s[0] == '+') { neg = s[0] == '-'; i = 1; if (n == 1) return false; }
    for (; i < n; ++i) { int c = s[i]; if (c < '0' || c > '9') return false; v = v * 10 + (c - '0'); if (v > (1LL << 40)) return false; }
    *out = neg ? -v : v; return true;
}
// leadprov.CIGAR_analyze
__device__ inline bool cigar_analyze_dev(const uint8_t* c, int n, long long* clip_start, long long* clip_end, long long* refspan, long long* readspan) {
    long long rs = 0, qs = 0, clip = 0, cstart = -1, val = 0; bool have = false;
    for (int i = 0; i < n; ++i) {
        int ch = c[i];
        if (ch >= '0' && ch <= '9') { val = val * 10 + (ch - '0'); have = true; if (val > (1LL << 40)) return false; continue; }
        if (!have) return false;
        bool h = false;
        if (ch == 'M' || ch == 'I' || ch == 'X' || ch == '=') { qs += val; h = true; }
        if (ch == 'M' || ch == 'D' || ch == 'X' || ch == '=' || ch == 'N') { rs += val; h = true; }
        if (!h) { if (ch == 'S' || ch == 'H') { if (cstart < 0 && qs + rs > 0) cstart = clip; clip += val; } else return false; }
        val = 0; have = false;
    }
    if (cstart < 0) cstart = clip;
    *clip_start = cstart; *clip_end = clip - cstart; *refspan = rs; *readspan = qs; return true;
}
struct SaEntry { int off[6]; int len[6]; };
__device__ inline bool sa_fields_dev(const uint8_t* s, int n, SaEntry* e) {
    int k = 0, st = 0;
    for (int i = 0; i <= n; ++i) if (i == n || s[i] == ',') { if (k == 6) return false; e->off[k] = st; e->len[k] = i - st; ++k; st = i + 1; }
    return k == 6;
}
__device__ inline int contig_lookup_dev(const snfb_contig* ct, uint32_t nct, const uint8_t* s, int n) {
    uint64_t h = fnv1a64(s, n);
    for (uint32_t i = 0; i < nct; ++i) if (ct[i].name_hash == h) return (int)i;
    return -1;
}
__device__ __forceinline__ void py_slice(long long L, long long a, long long b, int* off, int* len) {
    if (a > L) a = L; if (b > L) b = L; *off = (int)a; *len = b > a ? (int)(b - a) : 0;
}

// sv.classify_splits on the warp's shared segment list (lane-serial); returns the new count
__device__ inline int classify_splits_dev(const snfb_config& cfg, Seg* s, int n, int l_seq) {
    for (int pass = 0; pass < 2; ++pass) {
        for (int i = 1; i < n; ++i) { Seg x = s[i]; int j = i - 1; while (j >= 0 && s[j].qry_start > x.qry_start) { s[j + 1] = s[j]; --j; } s[j + 1] = x; }
        for (int i = 0; i < n; ++i) s[i].nhint = 0;
        int hints = 0; const int ms = cfg.minsvlen_screen;
        if ((double)s[0].qry_start >= (double)cfg.long_ins_length * 0.5) { s[0].h_type[0] = SNFB_INS; s[0].h_start[0] = s[0].ref_start; s[0].h_len[0] = 0; s[0].h_none[0] = 1; s[0].nhint = 1; }
        for (int i = 1; i < n; ++i) {
            Seg* cu = &s[i]; const Seg* la = &s[i - 1];
            if (cu->contig != la->contig) continue;
            const bool rev = cu->meta & 1, fwd = !rev; int ty = -1; long long st = 0, ln = 0;
            if ((cu->meta & 1) == (la->meta & 1)) {
                long long dq = (long long)cu->qry_start - la->qry_end;
                if (fwd && dq >= ms && dq - ((long long)cu->ref_start - la->ref_end) >= ms) {
                    ty = SNFB_INS; st = cu->ref_start; ln = dq;
                    if (ln <= cfg.dev_seq_cache_maxlen) { cu->meta |= 1 << 20; py_slice(l_seq, la->qry_end, cu->qry_start, &cu->seq_off, &cu->seq_len); } else cu->meta &= ~(1 << 20);
                } else if (rev && dq >= ms && dq - ((long long)la->ref_start - cu->ref_end) >= ms) {
                    ty = SNFB_INS; st = la->ref_start; ln = dq;
                    if (ln <= cfg.dev_seq_cache_maxlen) { cu->meta |= 1 << 20; py_slice(l_seq, la->qry_end, cu->qry_start, &cu->seq_off, &cu->seq_len); } else cu->meta &= ~(1 << 20);
                } else if (fwd && ((long long)cu->ref_start - la->ref_end) >= ms && ((long long)cu->ref_start - la->ref_end) - dq >= ms) {
                    ty = SNFB_DEL; st = cu->ref_start; ln = -((long long)cu->ref_start - la->ref_end);
                } else if (rev && ((long long)la->ref_start - cu->ref_end) >= ms && ((long long)la->ref_start - cu->ref_end) - dq >= ms) {
                    ty = SNFB_DEL; st = la->ref_start; ln = -((long long)la->ref_start - cu->ref_end);
                } else if (fwd && cu->ref_start <= la->ref_end) {
                    st = cu->ref_start; ln = (long long)la->ref_end - cu->ref_start; if (ln >= ms) ty = SNFB_DUP;
                } else if (rev && la->ref_start <= cu->ref_end) {
                    st = la->ref_start; ln = (long long)cu->ref_end - la->ref_start; if (ln >= ms) ty = SNFB_DUP;
                }
            } else {
                if (fwd && cu->ref_start <= la->ref_start) { st = cu->ref_start; ln = (long long)la->ref_start - cu->ref_start; if (ln >= ms) ty = SNFB_INV; }
                else if (fwd && cu->ref_start > la->ref_start) { st = la->ref_start; ln = (long long)cu->ref_start - la->ref_start; if (ln >= ms) ty = SNFB_INV; }
                else if (rev && cu->ref_end >= la->ref_end) { st = la->ref_end; ln = (long long)cu->ref_end - la->ref_end; if (ln >= ms) ty = SNFB_INV; }
                else if (rev && cu->ref_end < la->ref_end) { st = cu->ref_end; ln = (long long)la->ref_end - cu->ref_end; if (ln >= ms) ty = SNFB_INV; }
            }
            if (ty >= 0) { int k = cu->nhint++; cu->h_type[k] = ty; cu->h_start[k] = (int)st; cu->h_len[k] = (int)ln; cu->h_none[k] = 0; ++hints; }
        }
        if (!hints && n > 2) {
            int m = 0; const int c0 = s[0].contig, r0 = s[0].meta & 1;
            for (int i = 0; i < n; ++i) if (s[i].contig == c0 && (s[i].meta & 1) == r0) { Seg t = s[i]; s[m++] = t; }
            if (m == 2) { s[0].meta &= ~(1 << 20); s[1].meta &= ~(1 << 20); n = 2; continue; }   // one recursion level (sv.py:779-780)
            return m;
        }
        return n;
    }
    return n;
}

// ---- lead slot allocation.  A single global counter bumped once per lead serialises in L2; instead every thread reserves
//      SLOT_CHUNK slots at a time and hands them out locally.  Unused slots of a retired chunk are marked as holes
//      (rec == HOLE) and skipped later; canonical (record, k) order never depended on slot numbers.
constexpr unsigned SLOT_CHUNK = 8;          // per allocating thread: at most SLOT_CHUNK - 1 holes each
constexpr uint32_t HOLE = 0xffffffffu;
struct SlotState { unsigned long long cur, end; };
__device__ __forceinline__ unsigned long long alloc_slot_lane(SlotState& st, snfb_lead* leads, unsigned long long lead_cap, unsigned long long* n_slots) {   // one lane only
    if (st.cur + 1 > st.end) { const unsigned long long base = atomicAdd(n_slots, (unsigned long long)SLOT_CHUNK); st.cur = base; st.end = base + SLOT_CHUNK; }
    return st.cur++;
}

// ---- supplementary alignments (SA tag) of one record: Lead.for_bnd + read_itersplits, run by lane 0 ----
struct SaArgs {
    uint32_t rec; int qas, qae, alen, ref_end, hp; uint32_t base_flags; uint64_t qh; unsigned nlead; bool rev, is_supp;
    // the pieces of Params / snfb_rec / snfb_task the SA path needs, by value (keeps the caller's structs out of local memory)
    const uint8_t* sa; int sa_len; int clip_left, clip_right; int pos, l_seq, mapq, aux_flags, task;
    int tk_contig, tk_start, tk_end;
    const snfb_contig* contig; uint32_t n_contig; snfb_lead* leads; unsigned long long lead_cap; unsigned long long* n_slots; SlotState* slots;
    int mapq_min, dev_keep_lowqual_splits, max_splits_base; double max_splits_kb;
};
__device__ __noinline__ unsigned process_sa(const snfb_config* __restrict__ cfgp, Seg* sg, const SaArgs a, unsigned long long* soft_p, unsigned long long* overflow_p) {
    const snfb_config& cfg = *cfgp;
    const uint32_t rec = a.rec; const bool rev = a.rev;
    unsigned long long soft = 0, overflow = 0; unsigned added = 0;
    const uint8_t* sa = a.sa; const int sl = a.sa_len;
    struct { int pos, l_seq, mapq, aux_flags, task; } r = { a.pos, a.l_seq, a.mapq, a.aux_flags, a.task };
    struct { int contig, start, end; } tk = { a.tk_contig, a.tk_start, a.tk_end };
    struct { const snfb_contig* contig; uint32_t n_contig; snfb_lead* leads; unsigned long long lead_cap; } P = { a.contig, a.n_contig, a.leads, a.lead_cap };
    // pass 1: count the non-empty entries and locate the first one
    int ne = 0, f_off = 0, f_len = 0;
    for (int i = 0, st = 0; i <= sl; ++i) if (i == sl || sa[i] == ';') { if (i > st) { if (ne == 0) { f_off = st; f_len = i - st; } ++ne; } st = i + 1; }
    bool sa_ok = true; SaEntry e0;
    if (ne > 0 && !sa_fields_dev(sa + f_off, f_len, &e0)) { sa_ok = false; ++soft; }
    if (ne > 0 && sa_ok) {                                   // Lead.for_bnd: first entry only
        const uint8_t* e = sa + f_off;
        const int left = a.clip_left, right = a.clip_right;
        int bstart; bool is_first;
        if (left > right) { bstart = r.pos + 1; is_first = false; } else { bstart = a.ref_end; is_first = true; }
        const bool same = e0.len[2] == 1 && ((e[e0.off[2]] == '-' && rev) || (e[e0.off[2]] == '+' && !rev));
        if (!same) {
            long long p1, cs, ce, rs, qs, sanm = 0;
            if (!parse_int_dev(e + e0.off[1], e0.len[1], &p1)) ++soft;
            else if (!cigar_analyze_dev(e + e0.off[3], e0.len[3], &cs, &ce, &rs, &qs)) ++soft;
            else if ((r.aux_flags & SNFB_AUX_NM) && !parse_int_dev(e + e0.off[5], e0.len[5], &sanm)) ++soft;
            else {
                const long long p0 = p1 - 1; const bool is_reverse = ce > cs;
                const long long mate = is_reverse ? p0 + rs : (is_first ? p0 + 1 : p0 + 2);
                if (bstart >= tk.start && bstart < tk.end) {
                    snfb_lead L;
                    L.rec = rec; L.qname_hash = a.qh; L.read_len = 0; L.seq_off = -1; L.seq_len = 0;
                    L.ref_start = L.ref_end = bstart; L.qry_start = a.qas; L.qry_end = a.qae; L.svlen = 0;
                    L.mate_pos = (int)mate; L.mate_contig = contig_lookup_dev(P.contig, P.n_contig, e + e0.off[0], e0.len[0]);
                    if (L.mate_contig < 0) ++soft;
                    L.nm_sa = (int)sanm; L.task = (uint16_t)r.task; L.k = (uint16_t)(a.nlead + added);
                    L.flags = a.base_flags | SNFB_BND | ((uint32_t)SNFB_SRC_BND_SA << 3) | (is_first ? SNFB_LF_BND_FIRST : 0u) | (is_reverse ? SNFB_LF_BND_REVERSE : 0u)
                              | ((r.aux_flags & SNFB_AUX_NM) ? 0u : SNFB_LF_NM_NONE);
                    const unsigned long long slot = alloc_slot_lane(*a.slots, P.leads, P.lead_cap, a.n_slots);
                    if (slot < P.lead_cap) store_lead(P.leads + slot, L); else ++overflow;
                    ++added;
                }
            }
        }
    }
    // read_itersplits: primary alignments only
    if (!a.is_supp && sa_ok && ne > 0) {
        const double lim = __dadd_rn((double)cfg.max_splits_base, __dmul_rn(cfg.max_splits_kb, __ddiv_rn((double)r.l_seq, 1000.0)));
        if (!((double)ne > lim)) {
            if (ne + 1 > MAXSEG) ++soft;
            else {
                bool ok = true;
                sg[0].contig = tk.contig; sg[0].ref_start = r.pos; sg[0].ref_end = a.ref_end;
                sg[0].qry_start = rev ? r.l_seq - a.qae : a.qas; sg[0].qry_end = sg[0].qry_start + a.alen;
                sg[0].meta = (rev ? 1 : 0) | ((int)r.mapq << 8) | (SNFB_SRC_SPLIT_PRIM << 16); sg[0].nhint = 0;
                int ei = 0;
                for (int i = 0, st = 0; i <= sl && ok; ++i) if (i == sl || sa[i] == ';') {
                    if (i > st) {
                        SaEntry en; const uint8_t* e = sa + st; long long p1, cs, ce, rs, qs, mq;
                        if (!sa_fields_dev(e, i - st, &en) || !parse_int_dev(e + en.off[4], en.len[4], &mq)) { ok = false; ++soft; break; }
                        const bool srev = en.len[2] == 1 && e[en.off[2]] == '-';
                        if (!cigar_analyze_dev(e + en.off[3], en.len[3], &cs, &ce, &rs, &qs)) { ok = false; ++soft; break; }
                        if (!parse_int_dev(e + en.off[1], en.len[1], &p1)) { ok = false; ++soft; break; }
                        Seg* g = &sg[++ei];
                        g->contig = contig_lookup_dev(P.contig, P.n_contig, e + en.off[0], en.len[0]); if (g->contig < 0) { g->contig = -2 - ei; ++soft; }
                        g->ref_start = (int)(p1 - 1); g->ref_end = (int)(p1 - 1 + rs); g->qry_start = (int)(srev ? ce : cs); g->qry_end = g->qry_start + (int)qs;
                        g->meta = (srev ? 1 : 0) | ((int)mq << 8) | (SNFB_SRC_SPLIT_SUP << 16); g->nhint = 0;
                    }
                    st = i + 1;
                }
                if (ok) {
                    const int m = classify_splits_dev(cfg, sg, ne + 1, r.l_seq);
                    for (int i = 0; i < m; ++i) for (int h = 0; h < sg[i].nhint; ++h) {
                        const int mqc = (sg[i].meta >> 8) & 255, mqp = (sg[i > 0 ? i - 1 : 0].meta >> 8) & 255;
                        if (!cfg.dev_keep_lowqual_splits && (mqc < mqp ? mqc : mqp) < cfg.mapq) continue;
                        const int ty = sg[i].h_type[h]; const int hs = sg[i].h_start[h];
                        if (sg[i].contig != tk.contig || hs < tk.start || hs >= tk.end) continue;
                        snfb_lead L;
                        L.rec = rec; L.qname_hash = a.qh; L.read_len = 0; L.seq_off = -1; L.seq_len = 0; L.mate_contig = -1; L.mate_pos = 0; L.nm_sa = 0;
                        L.ref_start = hs; L.ref_end = (!sg[i].h_none[h] && ty != SNFB_INS) ? hs + sg[i].h_len[h] : hs;
                        L.qry_start = sg[i].qry_start; L.qry_end = sg[i].qry_end; L.svlen = sg[i].h_len[h];
                        uint32_t f = (uint32_t)ty | ((uint32_t)((sg[i].meta >> 16) & 3) << 3) | ((sg[i].meta & 1) ? SNFB_LF_REVERSE : 0u) | ((uint32_t)mqc << 16) | ((uint32_t)a.hp << 24);
                        if (sg[i].h_none[h]) f |= SNFB_LF_SVLEN_NONE;
                        if (ty == SNFB_INS && (sg[i].meta & (1 << 20))) { f |= SNFB_LF_HAS_SEQ; L.seq_off = sg[i].seq_off; L.seq_len = sg[i].seq_len; }
                        L.flags = f; L.task = (uint16_t)r.task; L.k = (uint16_t)(a.nlead + added);
                        const unsigned long long slot = alloc_slot_lane(*a.slots, P.leads, P.lead_cap, a.n_slots);
                        if (slot < P.lead_cap) store_lead(P.leads + slot, L); else ++overflow;
                        ++added;
                    }
                }
            }
        }
    }
    *soft_p += soft; *overflow_p += overflow;
    return added;
}

// ================================================================================================
// Stage A kernels:
//   k_rec_index (thread per record): the record's offset checks, task boundaries, sortedness, and everything that only needs the record core and the
//           clip ops at the two ends of its CIGAR: query_alignment_start/end, the read filters of iter_region, the
//           16-byte scan descriptor and the clip facts k_emit / k_sa use, the SA work list.
//   k_cigar_walk (hot, HBM-bound): the CIGAR walk, see "stage A streaming: the CIGAR walk" below: reference end, the NM correction,
//           lead counts, and one 32-byte Event per SV signature.  No lead is built here.
//   k_rec_post (thread per record): nm per read (the division), per-task read count / covered bases / longest span.
//   k_emit  one thread per Event: the 64-byte lead.
//   k_sa    one thread per record with an SA tag: Lead.for_bnd + read_itersplits.
// ================================================================================================

// the op at word h of the eight 16-bit words one lane holds (cls 0 / len 0 where a pad, P or extension word sits).  Groups never
// straddle a 16-byte boundary, so this is lane-local.
__device__ __forceinline__ void c16_op(const uint32_t (&ww)[4], int h, unsigned& cls, unsigned& len) {
    unsigned x[3];
    #pragma unroll
    for (int e = 0; e < 3; ++e) x[e] = h + e < 8 ? (ww[(h + e) >> 1] >> (16 * ((h + e) & 1))) & 0xffffu : 0u;
    unsigned c = 0, l = 0;
    if (!(x[0] & C16_EXT)) {
        c = c16_word_class(x[0]); l = x[0] & C16_LEN_MASK;
        if (x[1] & C16_EXT) {
            l += c16_ext_add(x[1]);
            if (x[2] & C16_EXT) l += c16_ext_add(x[2]);
        }
    }
    cls = c; len = l;
}
// all eight ops at their word positions
__device__ __forceinline__ void c16_decode8(const uint32_t (&ww)[4], unsigned (&cls)[8], unsigned (&len)[8]) {
    #pragma unroll
    for (int h = 0; h < 8; ++h) c16_op(ww, h, cls[h], len[h]);
}

struct RecScan { uint32_t cig8; uint32_t n_words; int32_t pos; uint32_t meta; };    // what the CIGAR walk needs of a record, one 16-byte load
constexpr int CH = 16;                                                              // 16-byte groups per chunk of the streaming pass (k_cigar_walk)
__host__ __device__ __forceinline__ uint32_t chunks_of(uint32_t n_words) { return (((n_words + 7u) >> 3) + (uint32_t)CH - 1u) / (uint32_t)CH; }
struct RecClip { int32_t alen, qas, clip_left, clip_right; };                        // query_alignment_length/start, first / last op if it is a clip
constexpr uint32_t RM_PASS = 1u << 24, RM_HAS_NM = 1u << 25, RM_HAS_SA = 1u << 26;   // RecScan.meta: task (0..15) | mapq (16..23) | flags | hp (27..28)

struct IndexParams {
    const snfb_rec* rec; const uint16_t* cigar; const snfb_task* task; uint32_t n_rec; uint32_t n_task; unsigned long long n_cigar, n_var, n_seq;
    int check_seq;                                    // the seq arena is resident: seq offsets are checked too
    int32_t* rec_pos; uint32_t* task_first; uint32_t* task_last;
    RecScan* scan; RecClip* clip; int32_t* rec_end; uint8_t* rec_flags; double* rec_nm; uint32_t* rec_nlead;
    uint32_t* sa_list; unsigned long long* n_sa;     // passing records with an SA tag (k_sa's work list)
    DevCounters* ctr; int mapq_min, alen_min, excl, want_nm;
    const snfb_region* region; const int32_t* last_region; uint32_t n_region;      // region table (null: none) and each task's last region
};

// the clip ops at the two ends of a CIGAR16 record of n words, word(k) = word k: query_alignment_start / end (qas, qae, starting from
// 0 and l_seq) and the first / last op's length when it is a clip.  Pad words (0) are skipped; an op's extension words follow its base word.
template <class Word>
__device__ __forceinline__ void clip_walk(uint32_t n, Word&& word, int& qas, int& qae, int& clip_left, int& clip_right) {
    uint32_t fe = 0;
    { bool first = true; uint32_t k = 0;
      while (k < n) {
          const unsigned w = word(k); if (w == 0) { ++k; continue; }
          unsigned len = w & C16_LEN_MASK; const unsigned cls = c16_word_class(w); uint32_t k2 = k + 1;
          while (k2 < n) { const unsigned e = word(k2); if (!(e & C16_EXT)) break; len += c16_ext_add(e); ++k2; }
          if (first) { if (cls == C16_S || cls == C16_H) clip_left = (int)len; first = false; fe = k2; }
          if (cls == C16_S) qas += (int)len; else if (cls != C16_H) break;
          k = k2;
      } }
    { bool last = true; long k = (long)n - 1;
      while (k >= (long)fe) {
          long b = k; while (b > (long)fe && (word((uint32_t)b) & C16_EXT)) --b;
          const unsigned w = word((uint32_t)b); if (w == 0) { k = b - 1; continue; }
          unsigned len = w & C16_LEN_MASK; const unsigned cls = c16_word_class(w);
          for (long e2 = b + 1; e2 <= k; ++e2) len += c16_ext_add(word((uint32_t)e2));
          if (last) { if (cls == C16_S || cls == C16_H) clip_right = (int)len; last = false; }
          if (cls == C16_S) qae -= (int)len; else if (cls != C16_H) break;
          k = b - 1;
      }
      if (last) clip_right = clip_left; }            // a single op is both the first and the last one
}
// word k of a record when it lies in its first group (f: words 0..7) or its last group (l: words l0..l0+7).  Otherwise `miss` is set and
// the word is a zero-length M, which ends either walk at once.  An op never straddles a group, so the clip walk stays inside these two
// groups unless the clips at an end take more than one group.
__device__ __forceinline__ unsigned end_word(const uint4& f, const uint4& l, uint32_t l0, uint32_t k, bool& miss) {
    const bool in_f = k < 8u, in_l = k >= l0;
    if (!in_f && !in_l) miss = true;
    const uint4 v = in_f ? f : l; const uint32_t h = (k & 7u) >> 1;
    const uint32_t x = h < 2u ? (h ? v.y : v.x) : (h == 2u ? v.z : v.w);
    return (in_f || in_l) ? (x >> (16u * (k & 1u))) & 0xffffu : C16_M << C16_CLASS_SHIFT;
}

// leadprov.py:488-516 (filters), pysam query_alignment_start / query_alignment_end; returns whether record i goes on the SA list.
// Also checks that every offset of the record stays inside its arena or table; a record that does not is counted in bad_records (the run fails).
__device__ __forceinline__ bool index_record(const IndexParams& P, uint32_t i) {
    const uint4* core = reinterpret_cast<const uint4*>(P.rec + i);
    const uint4 c0 = __ldg(core), c1 = __ldg(core + 1), c2 = __ldg(core + 2), c3 = __ldg(core + 3);
    const int task = (int)c0.x, pos = (int)c0.y; const unsigned flag = c0.z & 0xffffu, mapq = (c0.z >> 16) & 255u, aux = c0.z >> 24; unsigned hp = c0.w & 255u;
    const uint32_t l_qname = (c0.w >> 8) & 255u;
    const int nm = (int)c1.x; const uint32_t n = c1.z; const int l_seq = (int)c1.w; const uint32_t sa_len = c2.x;
    const unsigned long long cigar_off = (unsigned long long)c2.z | ((unsigned long long)c2.w << 32);
    const unsigned long long seq_off = (unsigned long long)c3.x | ((unsigned long long)c3.y << 32), var_off = (unsigned long long)c3.z | ((unsigned long long)c3.w << 32);
    const uint32_t rg = c2.y;
    const bool bad_core = (uint32_t)task >= P.n_task || (cigar_off & 7) || cigar_off + n > P.n_cigar || (P.region && (rg >= P.n_region || P.region[rg].task != task));
    const bool bad = bad_core || var_off + l_qname + sa_len > P.n_var || l_seq < 0
                     || (P.check_seq && seq_off + (unsigned long long)((l_seq + 1) / 2) > P.n_seq);
    if (bad) atomicAdd(&P.ctr->bad_records, 1ULL);
    if (bad_core) {                                  // touch nothing through its offsets
        RecScan s; s.cig8 = 0; s.n_words = 0; s.pos = pos; s.meta = 0; store16(P.scan + i, s);
        RecClip c; c.alen = 0; c.qas = 0; c.clip_left = 0; c.clip_right = 0; store16(P.clip + i, c);
        P.rec_pos[i] = pos; P.rec_flags[i] = 0; P.rec_nm[i] = -1.0; P.rec_end[i] = -1; P.rec_nlead[i] = 0; return false;
    }
    P.rec_pos[i] = pos;
    if (i == 0) P.task_first[task] = 0;
    else {
        const int2 pv = __ldg(reinterpret_cast<const int2*>(P.rec + i - 1));
        if (pv.x != task) { P.task_first[task] = i; if ((uint32_t)pv.x < P.n_task) P.task_last[pv.x] = i; }
        else if (pv.y > pos && (!P.region || __ldg(&P.rec[i - 1].region) == rg)) atomicAdd(&P.ctr->unsorted, 1ULL);     // sorted inside a region segment
    }
    if (i + 1 == P.n_rec) P.task_last[task] = P.n_rec;
    // clips at the two ends: from the first and the last group (two independent loads), word by word only when the clips leave them
    const uint16_t* cg = P.cigar + cigar_off;
    int qas = 0, qae = l_seq, clip_left = 0, clip_right = 0;
    const uint32_t G = (n + 7u) >> 3;
    bool miss = G == 0 || cigar_off + 8ull * G > P.n_cigar;          // the last group would end behind the arena: word by word
    if (!miss) {
        const uint4* g4 = reinterpret_cast<const uint4*>(cg);
        const uint4 f = __ldg(g4), l = __ldg(g4 + (G - 1u)); const uint32_t l0 = 8u * (G - 1u);
        clip_walk(n, [&](uint32_t k) { return end_word(f, l, l0, k, miss); }, qas, qae, clip_left, clip_right);
    }
    if (miss) { qas = 0; qae = l_seq; clip_left = 0; clip_right = 0; clip_walk(n, [&](uint32_t k) { return (unsigned)__ldg(cg + k); }, qas, qae, clip_left, clip_right); }
    const int alen = qae - qas;
    const int2 win = P.region ? make_int2(P.region[rg].start, P.region[rg].end) : make_int2(P.task[task].start, P.task[task].end);
    const bool pass = !((int)mapq < P.mapq_min || (flag & 256u) || alen < P.alen_min) && !(P.excl && (flag & (unsigned)P.excl)) && pos >= win.x && pos < win.y && n > 0;
    const bool has_nm = pass && P.want_nm && (aux & SNFB_AUX_NM);
    if (!(aux & SNFB_AUX_HP)) hp = 0;
    if (pass && hp > 2) { hp = 0; atomicAdd(&P.ctr->soft_errors, 1ULL); }
    RecScan s; s.cig8 = (uint32_t)(cigar_off >> 3); s.n_words = n; s.pos = pos;
    s.meta = ((uint32_t)task & 0xffffu) | (mapq << 16) | (pass ? RM_PASS : 0u) | (has_nm ? RM_HAS_NM : 0u) | ((pass && (aux & SNFB_AUX_SA)) ? RM_HAS_SA : 0u) | ((pass ? hp : 0u) << 27);
    store16(P.scan + i, s);
    RecClip c; c.alen = alen; c.qas = qas; c.clip_left = clip_left; c.clip_right = clip_right;
    store16(P.clip + i, c);
    const bool nm_mean = has_nm && (!P.region || P.last_region[task] == (int)rg);     // nm_sum is reset per region (leadprov.py:475-577)
    P.rec_flags[i] = pass ? (uint8_t)(RF_PASS | (has_nm ? RF_HAS_NM : 0) | (hp << 2) | (nm_mean ? RF_NM_MEAN : 0)) : (uint8_t)0;
    P.rec_nm[i] = has_nm ? (double)nm : -1.0;        // k_rec_post turns it into (nm - big) / (alen + 1)
    P.rec_end[i] = -1; P.rec_nlead[i] = 0;       // k_cigar_walk overwrites both for a passing record
    return pass && (aux & SNFB_AUX_SA);
}
__global__ void __launch_bounds__(256) k_rec_index(const IndexParams P) {
    __shared__ unsigned long long s_base;
    const uint32_t i = blockIdx.x * 256 + threadIdx.x;
    const uint32_t has_sa = i < P.n_rec && index_record(P, i) ? 1u : 0u;
    uint32_t tot; const uint32_t mine = prims::block_excl_scan(has_sa, &tot);     // one slot reservation per block
    if (threadIdx.x == 0) s_base = tot ? atomicAdd(P.n_sa, (unsigned long long)tot) : 0ull;
    __syncthreads();
    if (has_sa) P.sa_list[s_base + mine] = i;
}

// one SV signature found by k_cigar_walk (an I / D / S op of at least minsvlen_screen inside the task's region): all k_emit needs to build its lead
struct Event { uint32_t rec; uint32_t len; uint32_t pos_q; int32_t pos_r; uint32_t k_cls; uint32_t pad[3]; };   // k_cls: ordinal inside its record (16 bits) | class << 16; rec == HOLE: an unused slot

// ---- stage A streaming: the CIGAR walk --------------------------------------------------------------------------------------
// A passing record's CIGAR16 groups (16 bytes = 8 words) are cut into CHUNKS of up to CH groups (256 bytes); a chunk belongs to one
// record.  k_cigar_walk runs one WARP per tile of TILE consecutive records (persistent grid; 32, or 1 for a block too small to give every
// resident warp a 32-record tile: there the few busy warps would decode all flagged chunks one after the other).  A warp scan of the tile's chunk counts places
// every chunk of the tile; the warp then walks the chunks in rounds of 32, one chunk per lane:
//   - the lane sums its chunk's groups sequentially: per 32-bit word (two ops) two masked sums (read / reference advance, both halves
//     at once) and one OR (E / extension flags).  The loads of 8 groups (128 bytes) are issued before the first is used.
//   - a segmented warp scan of the sums (a segment starts at the first chunk of a record; a record that continues from the previous
//     round takes the carry) gives the absolute (query, reference) position at every chunk start.
//   - the round's chunks holding an E-flagged word are decoded together: their groups are laid out over the lanes in chunk order, one
//     group per lane, in passes of 32 groups (a chunk may continue into the next pass).  A shuffle binary search finds each group's
//     chunk; the lane reloads the group (just read: L1 / L2) and a scan segmented at chunk starts, seeded with the chunk's start position
//     (or the previous pass's carry), gives the group's position.  Only lanes whose group holds an E word decode, and only its E words
//     (group_events: the offset of a word is a masked sum of the words below it; a group with an extension word is decoded op by op),
//     apply the region test (leadprov.py:464-466), count signatures and big indels.  One scan of the counts over the pass gives the
//     event slots (one reservation per pass) and, segmented at record starts, each signature's final ordinal inside its record (a record
//     that continues from an earlier pass or round starts from the warp-uniform running count); the lanes then decode again and write
//     one Event per signature.  Each chunk's counts go back to the lane that owns it as the difference of the scans over its groups.
//     An extension word alone needs no decode: every I / D / S long enough to need one carries E, and so does every I / D / S of 11
//     bases or more (evt_need), which covers the big-indel sum.
//   - the lane holding a record's last chunk writes its reference end, lead count and "big indel" sum (get_cigar_indels).
// Event slots: a warp reserves WALK_SLOTS at a time and hands them out in order; what is left when it finishes is retired as holes.
struct WalkParams {
    const RecScan* scan; uint32_t n_rec;
    const uint16_t* cigar; const snfb_task* task;
    const snfb_rec* rec; const snfb_region* region;          // region table (null: none): a lead's window is its record's region
    int32_t* rec_end; uint32_t* rec_nlead; int32_t* rec_big;
    Event* ev; unsigned long long ev_cap; unsigned long long* n_ev;      // n_ev: event slots handed out, holes included
    DevCounters* ctr;
    int minsv;
};
constexpr int WALK_THREADS = 256, WALK_BLOCKS = NUM_SMS * 4;           // 4 blocks of 256 threads per SM are resident at <= 64 registers
constexpr unsigned long long WALK_WIDE_MIN = 32ull * WALK_BLOCKS * (WALK_THREADS / 32);   // records from which 32-record tiles fill the grid
constexpr unsigned WALK_SLOTS = 64;                                     // per warp: at most WALK_SLOTS - 1 holes each

// lowers the E-bit threshold of a CIGAR16 arena in place (a config that cares about shorter events than the block was packed for)
__global__ void k_reflag(uint16_t* __restrict__ cigar, unsigned long long n_words, unsigned evt_min) {
    for (unsigned long long i = blockIdx.x * (unsigned long long)blockDim.x + threadIdx.x; i < n_words; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned w = cigar[i]; if (w & (C16_EXT | C16_E)) continue;
        uint32_t len = w & C16_LEN_MASK;
        if (len < evt_min && (i & 7) != 7 && (cigar[i + 1] & C16_EXT)) len = 1u << C16_LEN_BITS;      // an extension word follows: the op is at least that long
        const unsigned e = c16_e_flag(c16_word_class(w), len, evt_min);
        if (e) cigar[i] = (uint16_t)(w | e);
    }
}

// read / reference advance of a lane's eight words when one of them is an extension word
__device__ __forceinline__ uint2 lane_sums_ext(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    const uint32_t ww[4] = { w0, w1, w2, w3 };
    unsigned cls[8], len[8]; c16_decode8(ww, cls, len);
    unsigned lq = 0, lr = 0;
    #pragma unroll
    for (int j = 0; j < 8; ++j) { lq += len[j] * (cls[j] & 1u); lr += len[j] * ((cls[j] >> 1) & 1u); }
    return make_uint2(lq, lr);
}

// per 32-bit word (two ops): the halves' lengths masked by "advances the read" (class bit 0 = word bit 11) / "advances the reference" (bit 12)
#define SNFB_WORD_BODY(w, aq, ar) { const uint32_t t_ = (w) >> 11; aq += (w) & ((t_ & 0x00010001u) * 0x7ffu); ar += (w) & (((t_ >> 1) & 0x00010001u) * 0x7ffu); }

// read / reference advance of one 16-byte group
__device__ __forceinline__ uint2 group_sums(const uint4 v) {
    if ((v.x | v.y | v.z | v.w) & 0x80008000u) return lane_sums_ext(v.x, v.y, v.z, v.w);       // an extension word: the group is decoded op by op
    uint32_t aq = 0, ar = 0;
    SNFB_WORD_BODY(v.x, aq, ar) SNFB_WORD_BODY(v.y, aq, ar) SNFB_WORD_BODY(v.z, aq, ar) SNFB_WORD_BODY(v.w, aq, ar)
    return make_uint2((aq & 0xffffu) + (aq >> 16), (ar & 0xffffu) + (ar >> 16));
}

// segmented inclusive sum over the warp: lane h (-1: none at or below this lane) starts this lane's segment, `init` is added to it
// (a carry when h < 0).  One plain scan; the prefix in front of the segment head is subtracted (exact in modular arithmetic).
__device__ __forceinline__ uint32_t seg_incl_sum(uint32_t v, int h, uint32_t init) {
    const uint32_t s = prims::warp_incl_scan(v);
    const uint32_t eh = __shfl_sync(FULL, s - v, h < 0 ? 0 : h);          // lane 0's exclusive prefix is 0
    return init + s - eh;
}

// the SV signatures of one 16-byte group that holds an E word, in op order: emit(cls, len, q, r) for every I / D / S of at least minsv
// whose signature lies inside [tk_start, tk_end) (leadprov.py:464-466); (q, r) = the op's read / reference position, the group starts at
// (q0, r0).  Adds the group's I / D ops above 10 bases to `big` (get_cigar_indels).  Every I / D / S of 11 bases or more carries E and
// minsv is at least the block's E threshold (evt_need), so the E words are all it has to look at:
//   - without an extension word, word h is op h: only the E words are visited, the offset of each is the masked sum of the words below it;
//   - with one, the group is decoded op by op (c16_op).
template <class Emit>
__device__ __forceinline__ void group_events(const uint4 v, uint32_t q0, int r0, int minsv, int tk_start, int tk_end, uint32_t& big, Emit&& emit) {
    const uint32_t ww[4] = { v.x, v.y, v.z, v.w };
    if ((v.x | v.y | v.z | v.w) & 0x80008000u) {
        uint32_t q = q0; int r = r0;
        #pragma unroll
        for (int x = 0; x < 8; ++x) {
            unsigned cls, len; c16_op(ww, x, cls, len);
            if (len > 10u && (cls == C16_I || cls == C16_D)) big += len;
            if (c16_is_event(cls) && (int)len >= minsv) {
                const int rsig = cls == C16_D ? r + (int)len : r;
                if (rsig >= tk_start && rsig < tk_end) emit(cls, len, q, r);
            }
            q += len * (cls & 1u); r += (int)(len * ((cls >> 1) & 1u));
        }
        return;
    }
    // E bit (word bit 14) of half h -> bit h
    uint32_t em = ((v.x >> 14) & 1u) | ((v.x >> 29) & 2u) | ((v.y >> 12) & 4u) | ((v.y >> 27) & 8u)
                | ((v.z >> 10) & 16u) | ((v.z >> 25) & 32u) | ((v.w >> 8) & 64u) | ((v.w >> 23) & 128u);
    for (; em; em &= em - 1u) {
        const uint32_t h = (uint32_t)__ffs(em) - 1u;
        const uint32_t w = h < 4u ? (h < 2u ? v.x : v.y) : (h < 6u ? v.z : v.w);
        const uint32_t x = (w >> (16u * (h & 1u))) & 0xffffu;
        const unsigned cls = c16_word_class(x), len = x & C16_LEN_MASK;
        if (len > 10u && (cls == C16_I || cls == C16_D)) big += len;
        if (!(c16_is_event(cls) && (int)len >= minsv)) continue;
        uint32_t aq = 0, ar = 0;                    // the words below h: whole 32-bit words, and the low half of h's own word when h is odd
        #pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t m = 2u * i + 2u <= h ? 0xffffffffu : (2u * i + 1u == h ? 0xffffu : 0u);
            SNFB_WORD_BODY(ww[i] & m, aq, ar)
        }
        const uint32_t q = q0 + (aq & 0xffffu) + (aq >> 16); const int r = r0 + (int)((ar & 0xffffu) + (ar >> 16));
        const int rsig = cls == C16_D ? r + (int)len : r;
        if (rsig >= tk_start && rsig < tk_end) emit(cls, len, q, r);
    }
}

// a read-only 16-byte load whose L2 miss fetches the whole 256-byte block around it: a lane's chunk is up to 256 contiguous bytes, so its first
// load brings the rest of the chunk into L2 at once instead of one 32-byte sector per later load
__device__ __forceinline__ uint4 ldg_l2_256(const uint4* p) {
    uint4 v; asm("ld.global.nc.L2::256B.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p)); return v;
}

template <int TILE>
__global__ void __launch_bounds__(WALK_THREADS, 4) k_cigar_walk(const __grid_constant__ WalkParams P) {
    // per warp, in shared memory to keep them out of the registers of the load loop: the tile's RecScans (cig8, n_words, pos, meta), and the
    // carry into the next round of a record that continues (query / reference position, events, big-indel sum; round 0 starts with a record)
    __shared__ uint4 s_rs[WALK_THREADS], s_carry[WALK_THREADS / 32];
    const uint4* __restrict__ cig4 = reinterpret_cast<const uint4*>(P.cigar);
    const uint32_t lane = lane_id();
    uint4* const rs = s_rs + (threadIdx.x & ~31u); uint4& carry = s_carry[threadIdx.x >> 5];
    const uint32_t warp = (blockIdx.x * WALK_THREADS + threadIdx.x) >> 5, n_warps = gridDim.x * (WALK_THREADS / 32);
    unsigned long long s_cur = 0; uint32_t s_left = 0;       // event slots [s_cur, s_cur + s_left) reserved by this warp and not handed out yet (warp-uniform)
    uint32_t run_rec = HOLE, run_cnt = 0;                    // record of the last decoded flagged chunk, its events so far (warp-uniform)
    uint32_t overflow = 0;
    for (uint32_t t0 = warp * TILE; t0 < P.n_rec; t0 += n_warps * TILE) {   // 64-byte records: n_rec is far below 2^32 - n_warps * 32
        uint4 d = make_uint4(0u, 0u, 0u, 0u);                // lanes >= TILE hold no record
        if (lane < (uint32_t)TILE && t0 + lane < P.n_rec) d = __ldg(reinterpret_cast<const uint4*>(P.scan + t0 + lane));
        __syncwarp();                                        // the previous tile's readers are done
        rs[lane] = d;
        __syncwarp();
        const uint32_t nch = (d.w & RM_PASS) ? chunks_of(d.y) : 0u;
        const uint32_t incl = prims::warp_incl_scan(nch), off = incl - nch, total = __shfl_sync(FULL, incl, 31);
        for (uint32_t c0 = 0; c0 < total; c0 += 32) {
            const uint32_t c = c0 + lane;
            int j = 0;                                       // the lane's record: the last one whose first chunk is <= c
            #pragma unroll
            for (int s = 16; s; s >>= 1) { const uint32_t o = __shfl_sync(FULL, off, j + s); if (o <= c) j += s; }
            const uint32_t k = c - __shfl_sync(FULL, off, j), G = (rs[j].y + 7u) >> 3;
            const bool valid = c < total, head = valid && k == 0, last = valid && (k + 1u) * CH >= G;
            const int ng = valid ? (int)min((uint32_t)CH, G - k * CH) : 0;
            const uint32_t g0 = rs[j].x + k * CH;
            // the chunk's read / reference advance and flags.  The packed half-word sums hold 32 values of at most 2047 before they could
            // carry into the neighbouring half: they are folded every 8 groups; groups behind the end of a short chunk read as pad words.
            uint32_t vq = 0, vr = 0, flags = 0;
            {
                const uint4* src = cig4 + g0;
                #pragma unroll 1
                for (int gb = 0; gb < ng; gb += 8) {
                    uint4 v[8];
                    #pragma unroll
                    for (int g = 0; g < 8; ++g) v[g] = gb + g < ng ? ldg_l2_256(src + gb + g) : make_uint4(0u, 0u, 0u, 0u);
                    uint32_t aq = 0, ar = 0, ext = 0;
                    #pragma unroll
                    for (int g = 0; g < 8; ++g) {
                        const uint32_t rb = v[g].x | v[g].y | v[g].z | v[g].w;
                        flags |= rb & 0x40004000u;
                        if (rb & 0x80008000u) ext |= 1u << g;
                        else { SNFB_WORD_BODY(v[g].x, aq, ar) SNFB_WORD_BODY(v[g].y, aq, ar) SNFB_WORD_BODY(v[g].z, aq, ar) SNFB_WORD_BODY(v[g].w, aq, ar) }
                    }
                    vq += (aq & 0xffffu) + (aq >> 16); vr += (ar & 0xffffu) + (ar >> 16);
                    // groups holding an extension word are decoded op by op, once the registers of the eight groups are free again (reloaded from L1)
                    for (; ext; ext &= ext - 1u) { const uint4 w = __ldg(src + gb + __ffs(ext) - 1); const uint2 t = lane_sums_ext(w.x, w.y, w.z, w.w); vq += t.x; vr += t.y; }
                }
            }
            // positions at the chunk start
            const unsigned hm = __ballot_sync(FULL, head) & (lanemask_lt() | (1u << lane));
            const int h = hm ? 31 - __clz(hm) : -1;
            const uint32_t pq = seg_incl_sum(vq, h, h < 0 ? carry.x : 0u) - vq, pr = seg_incl_sum(vr, h, h < 0 ? carry.y : rs[j].z) - vr;
            // the flagged chunks' groups, one per lane in chunk order, in passes of 32 (a chunk may continue into the next pass)
            uint32_t my_n = 0, my_big = 0;                   // events / big-indel sum of this lane's chunk
            const uint32_t fng = flags ? (uint32_t)ng : 0u;
            const uint32_t fin = prims::warp_incl_scan(fng), fex = fin - fng, ftot = __shfl_sync(FULL, fin, 31);
            uint32_t cq = 0, cr = 0;                         // group position at the end of the previous pass (warp-uniform)
            for (uint32_t p0 = 0; p0 < ftot; p0 += 32) {
                const uint32_t x = p0 + lane;
                const bool gv = x < ftot;
                int o = 0;                                   // the owner: the last lane whose first group is <= x (lanes without a flagged chunk own none)
                #pragma unroll
                for (int s = 16; s; s >>= 1) { const uint32_t e = __shfl_sync(FULL, fex, o + s); if (e <= x) o += s; }
                const uint32_t gi = x - __shfl_sync(FULL, fex, o), o_g0 = __shfl_sync(FULL, g0, o), o_pq = __shfl_sync(FULL, pq, o), o_pr = __shfl_sync(FULL, pr, o);
                const int o_j = __shfl_sync(FULL, j, o);
                const uint4 v = gv ? __ldg(cig4 + o_g0 + gi) : make_uint4(0u, 0u, 0u, 0u);     // just read by the owner: L1 / L2
                const uint2 a = group_sums(v);
                const unsigned gh = __ballot_sync(FULL, gv && gi == 0) & (lanemask_lt() | (1u << lane));
                const int hg = gh ? 31 - __clz(gh) : -1;
                const uint32_t q = seg_incl_sum(a.x, hg, hg < 0 ? cq : o_pq) - a.x, r = seg_incl_sum(a.y, hg, hg < 0 ? cr : o_pr) - a.y;
                cq = __shfl_sync(FULL, q + a.x, 31); cr = __shfl_sync(FULL, r + a.y, 31);
                const uint32_t f_rec = t0 + (uint32_t)o_j;
                int tk_start = 0, tk_end = 0; uint32_t n = 0, big = 0;
                if (gv && (((v.x | v.y | v.z | v.w) & 0x40004000u) != 0)) {      // count the group's signatures
                    const int2 win = rec_window(P.region, P.task, P.rec, f_rec, (int)(rs[o_j].w & 0xffffu));
                    tk_start = win.x; tk_end = win.y;
                    group_events(v, q, (int)r, P.minsv, tk_start, tk_end, big, [&](unsigned, unsigned, uint32_t, int) { ++n; });
                }
                const uint32_t n_incl = prims::warp_incl_scan(n), n_ex = n_incl - n, n_tot = __shfl_sync(FULL, n_incl, 31);
                const uint32_t b_incl = prims::warp_incl_scan(big);
                // this pass's share of each flagged chunk goes back to its owner lane: the scans' difference over the chunk's lanes
                const uint32_t lo = fex > p0 ? fex - p0 : 0u, hi = fin - p0 < 32u ? fin - p0 : 32u;          // lanes [lo, hi) of this pass
                const bool mine = fng && fin > p0 && fex < p0 + 32u;
                const uint32_t hi_n = __shfl_sync(FULL, n_incl, (hi - 1u) & 31u), lo_n = __shfl_sync(FULL, n_ex, lo & 31u);
                const uint32_t hi_b = __shfl_sync(FULL, b_incl, (hi - 1u) & 31u), lo_b = __shfl_sync(FULL, b_incl - big, lo & 31u);
                if (mine) { my_n += hi_n - lo_n; my_big += hi_b - lo_b; }
                if (n_tot) {
                    // ordinals: a segmented count that starts at every record's first group of the pass; a record that continues
                    // from an earlier pass or round starts from the running count
                    const uint32_t prev_rec = __shfl_up_sync(FULL, f_rec, 1);
                    const unsigned rh = __ballot_sync(FULL, gv && (lane == 0 ? f_rec != run_rec : f_rec != prev_rec)) & (lanemask_lt() | (1u << lane));
                    const int hr = rh ? 31 - __clz(rh) : -1;
                    const uint32_t ord = (hr < 0 ? run_cnt : 0u) + n_ex - __shfl_sync(FULL, n_ex, hr < 0 ? 0 : hr);
                    const uint32_t lastv = ftot - p0 < 32u ? ftot - p0 - 1u : 31u;
                    run_rec = __shfl_sync(FULL, f_rec, lastv); run_cnt = __shfl_sync(FULL, ord + n, lastv);
                    // the s_left reserved slots first, then a new reservation
                    const uint32_t avail = s_left;
                    unsigned long long nb = 0; uint32_t blk = 0;
                    if (n_tot > avail) {
                        blk = (n_tot - avail + WALK_SLOTS - 1) / WALK_SLOTS * WALK_SLOTS;
                        if (lane == 0) nb = atomicAdd(P.n_ev, (unsigned long long)blk);
                        nb = __shfl_sync(FULL, nb, 0);
                    }
                    if (n) {                                 // decode the group again and write its signatures
                        uint32_t t = n_ex, k = ord, big_again = 0;
                        group_events(v, q, (int)r, P.minsv, tk_start, tk_end, big_again, [&](unsigned cls, unsigned len, uint32_t eq, int er) {
                            const unsigned long long slot = t < avail ? s_cur + t : nb + (t - avail);
                            if (slot < P.ev_cap) { uint4* dst = reinterpret_cast<uint4*>(P.ev + slot); dst[0] = make_uint4(f_rec, len, eq, (uint32_t)er); dst[1] = make_uint4((k & 0xffffu) | (cls << 16), 0u, 0u, 0u); }
                            else ++overflow;
                            ++t; ++k;
                        });
                    }
                    if (n_tot > avail) { s_cur = nb + (n_tot - avail); s_left = blk - (n_tot - avail); } else { s_cur += n_tot; s_left -= n_tot; }
                }
            }
            // the record totals at its last chunk
            const uint32_t tn = seg_incl_sum(my_n, h, h < 0 ? carry.z : 0u), tb = seg_incl_sum(my_big, h, h < 0 ? carry.w : 0u);
            __syncwarp();
            if (lane == 31) carry = make_uint4(pq + vq, pr + vr, tn, tb);
            __syncwarp();
            if (last) {
                const uint32_t rec = t0 + (uint32_t)j;
                P.rec_end[rec] = (int)(pr + vr); P.rec_nlead[rec] = tn; P.rec_big[rec] = (int)tb;
                if (tn > 0xffffu) atomicAdd(&P.ctr->ordinal_overflow, 1ULL);
            }
        }
    }
    for (uint32_t x = lane; x < s_left; x += 32) if (s_cur + x < P.ev_cap) P.ev[s_cur + x].rec = HOLE;      // retire the unused slots
    if (overflow) atomicAdd(&P.ctr->lead_overflow, overflow);
}

// per read nm (leadprov.py:517-526) and the per-task bookkeeping of iter_region (read count, covered bases, longest span)
struct PostParams {
    const RecScan* scan; const RecClip* clip; const snfb_task* task; uint32_t n_rec;
    const int32_t* rec_end; const int32_t* rec_big; double* rec_nm;
    uint32_t* task_reads; unsigned long long* task_cov_bp; int32_t* task_maxspan;
};
__global__ void __launch_bounds__(256) k_rec_post(const PostParams P) {
    __shared__ unsigned s_reads; __shared__ unsigned long long s_bp; __shared__ int s_span; __shared__ int s_task;
    const uint32_t i0 = blockIdx.x * 256, i = i0 + threadIdx.x;
    if (threadIdx.x == 0) { s_reads = 0; s_bp = 0; s_span = 0; s_task = (int)(P.scan[i0].meta & 0xffffu); }
    __syncthreads();
    unsigned mine = 0; unsigned long long bp = 0; int span = 0;
    if (i < P.n_rec) {
        const RecScan s = P.scan[i];
        if (s.meta & RM_PASS) {
            const int task = (int)(s.meta & 0xffffu), ref_end = P.rec_end[i];
            if (s.meta & RM_HAS_NM) P.rec_nm[i] = __ddiv_rn(P.rec_nm[i] - (double)P.rec_big[i], (double)(P.clip[i].alen + 1));
            const int tk_len = P.task[task].contig_len;
            const int ce = ref_end < tk_len ? ref_end : tk_len;
            bp = ce > s.pos ? (unsigned long long)(ce - s.pos) : 0ull; span = ref_end - s.pos; if (span < 0) span = 0;
            if (task == s_task) mine = 1;
            else { atomicAdd(&P.task_reads[task], 1u); atomicAdd(&P.task_cov_bp[task], bp); atomicMax(&P.task_maxspan[task], span); bp = 0; span = 0; }   // block straddles a task boundary
        }
    }
    const unsigned wr = __reduce_add_sync(FULL, mine); const int ws = __reduce_max_sync(FULL, span);
    #pragma unroll
    for (int o = 16; o; o >>= 1) bp += __shfl_xor_sync(FULL, bp, o);
    if (lane_id() == 0 && wr) { atomicAdd(&s_reads, wr); atomicAdd(&s_bp, bp); atomicMax(&s_span, ws); }
    __syncthreads();
    if (threadIdx.x == 0 && s_reads) { atomicAdd(&P.task_reads[s_task], s_reads); atomicAdd(&P.task_cov_bp[s_task], s_bp); atomicMax(&P.task_maxspan[s_task], s_span); }
}

struct EmitParams {
    const snfb_rec* rec; const RecClip* clip; const uint8_t* var;
    const Event* ev; const unsigned long long* n_ev; unsigned long long ev_cap;
    snfb_lead* leads; DevCounters* ctr;
    int maxlen, detect_large_ins; double longinslen;
};
// qname_hash_warp (common.cuh) evaluated by one thread
__device__ inline uint64_t qname_hash_thread(const uint8_t* s, int n) {
    uint64_t acc = 0;
    for (int l = 0; l * 8 < n; ++l) {
        uint64_t w = 0; const int m = n - l * 8 < 8 ? n - l * 8 : 8;
        for (int j = 0; j < m; ++j) w |= (uint64_t)s[l * 8 + j] << (8 * j);
        acc += qname_word(w, (uint32_t)l);
    }
    return qname_finish(acc + (0x9E3779B97F4A7C15ull ^ (uint64_t)n));
}
// one thread per event: read_iterindels' lead construction (leadprov.py:583-670).  Event e becomes lead slot e (a hole stays one); the
// slots of the SA leads (k_sa) start behind the last event.
__global__ void __launch_bounds__(128) k_emit(const EmitParams P) {
    const unsigned long long n_all = *P.n_ev, n = n_all < P.ev_cap ? n_all : P.ev_cap;
    if (blockIdx.x == 0 && threadIdx.x == 0) P.ctr->n_slots = n_all;
    for (unsigned long long e = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (unsigned long long)gridDim.x * blockDim.x) {
        const uint4 e0 = __ldg(reinterpret_cast<const uint4*>(P.ev + e));
        if (e0.x == HOLE) { P.leads[e].rec = HOLE; continue; }
        const uint32_t kc = __ldg(&P.ev[e].k_cls);
        const uint32_t rec = e0.x; const int ln = (int)e0.y, pqi = (int)e0.z, pr = (int)e0.w; const unsigned op = kc >> 16;
        const uint4* core = reinterpret_cast<const uint4*>(P.rec + rec);
        const uint4 c0 = __ldg(core), c3 = __ldg(core + 3);
        const int r_task = (int)c0.x, r_pos = (int)c0.y; const unsigned flag = c0.z & 0xffffu, mapq = (c0.z >> 16) & 255u, aux = c0.z >> 24; const int l_qname = (int)((c0.w >> 8) & 255u);
        const unsigned long long var_off = (unsigned long long)c3.z | ((unsigned long long)c3.w << 32);
        const int alen = P.clip[rec].alen;
        const bool is_supp = flag & 2048u, rev = flag & 16u, has_sa = aux & SNFB_AUX_SA;
        unsigned hp = (aux & SNFB_AUX_HP) ? (c0.w & 255u) : 0u; if (hp > 2) hp = 0;
        const bool use_clips = P.detect_large_ins && !is_supp && !has_sa;
        snfb_lead L;
        L.rec = rec; L.qname_hash = qname_hash_thread(P.var + var_off, l_qname); L.read_len = alen; L.seq_off = -1; L.seq_len = 0; L.mate_contig = -1; L.mate_pos = 0; L.nm_sa = 0;
        L.task = (uint16_t)r_task; L.k = (uint16_t)(kc & 0xffffu);
        uint32_t f = (rev ? SNFB_LF_REVERSE : 0u) | (mapq << 16) | ((uint32_t)SNFB_SRC_INLINE << 3) | (hp << 24) | (is_supp ? SNFB_LF_IS_SA : 0u);
        if (op == C16_I) { f |= SNFB_INS; L.ref_start = pr; L.ref_end = pr; L.qry_start = pqi; L.qry_end = pqi + ln; L.svlen = ln;
            if (ln <= P.maxlen) { f |= SNFB_LF_HAS_SEQ; L.seq_off = pqi; L.seq_len = ln; } }
        else if (op == C16_D) { f |= SNFB_DEL; L.ref_start = pr + ln; L.ref_end = pr; L.qry_start = pqi; L.qry_end = pqi; L.svlen = -ln; }
        else if (use_clips && (double)ln >= P.longinslen) { f |= SNFB_INS | SNFB_LF_SVLEN_NONE; L.ref_start = L.ref_end = pr; L.qry_start = pqi; L.qry_end = pqi + ln; L.svlen = 0; }
        else { f |= (pr == r_pos) ? SNFB_SINGLE_LEFT : SNFB_SINGLE_RIGHT; L.ref_start = L.ref_end = pr; L.qry_start = pqi; L.qry_end = pqi + ln; L.svlen = 0; }
        L.flags = f;
        store_lead(P.leads + e, L);
    }
}

struct SaParams {
    const snfb_rec* rec; const RecClip* clip; const uint8_t* var; const snfb_task* task; const snfb_contig* contig; uint32_t n_contig;
    const uint32_t* sa_list; const unsigned long long* n_sa; const int32_t* rec_end; uint32_t* rec_nlead;
    snfb_lead* leads; unsigned long long lead_cap; DevCounters* ctr;
    Seg* seg_scratch;                 // MAXSEG segments per thread of the grid
    snfb_config cfg;
    const snfb_region* region;        // region table (null: none)
};
constexpr int SA_THREADS = 128, SA_BLOCKS = NUM_SMS * 8;
// one thread per record with an SA tag: the text parse is serial per record, so the parallelism is across records.
// Segments live in a per-thread slice of global scratch (a read has a handful of them; the touched part stays in L2).
__global__ void __launch_bounds__(SA_THREADS) k_sa(const SaParams P) {
    __shared__ snfb_config s_cfg;
    if (threadIdx.x < sizeof(snfb_config) / 4) reinterpret_cast<uint32_t*>(&s_cfg)[threadIdx.x] = reinterpret_cast<const uint32_t*>(&P.cfg)[threadIdx.x];
    __syncthreads();
    const unsigned long long n = *P.n_sa;
    const unsigned long long tid = (unsigned long long)blockIdx.x * SA_THREADS + threadIdx.x, nthr = (unsigned long long)gridDim.x * SA_THREADS;
    Seg* sg = P.seg_scratch + tid * MAXSEG;
    unsigned long long soft = 0, overflow = 0;
    SlotState slots; slots.cur = 0; slots.end = 0;
    for (unsigned long long e = tid; e < n; e += nthr) {
        const uint32_t rec = P.sa_list[e];
        const uint4* core = reinterpret_cast<const uint4*>(P.rec + rec);
        const uint4 c0 = __ldg(core), c1 = __ldg(core + 1), c3 = __ldg(core + 3);
        const int r_task = (int)c0.x, r_pos = (int)c0.y; const unsigned flag = c0.z & 0xffffu, mapq = (c0.z >> 16) & 255u, aux = c0.z >> 24; const int l_qname = (int)((c0.w >> 8) & 255u);
        const int l_seq = (int)c1.w; const unsigned long long var_off = (unsigned long long)c3.z | ((unsigned long long)c3.w << 32);
        const uint32_t sa_len = __ldg(reinterpret_cast<const uint32_t*>(core + 2));
        const snfb_task tk = P.task[r_task];
        const RecClip rc = P.clip[rec];
        int hp = (aux & SNFB_AUX_HP) ? (int)(c0.w & 255u) : 0; if (hp > 2) hp = 0;
        const bool rev = flag & 16u;
        SaArgs a; a.rec = rec; a.qas = rc.qas; a.qae = rc.qas + rc.alen; a.alen = rc.alen; a.ref_end = P.rec_end[rec]; a.hp = hp;
        a.base_flags = (rev ? SNFB_LF_REVERSE : 0u) | (mapq << 16); a.qh = qname_hash_thread(P.var + var_off, l_qname); a.nlead = P.rec_nlead[rec]; a.rev = rev; a.is_supp = flag & 2048u;
        a.sa = P.var + var_off + l_qname; a.sa_len = (int)sa_len; a.clip_left = rc.clip_left; a.clip_right = rc.clip_right; a.pos = r_pos; a.l_seq = l_seq; a.mapq = (int)mapq;
        a.aux_flags = (int)aux; a.task = r_task; a.tk_contig = tk.contig; const int2 win = rec_window(P.region, P.task, P.rec, rec, r_task); a.tk_start = win.x; a.tk_end = win.y; a.contig = P.contig; a.n_contig = P.n_contig;
        a.leads = P.leads; a.lead_cap = P.lead_cap; a.n_slots = &P.ctr->n_slots; a.slots = &slots;
        a.mapq_min = s_cfg.mapq; a.dev_keep_lowqual_splits = s_cfg.dev_keep_lowqual_splits; a.max_splits_base = s_cfg.max_splits_base; a.max_splits_kb = s_cfg.max_splits_kb;
        const unsigned added = process_sa(&s_cfg, sg, a, &soft, &overflow);
        if (added) { if (a.nlead + added > 0xffffu) atomicAdd(&P.ctr->ordinal_overflow, 1ULL); P.rec_nlead[rec] += added; }
    }
    for (unsigned long long sidx = slots.cur; sidx < slots.end; ++sidx) if (sidx < P.lead_cap) P.leads[sidx].rec = HOLE;   // retire the last chunk
    if (soft) atomicAdd(&P.ctr->soft_errors, soft);
    if (overflow) atomicAdd(&P.ctr->lead_overflow, overflow);
}

// deterministic per-task mean of the per-read nm values (config.average_regional_nm, leadprov.py:577).
// Fixed two-level reduction tree (4096-record chunks of each task, then the chunk partials in order): the result does
// not depend on scheduling; it can differ from the reference's sequential float accumulation in the last bits (DESIGN.md).
constexpr int NM_CHUNK = 4096;
__global__ void __launch_bounds__(256) k_nm_partial(const uint8_t* __restrict__ rec_flags, const double* __restrict__ rec_nm, const uint32_t* __restrict__ task_first,
                                                    const uint32_t* __restrict__ task_last, double* __restrict__ part_sum, unsigned* __restrict__ part_cnt) {
    __shared__ double ssum[256]; __shared__ unsigned scnt[256];
    const int t = blockIdx.y; const uint32_t lo = task_first[t] + blockIdx.x * NM_CHUNK, end = task_last[t];
    if (lo >= end) return;                                  // whole block exits together
    const uint32_t hi = lo + NM_CHUNK < end ? lo + NM_CHUNK : end;
    double s = 0; unsigned c = 0;
    for (uint32_t i = lo + threadIdx.x; i < hi; i += 256) if (rec_flags[i] & RF_NM_MEAN) { s += rec_nm[i]; ++c; }
    ssum[threadIdx.x] = s; scnt[threadIdx.x] = c; __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) { ssum[threadIdx.x] += ssum[threadIdx.x + o]; scnt[threadIdx.x] += scnt[threadIdx.x + o]; } __syncthreads(); }
    if (threadIdx.x == 0) { part_sum[(size_t)t * gridDim.x + blockIdx.x] = ssum[0]; part_cnt[(size_t)t * gridDim.x + blockIdx.x] = scnt[0]; }
}
__global__ void __launch_bounds__(256) k_task_nm(const uint32_t* __restrict__ task_first, const uint32_t* __restrict__ task_last, const double* __restrict__ part_sum,
                                                 const unsigned* __restrict__ part_cnt, int chunks_per_task, double* __restrict__ task_mean_nm) {
    __shared__ double ssum[256]; __shared__ unsigned long long scnt[256];
    const int t = blockIdx.x; const uint32_t lo = task_first[t], hi = task_last[t];
    const uint32_t nch = hi > lo ? (hi - lo + NM_CHUNK - 1) / NM_CHUNK : 0;
    double s = 0; unsigned long long c = 0;
    for (uint32_t ch = threadIdx.x; ch < nch; ch += 256) { s += part_sum[(size_t)t * chunks_per_task + ch]; c += part_cnt[(size_t)t * chunks_per_task + ch]; }
    ssum[threadIdx.x] = s; scnt[threadIdx.x] = c; __syncthreads();
    for (int o = 128; o; o >>= 1) { if (threadIdx.x < o) { ssum[threadIdx.x] += ssum[threadIdx.x + o]; scnt[threadIdx.x] += scnt[threadIdx.x + o]; } __syncthreads(); }
    if (threadIdx.x == 0) task_mean_nm[t] = ssum[0] / (double)(scnt[0] > 1 ? scnt[0] : 1);
}

}  // namespace extract
