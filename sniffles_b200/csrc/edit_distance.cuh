// edit_distance.cuh — the Levenshtein distance of edlib.align's defaults, shared by the combine grouping (group.align_call,
// combine.cuh) and the population match (PopulationVariant.match, population.cuh).
#pragma once
#include "common.cuh"

// Levenshtein distance (edlib.align(a, b) defaults: global alignment, task "distance") by one warp: Myers' bit-vector recurrence in 64-row blocks
// (Hyyro's block formulation, the one edlib implements), lane = block, the text streamed through the lanes as a wavefront (lane l works on column
// s - l at step s, its horizontal carry-in is lane l-1's carry-out of the step before); patterns of more than 32 blocks take several passes,
// the carries of a pass's last block wait in hs[].  The shorter string is the pattern.  The result is exact for any byte strings.
__device__ inline int edit_distance_warp(const uint8_t* a, int m, const uint8_t* b, int n, int8_t* hs) {
    const int lane = lane_id();
    if (m > n) { const uint8_t* t = a; a = b; b = t; const int ti = m; m = n; n = ti; }
    if (m == 0) return n;
    const int W = (m + 63) / 64; int score = m;
    for (int p0 = 0; p0 < W; p0 += 32) {
        const int blk = p0 + lane; const bool vb = blk < W; const bool last = blk == W - 1;
        unsigned long long eq[5] = { 0, 0, 0, 0, 0 };            // A C G T N
        const int rows = vb ? min(64, m - blk * 64) : 0;
        for (int k = 0; k < rows; ++k) { const uint8_t ch = a[blk * 64 + k]; const int idx = ch == 'A' ? 0 : ch == 'C' ? 1 : ch == 'G' ? 2 : ch == 'T' ? 3 : ch == 'N' ? 4 : -1;
            #pragma unroll
            for (int q = 0; q < 5; ++q) if (idx == q) eq[q] |= 1ull << k; }
        unsigned long long Pv = ~0ull, Mv = 0ull; int hout = 0;
        const unsigned long long top = last ? 1ull << ((m - 1) & 63) : 1ull << 63;
        // the text (and, after the first pass, the carries of the previous pass) reach the lanes through registers: lane l holds column
        // base + l of the current 32-column group and of the one before; the next group is loaded while this one is worked on
        int cprev = 0, ccur = lane < n ? (int)b[lane] : 0, hcur = (p0 && lane < n) ? (int)hs[lane] : 0;
        for (int base = 0; base < n + 31; base += 32) {
            const int nb = base + 32 + lane;
            const int cnext = nb < n ? (int)b[nb] : 0, hnext = (p0 && nb < n) ? (int)hs[nb] : 0;
            #pragma unroll 4
            for (int t = 0; t < 32; ++t) {
                const int s = base + t;
                const int hprev = __shfl_up_sync(FULL, hout, 1);
                const int j = s - lane;
                const int src = (t - lane) & 31;                                   // lane holding column j in its group
                const int c_a = __shfl_sync(FULL, ccur, src), c_b = __shfl_sync(FULL, cprev, src);
                const int h0 = __shfl_sync(FULL, hcur, t);                         // lane 0 works on column s
                const bool act = vb && j >= 0 && j < n;
                if (act) {
                    const uint8_t c = (uint8_t)(t >= lane ? c_a : c_b);
                    unsigned long long Eq;
                    if (c == 'A') Eq = eq[0]; else if (c == 'C') Eq = eq[1]; else if (c == 'G') Eq = eq[2]; else if (c == 'T') Eq = eq[3]; else if (c == 'N') Eq = eq[4];
                    else { Eq = 0; for (int k = 0; k < rows; ++k) if (a[blk * 64 + k] == c) Eq |= 1ull << k; }
                    const int hin = lane == 0 ? (p0 == 0 ? 1 : h0) : hprev;
                    const unsigned long long Xv = Eq | Mv;
                    if (hin < 0) Eq |= 1ull;
                    const unsigned long long Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
                    unsigned long long Ph = Mv | ~(Xh | Pv), Mh = Pv & Xh;
                    hout = (Ph & top) ? 1 : ((Mh & top) ? -1 : 0);
                    Ph <<= 1; Mh <<= 1;
                    if (hin < 0) Mh |= 1ull; else if (hin > 0) Ph |= 1ull;
                    Pv = Mh | ~(Xv | Ph); Mv = Ph & Xv;
                    if (last) score += hout; else if (lane == 31) hs[j] = (int8_t)hout;
                }
            }
            cprev = ccur; ccur = cnext; hcur = hnext;
        }
        __syncwarp();
    }
    return __shfl_sync(FULL, score, (W - 1) & 31);
}
