// cigar16.h — CIGAR16, the 2-byte CIGAR words the kernels read (include/snfb.h, SNFB_CIGAR_16, describes the format for users of
// the library).  This header is the one place that knows the bit layout, the op classes, how a BAM op becomes words and which ops
// carry E; the encoder (ingest::c16_convert) and the decoders (extract.cuh) take all of it from here.  It compiles under nvcc and
// under g++ (tests/native/ builds the one-lane encoder on the CPU).
#pragma once
#include <stdint.h>
#if defined(__CUDACC__)
#define SNFB_HD __host__ __device__ __forceinline__
#else
#define SNFB_HD inline
#endif

// ---- bit layout
// base word:      [15] 0 | [14] E | [13:11] class | [10:0] length & 0x7ff
// extension word: [15] 1 | [14:12] level (1, 2) | [11:0] payload, adding payload << (11 + 12 * (level - 1)) to the length of the base
//                 word it follows.  A base word and its extension words never straddle a 16-byte group.
constexpr unsigned C16_EXT = 0x8000u, C16_E = 0x4000u;
constexpr unsigned C16_CLASS_SHIFT = 11, C16_CLASS_MASK = 7u;
constexpr unsigned C16_LEN_BITS = 11, C16_LEN_MASK = 0x7ffu;
constexpr unsigned C16_EXT_LEVEL_SHIFT = 12, C16_EXT_LEVEL_MASK = 7u, C16_EXT_BITS = 12, C16_EXT_MASK = 0xfffu;

// ---- classes: bit 0 = the op advances the read, bit 1 = it advances the reference.  P and the zero pad word are class 0.
constexpr unsigned C16_P = 0, C16_I = 1, C16_D = 2, C16_M = 3, C16_H = 4, C16_S = 5, C16_N = 6;
// BAM op code (M I D N S H P = X = 0..8) -> class, one nibble per op; M, = and X are one class
constexpr uint64_t C16_OP_CLASSES = (uint64_t)C16_M | (uint64_t)C16_I << 4 | (uint64_t)C16_D << 8 | (uint64_t)C16_N << 12 | (uint64_t)C16_S << 16
                                  | (uint64_t)C16_H << 20 | (uint64_t)C16_P << 24 | (uint64_t)C16_M << 28 | (uint64_t)C16_M << 32;

// ---- encoding (BAM op -> words)
SNFB_HD unsigned c16_op_class(unsigned op) { return (unsigned)((C16_OP_CLASSES >> (4 * op)) & 15ull); }      // op <= 8
SNFB_HD int c16_op_words(uint32_t len) { return len < (1u << C16_LEN_BITS) ? 1 : (len < (1u << (C16_LEN_BITS + C16_EXT_BITS)) ? 2 : 3); }
// I, D and S are the ops an SV signature or an NM-corrected indel can come from
SNFB_HD bool c16_is_event(unsigned cls) { return (0x26u >> cls) & 1u; }
// E: an I / D / S of at least evt_min bases, what the streaming kernel has to look at (evt_min <= SNFB_CIGAR16_EVT_MIN)
SNFB_HD unsigned c16_e_flag(unsigned cls, uint32_t len, uint32_t evt_min) { return c16_is_event(cls) && len >= evt_min ? C16_E : 0u; }
SNFB_HD uint16_t c16_base_word(unsigned cls, uint32_t len, uint32_t evt_min) {
    return (uint16_t)(c16_e_flag(cls, len, evt_min) | (cls << C16_CLASS_SHIFT) | (len & C16_LEN_MASK));
}
SNFB_HD uint16_t c16_ext_word(uint32_t len, unsigned level) {       // level 1 or 2
    return (uint16_t)(C16_EXT | (level << C16_EXT_LEVEL_SHIFT) | ((len >> (C16_LEN_BITS + C16_EXT_BITS * (level - 1u))) & C16_EXT_MASK));
}

// ---- decoding
SNFB_HD unsigned c16_word_class(unsigned w) { return (w >> C16_CLASS_SHIFT) & C16_CLASS_MASK; }
SNFB_HD unsigned c16_ext_add(unsigned e) {
    return (e & C16_EXT_MASK) << (C16_LEN_BITS + C16_EXT_BITS * (((e >> C16_EXT_LEVEL_SHIFT) & C16_EXT_LEVEL_MASK) - 1u));
}
