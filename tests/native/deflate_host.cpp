// Test infrastructure (not part of the product): the BGZF encoder of sniffles_b200/csrc/deflate_core.h compiled with g++ as one
// thread (NT = 1) and one-lane warps (NL = 1), so the bytes k_deflate writes with a thread block per BGZF block can be checked against
// zlib on a machine without a GPU (tests/test_bgzf_write.py), and stand in for the device compressor in the VCF output tests.
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../sniffles_b200/csrc/deflate_core.h"

extern "C" {

// the BGZF members of in[0 .. n_in), back to back, no EOF marker; coffset[k] = offset of member k.  Returns the bytes written, or -1
// when out_cap is below ceil(n_in / 0xff00) * 65536.
int64_t deflate_host_bgzf(const uint8_t* in, uint64_t n_in, uint8_t* out, uint64_t out_cap, uint64_t* coffset) {
    const uint64_t nb = (n_in + deflate::BLOCK_IN - 1) / deflate::BLOCK_IN;
    if (out_cap < nb * deflate::MEMBER_MAX) return -1;
    deflate::Shared* S = new deflate::Shared;
    std::vector<uint16_t> cand(deflate::BLOCK_IN), dist(deflate::BLOCK_IN);
    ingest::crc_tables_fill(&S->crc, 0, 1);
    uint64_t o = 0;
    for (uint64_t k = 0; k < nb; ++k) {
        const uint64_t off = k * deflate::BLOCK_IN;
        const uint32_t n = (uint32_t)(n_in - off < deflate::BLOCK_IN ? n_in - off : deflate::BLOCK_IN);
        deflate::stage(S, in + off, n, 0, 1);
        deflate::find_candidates<1>(S, cand.data(), 0);
        S->crc_val = ingest::crc32_group<1>(S->data, n, &S->crc, 0, 1u);
        deflate::longest_matches(S, cand.data(), dist.data(), 0, 1);
        deflate::greedy_parse<1>(S, 0);
        deflate::histogram(S, dist.data(), 0, 1);
        deflate::plan(S);
        if (S->btype != 0) {
            deflate::count_bits(S, dist.data(), 0, 1);
            deflate::write_header(S, 1);
            deflate::write_tokens(S, dist.data(), 0);
        }
        if (coffset) coffset[k] = o;
        o += deflate::write_member(S, out + o, 0, 1);
    }
    delete S;
    return (int64_t)o;
}

}
