// Test infrastructure (not part of the product): the BGZF CRC-32 of sniffles_b200/csrc/ingest_core.h compiled with g++ as a one-lane
// group, so the code k_inflate runs with 16 lanes can be checked against zlib on a machine without a GPU (tests/test_bgzf_crc.py).
#include <stdint.h>
#include "../../sniffles_b200/csrc/ingest_core.h"

extern "C" {

// CRC-32 of p[0 .. n) by a one-lane group (crc32_group<1>: one slice, no combine step)
uint32_t crc_host_crc32(const uint8_t* p, uint32_t n) {
    ingest::CrcTables C; ingest::crc_tables_fill(&C, 0, 1);
    return ingest::crc32_group<1>(p, n, &C, 0, 1u);
}

// CRC of A || B from crc(A), crc(B) and len(B): the step that joins the lanes' slices
uint32_t crc_host_crc32_combine(uint32_t crc_a, uint32_t crc_b, uint32_t len_b) {
    ingest::CrcTables C; ingest::crc_tables_fill(&C, 0, 1);
    return ingest::crc32_combine(crc_a, crc_b, len_b, C.x8pow);
}

}
