// host_math.h — host-side scalar mathematics of the engine (no data-path work):
// GF(2^8)/0x11d arithmetic, generator / recovery matrices, CRC-32 polynomial algebra, goal geometry.
// These are O(k^3) byte operations per call (k <= 32) and stay on the host by design
// (SURVEY.md §8 a4/a5/a14: "negligible; host-side in the new design").
#pragma once
#include <cstddef>
#include <cstdint>

#include "lzgpu.h"

namespace lz {

// GF(2^8), x^8+x^4+x^3+x^2+1 (reference: src/common/galois_coeff.h:30-32)
uint8_t gf_mul_host(uint8_t a, uint8_t b);
uint8_t gf_inv_host(uint8_t a);

// generator matrix selection rule of ReedSolomon::createRSMatrix (src/common/reed_solomon.h:163-178)
bool uses_cauchy(int k, int m);
int rs_generator(int k, int m, uint8_t *matrix);
// rows computing `wanted` erased parts from the k non-erased parts (reed_solomon.h:189-281)
int rs_recovery_matrix(int k, int m, const uint8_t *erased, const uint8_t *wanted, uint8_t *matrix, bool *singular);

// CRC-32 algebra in the reflected domain (bit 31 = x^0), polynomial 0xEDB88320
// (src/protocol/MFSCommunication.h:81)
constexpr uint32_t kCrcPolyReflected = 0xEDB88320u;
uint32_t crc_mulmod(uint32_t a, uint32_t b);
uint32_t crc_xpow_bytes(uint64_t nbytes);            // x^(8*nbytes) mod P
void crc_xpow2_table(uint32_t pow2[32]);             // pow2[i] = x^(8 * 2^i) mod P
uint32_t crc_of_zeros(uint64_t nbytes);              // mycrc32(0, zeros, nbytes)
uint32_t crc_combine(uint32_t crc1, uint32_t crc2, uint64_t len2);
void crc_make_tables(uint32_t tab[4][256]);          // slicing-by-4 tables for x^32..x^56 steps

}  // namespace lz
