// repair_rows.h — the recovery rows of lzgpu_repair_stripes, derived per stripe: the blocks of the parts in `wanted` as GF(2^8)
// combinations of the k input blocks.  The erasure pattern depends on which blocks fail their stored CRCs, so the rows cannot come
// from a host table built before the call: repair_map_kernel (correct_kernel.cuh) derives them in shared memory, and host_math.cc
// runs the host build of the same function (lzgpu_debug_repair_rows), which tests/test_repair_rows.py pins against
// lzgpu_rs_recovery_matrix.
//
// With A = the generator rows of the k inputs (a unit row for a data part, the parity row for a parity part), the data are A^-1 times
// the inputs, so part p is G[p] A^-1 times the inputs: the unique combination, hence byte for byte lz::rs_recovery_matrix's.  A^-1
// comes from Gauss-Jordan elimination of [A | I], one column at a time: the pivot row (thread 0), the swap and scale of the pivot row
// (one thread per column), the elimination of every other row (one thread per byte).  Column c of the left half is left as it is
// after its own step: nothing reads it again.
#pragma once
#include <cstdint>

#include "bitslice.cuh"  // LZ_HD

namespace lzd {

struct GfTables {
	uint8_t log[256], exp[512];  // x^8 = x^4+x^3+x^2+1 (0x11d); exp is doubled, so log[a] + log[b] needs no reduction
};

LZ_HD inline void gf_tables_build(GfTables &t) {
	uint32_t x = 1;
	for (int i = 0; i < 255; ++i) {
		t.exp[i] = t.exp[i + 255] = static_cast<uint8_t>(x);
		t.log[x] = static_cast<uint8_t>(i);
		x = (x << 1) ^ ((x & 0x80u) ? 0x11du : 0u);
	}
	t.exp[510] = t.exp[511] = 0;
	t.log[0] = 0;
}

LZ_HD inline uint8_t gf_mul_t(uint32_t a, uint32_t b, const GfTables &t) { return (a && b) ? t.exp[t.log[a] + t.log[b]] : 0; }

// Every thread t of nt calls it (device: the CTA, sync = __syncthreads; host: t = 0, nt = 1, sync does nothing).
//   k        data parts (<= 32); gen + 32 r: parity row r of the generator
//   inputs   the k input parts, wanted: the n_wanted parts to rebuild (this API's numbering, none of them an input)
//   mat      [32][64] scratch, *pivot one shared word
//   rows     rows[32 w + j]: the coefficient of input j in the block of part wanted[w]
// Returns false, in every thread, when the inputs' submatrix is singular (rows then unset).
#ifdef __CUDACC__
#pragma nv_exec_check_disable  // Sync is __syncthreads on the device, a host no-op on the host
#endif
template <class Sync>
LZ_HD inline bool repair_rows(uint32_t k, const uint8_t *gen, const uint8_t *inputs, const uint8_t *wanted, uint32_t n_wanted, const GfTables &tb,
                              uint8_t (*mat)[64], uint32_t *pivot, uint8_t *rows, uint32_t t, uint32_t nt, Sync sync) {
	const uint32_t w2 = 2 * k;
	for (uint32_t x = t; x < k * w2; x += nt) {
		const uint32_t i = x / w2, j = x % w2, p = inputs[i];
		mat[i][j] = j < k ? (p < k ? (p == j ? 1 : 0) : gen[32 * (p - k) + j]) : (j - k == i ? 1 : 0);
	}
	sync();
	for (uint32_t c = 0; c < k; ++c) {
		if (t == 0) {
			uint32_t r = 0xffu;
			for (uint32_t i = c; i < k && r == 0xffu; ++i)
				if (mat[i][c]) r = i;
			*pivot = r == 0xffu ? 0xffffffffu : (r | static_cast<uint32_t>(tb.exp[255 - tb.log[mat[r][c]]]) << 8);  // row, 1 / pivot
		}
		sync();
		const uint32_t pv = *pivot;
		if (pv == 0xffffffffu) return false;
		const uint32_t r = pv & 0xffu, inv = pv >> 8;
		for (uint32_t j = t; j < w2; j += nt) {  // swap rows r and c, scale the pivot row to a 1 in column c
			const uint8_t x = mat[r][j];
			mat[r][j] = mat[c][j];
			mat[c][j] = gf_mul_t(x, inv, tb);
		}
		sync();
		for (uint32_t x = t; x < k * w2; x += nt) {  // every other row: minus its column-c multiple of the pivot row (column c not written)
			const uint32_t i = x / w2, j = x % w2;
			if (i != c && j != c) mat[i][j] ^= gf_mul_t(mat[i][c], mat[c][j], tb);
		}
		sync();
	}
	for (uint32_t x = t; x < n_wanted * k; x += nt) {  // rows = G[wanted] A^-1 (the right half)
		const uint32_t w = x / k, j = x % k, p = wanted[w];
		uint32_t v = 0;
		if (p < k) v = mat[p][k + j];
		else
			for (uint32_t i = 0; i < k; ++i) v ^= gf_mul_t(gen[32 * (p - k) + i], mat[i][k + j], tb);
		rows[32 * w + j] = static_cast<uint8_t>(v);
	}
	sync();
	return true;
}

}  // namespace lzd
