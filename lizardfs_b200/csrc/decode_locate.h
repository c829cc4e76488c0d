// decode_locate.h — the error locator of lzgpu_decode_stripes: which one or two blocks of a stripe, with valid CRCs and wrong bytes,
// explain its syndromes in the code punctured by the blocks that fail their CRCs.  decode_map_kernel (correct_kernel.cuh) runs it
// with the CTA, host_math.cc runs the host build of the same function (lzgpu_debug_locate_errors), which
// tests/test_decode_locate.py pins against a brute force.
//
// The punctured code: the n given parts outside F, as blk[0 .. n-1]; blk[0 .. k-1] are the inputs, blk[k .. n-1] the s = n - k
// spares.  rows[32 j + i] = M[j][i], the coefficient of input i in spare j (repair_rows).  The syndrome of byte b is
// S_j = spare_j[b] ^ sum_i M[j][i] input_i[b]; column q of the check matrix H = [M | I] is M[., q] for an input, the unit vector
// e_(q-k) for a spare.  Every goal is MDS, so any s columns of H are independent: a non-zero S is a multiple of at most one column
// (s >= 2), and lies in the span of at most one pair of columns when it is not a multiple of one (s >= 4).
//
// So the locator classifies each byte as zero, a multiple of one column c ("single"), or neither ("multi", s >= 4 only; with s < 4 such
// a byte is beyond the radius).  The singles of all bytes are ORed.  Without multi bytes the located set is that union (at most one
// column for s < 4, at most two for s >= 4).  With multi bytes, the first one names its unique pair P (every pair of columns tried
// against it); every single must lie in P, and a second pass requires every byte to lie in the span of P.  A pair is never taken from
// a single byte, which fits every pair that contains its column: two bad blocks whose differing bytes are disjoint give two singles
// and no multi byte.
#pragma once
#include <cstdint>

#include "repair_rows.h"

namespace lzd {

struct LocateScratch {
	uint8_t syn[32][256];      // S of this thread's current byte, one column per thread (the host build: column 0)
	uint8_t ratio[256];        // M[1][i] / M[0][i] -> i + 1 (0: no input column has that ratio)
	unsigned long long singles, pair;
	uint32_t multi, none, n_pairs, bad, ambiguous;
};

LZ_HD inline void loc_or(unsigned long long *p, unsigned long long v) {
#ifdef __CUDA_ARCH__
	if (v) atomicOr(p, v);
#else
	*p |= v;
#endif
}
LZ_HD inline void loc_or32(uint32_t *p, uint32_t v) {
#ifdef __CUDA_ARCH__
	if (v) atomicOr(p, v);
#else
	*p |= v;
#endif
}
LZ_HD inline void loc_min(uint32_t *p, uint32_t v) {
#ifdef __CUDA_ARCH__
	if (v != 0xffffffffu) atomicMin(p, v);
#else
	*p = v < *p ? v : *p;
#endif
}
LZ_HD inline uint32_t loc_popc(unsigned long long x) {
	uint32_t n = 0;
	for (; x; x &= x - 1) ++n;
	return n;
}
LZ_HD inline uint32_t gf_div_t(uint32_t a, uint32_t b, const GfTables &t) { return a ? t.exp[t.log[a] + 255 - t.log[b]] : 0; }

// column q of H at row j
LZ_HD inline uint32_t loc_col(const uint8_t *rows, uint32_t k, uint32_t q, uint32_t j) { return q < k ? rows[32 * j + q] : (q - k == j ? 1u : 0u); }

// S of byte b into syn[.][t]; true when it is not zero
LZ_HD inline bool loc_syndrome(uint32_t k, uint32_t s, const uint8_t *rows, const uint8_t *const *blk, uint32_t b, const GfTables &tb,
                               LocateScratch &sc, uint32_t t) {
	bool any = false;
	for (uint32_t j = 0; j < s; ++j) {
		uint32_t v = blk[k + j][b];
		for (uint32_t i = 0; i < k; ++i) v ^= gf_mul_t(rows[32 * j + i], blk[i][b], tb);
		sc.syn[j][t] = static_cast<uint8_t>(v);
		any |= v != 0;
	}
	return any;
}

// a non-zero S: the one column it is a multiple of, or -1
LZ_HD inline int loc_single(uint32_t k, uint32_t s, const uint8_t *rows, const GfTables &tb, const LocateScratch &sc, uint32_t t) {
	uint32_t nz = 0, last = 0;
	for (uint32_t j = 0; j < s; ++j)
		if (sc.syn[j][t]) {
			++nz;
			last = j;
		}
	if (nz == 1) return static_cast<int>(k + last);
	const uint32_t s0 = sc.syn[0][t], s1 = sc.syn[1][t];
	if (!s0 || !s1) return -1;  // every entry of M is non-zero: an input's multiple has no zero row
	const uint32_t q = sc.ratio[gf_div_t(s1, s0, tb)];
	if (!q) return -1;
	const uint32_t x = gf_div_t(s0, rows[q - 1], tb);
	for (uint32_t j = 2; j < s; ++j)
		if (sc.syn[j][t] != gf_mul_t(x, rows[32 * j + q - 1], tb)) return -1;
	return static_cast<int>(q - 1);
}

// S in the span of columns c and d (solved on the first two rows where they are independent, checked on every row)
LZ_HD inline bool loc_pair_fits(uint32_t k, uint32_t s, const uint8_t *rows, uint32_t c, uint32_t d, const GfTables &tb, const LocateScratch &sc,
                                uint32_t t) {
	for (uint32_t r0 = 0; r0 < s; ++r0)
		for (uint32_t r1 = r0 + 1; r1 < s; ++r1) {
			const uint32_t c0 = loc_col(rows, k, c, r0), c1 = loc_col(rows, k, c, r1), d0 = loc_col(rows, k, d, r0), d1 = loc_col(rows, k, d, r1);
			const uint32_t det = gf_mul_t(c0, d1, tb) ^ gf_mul_t(c1, d0, tb);
			if (!det) continue;
			const uint32_t s0 = sc.syn[r0][t], s1 = sc.syn[r1][t];
			const uint32_t x = gf_div_t(gf_mul_t(s0, d1, tb) ^ gf_mul_t(s1, d0, tb), det, tb);
			const uint32_t y = gf_div_t(gf_mul_t(c0, s1, tb) ^ gf_mul_t(c1, s0, tb), det, tb);
			for (uint32_t j = 0; j < s; ++j)
				if (sc.syn[j][t] != (gf_mul_t(x, loc_col(rows, k, c, j), tb) ^ gf_mul_t(y, loc_col(rows, k, d, j), tb))) return false;
			return true;
		}
	return false;
}

// Every thread t of nt calls it (device: the CTA, sync = __syncthreads; host: t = 0, nt = 1, sync does nothing).
//   k, s      inputs and spares of the punctured code; rows: M (repair_rows); blk[q]: the block of column q, len bytes
// Returns, in every thread, the number of located columns (0: the punctured stripe is a codeword) with *located = their bits
// (column indices), or -1 when no unique set of at most two columns with 2 |E| <= s explains every byte.  The caller's barrier must
// come before sc is used again.
#ifdef __CUDACC__
#pragma nv_exec_check_disable  // Sync is __syncthreads on the device, a host no-op on the host
#endif
template <class Sync>
LZ_HD inline int locate_errors(uint32_t k, uint32_t s, const uint8_t *rows, const uint8_t *const *blk, uint32_t len, const GfTables &tb,
                               LocateScratch &sc, uint32_t t, uint32_t nt, Sync sync, unsigned long long *located) {
	if (t == 0) {
		for (uint32_t x = 0; x < 256; ++x) sc.ratio[x] = 0;
		sc.ambiguous = 0;
		for (uint32_t i = 0; s >= 2 && i < k; ++i) {  // a zero entry or a repeated ratio would break the single test: locate nothing
			const uint32_t r = rows[i] && rows[32 + i] ? gf_div_t(rows[32 + i], rows[i], tb) : 0;
			if (!r || sc.ratio[r]) sc.ambiguous = 1;
			else sc.ratio[r] = static_cast<uint8_t>(i + 1);
		}
		sc.singles = sc.pair = 0;
		sc.multi = 0xffffffffu;
		sc.none = sc.n_pairs = sc.bad = 0;
	}
	sync();
	if (sc.ambiguous) return -1;
	unsigned long long singles = 0;
	uint32_t none = 0, multi = 0xffffffffu;
	for (uint32_t b = t; b < len; b += nt) {
		if (!loc_syndrome(k, s, rows, blk, b, tb, sc, t)) continue;
		const int q = s >= 2 ? loc_single(k, s, rows, tb, sc, t) : -1;
		if (q >= 0) singles |= 1ull << q;
		else if (s >= 4) multi = b < multi ? b : multi;
		else none = 1;
	}
	loc_or(&sc.singles, singles);
	loc_or32(&sc.none, none);
	loc_min(&sc.multi, multi);
	sync();
	singles = sc.singles;
	multi = sc.multi;
	const uint32_t n1 = loc_popc(singles);
	if (sc.none || n1 > 2 || (n1 == 2 && s < 4)) return -1;
	if (multi == 0xffffffffu) {
		*located = singles;
		return static_cast<int>(n1);
	}
	// the pair of the first multi byte: every thread has its syndromes, and tries its share of the pairs
	const uint32_t n = k + s;
	loc_syndrome(k, s, rows, blk, multi, tb, sc, t);
	unsigned long long pair = 0;
	uint32_t n_pairs = 0;
	for (uint32_t x = t; x < n * n; x += nt) {
		const uint32_t c = x / n, d = x % n;
		if (c < d && loc_pair_fits(k, s, rows, c, d, tb, sc, t)) {
			pair = 1ull << c | 1ull << d;
			++n_pairs;
		}
	}
	loc_or(&sc.pair, pair);
#ifdef __CUDA_ARCH__
	if (n_pairs) atomicAdd(&sc.n_pairs, n_pairs);
#else
	sc.n_pairs += n_pairs;
#endif
	sync();
	pair = sc.pair;
	if (sc.n_pairs != 1 || (singles & ~pair)) return -1;
	uint32_t c = 0, d;
	while (!((pair >> c) & 1ull)) ++c;
	for (d = c + 1; !((pair >> d) & 1ull); ++d) {}
	uint32_t bad = 0;
	for (uint32_t b = t; b < len && !bad; b += nt)
		if (loc_syndrome(k, s, rows, blk, b, tb, sc, t) && !loc_pair_fits(k, s, rows, c, d, tb, sc, t)) bad = 1;
	loc_or32(&sc.bad, bad);
	sync();
	if (sc.bad) return -1;
	*located = pair;
	return 2;
}

}  // namespace lzd
