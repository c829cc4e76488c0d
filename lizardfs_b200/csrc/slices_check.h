// slices_check.h — the host side of lzgpu_check_slices: the checks of one stripe shape of a multi-slice goal, as rows over its given
// blocks, and what the locate pass needs to name a suspect part.  Pure host code, like slices_solve.h; lzgpu_plan_check_slices and
// lzgpu_debug_check_slices_rows run it without a GPU.
//
// The given blocks of a shape are every block of a given parity part in a slice stripe that exists and every block of a given data
// part at a position < valid (a data block past the chunk's end is padding, never a check).  The basis is what lzgpu_recover_slices
// solves from: the first given copy, in flat order, of each known position, and the independent parity equations slice_solve chose.
// Every other given block defines one check: the block XOR what the basis predicts for it.  A further copy of a known position is
// predicted by the first copy; a parity block by the re-encoding of its slice stripe from the basis, with the unknowns taken from a
// particular solution of the chosen equations (every pivot unknown its row of T, every free unknown 0), which slice_solve leaves out
// for the unknowns it does not determine.  Checks are numbered in flat order of their defining block (part, then stripe); there are
// given blocks - rank of them, whatever the basis.
//
// A part g explains a syndrome vector S when S lies in the span of the columns of g's blocks in the check matrix H.  The locate pass
// tests that with an annihilator per part: rows spanning {w : w H_g = 0}, so S is in the span exactly when every row maps it to 0.
//
// lzgpu_correct_slices corrects a named part g when its columns H_g have full rank (g is `correctable`): then H_g e = S has exactly one
// solution, the error of g's blocks, and e = P_g S for any left inverse P_g (P_g H_g = I).  P_g is the top of the row operations that
// bring H_g to [I; 0] (Gauss-Jordan of [H_g | I]); the rank test is the same elimination.
#pragma once
#include <cstdint>
#include <cstring>
#include <vector>

#include "slices_solve.h"

namespace lzd {

constexpr uint32_t kScMaxChecks = 64;   // bad_checks is a 64-bit mask

struct SliceChecks {
	uint32_t valid = 0, n_blocks = 0, rank = 0, n_checks = 0;   // n_checks may exceed kScMaxChecks: then only the counts are filled
	uint64_t parts = 0;                      // given parts with a block in this shape
	uint64_t checked = 0, locatable = 0;     // lzgpu_slices_check_plan's masks (locatable only when asked for)
	uint64_t correctable = 0;                // given parts with a block in the shape whose columns of H have full rank
	std::vector<uint8_t> pinv;               // [b * kScMaxChecks + h]: block b of a correctable part, coefficient of S_h in its error
	std::vector<uint8_t> blk_part, blk_s;    // given block b: flat part, stripe of the part's slice in the combined stripe
	std::vector<uint32_t> def;               // check h: its defining block
	std::vector<uint8_t> H;                  // [h * n_blocks + b]: coefficient of given block b in check h
	uint8_t prow[kRsMaxL][kRsMaxL] = {};     // [x][e]: unknown x of the particular solution from the chosen equations' syndromes
	int8_t check_of[LZGPU_MAX_PARTS][kRsMaxL];   // [g][s]: the check block s of part g defines, -1 none
	std::vector<uint8_t> ann;                // annihilator rows, kScMaxChecks bytes each (entry h: coefficient of S_h)
	uint16_t ann_first[LZGPU_MAX_PARTS + 1] = {0};   // part g's rows: ann_first[g] .. ann_first[g + 1] - 1 (none for a part not in `parts`)
};

// rank over GF(2^8) of n vectors of length len (destroys them)
inline uint32_t sc_rank(std::vector<uint8_t> &m, uint32_t n, uint32_t len) {
	uint32_t r = 0;
	for (uint32_t c = 0; c < len && r < n; ++c) {
		uint32_t p = r;
		while (p < n && !m[p * len + c]) ++p;
		if (p == n) continue;
		if (p != r)
			for (uint32_t j = 0; j < len; ++j) std::swap(m[p * len + j], m[r * len + j]);
		const uint8_t inv = lz::gf_inv_host(m[r * len + c]);
		for (uint32_t j = 0; j < len; ++j) m[r * len + j] = lz::gf_mul_host(m[r * len + j], inv);
		for (uint32_t i = 0; i < n; ++i) {
			const uint8_t f = m[i * len + c];
			if (i == r || !f) continue;
			for (uint32_t j = 0; j < len; ++j) m[i * len + j] ^= lz::gf_mul_host(f, m[r * len + j]);
		}
		++r;
	}
	return r;
}

// The columns of H for the blocks of the parts in mask, as rows of length n_checks
inline std::vector<uint8_t> sc_columns(const SliceChecks &o, uint64_t mask, uint32_t *n) {
	std::vector<uint8_t> m;
	*n = 0;
	for (uint32_t b = 0; b < o.n_blocks; ++b) {
		if (!((mask >> o.blk_part[b]) & 1ull)) continue;
		for (uint32_t h = 0; h < o.n_checks; ++h) m.push_back(o.H[h * o.n_blocks + b]);
		++*n;
	}
	return m;
}

// The checks of the shape sv (slice_solve of the same given parts).  locatable: also fill the locatable mask (pairwise rank tests; the
// call itself does not need it).
inline void slice_checks(const SliceLayout &lay, const uint8_t *given, const SliceSolve &sv, SliceChecks &o, bool locatable = false) {
	o = SliceChecks();
	std::memset(o.check_of, -1, sizeof(o.check_of));
	const uint32_t L = lay.L, valid = sv.valid, E = sv.n_eq, U = sv.n_unknown;
	o.valid = valid;
	int first[kRsMaxL], eq_blk[kRsMaxL];
	for (uint32_t q = 0; q < kRsMaxL; ++q) first[q] = eq_blk[q] = -1;
	for (uint32_t i = 0; i < lay.n_slices; ++i)
		for (uint32_t p = 0; p < lay.k[i] + lay.m[i]; ++p) {
			const uint32_t g = lay.base[i] + p;
			if (!given[g]) continue;
			for (uint32_t s = 0; s < L / lay.k[i]; ++s) {
				if (!stripe_exists(lay, i, s, valid)) continue;
				const uint32_t b = static_cast<uint32_t>(o.blk_part.size());
				if (p < lay.k[i]) {
					const uint32_t q = s * lay.k[i] + p;
					if (q >= valid) continue;   // padding
					if (first[q] < 0) first[q] = static_cast<int>(b);
				} else {
					for (uint32_t e = 0; e < E; ++e)
						if (sv.eq_slice[e] == i && sv.eq_row[e] == p - lay.k[i] && sv.eq_stripe[e] == s) eq_blk[e] = static_cast<int>(b);
				}
				o.blk_part.push_back(static_cast<uint8_t>(g));
				o.blk_s.push_back(static_cast<uint8_t>(s));
				o.parts |= 1ull << g;
			}
		}
	const uint32_t n = o.n_blocks = static_cast<uint32_t>(o.blk_part.size());
	o.rank = static_cast<uint32_t>(__builtin_popcountll(sv.known)) + E;
	o.n_checks = n - o.rank;
	if (o.n_checks > kScMaxChecks) return;

	// the particular solution: Gauss-Jordan of [A | I] over the chosen equations, as slice_solve does, keeping every pivot row
	int col_of[kRsMaxL];
	for (uint32_t q = 0; q < kRsMaxL; ++q) col_of[q] = -1;
	for (uint32_t x = 0; x < U; ++x) col_of[sv.unk_pos[x]] = static_cast<int>(x);
	std::vector<uint8_t> M(static_cast<size_t>(E) * (U + E), 0);
	const uint32_t W = U + E;
	for (uint32_t e = 0; e < E; ++e) {
		const uint32_t i = sv.eq_slice[e], r = sv.eq_row[e], s = sv.eq_stripe[e];
		for (uint32_t j = 0; j < lay.k[i]; ++j) {
			const int c = col_of[s * lay.k[i] + j];
			if (c >= 0) M[e * W + c] = lay.gen[i][r][j];
		}
		M[e * W + U + e] = 1;
	}
	uint32_t row = 0, pivot_col[kRsMaxL];
	for (uint32_t c = 0; c < U && row < E; ++c) {
		uint32_t pr = row;
		while (pr < E && !M[pr * W + c]) ++pr;
		if (pr == E) continue;
		if (pr != row)
			for (uint32_t j = 0; j < W; ++j) std::swap(M[pr * W + j], M[row * W + j]);
		const uint8_t inv = lz::gf_inv_host(M[row * W + c]);
		for (uint32_t j = 0; j < W; ++j) M[row * W + j] = lz::gf_mul_host(M[row * W + j], inv);
		for (uint32_t e = 0; e < E; ++e) {
			const uint8_t f = M[e * W + c];
			if (e == row || !f) continue;
			for (uint32_t j = 0; j < W; ++j) M[e * W + j] ^= lz::gf_mul_host(f, M[row * W + j]);
		}
		pivot_col[row++] = c;
	}
	for (uint32_t e = 0; e < row; ++e)
		for (uint32_t f = 0; f < E; ++f) o.prow[pivot_col[e]][f] = M[e * W + U + f];

	// every position of the combined stripe as a row over the given blocks: a known one its first copy, an unknown one its
	// particular solution from the syndromes S_e = (parity block of e) + (the known share of e's slice stripe), the rest 0
	std::vector<uint8_t> xh(static_cast<size_t>(L) * n, 0), syn(static_cast<size_t>(E) * n, 0);
	for (uint32_t q = 0; q < valid; ++q)
		if (first[q] >= 0) xh[q * n + first[q]] = 1;
	for (uint32_t e = 0; e < E; ++e) {
		const uint32_t i = sv.eq_slice[e], r = sv.eq_row[e], s = sv.eq_stripe[e];
		syn[e * n + eq_blk[e]] = 1;
		for (uint32_t j = 0; j < lay.k[i]; ++j) {
			const uint32_t q = s * lay.k[i] + j;
			if (q < valid && first[q] >= 0) syn[e * n + first[q]] ^= lay.gen[i][r][j];
		}
	}
	for (uint32_t x = 0; x < U; ++x)
		for (uint32_t e = 0; e < E; ++e)
			if (o.prow[x][e])
				for (uint32_t b = 0; b < n; ++b) xh[sv.unk_pos[x] * n + b] ^= lz::gf_mul_host(o.prow[x][e], syn[e * n + b]);

	// the checks, in flat order of their defining blocks
	std::vector<bool> basis(n, false);
	for (uint32_t q = 0; q < valid; ++q)
		if (first[q] >= 0) basis[first[q]] = true;
	for (uint32_t e = 0; e < E; ++e) basis[eq_blk[e]] = true;
	o.H.assign(static_cast<size_t>(o.n_checks) * n, 0);
	for (uint32_t b = 0; b < n; ++b) {
		if (basis[b]) continue;
		const uint32_t h = static_cast<uint32_t>(o.def.size());
		o.def.push_back(b);
		const uint32_t g = o.blk_part[b], s = o.blk_s[b], i = static_cast<uint32_t>(lay.slice_of(g)), p = g - lay.base[i];
		o.check_of[g][s] = static_cast<int8_t>(h);
		uint8_t *hr = &o.H[static_cast<size_t>(h) * n];
		if (p < lay.k[i]) {
			std::memcpy(hr, &xh[(s * lay.k[i] + p) * n], n);
		} else {
			for (uint32_t j = 0; j < lay.k[i]; ++j) {
				const uint32_t q = s * lay.k[i] + j;
				const uint8_t c = lay.gen[i][p - lay.k[i]][j];
				if (q < valid && c)
					for (uint32_t a = 0; a < n; ++a) hr[a] ^= lz::gf_mul_host(c, xh[q * n + a]);
			}
		}
		hr[b] ^= 1;
	}

	// checked, the annihilators, locatable
	const uint32_t nc = o.n_checks;
	for (uint32_t g = 0; g < LZGPU_MAX_PARTS; ++g) {
		o.ann_first[g + 1] = o.ann_first[g];
		if (!((o.parts >> g) & 1ull)) continue;
		bool all = true;
		for (uint32_t b = 0; b < n; ++b) {
			if (o.blk_part[b] != g) continue;
			bool any = false;
			for (uint32_t h = 0; h < nc && !any; ++h) any = o.H[h * n + b] != 0;
			all = all && any;
		}
		if (all) o.checked |= 1ull << g;
		// RREF of C = H_g^T (c x nc); the null space of C, one vector per free column, annihilates the span of g's columns
		uint32_t c;
		std::vector<uint8_t> C = sc_columns(o, 1ull << g, &c);
		const uint32_t r = sc_rank(C, c, nc);
		std::vector<int> pivot(r);
		for (uint32_t i = 0, col = 0; i < r; ++i) {
			while (!C[i * nc + col]) ++col;
			pivot[i] = static_cast<int>(col);
		}
		for (uint32_t f = 0; f < nc; ++f) {
			bool is_pivot = false;
			for (uint32_t i = 0; i < r; ++i) is_pivot |= pivot[i] == static_cast<int>(f);
			if (is_pivot) continue;
			uint8_t w[kScMaxChecks] = {0};
			w[f] = 1;
			for (uint32_t i = 0; i < r; ++i) w[pivot[i]] = C[i * nc + f];
			o.ann.insert(o.ann.end(), w, w + kScMaxChecks);
			++o.ann_first[g + 1];
		}
	}

	// correctable, the left inverses: Gauss-Jordan of [H_g | I] (nc rows), the first c rows of the right half are P_g
	o.pinv.assign(static_cast<size_t>(n) * kScMaxChecks, 0);
	for (uint32_t g = 0; g < LZGPU_MAX_PARTS; ++g) {
		if (!((o.parts >> g) & 1ull)) continue;
		uint32_t b0 = 0;
		while (o.blk_part[b0] != g) ++b0;
		uint32_t c = 0;
		while (b0 + c < n && o.blk_part[b0 + c] == g) ++c;
		if (c > nc) continue;
		const uint32_t W = c + nc;
		std::vector<uint8_t> M(static_cast<size_t>(nc) * W, 0);
		for (uint32_t h = 0; h < nc; ++h) {
			for (uint32_t j = 0; j < c; ++j) M[h * W + j] = o.H[h * n + b0 + j];
			M[h * W + c + h] = 1;
		}
		bool full = true;
		for (uint32_t j = 0; j < c && full; ++j) {
			uint32_t pr = j;
			while (pr < nc && !M[pr * W + j]) ++pr;
			if (pr == nc) { full = false; break; }
			if (pr != j)
				for (uint32_t x = 0; x < W; ++x) std::swap(M[pr * W + x], M[j * W + x]);
			const uint8_t inv = lz::gf_inv_host(M[j * W + j]);
			for (uint32_t x = 0; x < W; ++x) M[j * W + x] = lz::gf_mul_host(M[j * W + x], inv);
			for (uint32_t h = 0; h < nc; ++h) {
				const uint8_t f = M[h * W + j];
				if (h == j || !f) continue;
				for (uint32_t x = 0; x < W; ++x) M[h * W + x] ^= lz::gf_mul_host(f, M[j * W + x]);
			}
		}
		if (!full) continue;
		o.correctable |= 1ull << g;
		for (uint32_t j = 0; j < c; ++j) std::memcpy(&o.pinv[static_cast<size_t>(b0 + j) * kScMaxChecks], &M[j * W + c], nc);
	}
	if (!locatable) return;
	for (uint32_t g = 0; g < LZGPU_MAX_PARTS; ++g) {
		if (!((o.parts >> g) & 1ull)) continue;
		uint32_t cg;
		std::vector<uint8_t> Cg = sc_columns(o, 1ull << g, &cg);
		const uint32_t rg = sc_rank(Cg, cg, nc);
		bool ok = rg == cg;
		for (uint32_t g2 = 0; g2 < LZGPU_MAX_PARTS && ok; ++g2) {
			if (g2 == g || !((o.parts >> g2) & 1ull)) continue;
			uint32_t c2, c12;
			std::vector<uint8_t> C2 = sc_columns(o, 1ull << g2, &c2), C12 = sc_columns(o, (1ull << g) | (1ull << g2), &c12);
			ok = sc_rank(C12, c12, nc) == rg + sc_rank(C2, c2, nc);
		}
		if (ok) o.locatable |= 1ull << g;
	}
}

// The stripe shapes of a batch of nb blocks per chunk, for a call of `mode` and for its plan: the solve of a full combined stripe
// (shapes[0]) and of the chunk's last one when L does not divide nb (shapes[1]); for CHECK and CORRECT the checks of each shape a chunk
// has; and the launch geometry of those shapes.  plan: what the lzgpu_plan_*_slices report beyond what the call needs: the full shape's
// checks even when nb < L, and the locatable masks.
struct SliceShapes {
	SliceSolve shapes[2];
	SliceChecks checks[2];
	RsGeometry geo;
};

inline void slice_shapes(const SliceLayout &lay, const uint8_t *given, uint32_t nb, RsMode mode, SliceShapes &o, bool plan = false) {
	const uint32_t tail = nb % lay.L;
	slice_solve(lay, given, lay.L, o.shapes[0]);
	if (tail) slice_solve(lay, given, tail, o.shapes[1]);
	for (int t = 0; t < 2 && (mode == RsMode::CHECK || mode == RsMode::CORRECT); ++t)
		if (t == 0 ? plan || nb >= lay.L : tail != 0) slice_checks(lay, given, o.shapes[t], o.checks[t], plan);
	const SliceSolve used[2] = {nb >= lay.L ? o.shapes[0] : o.shapes[1], tail ? o.shapes[1] : o.shapes[0]};
	o.geo = rs_geometry(lay, given, used, 2, mode);
}

}  // namespace lzd
