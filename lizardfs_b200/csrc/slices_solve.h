// slices_solve.h — the host solve of lzgpu_recover_slices: which blocks of a combined stripe the given parts of every slice of a
// goal determine, and for each determined unknown block one GF(2^8) row over a fixed set of independent parity equations.  Pure host
// code, like repair_rows.h and decode_locate.h; lzgpu_plan_recover_slices and lzgpu_debug_recover_slices_rows run it without a GPU.
//
// All slices store the same chunk, so a combined stripe of L = lcm(k_i) chunk blocks is one vector of L unknowns over GF(2^8).  A data
// part of any slice that is given pins the positions it holds (known); every given parity block of every slice stripe is one linear
// equation over the L positions (row r of that slice's generator, lz::rs_generator: Vandermonde or Cauchy).  The unknowns are the
// positions not known.  The equations restricted to the unknowns are reduced greedily to an independent set A (at most one equation
// per unknown, so at most 64), and Gauss-Jordan elimination of [A | I] gives T with T A = R in reduced row echelon form.  Unknown x is
// determined exactly when some row of R is the unit vector e_x; that row of T then maps the syndromes of A (each given parity block
// minus the known positions' share) to the block: u_x = sum_e T[x][e] S_e.
//
// The chunk's last combined stripe is short when L does not divide nb: its positions at or past `valid` are known zeros, and a slice
// stripe exists there only if its first block is a chunk block.  That shape is solved separately (the tail), and can determine more.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>

#include "fused_plan.h"  // slice_is_std, kSlicesMax
#include "host_math.h"

namespace lzd {

constexpr uint32_t kRsMaxL = 64;   // combined stripe length limit, the same as StripeBatcher's and the one-pass encoder's

// A goal set's flat part numbering: slice i's parts are base[i] .. base[i] + k[i] + m[i] - 1 (the standard slice: k = 1, m = 0)
struct SliceLayout {
	uint32_t n_slices = 0, L = 1, n_parts = 0;
	uint32_t k[kSlicesMax] = {0}, m[kSlicesMax] = {0}, base[kSlicesMax] = {0};
	uint8_t gen[kSlicesMax][32][32] = {};   // gen[i][r][j]: coefficient of data block j in parity row r of slice i
	int slice_of(uint32_t g) const {
		for (uint32_t i = 0; i < n_slices; ++i)
			if (g >= base[i] && g < base[i] + k[i] + m[i]) return static_cast<int>(i);
		return -1;
	}
};

// LZGPU_OK, or LZGPU_ERR_ARG with *why set: n_slices outside 1..4, a goal that is neither xor/ec nor the standard slice, a repeated
// slice type, no xor/ec slice, L > 64, or more than 64 parts in all
inline int slice_layout(const lzgpu_goal *goals, uint32_t n_slices, SliceLayout &out, const char **why) {
	out = SliceLayout();
	if (!goals || n_slices < 1 || n_slices > static_cast<uint32_t>(kSlicesMax)) { *why = "n_slices must be 1..4"; return LZGPU_ERR_ARG; }
	bool striped = false;
	for (uint32_t i = 0; i < n_slices; ++i) {
		const lzgpu_goal &g = goals[i];
		const bool std_slice = slice_is_std(g);
		if (!std_slice && !lzgpu_goal_valid(&g)) { *why = "a goal is neither an xor/ec goal nor the standard slice"; return LZGPU_ERR_ARG; }
		for (uint32_t j = 0; j < i; ++j)
			if (goals[j].kind == g.kind && goals[j].k == g.k && goals[j].m == g.m) { *why = "a slice type is repeated"; return LZGPU_ERR_ARG; }
		out.k[i] = static_cast<uint32_t>(g.k);
		out.m[i] = std_slice ? 0 : static_cast<uint32_t>(g.m);
		out.base[i] = out.n_parts;
		out.n_parts += out.k[i] + out.m[i];
		if (std_slice) continue;
		striped = true;
		uint32_t a = out.L, b = out.k[i];
		while (b) { const uint32_t t = a % b; a = b; b = t; }
		out.L = out.L / a * out.k[i];
		if (out.L > kRsMaxL) { *why = "the combined stripe lcm(k) is longer than 64 blocks"; return LZGPU_ERR_ARG; }
		uint8_t full[(LZGPU_MAX_DATA + LZGPU_MAX_PARITY) * LZGPU_MAX_DATA];
		lz::rs_generator(g.k, g.m, full);
		for (uint32_t r = 0; r < out.m[i]; ++r)
			for (uint32_t j = 0; j < out.k[i]; ++j) out.gen[i][r][j] = full[(out.k[i] + r) * out.k[i] + j];
	}
	if (!striped) { *why = "no xor/ec slice"; return LZGPU_ERR_ARG; }
	if (out.n_parts > LZGPU_MAX_PARTS) { *why = "more than 64 parts in all"; return LZGPU_ERR_ARG; }
	out.n_slices = n_slices;
	return LZGPU_OK;
}

// One stripe shape: positions < valid are chunk blocks, the rest known zeros
struct SliceSolve {
	uint32_t valid = 0;
	uint64_t known = 0;        // positions < valid held by a given data part
	uint64_t determined = 0;   // known, the solved unknowns, and the known zeros at or past valid
	uint32_t n_unknown = 0, n_eq = 0;
	uint8_t unk_pos[kRsMaxL] = {0};                                    // unknown x -> position, ascending
	uint8_t eq_slice[kRsMaxL] = {0}, eq_row[kRsMaxL] = {0}, eq_stripe[kRsMaxL] = {0};  // chosen equation e: slice, parity row, stripe of the slice
	uint8_t rows[kRsMaxL][kRsMaxL] = {};                               // rows[x][e]; all zero for an undetermined unknown
};

// slice i's stripe s (in the combined stripe) has a block in this shape
inline bool stripe_exists(const SliceLayout &lay, uint32_t i, uint32_t s, uint32_t valid) { return s * lay.k[i] < valid; }

inline void slice_solve(const SliceLayout &lay, const uint8_t *given, uint32_t valid, SliceSolve &out) {
	out = SliceSolve();
	out.valid = valid;
	const uint32_t L = lay.L;
	for (uint32_t i = 0; i < lay.n_slices; ++i)
		for (uint32_t j = 0; j < lay.k[i]; ++j)
			if (given[lay.base[i] + j])
				for (uint32_t q = j; q < valid; q += lay.k[i]) out.known |= 1ull << q;
	int col_of[kRsMaxL];
	for (uint32_t q = 0; q < L; ++q) {
		col_of[q] = -1;
		if (q < valid && !((out.known >> q) & 1ull)) {
			col_of[q] = static_cast<int>(out.n_unknown);
			out.unk_pos[out.n_unknown++] = static_cast<uint8_t>(q);
		}
	}
	const uint32_t U = out.n_unknown;
	// greedy independent set: basis rows kept reduced, pivot column piv[b] (its entry 1)
	uint8_t basis[kRsMaxL][kRsMaxL], A[kRsMaxL][kRsMaxL];
	int piv[kRsMaxL];
	uint32_t nb_ = 0;
	for (uint32_t i = 0; i < lay.n_slices && nb_ < U; ++i)
		for (uint32_t r = 0; r < lay.m[i] && nb_ < U; ++r) {
			if (!given[lay.base[i] + lay.k[i] + r]) continue;
			for (uint32_t s = 0; s < L / lay.k[i] && nb_ < U; ++s) {
				if (!stripe_exists(lay, i, s, valid)) continue;
				uint8_t v[kRsMaxL] = {0};
				bool any = false;
				for (uint32_t j = 0; j < lay.k[i]; ++j) {
					const int c = col_of[s * lay.k[i] + j];
					if (c >= 0 && lay.gen[i][r][j]) { v[c] = lay.gen[i][r][j]; any = true; }
				}
				if (!any) continue;
				std::memcpy(A[nb_], v, U);
				for (uint32_t b = 0; b < nb_; ++b) {
					const uint8_t f = v[piv[b]];
					if (f)
						for (uint32_t c = 0; c < U; ++c) v[c] ^= lz::gf_mul_host(f, basis[b][c]);
				}
				int p = -1;
				for (uint32_t c = 0; c < U && p < 0; ++c)
					if (v[c]) p = static_cast<int>(c);
				if (p < 0) continue;   // dependent on the equations already chosen
				const uint8_t inv = lz::gf_inv_host(v[p]);
				for (uint32_t c = 0; c < U; ++c) v[c] = lz::gf_mul_host(v[c], inv);
				std::memcpy(basis[nb_], v, U);
				piv[nb_] = p;
				out.eq_slice[nb_] = static_cast<uint8_t>(i);
				out.eq_row[nb_] = static_cast<uint8_t>(r);
				out.eq_stripe[nb_] = static_cast<uint8_t>(s);
				++nb_;
			}
		}
	const uint32_t E = nb_;
	out.n_eq = E;
	// Gauss-Jordan of [A | I] (E x (U + E)), rows of full rank
	uint8_t M[kRsMaxL][2 * kRsMaxL];
	for (uint32_t e = 0; e < E; ++e) {
		std::memset(M[e], 0, sizeof(M[e]));
		std::memcpy(M[e], A[e], U);
		M[e][U + e] = 1;
	}
	int pivot_col[kRsMaxL];
	uint32_t row = 0;
	for (uint32_t c = 0; c < U && row < E; ++c) {
		uint32_t pr = row;
		while (pr < E && !M[pr][c]) ++pr;
		if (pr == E) continue;
		if (pr != row)
			for (uint32_t j = 0; j < U + E; ++j) { const uint8_t t = M[pr][j]; M[pr][j] = M[row][j]; M[row][j] = t; }
		const uint8_t inv = lz::gf_inv_host(M[row][c]);
		for (uint32_t j = 0; j < U + E; ++j) M[row][j] = lz::gf_mul_host(M[row][j], inv);
		for (uint32_t e = 0; e < E; ++e) {
			if (e == row || !M[e][c]) continue;
			const uint8_t f = M[e][c];
			for (uint32_t j = 0; j < U + E; ++j) M[e][j] ^= lz::gf_mul_host(f, M[row][j]);
		}
		pivot_col[row++] = static_cast<int>(c);
	}
	out.determined = out.known;
	for (uint32_t q = valid; q < L; ++q) out.determined |= 1ull << q;
	for (uint32_t e = 0; e < row; ++e) {
		const uint32_t x = static_cast<uint32_t>(pivot_col[e]);
		bool unit = true;
		for (uint32_t c = 0; c < U && unit; ++c) unit = c == x || !M[e][c];
		if (!unit) continue;
		for (uint32_t f = 0; f < E; ++f) out.rows[x][f] = M[e][U + f];
		out.determined |= 1ull << out.unk_pos[x];
	}
}

// The positions of a shape the call writes: the image's, those of every block of a wanted data part, and the whole stripe of a
// wanted parity block (a parity block is computed from its stripe's data blocks)
inline uint64_t slice_needed(const SliceLayout &lay, const uint8_t *want, bool image, uint32_t valid) {
	uint64_t need = 0;
	if (image) need |= valid >= 64 ? ~0ull : ((1ull << valid) - 1ull);
	for (uint32_t i = 0; i < lay.n_slices; ++i)
		for (uint32_t g = 0; g < lay.k[i] + lay.m[i]; ++g) {
			if (!want[lay.base[i] + g]) continue;
			for (uint32_t s = 0; s < lay.L / lay.k[i]; ++s) {
				if (!stripe_exists(lay, i, s, valid)) continue;
				for (uint32_t j = 0; j < lay.k[i]; ++j) {
					const uint32_t q = s * lay.k[i] + j;
					if (q < valid && (g >= lay.k[i] || g == j)) need |= 1ull << q;
				}
			}
		}
	return need;
}

// Launch geometry of recover_slices_kernel (recover_slices_kernel.cuh), sized for the largest request the given parts allow (every
// part that is not given wanted, with its CRCs, and the image), so that it does not depend on `want`: one 256-thread CTA per SM, a
// unit of G combined stripes, shared memory = the CRC tables + one 1 KiB slab per staged block + 128 bytes per CRC stream.  SALVAGE:
// the largest salvage request instead (lzgpu_salvage_slices: nothing wanted, every given part verified, the image with its CRCs).
// CHECK (lzgpu_check_slices): every given part verified, nothing written, a slab per check's defining block (slice_check_count);
// CORRECT (lzgpu_correct_slices) stages what CHECK stages.
enum class RsMode : int { RECOVER, SALVAGE, CHECK, CORRECT };
constexpr uint32_t kRsThreadsPerCta = 256, kRsEntryCap = 192, kRsOutCap = 64;
constexpr size_t kRsSmemCap = 220 * 1024;
struct RsGeometry {
	bool ok = false;
	uint32_t G = 0, threads = 0, stages = 1, slots = 0, states = 0;
	size_t smem = 0;
};

// The checks of a shape (lzgpu_check_slices, slices_check.h): its given blocks (a data block past the chunk's end is padding, not
// one of them) less the rank, |known| + E
inline uint32_t slice_check_count(const SliceLayout &lay, const uint8_t *given, const SliceSolve &sv) {
	uint32_t n = 0;
	for (uint32_t i = 0; i < lay.n_slices; ++i)
		for (uint32_t p = 0; p < lay.k[i] + lay.m[i]; ++p) {
			if (!given[lay.base[i] + p]) continue;
			for (uint32_t s = 0; s < lay.L / lay.k[i]; ++s)
				if (stripe_exists(lay, i, s, sv.valid) && (p >= lay.k[i] || s * lay.k[i] + p < sv.valid)) ++n;
		}
	return n - static_cast<uint32_t>(__builtin_popcountll(sv.known)) - sv.n_eq;
}

inline RsGeometry rs_geometry(const SliceLayout &lay, const uint8_t *given, const SliceSolve *shapes, int n_shapes, RsMode mode = RsMode::RECOVER) {
	const bool salvage = mode == RsMode::SALVAGE, check = mode == RsMode::CHECK || mode == RsMode::CORRECT;
	RsGeometry g;
	g.G = lay.L >= 8 ? 1 : 8 / lay.L;
	g.threads = kRsThreadsPerCta;
	bool fits = true;
	for (int t = 0; t < n_shapes; ++t) {
		const SliceSolve &sv = shapes[t];
		uint32_t reads = 0, writes = sv.valid, outs = 0;
		for (uint32_t i = 0; i < lay.n_slices; ++i)
			for (uint32_t s = 0; s < lay.L / lay.k[i]; ++s) {
				if (!stripe_exists(lay, i, s, sv.valid)) continue;
				for (uint32_t p = 0; p < lay.k[i] + lay.m[i]; ++p) {
					if (given[lay.base[i] + p]) ++reads;
					else if (!salvage && !check) { ++writes; outs += p >= lay.k[i] ? 1 : 0; }
				}
			}
		if (check) {
			writes = 0;
			outs = slice_check_count(lay, given, sv);
		}
		const uint32_t states = salvage ? reads + sv.valid : check ? reads : reads + writes - sv.valid;
		fits = fits && reads <= kRsEntryCap && writes <= kRsEntryCap && states <= kRsEntryCap && outs <= kRsOutCap;
		g.slots = std::max(g.slots, lay.L + sv.n_eq + outs);
		g.states = std::max(g.states, states);
	}
	g.smem = 4096 + static_cast<size_t>(g.slots) * 1024 + static_cast<size_t>(g.states) * 128;
	g.ok = fits && g.smem <= kRsSmemCap;
	return g;
}

}  // namespace lzd
