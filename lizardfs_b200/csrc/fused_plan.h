// fused_plan.h — geometry of the fused encode kernel as pure functions (no CUDA calls): which unit mode a batch gets, how many
// stripes a unit holds, how many units there are; the same for the one-pass slice conversion (convert_plan), the router of the
// degraded read (recover_plan), the stripe check (check_plan) and the one-pass multi-slice encode (slices_plan).  Shared by the
// launchers (fused.cu) and the diagnostics entry points lzgpu_plan_encode, lzgpu_plan_convert, lzgpu_plan_recover, lzgpu_plan_check
// and lzgpu_plan_encode_slices (host_math.cc), so the decisions are
// unit-tested on a machine without a GPU (tests/test_host_math.py, tests/test_gpu_convert_geometry.py,
// tests/test_gpu_recover_geometry.py, tests/test_gpu_check_geometry.py).
#pragma once
#include <cstddef>
#include <cstdint>

#include "lzgpu.h"

#ifndef __CUDACC__
#define LZ_HD
#else
#define LZ_HD __host__ __device__
#endif

namespace lzd {

constexpr int kStepBytes = 128;
constexpr int kRowBytes = 16384;
constexpr int kStepsPerUnit = kRowBytes / kStepBytes;  // 128
constexpr int kConsumers = 288;                        // recover kernel: 9 warps, all consumers
constexpr int kFusedThreads = kConsumers;
constexpr int kMaxRows = 256;                          // TMA box limit per dimension
constexpr int kMaxParityRows = 128;
constexpr int kSmemCap = 113 * 1024;                   // dynamic shared memory per CTA with two CTAs per SM

// Three or four parity rows keep 12-16 Horner accumulators live next to the 64-word CRC window: at 96 registers the kernel
// spills into its inner loop (ncu: long-scoreboard stalls on the local loads).  Those
// shapes run with 8 warps instead of 9, which lets two CTAs per SM have 128 registers per thread.
// CTA shape per instantiation (parity rows M, Vandermonde or generic coefficients), each the faster one in A/B measurements on the
// previous target (same per-SM shared memory, registers and schedulers as the H100; not re-swept on the H100):
//   M <= 2            two 8-warp CTAs per SM (ec(8,2): G = 7, 252 of 256 threads carry a stream; faster than the 9-warp CTA whose
//                     ninth warp — parity CRC only — unbalances the four schedulers)
//   M == 3            two 8-warp CTAs per SM, 128 registers (12 Horner accumulators next to the 64-word CRC window spill at 96)
//   M == 4            ONE 16-warp CTA per SM (ec(8,4): G = 8, every scheduler gets two item warps and three row warps; faster than
//                     two 8-warp CTAs whose five item warps load the schedulers 2:1:1:1), deeper stage ring instead
//   generic (Cauchy)  two 9-warp CTAs; item width chosen per launch (fused_generic_item_words)
// Every value can be overridden at build time (-DLZ_T2=..., experiment builds next to the production library).
#ifndef LZ_T2
#define LZ_T2 256
#endif
#ifndef LZ_T3
#define LZ_T3 256
#endif
#ifndef LZ_T4
#define LZ_T4 512
#endif
#ifndef LZ_TGEN
#define LZ_TGEN 288      // nine warps: ec(29,4) and ec(31,4) need 2 stripes x (4k data + 16 parity) rows = 264 / 280 threads
#endif
#ifndef LZ_W3
#define LZ_W3 4
#endif
#ifndef LZ_W4
#define LZ_W4 2           // ec(8,4): 512 eight-byte items fill the 16 warps (measured faster than 16-byte items)
#endif
// Bit-sliced GF role (bitslice.cuh; measured faster than packed-word Horner for every four-row goal and for three rows on wide
// stripes): three or four Vandermonde rows on ONE 16-warp CTA per SM whose last
// ceil(16 G / 32) <= 4 warps only do the GF items (32-byte items on bit planes); the warps before them own the CRC streams.
// LZGPU_BITSLICE / LZ_BITSLICE_DEFAULT: bit 0 = four parity rows, bit 1 = three parity rows with k >= 7 (narrower stripes — ec(4,3),
// ec(5,3), ec(6,3) — measured slightly slower than the two 8-warp CTAs of the packed-byte route),
// bit 2 = three parity rows with any k (A/B).
#ifndef LZ_BITSLICE_DEFAULT
#define LZ_BITSLICE_DEFAULT 3
#endif
constexpr int kBsThreads = 512;
LZ_HD constexpr bool fused_bitslice(int m, bool generic, int mask, uint32_t k) {
	return !generic && ((m == 4 && (mask & 1)) || (m == 3 && (((mask & 2) && k >= 7) || (mask & 4))));
}
LZ_HD constexpr int fused_threads(int m, bool generic, bool bs = false) { return bs ? kBsThreads : generic ? LZ_TGEN : m <= 2 ? LZ_T2 : m == 3 ? LZ_T3 : LZ_T4; }
// packed words per GF item (4 = 16 bytes); narrower items = more, lighter items per step
// (generic coefficients: chosen per launch by fused_generic_item_words — both widths are instantiated)
LZ_HD constexpr int fused_item_words(int m, bool generic) { return generic ? 4 : m == 3 ? LZ_W3 : m == 4 ? LZ_W4 : 4; }
// Generic (Cauchy) coefficients: 16-byte items when a step has at least three warps of them (the fixed cost per item — addresses,
// narrow loads and stores — dominates otherwise: 16-byte items measured faster for ec(8,6) and ec(16,8)),
// 4-byte items when k > 20 leaves only two stripes per unit (ec(21,4): 64 sixteen-byte items would put every multiply on two warps;
// 4-byte items measured faster)
LZ_HD constexpr int fused_generic_item_words(uint32_t G) { return 32 * G >= 96 ? 4 : 1; }
// CTAs per SM: two, except for the 128-word fold window and for CTAs of more than nine warps (16 warps x 128 registers fill the
// register file on their own; their stage ring is deeper instead)
LZ_HD constexpr int fused_ctas_per_sm(int m, bool generic, int fw, bool bs = false) { return (fw != 64 || fused_threads(m, generic, bs) > 320) ? 1 : 2; }

// pipeline depth by fold window: FW = 64 -> 2 CTAs/SM (96-128 registers), 3 data stages + 4-deep parity ring (4 stages for the
// one-CTA shapes); FW = 128 -> 1 CTA/SM (the 128-word window needs ~170 registers), 6 data stages + 6-deep parity ring
#ifndef LZ_NPST
#define LZ_NPST 4
#endif
#ifndef LZ_NST_BIG
#define LZ_NST_BIG 4
#endif
LZ_HD constexpr int fused_nst(int fw, int m, bool generic, bool bs = false) { return fw != 64 ? 6 : (fused_ctas_per_sm(m, generic, fw, bs) == 1 ? LZ_NST_BIG : 3); }
LZ_HD constexpr int fused_npst(int fw, int m, bool generic) { return fw == 64 ? LZ_NPST : 6; }
LZ_HD constexpr int fused_smem_cap(int m, bool generic, int fw, bool bs = false) { return fused_ctas_per_sm(m, generic, fw, bs) == 1 ? 200 * 1024 : kSmemCap; }

inline size_t fused_smem_bytes_n(uint32_t rows, uint32_t prows, size_t nst, size_t npst) {
	const size_t pstage = (static_cast<size_t>(prows) * kStepBytes + 1023) & ~size_t(1023);
	return nst * rows * kStepBytes + npst * pstage + 520 + 8 * (2 * nst + 2 * npst);
}
inline size_t fused_smem_bytes(uint32_t rows, uint32_t prows, int fw, int m, bool generic, bool bs = false) {
	return fused_smem_bytes_n(rows, prows, fused_nst(fw, m, generic, bs), fused_npst(fw, m, generic));
}
// The bit-sliced kernels take their stage count at run time: as many stages as fit (their G is capped at 8 by the 128 GF threads,
// so narrow stripes leave shared memory for a deeper ring — more bytes in flight per SM)
#ifndef LZ_BS_MAX_STAGES
#define LZ_BS_MAX_STAGES 4   // (4 / 6 / 8 stages, 200 / 224 KB measured alike for every goal; LZGPU_BS_STAGES, LZGPU_BS_SMEM_KB)
#endif

// Largest stripe group G such that data + parity-CRC rows fit the consumer threads, the data rows fit
// one TMA box (<= 256 rows, a multiple of 8 for the 1024-byte stage alignment) and the stages fit shared memory.
#ifndef LZ_GCAP
#define LZ_GCAP 1         // on the one-CTA shapes never plan more GF items per step than the CTA has threads (ec(4,4): G = 16 would
#endif                    // give every thread two items and leave half the warps without a stream; G = 8 measured faster)
// (bit-sliced: 16 items of 32 bytes per stripe and step on the last ceil(16 g / 32) warps — at most bs_max_gf_warps of them —, the
// streams on the warps before them.  The encoders are ALU bound: a fifth or sixth GF warp only unbalances the four
// schedulers — measured slower for ec(4,4) and ec(6,4) — so four is the default;
// LZGPU_BS_GFW raises it for A/B runs.)
#ifndef LZ_BS_MAX_GF_WARPS
#define LZ_BS_MAX_GF_WARPS 4
#endif
inline uint32_t pick_group(uint32_t K, uint32_t PC, int max_smem_per_cta, int fw, uint32_t threads, int m, bool generic, bool bs = false,
                           int bs_max_gf_warps = LZ_BS_MAX_GF_WARPS) {
	uint32_t best = 0;
	const uint32_t items_per_stripe = bs ? 16u : 128u / static_cast<uint32_t>(fused_item_words(m, generic));
	for (uint32_t g = 1; g <= 64; ++g) {
		const uint32_t gf_warps = bs ? (g * items_per_stripe + 31) / 32 : 0;
		if (bs ? gf_warps > static_cast<uint32_t>(bs_max_gf_warps) : (LZ_GCAP && (threads > 288 || m >= 3) && m > 0 && best && g * items_per_stripe > threads)) break;
		const uint32_t rows = g * K * 4, prows = g * PC * 4;
		if (rows > kMaxRows || rows + prows > threads - 32 * gf_warps || prows > kMaxParityRows || g * K > 64) break;
		if (rows % 8) continue;
		if (fused_smem_bytes(rows, prows, fw, m, generic, bs) > static_cast<size_t>(max_smem_per_cta)) break;
		best = g;
	}
	return best;
}

// Unit geometry of one launch.  mode 0: a unit is G stripes of ONE chunk (out-of-range rows zero-filled by TMA);
// mode 1 ("flat"): chunks are contiguous and made of whole stripes, the batch is one run of n_chunks*pb stripes in one
// 2-D tensor; mode 2 ("striped"): the same run of global stripes for any nb / stride, one TMA box per stripe.
struct FusedPlan {
	uint32_t G = 0, pb = 0, mode = 0, units_per_chunk = 0, total_units = 0, threads = 0, rows = 0, prows = 0, n_stages = 0;
	size_t smem = 0;
	bool ok = false;  // false: the fused kernel does not take this shape (generic kernels do)
	bool bs = false;  // bit-sliced geometry (16 warps, four of them GF warps)
};

// striped_policy: -1 automatic (striped when per-chunk units would leave more than 12 % of their stripe slots empty — measured:
// G boxes per step instead of one cost a few per cent at 64 MiB and win by a wide margin at 1-4 MiB), 0 never, 1 always
inline FusedPlan fused_plan(int M, bool generic, uint32_t K, uint32_t n_chunks, uint32_t nb, size_t chunk_stride, int smem_cap, int fw,
                            int striped_policy, bool bs = false, int bs_max_stages = LZ_BS_MAX_STAGES, int bs_max_gf_warps = LZ_BS_MAX_GF_WARPS) {
	FusedPlan pl;
	const uint32_t PC = M == 0 ? 0 : (generic ? M : M - 1);
	const int mm = M;  // the instantiation's M (thread count, stage depth); a Cauchy generator is encoded in passes of <= 4 rows
	pl.threads = static_cast<uint32_t>(fused_threads(mm, generic, bs));
	pl.bs = bs;
	pl.G = pick_group(K, PC, smem_cap, fw, pl.threads, mm, generic, bs, bs_max_gf_warps);
	if (pl.G == 0 || (chunk_stride % 16)) return pl;
	const uint32_t G = pl.G;
	pl.pb = (nb + K - 1) / K;
	const bool flat = n_chunks > 1 && chunk_stride == static_cast<size_t>(nb) * 65536u && nb % K == 0 &&
	                  static_cast<uint64_t>(n_chunks) * pl.pb < (1ull << 31) && static_cast<uint64_t>(n_chunks) * nb * 4 < (1ull << 31);  // TMA coordinates are int32
	pl.mode = flat ? 1u : 0u;
	if (!flat && M > 0 && static_cast<uint64_t>(n_chunks) * pl.pb < (1ull << 31) && static_cast<uint64_t>(nb) * 4 < (1ull << 31)) {
		const uint64_t per_chunk_slots = static_cast<uint64_t>((pl.pb + G - 1) / G) * G * n_chunks;
		const uint64_t stripes = static_cast<uint64_t>(n_chunks) * pl.pb;
		const bool wasteful = per_chunk_slots * 100 > stripes * 112;
		if (striped_policy == 1 || (striped_policy < 0 && wasteful)) pl.mode = 2u;
	}
	uint64_t total;
	if (pl.mode != 0) {
		pl.units_per_chunk = static_cast<uint32_t>((static_cast<uint64_t>(n_chunks) * pl.pb + G - 1) / G);
		total = pl.units_per_chunk;
	} else {
		pl.units_per_chunk = (pl.pb + G - 1) / G;
		total = static_cast<uint64_t>(pl.units_per_chunk) * n_chunks;
	}
	if (total > 0x7fffffffull) return pl;
	pl.total_units = static_cast<uint32_t>(total);
	pl.rows = G * K * 4;
	pl.prows = G * PC * 4;
	pl.n_stages = static_cast<uint32_t>(fused_nst(fw, mm, generic, bs));
	const size_t npst = fused_npst(fw, mm, generic);
	if (bs)
		while (static_cast<int>(pl.n_stages) < bs_max_stages && fused_smem_bytes_n(pl.rows, pl.prows, pl.n_stages + 1, npst) <= static_cast<size_t>(smem_cap)) ++pl.n_stages;
	pl.smem = fused_smem_bytes_n(pl.rows, pl.prows, pl.n_stages, npst);
	pl.ok = true;
	return pl;
}

// ---------------------------------------------------------------------------------------------------
// One-pass slice conversion (convert_kernel.cuh): geometry as a pure function, shared by lz_fused_convert and lzgpu_plan_convert.
// A unit is G destination stripes = T source stripes (G*Kd == T*Ks chunk blocks); worker warps own one CRC row per thread (the R*4
// data rows, e*T*4 source parity rows, G*(Md-1)*4 staged destination parity rows) and the 32 G destination items, with lost parts
// the remaining warps only rebuild.  G is the candidate with the lowest estimated instruction count per chunk block on the busier role.
// ---------------------------------------------------------------------------------------------------
constexpr int kConvertThreads = 256;
constexpr int kConvertNPST = 4;

struct ConvertPlan {
	bool ok = false;
	uint32_t G = 0, T = 0, region_rows = 0, n_stages = 0, n_workers = 0;
	uint32_t e = 0;            // lost source data parts (0..2)
	uint8_t erased[2] = {0, 0};
	size_t smem = 0;
};

// available[i] != 0: part i of the source slice (data parts first, then parity parts) can be read.  The kernel takes Vandermonde
// sources with at most two data parts lost whose first-k-available rule (ec_read_plan.h:126-133) brings in parity rows 0 .. e-1 in
// this order, and Vandermonde destinations with one to three parity parts.
inline ConvertPlan convert_plan(int Ks, int Ms, bool src_cauchy, int Kd, int Md, bool dst_cauchy, const uint8_t *available, int max_smem) {
	ConvertPlan pl;
	if (src_cauchy || dst_cauchy || Md < 1 || Md > 3 || Ks < 1 || Ks > 32 || Kd < 1 || Kd > 32) return pl;
	int n_used = 0, n_par = 0;
	bool present[32] = {false};
	for (int i = 0; i < Ks + Ms && n_used < Ks; ++i) {
		if (!available[i]) continue;
		++n_used;
		if (i < Ks) present[i] = true;
		else if (i == Ks + n_par && n_par < 2) ++n_par;   // parity rows 0, 1 in this order only
		else return pl;
	}
	if (n_used < Ks) return pl;
	uint32_t e = 0;
	for (int j = 0; j < Ks; ++j)
		if (!present[j]) {
			if (e >= 2) return pl;
			pl.erased[e++] = static_cast<uint8_t>(j);
		}
	if (static_cast<int>(e) != n_par) return pl;
	pl.e = e;
	uint32_t a = static_cast<uint32_t>(Ks), b = static_cast<uint32_t>(Kd);
	while (b) { const uint32_t t = a % b; a = b; b = t; }
	const uint32_t g0 = static_cast<uint32_t>(Ks) / a, PC = static_cast<uint32_t>(Md - 1);
	const size_t cap = static_cast<size_t>(max_smem < kSmemCap ? max_smem : kSmemCap);
	double best_cost = 0;
	for (uint32_t g = g0; g <= 64; g += g0) {
		const uint32_t R = g * Kd, t = R / Ks;
		const uint32_t rows = R * 4 + e * t * 4 + g * PC * 4;
		// worker warps own the rows; with lost parts at least one warp is left for the rebuild
		if (R > 64 || t * 4 > 256 || rows > static_cast<uint32_t>(kConvertThreads) - (e ? 32u : 0u)) break;
		const uint32_t rr = (t * 4 + 7) & ~7u;
		const size_t stage = static_cast<size_t>(Ks + e) * rr * kStepBytes;
		const size_t pstage = (static_cast<size_t>(g) * PC * 4 * kStepBytes + 1023) & ~size_t(1023);
		const size_t fixed = kConvertNPST * pstage + 520 + 8 * (2 * kConvertNPST) + 64;
		uint32_t ns = 0;
		for (uint32_t n = 4; n >= 2; --n)
			if (n * stage + 24 * n + fixed <= cap) { ns = n; break; }
		if (!ns) break;
		// instructions per thread and step of the busier role, per chunk block of the unit (rough counts; only the ordering matters):
		// a worker thread folds one row (~140) and takes its share of the 32 g destination items (~35 per block of the stripe + stores),
		// a rebuild thread its share of the 32 t source-stripe items (Horner over Ks columns; two syndromes and the solve when e = 2)
		const uint32_t n_wk = e ? (rows + 31) / 32 : kConvertThreads / 32, n_rb = kConvertThreads / 32 - n_wk;
		const double worker = 140.0 + static_cast<double>((g + n_wk - 1) / n_wk) * (35.0 * Kd + 20.0);
		const double rebuild = e ? static_cast<double>((t + n_rb - 1) / n_rb) * (e == 2 ? 30.0 * Ks + 150.0 : 6.0 * Ks + 20.0) : 0.0;
		const double cost = (worker > rebuild ? worker : rebuild) / R;
		if (!pl.ok || cost < best_cost) {
			best_cost = cost;
			pl.ok = true;
			pl.G = g; pl.T = t; pl.region_rows = rr; pl.n_stages = ns; pl.n_workers = n_wk;
			pl.smem = ns * stage + 24 * ns + fixed;
		}
	}
	return pl;
}

// ---------------------------------------------------------------------------------------------------
// One-pass encode of every slice of a goal (slices_kernel.cuh): geometry as a pure function, shared by lz_fused_encode_slices and
// lzgpu_plan_encode_slices.  A unit is G combined stripes of one chunk, R = G*L consecutive chunk blocks (L = lcm of the striped
// slices' k), one TMA box of 4R quarter-rows per step (4R <= 256).  One 16-warp CTA per SM: thread t < 4R owns data row t, the
// next rows are the staged parity rows 1 .. m_i - 1 of every stripe of every slice; every thread takes GF items.
// G: the largest whose CRC rows fit the CTA and whose stages fit the shared memory, capped by ceil(nb / L) so that a batch of
// short chunks gets no units it cannot fill; then as many stages as fit, at most four.
// ---------------------------------------------------------------------------------------------------
constexpr int kSlicesThreads = 512;
constexpr int kSlicesNPST = 4;                 // parity staging ring
constexpr int kSlicesMaxStages = 4;
constexpr int kSlicesSmemCap = 200 * 1024;
constexpr int kSlicesMax = 4;                  // slices per call: the size of the parameter block's per-slice arrays
constexpr int kSlicesMaxStripes = 128;         // stripes of all slices per unit: at most 4 x 64 / 2
LZ_HD constexpr int slices_item_words(int m) { return m >= 3 ? 2 : 4; }   // 8-byte items for three or four rows (16 accumulators next to the CRC window spill)

inline size_t slices_smem_bytes(uint32_t R, uint32_t prows, uint32_t nst) {
	const size_t stage = (static_cast<size_t>(R) * 4 * kStepBytes + 1023) & ~size_t(1023);
	const size_t pstage = (static_cast<size_t>(prows) * kStepBytes + 1023) & ~size_t(1023);
	return nst * stage + kSlicesNPST * pstage + 520 + 8 * (2 * nst + 2 * kSlicesNPST);
}

inline bool slice_is_std(const lzgpu_goal &g) { return g.kind == LZGPU_KIND_STD && g.k == 1 && g.m == 0; }

struct SlicesPlan {
	lzgpu_slices_plan out{};
	uint32_t m = 0;                 // the instantiation: the largest m of the striped slices
	uint32_t R = 0, prows = 0;      // chunk blocks per unit, staged parity rows
	uint32_t S[kSlicesMax] = {0};   // stripes of slice i per unit (0: standard slice)
};

// goals: valid xor/ec goals or the standard slice, at least one striped (the caller checks); cauchy[i]: slice i has a Cauchy generator
inline SlicesPlan slices_plan(const lzgpu_goal *goals, const bool *cauchy, uint32_t n_slices, uint32_t n_chunks, uint32_t nb) {
	SlicesPlan pl;
	lzgpu_slices_plan &o = pl.out;
	uint32_t n_striped = 0, L = 1;
	bool any_cauchy = false;
	for (uint32_t i = 0; i < n_slices; ++i) {
		if (slice_is_std(goals[i])) continue;
		++n_striped;
		any_cauchy |= cauchy[i];
		const uint32_t k = static_cast<uint32_t>(goals[i].k);
		uint32_t a = L, b = k;
		while (b) { const uint32_t t = a % b; a = b; b = t; }
		L = L / a * k;                     // k <= 32 and at most four slices: no overflow
		pl.m = pl.m > static_cast<uint32_t>(goals[i].m) ? pl.m : static_cast<uint32_t>(goals[i].m);
	}
	o.L = L;
	if (n_striped < 2) { o.refusal = LZGPU_SLICES_REFUSED_SINGLE; return pl; }
	if (any_cauchy) { o.refusal = LZGPU_SLICES_REFUSED_CAUCHY; return pl; }
	if (L > 64) { o.refusal = LZGPU_SLICES_REFUSED_WIDE; return pl; }
	auto prows_of = [&](uint32_t R) {
		uint32_t rows = 0;
		for (uint32_t i = 0; i < n_slices; ++i)
			if (!slice_is_std(goals[i])) rows += R / static_cast<uint32_t>(goals[i].k) * static_cast<uint32_t>(goals[i].m - 1) * 4;
		return rows;
	};
	uint32_t G = 0;
	for (uint32_t g = 1; g * L <= 64; ++g) {
		const uint32_t R = g * L, prows = prows_of(R);
		if (4 * R + prows > static_cast<uint32_t>(kSlicesThreads) || slices_smem_bytes(R, prows, 2) > static_cast<size_t>(kSlicesSmemCap)) break;
		G = g;
	}
	if (G == 0) { o.refusal = LZGPU_SLICES_REFUSED_NO_GEOMETRY; return pl; }
	const uint32_t per_chunk = (nb + L - 1) / L;
	if (G > per_chunk) G = per_chunk;
	pl.R = G * L;
	pl.prows = prows_of(pl.R);
	uint32_t nst = 2;
	while (nst < static_cast<uint32_t>(kSlicesMaxStages) && slices_smem_bytes(pl.R, pl.prows, nst + 1) <= static_cast<size_t>(kSlicesSmemCap)) ++nst;
	const uint64_t units = static_cast<uint64_t>((nb + pl.R - 1) / pl.R) * n_chunks;
	if (units > 0x7fffffffull) { o.refusal = LZGPU_SLICES_REFUSED_NO_GEOMETRY; return pl; }
	for (uint32_t i = 0; i < n_slices; ++i) pl.S[i] = slice_is_std(goals[i]) ? 0 : pl.R / static_cast<uint32_t>(goals[i].k);
	o.fused = 1;
	o.G = G;
	o.threads = kSlicesThreads;
	o.stages = nst;
	o.crc_rows = 4 * pl.R + pl.prows;
	o.smem_bytes = static_cast<uint32_t>(slices_smem_bytes(pl.R, pl.prows, nst));
	o.units = static_cast<uint32_t>(units);
	return pl;
}

// ---------------------------------------------------------------------------------------------------
// Fused degraded read (fused_recover_kernel, fused_kernel.cuh; bs_recover3_kernel, bs_recover_kernel.cuh): the router as a pure
// function, shared by lz_fused_recover (which dispatches on its fields alone) and lzgpu_plan_recover.
// ---------------------------------------------------------------------------------------------------
constexpr int kRecoverSmemCap = 200 * 1024;     // GEO 0: one 9-warp CTA per SM, 6 stages
constexpr int kRecoverSmemCap2 = 100 * 1024;    // GEO 1: two 9-warp CTAs per SM, 3 stages (E <= 2)
constexpr int kRecoverSmemCapBig = 208 * 1024;  // GEO 2, DIRECT, bs_recover3: one 16-warp CTA per SM
constexpr int kBsRecoverThreads = 512;
LZ_HD constexpr int recover_stages(int geo) { return geo == 1 ? 3 : 6; }
LZ_HD constexpr int recover_threads(int geo) { return geo == 2 ? 512 : kFusedThreads; }
#ifndef LZ_RW3
#define LZ_RW3 2   // words per GF item for three or four erased parts on the 16-warp geometry (narrower items = fewer live accumulators)
#endif
LZ_HD constexpr int recover_item_words(int e, int geo) { return (geo == 2 && e >= 3) ? LZ_RW3 : 4; }
// wide items of the DIRECT degraded read: 16 bytes for one rebuilt part, 8 for more (e x 4 accumulators next to the CRC window spill at 128 registers)
LZ_HD constexpr int direct_wide_words(int e) { return e >= 2 ? 2 : 4; }

// the one-CTA 16-warp routes (GEO 2, DIRECT, bs_recover3): as many stages as fit 208 KiB, at most six
inline uint32_t recover_big_stages(uint32_t K, uint32_t G) {
	const size_t fit = (kRecoverSmemCapBig - 256) / (static_cast<size_t>(K) * G * 4 * kStepBytes);
	return static_cast<uint32_t>(fit < 6 ? fit : 6);
}

#ifndef LZ_BS_RECOVER_DEFAULT
#define LZ_BS_RECOVER_DEFAULT 1
#endif
// the context switches the router reads (lzgpu_recover_switches; the defaults are the build's)
inline lzgpu_recover_switches recover_switches_default() {
	lzgpu_recover_switches s;
	s.recover_geo = -1;
	s.recover_two = -1;
	s.recover_k3 = 1;
	s.bs_recover = LZ_BS_RECOVER_DEFAULT;
	s.bs_recover_gf_warps = 8;
	s.direct_wide = -1;
	return s;
}

struct RecoverPlan {
	lzgpu_recover_plan out{};         // what lzgpu_plan_recover reports (refusal, kernel, instantiation, geometry)
	int used[LZGPU_MAX_DATA] = {0};   // slot a -> part index: the first k available parts (ec_read_plan.h:126-133)
	uint8_t erased_idx[4] = {0};      // data index of lost part x, ascending
	uint8_t par_slot[4] = {0}, par_row[4] = {0};  // parity parts in use: slot and generator row, ascending
	int geo = 0;                      // packed-word geometry (0, 1, 2) of the fused_recover_kernel routes
	bool wide = false;                // DIRECT: 8- / 16-byte items (else 4)
};

// available[i]: part i (data parts first) can be read.  want_missing_parity: a wanted parity part that is not available has an
// output buffer (only lost data parts are rebuilt here).  verify: some part read has stored CRCs.  image: a chunk-order image is
// written.
inline RecoverPlan recover_plan(int K, int M, bool cauchy, const uint8_t *available, bool want_missing_parity, bool verify, bool image,
                                const lzgpu_recover_switches &sw) {
	RecoverPlan pl;
	lzgpu_recover_plan &o = pl.out;
	o.doublings = -1;
	const bool direct = cauchy;   // no Horner syndromes for a Cauchy generator: general rows over the k inputs
	if (direct && sw.direct_wide == -2) { o.refusal = LZGPU_RECOVER_REFUSED_DIRECT_OFF; return pl; }   // A/B against the generic route
	const bool direct_forced = direct && sw.direct_wide >= 0;
	int n_used = 0;
	for (int i = 0; i < K + M && n_used < K; ++i)
		if (available[i]) pl.used[n_used++] = i;
	if (n_used < K) { o.refusal = LZGPU_RECOVER_REFUSED_TOO_FEW_PARTS; return pl; }
	bool present[LZGPU_MAX_DATA] = {false};
	uint32_t e = 0, n_par = 0;
	for (int a = 0; a < K; ++a) {
		const int idx = pl.used[a];
		if (idx < K) present[idx] = true;
		else if (n_par < 4) { pl.par_slot[n_par] = static_cast<uint8_t>(a); pl.par_row[n_par] = static_cast<uint8_t>(idx - K); ++n_par; }
		else { o.refusal = LZGPU_RECOVER_REFUSED_OVER_FOUR_LOST; return pl; }
	}
	for (int j = 0; j < K; ++j)
		if (!present[j]) {
			if (e >= 4) { o.refusal = LZGPU_RECOVER_REFUSED_OVER_FOUR_LOST; return pl; }
			pl.erased_idx[e++] = static_cast<uint8_t>(j);
		}
	o.lost_data_parts = e;
	if (e == 0 || e != n_par) { o.refusal = LZGPU_RECOVER_REFUSED_NO_LOST_DATA; return pl; }
	// Measured: with general coefficients the rebuild is bound by the bit-plane multiplies, not by HBM, and
	// the grid-stride gf_dot_kernel (full occupancy, no stage barriers) does e >= 2 rows faster than this kernel's 16 warps per SM
	// even though it needs separate CRC and image passes.  One lost part, and two lost parts when the call verifies and wants the
	// image, measured faster here and stay here.
	if (direct && !direct_forced && !(e == 1 || (e == 2 && verify && image))) { o.refusal = LZGPU_RECOVER_REFUSED_DIRECT_SLOWER; return pl; }
	// every requested missing part must be a data part
	if (want_missing_parity) { o.refusal = LZGPU_RECOVER_REFUSED_PARITY_WANTED; return pl; }
	// geometry: even G (1024-byte aligned slot regions), K*G*4 rows <= 256
	// Two CTAs per SM with a 3-stage ring, or one CTA with 6 stages?  Measured with 64 MiB chunks: two CTAs win for the runtime-k
	// shapes, except the single-erasure case that also writes the image; the k = 8 instantiation keeps one.  LZGPU_RECOVER_TWO=0|1 forces either.
	const bool two_auto = K != 8 && (e == 2 || (e == 1 && !image));
	const bool two = e <= 2 && (sw.recover_two < 0 ? two_auto : sw.recover_two != 0);
	// Measured (recover only and verify + image): the 16-warp CTA wins for the runtime-k shapes with two or more erased parts, against
	// two 9-warp CTAs and against one, while the k = 8 instantiation keeps one 9-warp CTA with six stages.  LZGPU_RECOVER_GEO=0|1|2 forces one.
	int geo = sw.recover_geo >= 0 ? sw.recover_geo : (K != 8 && e >= 2) ? 2 : (two ? 1 : 0);
	if (direct) geo = 2;
	if (geo == 1 && e > 2) geo = 0;
	// three lost data parts with parity rows 0, 1, 2 in use: bit planes + dedicated GF warps (bs_recover_kernel.cuh) — geometry: G even,
	// the 16 G items of a step on the last ceil(16 G / 32) warps, the k G 4 input rows on the warps before them when the call verifies
	// stored CRCs (no stream warps otherwise), one TMA box per part (G 4 <= 256 rows), at least three stages
	bool bs3 = !direct && e == 3 && sw.bs_recover && pl.par_row[0] == 0 && pl.par_row[1] == 1 && pl.par_row[2] == 2;
	uint32_t G = 0, n_stages = 0;
	const uint32_t UK = static_cast<uint32_t>(K);
	if (bs3) {
		// Measured with at most four against at most eight GF warps: more GF warps win for rebuild only (no stream warps, G = 16, eight
		// GF warps) and with verification and image for ec(5,3) (seven) and ec(6,3) (six), but ec(8,3) loses with five (one scheduler
		// gets two of them).  So: the largest G, unless it only buys a fifth GF warp.
		uint32_t g4 = 0;
		for (uint32_t g = 2; g <= 64; g += 2) {
			const size_t stage = static_cast<size_t>(UK) * g * 4 * kStepBytes;
			const uint32_t gf_warps = (16 * g + 31) / 32, stream_warps = verify ? (UK * g * 4 + 31) / 32 : 0;
			if (gf_warps > static_cast<uint32_t>(sw.bs_recover_gf_warps) || gf_warps + stream_warps > kBsRecoverThreads / 32 || 3 * stage + 256 > static_cast<size_t>(kRecoverSmemCapBig)) break;
			G = g;
			if (gf_warps <= 4) g4 = g;
		}
		if (G && g4 && (16 * G + 31) / 32 == 5) G = g4;
		if (G) n_stages = recover_big_stages(UK, G);
		else bs3 = false;
	}
	if (bs3) {
		// (geometry chosen above)
	} else if (geo == 2) {
		// one 16-warp CTA: the largest G whose K*G*4 input rows fit 512 threads (one TMA box per part: G*4 <= 256 rows) and whose
		// 32*G items fill whole rounds of the CTA (G a multiple of 16) where K allows, with at least three stages in 208 KiB
		uint32_t best = 0, best16 = 0;
		for (uint32_t g = 2; g <= 64; g += 2) {
			const uint32_t rows = UK * g * 4;
			if (rows > 512 || 3 * static_cast<size_t>(rows) * kStepBytes + 256 > kRecoverSmemCapBig) break;
			best = g;
			if (g % 16 == 0) best16 = g;
		}
		G = best16 ? best16 : best;
		if (G) n_stages = recover_big_stages(UK, G);
	} else {
		n_stages = static_cast<uint32_t>(recover_stages(geo));
		const size_t smem_cap = geo == 1 ? kRecoverSmemCap2 : kRecoverSmemCap;
		for (uint32_t g = 2; g <= 64; g += 2) {
			const uint32_t rows = UK * g * 4;
			if (rows > kMaxRows || static_cast<size_t>(n_stages) * rows * kStepBytes + 256 > smem_cap) break;
			G = g;
		}
	}
	if (G == 0) { o.refusal = LZGPU_RECOVER_REFUSED_NO_GEOMETRY; return pl; }
	pl.geo = geo;
	o.fused = 1;
	o.G = G;
	o.stages = n_stages;
	o.smem_bytes = static_cast<uint32_t>(static_cast<size_t>(n_stages) * UK * G * 4 * kStepBytes + 16 * n_stages + 64);
	bool consecutive = true;   // parity rows 0, 1, .., e-1 in use (the first e parity parts are the available ones — the common case)
	for (uint32_t r = 0; r < e; ++r) consecutive &= pl.par_row[r] == r;
	const bool row0 = pl.par_row[0] == 0, row01 = e >= 2 && consecutive;
	const int x0 = pl.erased_idx[0];
	if (bs3) {
		o.kernel = LZGPU_KERNEL_RECOVER_BS3;
		o.kt = (K == 5 || K == 8) ? static_cast<uint32_t>(K) : 0;
		o.rows = LZGPU_RECOVER_ROWS_FIRST_E;
		o.item_bytes = 32;
		o.solve = LZGPU_RECOVER_SOLVE_ELIM3;
		o.doublings = x0 <= 3 ? x0 : -1;
		o.threads = kBsRecoverThreads;
		o.gf_warps = (16 * G + 31) / 32;
		return pl;
	}
	if (direct) {
		// item width: 16-byte items leave most of the 16 warps without work when k is large (G small)
		// the 8 / 16-byte items measured faster on every shape; 4-byte items stay for A/B
		pl.wide = sw.direct_wide >= 0 ? sw.direct_wide != 0 : true;
		o.kernel = LZGPU_KERNEL_RECOVER_DIRECT;
		o.rows = LZGPU_RECOVER_ROWS_DIRECT;
		o.item_bytes = 4 * (pl.wide ? direct_wide_words(static_cast<int>(e)) : 1);
		o.solve = LZGPU_RECOVER_SOLVE_DIRECT;
		o.threads = recover_threads(2);
		return pl;
	}
	o.kernel = geo == 2 ? LZGPU_KERNEL_RECOVER_GEO2 : geo == 1 ? LZGPU_KERNEL_RECOVER_GEO1 : LZGPU_KERNEL_RECOVER_GEO0;
	o.threads = static_cast<uint32_t>(recover_threads(geo));
	o.item_bytes = 4 * recover_item_words(static_cast<int>(e), geo);
	o.rows = e == 1 ? (row0 ? LZGPU_RECOVER_ROWS_FIRST_E : LZGPU_RECOVER_ROWS_GENERAL) : (row01 ? LZGPU_RECOVER_ROWS_FIRST_E : LZGPU_RECOVER_ROWS_GENERAL);
	// compile-time k (the walk over the columns unrolls, parameter loads become immediates):
	// ec(3,2) / ec(5,3) on the 16-warp geometry, measured faster than the runtime-k kernel for ec(3,2), most of all for rebuild only.
	// ec(5,3): two lost, faster for rebuild only but slower with verification and image (the unrolled walk costs the CRC role
	// registers), so that combination keeps the runtime-k kernel; three lost faster either way.  ec(4,2), ec(6,2), ec(6,3): the same
	// rule as for k = 5.  k = 8 (G = 8 or the 16-warp geometry): one and two lost parts with rows 0 (0, 1) in use.
	const bool k8 = K == 8 && (G == 8 || geo == 2);
	const bool vi = verify && image;
	if (geo == 2 && sw.recover_k3 && ((K == 3 && ((e == 1 && row0) || (e == 2 && row01))) || ((K == 4 || K == 5 || K == 6) && e == 2 && row01 && !vi) ||
	                                  ((K == 5 || K == 6) && e == 3 && row01)))
		o.kt = static_cast<uint32_t>(K);
	else if (k8 && e <= 2 && o.rows == LZGPU_RECOVER_ROWS_FIRST_E)
		o.kt = 8;
	// the form of the solve (fused_recover_kernel): RAID-6 elimination for two unknowns with rows 0, 1 (not the k = 8 instantiation:
	// there the two bit-plane multiplies measured faster), x0 doublings for 2^x0 S0 up to x0 = 4, else the multiply by w[0]; the
	// three-unknown elimination with rows 0, 1, 2, x0 doublings up to x0 = 3, else the multiplies by w[4], w[5]; otherwise
	// d = V^-1 S, where row 0 known at compile time makes the last unknown S0 ^ (the others)
	if (e == 2 && row01 && o.kt != 8) {
		o.solve = LZGPU_RECOVER_SOLVE_RAID6;
		o.doublings = x0 <= 4 ? x0 : -1;
	} else if (e == 3 && row01) {
		o.solve = LZGPU_RECOVER_SOLVE_ELIM3;
		o.doublings = x0 <= 3 ? x0 : -1;
	} else {
		o.solve = o.rows == LZGPU_RECOVER_ROWS_FIRST_E ? LZGPU_RECOVER_SOLVE_INVERSE_ROW0 : LZGPU_RECOVER_SOLVE_INVERSE;
	}
	return pl;
}

// ---------------------------------------------------------------------------------------------------
// Fused stripe check (fused_check_kernel / fused_check_map_kernel, check_kernel.cuh): the geometry as a pure function, shared by
// lz_fused_check (which launches exactly what it returns) and lzgpu_plan_check.
// ---------------------------------------------------------------------------------------------------
constexpr int kCheckThreads = 512;

struct CheckPlan {
	lzgpu_check_plan out{};      // what lzgpu_plan_check reports
	uint8_t row[4] = {0};        // generator row of checked parity slot K + r (fused only)
};

// given[i]: part i is given (data parts first).  A missing data part has no slot (fused_check_degraded_kernel; the degraded calls
// guarantee more given parity rows than lost data parts).  One 16-warp CTA per SM: the largest even G whose NSLOT*G*4 rows give
// every row a thread (one TMA box per part: G*4 <= 256 rows), NSLOT = given data parts + R, with at least three stages in the
// shared-memory budget; then as many stages as fit, at most six.
inline CheckPlan check_plan(int K, int M, bool cauchy, const uint8_t *given) {
	CheckPlan pl;
	lzgpu_check_plan &o = pl.out;
	uint32_t D = 0, R = 0;
	for (int j = 0; j < K; ++j) D += given[j] ? 1u : 0u;
	bool consecutive = true;
	for (int r = 0; r < M; ++r) {
		if (!given[K + r]) continue;
		consecutive &= static_cast<int>(R) == r;
		if (R < 4) pl.row[R] = static_cast<uint8_t>(r);
		++R;
	}
	o.rows = R;
	o.consecutive = consecutive ? 1 : 0;
	if (cauchy || R == 0 || R > 4 || D + R <= static_cast<uint32_t>(K)) return pl;
	const uint32_t NSLOT = D + R;
	uint32_t G = 0;
	for (uint32_t g = 2; g <= 64; g += 2) {
		const uint32_t rows = NSLOT * g * 4;
		if (rows > static_cast<uint32_t>(kCheckThreads) || 3 * static_cast<size_t>(rows) * kStepBytes + 256 > static_cast<size_t>(kRecoverSmemCapBig)) break;
		G = g;
	}
	if (G == 0) return pl;
	const size_t fit = (kRecoverSmemCapBig - 256) / (static_cast<size_t>(NSLOT) * G * 4 * kStepBytes);
	const uint32_t n_stages = static_cast<uint32_t>(fit < 6 ? fit : 6);
	o.fused = 1;
	o.G = G;
	o.stages = n_stages;
	o.threads = kCheckThreads;
	o.item_passes = (32 * G + kCheckThreads - 1) / kCheckThreads;
	o.smem_bytes = static_cast<uint32_t>(static_cast<size_t>(n_stages) * NSLOT * G * 4 * kStepBytes + 16 * n_stages + 64);
	return pl;
}

}  // namespace lzd
