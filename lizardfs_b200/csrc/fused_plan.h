// fused_plan.h — geometry of the fused encode kernel as pure functions (no CUDA calls): which unit mode a batch gets, how many
// stripes a unit holds, how many units there are.  Shared by the launcher (fused.cu) and the diagnostics entry point
// lzgpu_plan_encode (engine side), so the decisions are unit-tested on a machine without a GPU (tests/test_host_math.py).
#pragma once
#include <cstddef>
#include <cstdint>

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

}  // namespace lzd
