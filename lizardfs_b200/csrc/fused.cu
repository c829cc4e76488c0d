// fused.cu — host side of the TMA-streamed fused kernels (fused_kernel.cuh): tensor-map creation,
// work-unit geometry, launch.  Returns LZGPU_NOT_HANDLED for shapes the fused path does not cover
// (engine.cu then uses the generic kernels).
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <numeric>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>

#include "engine_internal.h"
#include "fused_kernel.cuh"
#include "convert_kernel.cuh"
#include "bs_recover_kernel.cuh"
#include "check_kernel.cuh"
#include "slices_kernel.cuh"
#include "recover_slices_kernel.cuh"
#include "slices_check.h"
#include "host_math.h"

using namespace lzd;

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct FusedState {
	EncodeTiledFn encode_tiled = nullptr;
	uint32_t qmult[4];
	int max_smem = 0;
	bool disabled = false;
	uint32_t probe = 0;
	uint32_t *d_sm_ctr = nullptr;
	int evict_first = 0;
	int striped = -1;
	// LZGPU_RECOVER_TWO, LZGPU_RECOVER_GEO, LZGPU_RECOVER_K3, LZGPU_BS_RECOVER, LZGPU_BS_RECOVER_GFW, LZGPU_DIRECT_WIDE: the degraded read's
	// router switches (lzgpu_recover_switches, lzgpu.h)
	lzgpu_recover_switches recover = recover_switches_default();
	int cauchy_encode_off = 0;   // LZGPU_CAUCHY_FUSED=0: Cauchy-generator encodes on gf_dot_kernel + CRC passes instead of the fused kernel
	int convert_off = 0;   // LZGPU_CONVERT_FUSED=0: slice conversion through the two-pass route (image, then SPLIT encode)
	int bs_max_gf_warps = LZ_BS_MAX_GF_WARPS;  // LZGPU_BS_GFW: most GF warps of a bit-sliced encoder CTA (default 4, fused_plan.h)
	int bs_max_stages = LZ_BS_MAX_STAGES;  // LZGPU_BS_STAGES: deepest data stage ring of the bit-sliced kernels
	int bs_smem_cap = 200 * 1024;          // LZGPU_BS_SMEM_KB: their shared memory budget (one CTA per SM)
	int bitslice = LZ_BITSLICE_DEFAULT;  // LZGPU_BITSLICE: Vandermonde parity rows on bit planes (W = 8 items, bitslice.cuh) — bit 0: four rows, bit 1: three rows with k >= 7, bit 2: three rows with any k; 0 = packed-byte Horner
	int promo = 3;  // CU_TENSOR_MAP_L2_PROMOTION_L2_256B: measured faster streaming than 128B/none
	uint32_t grid_cap = 0;  // LZGPU_GRID_CAP (testing): at most this many CTAs per persistent launch, so that every CTA walks several units; 0 = no cap
	std::mutex last_mu;                     // guards the three below: they are recorded and read as one snapshot
	lzgpu_launch_geometry last_geo{};       // the latest persistent launch (lzgpu_debug_last_launch, lzgpu_debug_last_geometry)
	int32_t last_encoder = -1;              // its encoder instantiation and unit mode (lzgpu_debug_last_encoder); -1: not an encoder
	uint32_t last_mode = 0;
};

// what a launch site knows of its kernel's geometry before the grid is chosen (persistent_grid adds grid and units)
static lzgpu_launch_geometry launch_geo(int kernel, uint32_t threads, uint32_t G, uint32_t stages, uint32_t gf_warps, size_t smem) {
	lzgpu_launch_geometry g{};
	g.kernel = kernel;
	g.threads = threads;
	g.G = G;
	g.stages = stages;
	g.gf_warps = gf_warps;
	g.smem_bytes = static_cast<uint32_t>(smem);
	return g;
}

// What a launch records as the context's latest: its geometry, and for an encoder kernel (fused_run) the kernel's position in the
// list lzgpu_debug_encoder_kernels reports and the unit mode; every other launch records encoder -1
struct LaunchRecord {
	lzgpu_launch_geometry geo;
	int32_t encoder;
	uint32_t mode;
	LaunchRecord(const lzgpu_launch_geometry &g, int32_t e = -1, uint32_t m = 0) : geo(g), encoder(e), mode(m) {}
};

// CTAs of a persistent launch (each CTA starts at unit blockIdx.x and steps by gridDim.x): one per unit, at most `per_sm` per SM,
// and at most LZGPU_GRID_CAP when that is set.  Records the launch (geo, completed with grid and units) as the context's latest.
static int persistent_grid(lzgpu_ctx *ctx, uint64_t total_units, int per_sm, const LaunchRecord &rec) {
	FusedState *fs = ctx->fused;
	uint64_t grid = std::min<uint64_t>(total_units, static_cast<uint64_t>(ctx->sm_count) * per_sm);
	if (fs->grid_cap) grid = std::min<uint64_t>(grid, fs->grid_cap);
	lzgpu_launch_geometry geo = rec.geo;
	geo.grid = static_cast<uint32_t>(grid);
	geo.units = static_cast<uint32_t>(total_units);
	std::lock_guard<std::mutex> lock(fs->last_mu);
	fs->last_geo = geo;
	fs->last_encoder = rec.encoder;
	fs->last_mode = rec.mode;
	return static_cast<int>(grid);
}

// x^n mod P for a possibly negative n (x has multiplicative order dividing 2^32 - 1)
static uint32_t crc_xpow_bits_signed(long long n) {
	const long long ord = 0xFFFFFFFFll;
	n %= ord;
	if (n < 0) n += ord;
	uint32_t acc = 0x80000000u, sq = 0x40000000u;  // 1, x
	for (; n; n >>= 1) {
		if (n & 1) acc = lz::crc_mulmod(acc, sq);
		sq = lz::crc_mulmod(sq, sq);
	}
	return acc;
}

static uint8_t gf_pow2(int n) {
	uint8_t v = 1;
	for (int i = 0; i < n; ++i) v = lz::gf_mul_host(v, 2);
	return v;
}

// RAID-6 solve of lost data parts x0, x1 from parity rows 0 and 1 (fused_recover_kernel, fused_convert_kernel): w[0] = planes of
// 2^x0, w[1] = planes of (2^x0 ^ 2^x1)^-1
static void set_raid6_pair(CoefPlanes *w, int x0, int x1) {
	const uint8_t g0 = gf_pow2(x0);
	coef_planes_set(w[0], g0);
	coef_planes_set(w[1], lz::gf_inv_host(g0 ^ gf_pow2(x1)));
}

// the three-unknown elimination with parity rows 0, 1, 2 (the fused_recover_kernel comment; bs_recover3_kernel): alpha, beta, gamma,
// delta, then 2^x0 and 4^x0.  p, q, p^q are non-zero because 2 has order 255 and the positions differ by less than 32.
static void elim3_constants(int x0, int x1, int x2, uint8_t c[6]) {
	const uint8_t A = gf_pow2(x0), pp = A ^ gf_pow2(x1), qq = A ^ gf_pow2(x2);
	c[0] = lz::gf_inv_host(lz::gf_mul_host(qq, pp ^ qq));
	c[1] = lz::gf_mul_host(pp, c[0]);
	c[2] = lz::gf_inv_host(pp);
	c[3] = lz::gf_mul_host(qq, c[2]);
	c[4] = A;
	c[5] = lz::gf_mul_host(A, A);
}

// One persistent launch: geo.threads threads and geo.smem_bytes bytes of shared memory per CTA, the grid from persistent_grid
template <class... P, class... A>
static int launch(lzgpu_ctx *ctx, void (*kernel)(P...), const LaunchRecord &rec, int per_sm, uint64_t units, cudaStream_t st,
                  const A &...args) {
	const int grid = persistent_grid(ctx, units, per_sm, rec);
	kernel<<<grid, rec.geo.threads, rec.geo.smem_bytes, st>>>(args...);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

template <class F>
static int set_smem(F *kernel, int bytes) {
	CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
	return LZGPU_OK;
}

// ---------------------------------------------------------------------------------------------------
// Every kernel instantiation, one table per family.  lz_fused_init sets the shared-memory limit of each entry; the launch sites
// take the entry their plan names.  A kernel missing here is neither compiled nor launched.
// ---------------------------------------------------------------------------------------------------
// Encoders (fused_stream_kernel): packed-word items, or bit-sliced ones (bs: W = 8, one 16-warp CTA per SM, the last
// ceil(16 G / 32) warps take the 16 G items of a step, the warps before them the G (K + M - 1) * 4 streams; the plan made with
// bs = true guarantees both fit).  k = g = 0: runtime k and G.
using EncodeKernel = void (*)(CUtensorMap, FusedParams);
struct EncodeKernelEntry {
	int m;
	bool generic, striped, split, bs;
	uint32_t k, g;
	EncodeKernel fn;
	EncodeKernel narrow;  // generic coefficients: the 4-byte-item twin (fused_generic_item_words)
};
template <int M, bool GENERIC, int KT = 0, int GT = 0, bool STRIPED = false, bool SPLIT = false>
static EncodeKernelEntry encoder() {
	EncodeKernelEntry k{M, GENERIC, STRIPED, SPLIT, false, KT, GT, fused_stream_kernel<M, GENERIC, KT, GT, 64, STRIPED, SPLIT>, nullptr};
	if constexpr (GENERIC) k.narrow = fused_stream_kernel<M, GENERIC, KT, GT, 64, STRIPED, SPLIT, 1>;
	return k;
}
template <int M, int KT = 0, int GT = 0, bool STRIPED = false>
static EncodeKernelEntry bitsliced() {
	return {M, false, STRIPED, false, true, KT, GT, fused_stream_kernel<M, false, KT, GT, 64, STRIPED, false, 8>, nullptr};
}
static const EncodeKernelEntry kEncoders[] = {
	// runtime k and G: the CRC pass alone (M = 0), Vandermonde and generic (Cauchy) coefficients, the conversion form, striped units
	encoder<0, false>(), encoder<1, false>(), encoder<2, false>(), encoder<3, false>(), encoder<4, false>(),
	encoder<1, true>(), encoder<2, true>(), encoder<3, true>(), encoder<4, true>(),
	encoder<1, false, 0, 0, false, true>(), encoder<2, false, 0, 0, false, true>(), encoder<3, false, 0, 0, false, true>(),
	encoder<4, false, 0, 0, false, true>(), encoder<4, true, 0, 0, false, true>(),
	encoder<1, false, 0, 0, true>(), encoder<2, false, 0, 0, true>(), encoder<3, false, 0, 0, true>(), encoder<4, false, 0, 0, true>(),
	encoder<4, true, 0, 0, true>(),
	// constant-folded (M, K, G) for the common goals (K, G from pick_group)
	encoder<2, false, 8, 7>(),    // ec(8,2)
	encoder<1, false, 2, 32>(),   // xor2
	encoder<1, false, 3, 20>(),   // xor3
	encoder<2, false, 3, 16>(),   // ec(3,2)
	encoder<2, false, 4, 12>(),   // ec(4,2)
	encoder<2, false, 6, 9>(),    // ec(6,2)
	encoder<3, false, 5, 8>(),    // ec(5,3)
	encoder<3, false, 6, 8>(),    // ec(6,3)
	encoder<4, false, 8, 8>(),    // ec(8,4) on one 16-warp CTA per SM
	// more goals folded (the runtime-k instantiation measured markedly slower for ec(8,3), ec(6,4), ec(4,4))
	encoder<3, false, 8, 6>(),    // ec(8,3)
	encoder<1, false, 4, 16>(),   // xor4 / ec(4,1)
	encoder<2, false, 5, 10>(),   // ec(5,2)
	encoder<2, false, 10, 5>(),   // ec(10,2)
	encoder<3, false, 4, 8>(),    // ec(4,3)
	encoder<4, false, 10, 6>(),   // ec(10,4)
	encoder<4, false, 12, 5>(),   // ec(12,4)
	encoder<4, false, 6, 8>(),    // ec(6,4)
	encoder<4, false, 4, 8>(),    // ec(4,4)
	encoder<2, false, 8, 7, true>(), encoder<1, false, 2, 32, true>(), encoder<1, false, 3, 20, true>(), encoder<2, false, 3, 16, true>(),
	encoder<3, false, 5, 8, true>(), encoder<4, false, 8, 8, true>(),
	// bit-sliced: runtime k and G, then the constant-folded (M, K, G), G from pick_group(.., bs = true)
	bitsliced<3>(), bitsliced<4>(), bitsliced<3, 0, 0, true>(), bitsliced<4, 0, 0, true>(),
	bitsliced<4, 8, 8>(), bitsliced<4, 10, 6>(), bitsliced<4, 12, 5>(), bitsliced<4, 6, 8>(), bitsliced<4, 4, 8>(),
	bitsliced<3, 8, 8>(), bitsliced<3, 9, 6>(), bitsliced<3, 10, 6>(), bitsliced<3, 12, 5>(), bitsliced<4, 8, 8, true>(),
};

// the folded entry of (M, K, G) where there is one, else the runtime-k one; nullptr: the fused path does not take the shape
static const EncodeKernelEntry *find_encoder(int M, bool generic, uint32_t K, uint32_t G, bool striped, bool split, bool bs) {
	const EncodeKernelEntry *runtime_k = nullptr;
	for (const EncodeKernelEntry &k : kEncoders) {
		if (k.m != M || k.generic != generic || k.striped != striped || k.split != split || k.bs != bs) continue;
		if (k.k == K && k.g == G) return &k;
		if (k.k == 0) runtime_k = &k;
	}
	return runtime_k;
}

// position of entry k's kernel (narrow: its 4-byte-item twin, right after it) in the list lzgpu_debug_encoder_kernels reports
static int32_t encoder_index(const EncodeKernelEntry *k, bool narrow) {
	int32_t i = 0;
	for (const EncodeKernelEntry *e = kEncoders; e != k; ++e) i += e->narrow ? 2 : 1;
	return i + (narrow ? 1 : 0);
}

// Degraded read (fused_recover_kernel), keyed by the plan's kernel, lost data parts, compile-time k (0: runtime) and parity rows:
// 0 .. e-1 (first_e: R0 = 0, R1 = 1) or any.  DIRECT (any generator; the Cauchy codes): 16-warp geometry, 4-byte or wide items.
using RecoverKernel = void (*)(TmapArray, RecoverParams);
struct RecoverKernelEntry {
	int kernel;  // LZGPU_KERNEL_RECOVER_GEO0 / _GEO1 / _GEO2 / _DIRECT
	uint32_t e, kt;
	bool first_e, wide;
	RecoverKernel fn;
};
template <int GEO, int E, int KT, int R0 = -1, int R1 = -1>
static RecoverKernelEntry recoverer() {
	constexpr int kernel = GEO == 2 ? LZGPU_KERNEL_RECOVER_GEO2 : GEO == 1 ? LZGPU_KERNEL_RECOVER_GEO1 : LZGPU_KERNEL_RECOVER_GEO0;
	return {kernel, E, KT, R0 == 0, false, fused_recover_kernel<E, KT, R0, R1, 64, GEO>};
}
template <int E, bool WIDE>
static RecoverKernelEntry direct() {
	return {LZGPU_KERNEL_RECOVER_DIRECT, E, 0, false, WIDE, fused_recover_kernel<E, 0, kRecoverDirect, -1, 64, 2, WIDE ? direct_wide_words(E) : 1>};
}
static const RecoverKernelEntry kRecoverers[] = {
	// every geometry (two 9-warp CTAs per SM only for e <= 2); k = 8 with rows 0 .. e-1 for e <= 2
	recoverer<0, 1, 8, 0>(), recoverer<1, 1, 8, 0>(), recoverer<2, 1, 8, 0>(),
	recoverer<0, 1, 0, 0>(), recoverer<1, 1, 0, 0>(), recoverer<2, 1, 0, 0>(),
	recoverer<0, 1, 0>(), recoverer<1, 1, 0>(), recoverer<2, 1, 0>(),
	recoverer<0, 2, 8, 0, 1>(), recoverer<1, 2, 8, 0, 1>(), recoverer<2, 2, 8, 0, 1>(),
	recoverer<0, 2, 0, 0, 1>(), recoverer<1, 2, 0, 0, 1>(), recoverer<2, 2, 0, 0, 1>(),
	recoverer<0, 2, 0>(), recoverer<1, 2, 0>(), recoverer<2, 2, 0>(),
	recoverer<0, 3, 0, 0, 1>(), recoverer<2, 3, 0, 0, 1>(), recoverer<0, 3, 0>(), recoverer<2, 3, 0>(),
	recoverer<0, 4, 0, 0, 1>(), recoverer<2, 4, 0, 0, 1>(), recoverer<0, 4, 0>(), recoverer<2, 4, 0>(),
	// a compile-time k other than 8 (ec(3,2), the BASELINE configs[1] goal; ec(4,2), ec(5,3), ec(6,2), ec(6,3)): the 16-warp geometry
	// only, rows 0 .. e-1
	recoverer<2, 1, 3, 0>(), recoverer<2, 2, 3, 0, 1>(), recoverer<2, 2, 4, 0, 1>(), recoverer<2, 2, 5, 0, 1>(),
	recoverer<2, 3, 5, 0, 1>(), recoverer<2, 2, 6, 0, 1>(), recoverer<2, 3, 6, 0, 1>(),
	direct<1, false>(), direct<2, false>(), direct<3, false>(), direct<4, false>(),
	direct<1, true>(), direct<2, true>(), direct<3, true>(), direct<4, true>(),
};
static int recover_smem_cap(int kernel) {
	return kernel == LZGPU_KERNEL_RECOVER_GEO0 ? kRecoverSmemCap : kernel == LZGPU_KERNEL_RECOVER_GEO1 ? kRecoverSmemCap2 : kRecoverSmemCapBig;
}

// three lost data parts on bit planes (bs_recover3_kernel), keyed by the compile-time k (0: runtime)
using BsRecoverKernel = void (*)(TmapArray, RecoverParams, BsRecoverMasks);
static const struct {
	uint32_t kt;
	BsRecoverKernel fn;
} kBsRecoverers[] = {{0, bs_recover3_kernel<0>}, {5, bs_recover3_kernel<5>}, {8, bs_recover3_kernel<8>}};

// Stripe checks (check_kernel.cuh), keyed by the checked parity rows R, whether they are rows 0 .. R-1, and for the degraded forms
// the lost data parts E.  check_plan gives E < R <= 4, and rows other than 0 .. R-1 only with m <= 4, so R <= 3 (m >= 5 is Cauchy).
using CheckKernel = void (*)(CheckTmaps, CheckParams);
using CheckMapKernel = void (*)(CheckTmaps, CheckParams, uint32_t *);
using CheckRepairKernel = void (*)(CheckTmaps, CheckParams, uint32_t *, unsigned long long *);
using CheckDegradedKernel = void (*)(CheckTmaps, CheckParams, uint32_t *, CheckLost);
using CheckRepairDegradedKernel = void (*)(CheckTmaps, CheckParams, uint32_t *, CheckLost, unsigned long long *);
struct CheckKernels {
	uint32_t r;
	bool consecutive;
	CheckKernel check;
	CheckMapKernel map;
	CheckRepairKernel repair;
};
struct CheckDegradedKernels {
	uint32_t e, r;
	bool consecutive;
	CheckDegradedKernel map;
	CheckRepairDegradedKernel repair;
};
template <int R, bool C>
static CheckKernels checkers() {
	return {R, C, fused_check_kernel<R, C>, fused_check_map_kernel<R, C>, fused_check_repair_kernel<R, C>};
}
template <int E, int R, bool C>
static CheckDegradedKernels degraded_checkers() {
	return {E, R, C, fused_check_degraded_kernel<E, R, C>, fused_check_repair_degraded_kernel<E, R, C>};
}
static const CheckKernels kCheckers[] = {checkers<1, true>(),  checkers<2, true>(),  checkers<3, true>(), checkers<4, true>(),
                                         checkers<1, false>(), checkers<2, false>(), checkers<3, false>()};
static const CheckDegradedKernels kDegradedCheckers[] = {
	degraded_checkers<1, 2, true>(),  degraded_checkers<1, 3, true>(),  degraded_checkers<1, 4, true>(),
	degraded_checkers<2, 3, true>(),  degraded_checkers<2, 4, true>(),  degraded_checkers<3, 4, true>(),
	degraded_checkers<1, 2, false>(), degraded_checkers<1, 3, false>(), degraded_checkers<2, 3, false>()};

// Slice conversion (fused_convert_kernel), keyed by the destination's parity parts, the lost source data parts and a compile-time
// destination k (0: runtime; 3 for the xor3 / ec(3,2) destinations)
using ConvertKernel = void (*)(TmapArray, ConvertParams);
static const struct {
	int m;
	uint32_t e;
	int kd;
	ConvertKernel fn;
} kConverters[] = {
	{1, 0, 0, fused_convert_kernel<1, 0>}, {1, 1, 0, fused_convert_kernel<1, 1>}, {1, 2, 0, fused_convert_kernel<1, 2>},
	{2, 0, 0, fused_convert_kernel<2, 0>}, {2, 1, 0, fused_convert_kernel<2, 1>}, {2, 2, 0, fused_convert_kernel<2, 2>},
	{3, 0, 0, fused_convert_kernel<3, 0>}, {3, 1, 0, fused_convert_kernel<3, 1>}, {3, 2, 0, fused_convert_kernel<3, 2>},
	{1, 0, 3, fused_convert_kernel<1, 0, 3>}, {1, 1, 3, fused_convert_kernel<1, 1, 3>}, {1, 2, 3, fused_convert_kernel<1, 2, 3>},
	{2, 0, 3, fused_convert_kernel<2, 0, 3>}, {2, 1, 3, fused_convert_kernel<2, 1, 3>}, {2, 2, 3, fused_convert_kernel<2, 2, 3>},
};

// One-pass encode for several slices (fused_slices_kernel), keyed by the largest m of the slices
using SlicesKernel = void (*)(CUtensorMap, SlicesParams);
static const struct {
	uint32_t m;
	SlicesKernel fn;
} kSlicers[] = {{1, fused_slices_kernel<1>}, {2, fused_slices_kernel<2>}, {3, fused_slices_kernel<3>}, {4, fused_slices_kernel<4>}};

// Recovery from the parts of every slice together (recover_slices_kernel): one instantiation for any goal set, and its SALVAGE,
// CHECK and CORRECT twins, indexed by RsMode
using RecoverSlicesKernel = void (*)(RecoverSlicesParams);
static const RecoverSlicesKernel kRecoverSlicers[] = {recover_slices_kernel<RsMode::RECOVER>, recover_slices_kernel<RsMode::SALVAGE>,
                                                      recover_slices_kernel<RsMode::CHECK>, recover_slices_kernel<RsMode::CORRECT>};
static_assert(sizeof(RsFixEntry) == sizeof(lzgpu_slices_fix) && sizeof(RsCheckEntry) == sizeof(lzgpu_slices_check), "entry layouts");

// function attributes are per device: set once per context
static int set_all_smem_attrs(const FusedState *fs) {
	int rc;
	const int smem = std::min(fs->max_smem, kSmemCap);
	for (const EncodeKernelEntry &k : kEncoders) {
		const int bytes = k.bs ? 226 * 1024 : std::max(smem, fused_smem_cap(k.m, k.generic, 64));  // one-CTA-per-SM shapes use a deeper ring
		if ((rc = set_smem(k.fn, bytes)) || (k.narrow && (rc = set_smem(k.narrow, bytes)))) return rc;
	}
	for (const RecoverKernelEntry &k : kRecoverers)
		if ((rc = set_smem(k.fn, recover_smem_cap(k.kernel)))) return rc;
	for (const auto &k : kBsRecoverers)
		if ((rc = set_smem(k.fn, kRecoverSmemCapBig))) return rc;
	for (const CheckKernels &k : kCheckers)
		if ((rc = set_smem(k.check, kRecoverSmemCapBig)) || (rc = set_smem(k.map, kRecoverSmemCapBig)) || (rc = set_smem(k.repair, kRecoverSmemCapBig))) return rc;
	for (const CheckDegradedKernels &k : kDegradedCheckers)
		if ((rc = set_smem(k.map, kRecoverSmemCapBig)) || (rc = set_smem(k.repair, kRecoverSmemCapBig))) return rc;
	for (const auto &k : kConverters)
		if ((rc = set_smem(k.fn, kSmemCap))) return rc;
	for (const auto &k : kSlicers)
		if ((rc = set_smem(k.fn, kSlicesSmemCap))) return rc;
	for (const RecoverSlicesKernel k : kRecoverSlicers)
		if ((rc = set_smem(k, static_cast<int>(kRsSmemCap)))) return rc;
	if ((rc = set_smem(correct_slices_kernel, static_cast<int>(rsc_smem_bytes(kScMaxChecks, kRsMaxL))))) return rc;
	return LZGPU_OK;
}

int lz_fused_init(lzgpu_ctx *ctx) {
	auto *fs = new FusedState();
	ctx->fused = fs;
	if (const char *e = std::getenv("LZGPU_DISABLE_FUSED")) fs->disabled = std::atoi(e) != 0;
	if (const char *e = std::getenv("LZGPU_PROBE")) fs->probe = static_cast<uint32_t>(std::atoi(e));
	if (const char *e = std::getenv("LZGPU_L2_PROMO")) fs->promo = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_EVICT_FIRST")) fs->evict_first = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_RECOVER_TWO")) fs->recover.recover_two = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_RECOVER_GEO")) fs->recover.recover_geo = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_DIRECT_WIDE")) fs->recover.direct_wide = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_CONVERT_FUSED")) fs->convert_off = std::atoi(e) == 0;
	if (const char *e = std::getenv("LZGPU_CAUCHY_FUSED")) fs->cauchy_encode_off = std::atoi(e) == 0;
	if (const char *e = std::getenv("LZGPU_RECOVER_K3")) fs->recover.recover_k3 = std::atoi(e) != 0;
	if (const char *e = std::getenv("LZGPU_STRIPED")) fs->striped = std::atoi(e);  // 0 never, 1 whenever possible, unset = automatic
	if (const char *e = std::getenv("LZGPU_BITSLICE")) fs->bitslice = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_BS_RECOVER")) fs->recover.bs_recover = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_BS_GFW")) fs->bs_max_gf_warps = std::max(1, std::min(12, std::atoi(e)));
	if (const char *e = std::getenv("LZGPU_BS_RECOVER_GFW")) fs->recover.bs_recover_gf_warps = std::max(1, std::min(16, std::atoi(e)));
	if (const char *e = std::getenv("LZGPU_BS_STAGES")) fs->bs_max_stages = std::max(2, std::min(16, std::atoi(e)));
	if (const char *e = std::getenv("LZGPU_BS_SMEM_KB")) fs->bs_smem_cap = std::max(64, std::min(226, std::atoi(e))) * 1024;
	if (const char *e = std::getenv("LZGPU_GRID_CAP")) fs->grid_cap = static_cast<uint32_t>(std::max(0, std::atoi(e)));
	void *fn = nullptr;
	cudaDriverEntryPointQueryResult qres;
	cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
	if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn) {
		cudaGetLastError();
		lz_set_error("cuTensorMapEncodeTiled is not available from the driver");
		return LZGPU_ERR_CUDA;
	}
	fs->encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
	for (int q = 0; q < 4; ++q) fs->qmult[q] = crc_xpow_bits_signed(32ll * (4096ll * (3 - q) - FoldSpec<64>::deg));
	CUDA_TRY(cudaDeviceGetAttribute(&fs->max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, ctx->device));
	CUDA_TRY(cudaMalloc(&fs->d_sm_ctr, 256 * sizeof(uint32_t)));
	CUDA_TRY(cudaMemset(fs->d_sm_ctr, 0, 256 * sizeof(uint32_t)));
	return set_all_smem_attrs(fs);
}

void lz_fused_destroy(lzgpu_ctx *ctx) {
	if (ctx->fused && ctx->fused->d_sm_ctr) cudaFree(ctx->fused->d_sm_ctr);
	delete ctx->fused;
	ctx->fused = nullptr;
}

extern "C" int lzgpu_debug_last_launch(lzgpu_ctx *ctx, uint32_t *grid, uint32_t *units) {
	if (!ctx || !ctx->fused || !grid || !units) return LZGPU_ERR_ARG;
	std::lock_guard<std::mutex> lock(ctx->fused->last_mu);
	*grid = ctx->fused->last_geo.grid;
	*units = ctx->fused->last_geo.units;
	return LZGPU_OK;
}

extern "C" int lzgpu_debug_last_geometry(lzgpu_ctx *ctx, lzgpu_launch_geometry *out) {
	if (!ctx || !ctx->fused || !out) return LZGPU_ERR_ARG;
	std::lock_guard<std::mutex> lock(ctx->fused->last_mu);
	*out = ctx->fused->last_geo;
	return LZGPU_OK;
}

extern "C" int lzgpu_debug_last_encoder(lzgpu_ctx *ctx, int32_t *index, uint32_t *mode) {
	if (!ctx || !ctx->fused || !index || !mode) return LZGPU_ERR_ARG;
	std::lock_guard<std::mutex> lock(ctx->fused->last_mu);
	*index = ctx->fused->last_encoder;
	*mode = ctx->fused->last_mode;
	return LZGPU_OK;
}

extern "C" int lzgpu_debug_encoder_kernels(lzgpu_encoder_kernel *out, uint32_t capacity) {
	uint32_t n = 0;
	for (const EncodeKernelEntry &k : kEncoders)
		for (int narrow = 0; narrow <= (k.narrow ? 1 : 0); ++narrow, ++n) {
			if (!out || n >= capacity) continue;
			lzgpu_encoder_kernel &o = out[n];
			o.m = k.m;
			o.generic = k.generic;
			o.bitsliced = k.bs;
			o.striped = k.striped;
			o.split = k.split;
			o.kt = k.k;
			o.gt = k.g;
			o.item_bytes = k.bs ? 32u : narrow ? 4u : 4u * static_cast<uint32_t>(fused_item_words(k.m, k.generic));  // (the W of each instantiation)
		}
	return static_cast<int>(n);
}

// rows_per_chunk rows of kRowBytes per chunk, chunk c at base + c * chunk_stride (0: contiguous), boxes of box_rows rows
static CUresult make_tensor_map(const FusedState *fs, CUtensorMap *map, const void *base, uint64_t rows_per_chunk, uint64_t n_chunks,
                                uint64_t chunk_stride, uint32_t box_rows) {
	const cuuint64_t dims[3] = {static_cast<cuuint64_t>(kRowBytes), rows_per_chunk, n_chunks};
	const cuuint64_t strides[2] = {static_cast<cuuint64_t>(kRowBytes), chunk_stride ? chunk_stride : rows_per_chunk * kRowBytes};
	const cuuint32_t box[3] = {kStepBytes, box_rows, 1};
	const cuuint32_t estr[3] = {1, 1, 1};
	return fs->encode_tiled(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
	                        CU_TENSOR_MAP_SWIZZLE_128B, static_cast<CUtensorMapL2promotion>(fs->promo), CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// split_out != nullptr: the conversion form — K + M destination part buffers (nullptr = part not wanted), data parts stored by the
// BlockConverter pick and parity parts stored separately, chunk c at + c*split_stride; d_parity is then unused
static int fused_run(lzgpu_ctx *ctx, int M, bool generic, const uint8_t *coef_rows, uint32_t K, uint32_t n_chunks, uint32_t nb,
                     const void *d_data, size_t chunk_stride, void *d_parity, size_t parity_stride, void *d_crc, size_t crc_stride,
                     cudaStream_t st, void *const *split_out = nullptr, size_t split_stride = 0, uint32_t crc_row_base = 0, bool skip_data_crc = false,
                     int striped_policy = -2 /* -2: the context's setting */) {
	FusedState *fs = ctx->fused;
	// unit geometry: per-chunk, flat or striped units, stripes per unit (fused_plan.h; unit-tested without a GPU); the bit-sliced
	// geometry first where it is switched on, the packed-byte one if a shape does not fit it
	const int spol = split_out ? 0 : (striped_policy == -2 ? fs->striped : striped_policy);
	FusedPlan pl;
	if (!split_out && fused_bitslice(M, generic, fs->bitslice, K))
		pl = fused_plan(M, generic, K, n_chunks, nb, chunk_stride, std::min(fs->max_smem, fs->bs_smem_cap), 64, spol, true, fs->bs_max_stages, fs->bs_max_gf_warps);
	if (!pl.ok) pl = fused_plan(M, generic, K, n_chunks, nb, chunk_stride, std::min(fs->max_smem, fused_smem_cap(M, generic, 64)), 64, spol);
	if (!pl.ok || (reinterpret_cast<uintptr_t>(d_data) % 16)) return LZGPU_NOT_HANDLED;
	const uint32_t G = pl.G;
	const bool flat = pl.mode == 1u, striped = pl.mode == 2u;
	FusedParams p{};
	p.parity = static_cast<uint8_t *>(d_parity);
	p.crc = static_cast<uint32_t *>(d_crc);
	p.tables = ctx->d_crc_tables;
	p.parity_stride = parity_stride;
	p.crc_stride = crc_stride;
	p.n_chunks = n_chunks;
	p.nb = nb;
	p.pb = pl.pb;
	p.K = K;
	p.G = G;
	p.n_stages = pl.n_stages;
	p.flat = pl.mode;
	p.flat_magic = (1ull << 40) / p.pb + 1;
	p.units_per_chunk = pl.units_per_chunk;
	p.total_units = pl.total_units;
	std::memcpy(p.qmult, fs->qmult, sizeof(p.qmult));
	p.zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	p.probe = fs->probe;
	p.evict_first = static_cast<uint32_t>(fs->evict_first);
	p.crc_row_base = crc_row_base;
	p.skip_data_crc = skip_data_crc ? 1u : 0u;
	if (generic) {
		for (int r = 0; r < M; ++r)
			for (uint32_t j = 0; j < K; ++j) {
				coef_planes_set(p.coef[r * 32 + j], coef_rows[r * K + j]);
			}
	}
	// flat: the batch is one run of stripes; striped: one box per stripe
	const uint64_t map_rows = flat ? static_cast<uint64_t>(n_chunks) * nb * 4 : static_cast<uint64_t>(nb) * 4, map_chunks = flat ? 1 : n_chunks;
	const uint64_t map_stride = flat ? 0 : chunk_stride;
	const uint32_t box_rows = striped ? K * 4 : G * K * 4;
	CUtensorMap map;
	const CUresult r = make_tensor_map(fs, &map, d_data, map_rows, map_chunks, map_stride, box_rows);
	if (r != CUDA_SUCCESS) {
		lz_set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows/chunk %llu, chunks %llu, stride %llu, box rows %u)", static_cast<int>(r),
		             static_cast<unsigned long long>(map_rows), static_cast<unsigned long long>(map_chunks), static_cast<unsigned long long>(map_stride), box_rows);
		return LZGPU_ERR_CUDA;
	}
	if (split_out) {
		if (striped || (split_stride % 16)) return LZGPU_NOT_HANDLED;
		for (uint32_t j = 0; j < K; ++j) p.data_out[j] = static_cast<uint8_t *>(split_out[j]);
		for (int r = 0; r < M; ++r) p.par_out[r] = static_cast<uint8_t *>(split_out[K + r]);
		p.part_out_stride = split_stride;
	}
	const EncodeKernelEntry *k = find_encoder(M, generic, K, G, striped, split_out != nullptr, pl.bs);
	if (!k) return LZGPU_NOT_HANDLED;
	const lzgpu_launch_geometry geo = launch_geo(pl.bs ? LZGPU_KERNEL_ENCODE_BITSLICE : LZGPU_KERNEL_ENCODE, pl.threads, G, pl.n_stages,
	                                             pl.bs ? (16 * G + 31) / 32 : 0, pl.smem);
	const bool narrow = k->narrow && fused_generic_item_words(G) == 1;
	return launch(ctx, narrow ? k->narrow : k->fn, LaunchRecord(geo, encoder_index(k, narrow), pl.mode), fused_ctas_per_sm(M, generic, 64, pl.bs),
	              p.total_units, st, map, p);
}

int lz_fused_encode(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_data, size_t chunk_stride,
                    void *d_parity, size_t parity_stride, void *d_crc, size_t crc_stride, cudaStream_t st) {
	FusedState *fs = ctx->fused;
	if (!fs || fs->disabled) return LZGPU_NOT_HANDLED;
	const int K = goal->k, M = goal->m;
	if (lz::uses_cauchy(K, M)) {
		if (fs->cauchy_encode_off) return LZGPU_NOT_HANDLED;   // LZGPU_CAUCHY_FUSED=0: gf_dot_kernel + the fused CRC kernel (A/B)
		// Cauchy generator (m >= 5, or m == 4 and k > 20; reed_solomon.h:168-172): arbitrary coefficients, bit-plane multiply inside
		// the fused kernel, in passes of up to four parity rows over the same data (the TMA stream, the fused parity CRCs and the
		// part-major stores stay; the first pass also checksums the data blocks).  A shape one pass cannot take leaves the whole
		// encode to the generic kernels — decided before anything is launched (the plan is pure host logic).
		uint8_t gen[LZGPU_MAX_PARTS * LZGPU_MAX_DATA];
		lz::rs_generator(K, M, gen);
		if (M == 4) return fused_run(ctx, 4, true, gen + K * K, K, n_chunks, nb, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, st);
		const uint32_t pb = (nb + K - 1) / K;
		for (int rows : {4, M % 4})
			if (rows && !fused_plan(rows, true, K, n_chunks, nb, chunk_stride, std::min(fs->max_smem, fused_smem_cap(rows, true, 64)), 64, 0).ok) return LZGPU_NOT_HANDLED;
		if (reinterpret_cast<uintptr_t>(d_data) % 16) return LZGPU_NOT_HANDLED;
		for (int r0 = 0; r0 < M; r0 += 4) {
			// per-chunk / flat units only: the passes share one geometry rule (striped policy 0)
			int rc = fused_run(ctx, std::min(4, M - r0), true, gen + (K + r0) * K, K, n_chunks, nb, d_data, chunk_stride,
			                   static_cast<uint8_t *>(d_parity) + static_cast<size_t>(r0) * pb * LZGPU_BLOCK_SIZE, parity_stride, d_crc, crc_stride, st, nullptr, 0,
			                   static_cast<uint32_t>(r0), r0 > 0, 0);
			if (rc != LZGPU_OK) return rc == LZGPU_NOT_HANDLED ? LZGPU_ERR_CUDA : rc;  // (cannot happen: the plans were checked above)
		}
		return LZGPU_OK;
	}
	if (M > 4) return LZGPU_NOT_HANDLED;
	// xorN is ec(N,1): parity row 0 of the Vandermonde generator is all ones (chunk_writer.cc:373-381)
	int rc = fused_run(ctx, M, false, nullptr, K, n_chunks, nb, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, st);
	if (rc == LZGPU_NOT_HANDLED && goal->kind == LZGPU_KIND_EC) {
		// a Vandermonde shape whose two-stripe unit does not fit the 8-warp CTA (ec(31,3): 264 rows) still fits the nine warps of
		// the generic-coefficient instantiation: same rows, taken as general coefficients (slower multiplies, same TMA stream)
		uint8_t gen[LZGPU_MAX_PARTS * LZGPU_MAX_DATA];
		lz::rs_generator(K, M, gen);
		rc = fused_run(ctx, M, true, gen + K * K, K, n_chunks, nb, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, st, nullptr, 0, 0, false, 0);
	}
	return rc;
}

// conversion form of the encode (SliceRecoveryPlanner: BlockConverter for the data parts + RecoverParity for the parity parts in
// ONE pass over the chunk image): d_out[i], i < k+m, nullptr = part not wanted; CRC array as in lz_fused_encode
int lz_fused_encode_split(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_data, size_t chunk_stride,
                          void *const *d_out, size_t out_stride, void *d_crc, size_t crc_stride, cudaStream_t st) {
	FusedState *fs = ctx->fused;
	if (!fs || fs->disabled) return LZGPU_NOT_HANDLED;
	const int K = goal->k, M = goal->m;
	if (M > 4) return LZGPU_NOT_HANDLED;
	if (lz::uses_cauchy(K, M)) {
		uint8_t gen[LZGPU_MAX_PARTS * LZGPU_MAX_DATA];
		lz::rs_generator(K, M, gen);
		return fused_run(ctx, 4, true, gen + K * K, K, n_chunks, nb, d_data, chunk_stride, nullptr, 0, d_crc, crc_stride, st, d_out, out_stride);
	}
	return fused_run(ctx, M, false, nullptr, K, n_chunks, nb, d_data, chunk_stride, nullptr, 0, d_crc, crc_stride, st, d_out, out_stride);
}

int lz_fused_crc(lzgpu_ctx *ctx, const void *base, unsigned long long n_blocks, unsigned long long blocks_per_chunk,
                 unsigned long long chunk_stride, void *out, unsigned long long out_chunk_stride, cudaStream_t st) {
	FusedState *fs = ctx->fused;
	if (!fs || fs->disabled || n_blocks == 0) return LZGPU_NOT_HANDLED;
	if (blocks_per_chunk == 0) blocks_per_chunk = n_blocks;
	if (n_blocks % blocks_per_chunk) return LZGPU_NOT_HANDLED;
	const unsigned long long n_chunks = n_blocks / blocks_per_chunk;
	if (blocks_per_chunk > 0x3fffffffull || n_chunks > 0x7fffffffull) return LZGPU_NOT_HANDLED;
	if (n_chunks == 1) chunk_stride = blocks_per_chunk * LZGPU_BLOCK_SIZE;
	// CRC only, no parity: a unit is 64 blocks.  Contiguous "chunks" (parts) whose block count is not a multiple of 64 are
	// taken as one run of single-block stripes (K = 1, G = 64, flat units crossing the part boundaries) instead of
	// K = 64 blocks per unit inside each part, which would leave the last unit of every part partly empty.
	const bool contiguous = n_chunks > 1 && chunk_stride == blocks_per_chunk * LZGPU_BLOCK_SIZE;
	const uint32_t K = (contiguous && blocks_per_chunk % 64) ? 1 : 64;
	return fused_run(ctx, 0, false, nullptr, K, static_cast<uint32_t>(n_chunks), static_cast<uint32_t>(blocks_per_chunk), base, chunk_stride,
	                 nullptr, 0, out, out_chunk_stride, st);
}

// ---------------------------------------------------------------------------------------------------
// fused degraded read
// ---------------------------------------------------------------------------------------------------
int lz_fused_recover(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                     const void *const *d_part_crc, const uint8_t *want, void *const *d_out, void *d_chunk_out, size_t chunk_out_stride,
                     cudaStream_t st, unsigned long long *d_first_bad) {
	FusedState *fs = ctx->fused;
	if (!fs || fs->disabled) return LZGPU_NOT_HANDLED;
	const int K = goal->k, M = goal->m, N = K + M;
	const bool direct = lz::uses_cauchy(K, M);
	if ((part_stride % 16) || (chunk_out_stride % 16)) return LZGPU_NOT_HANDLED;
	// the router (recover_plan, fused_plan.h): inputs are the first k available parts (ec_read_plan.h:126-133), of which the ones
	// with stored CRCs are verified
	uint8_t available[LZGPU_MAX_PARTS];
	bool want_missing_parity = false, verifying = false;
	for (int i = 0, n_used = 0; i < N; ++i) {
		available[i] = d_parts[i] != nullptr;
		if (available[i] && n_used < K) { verifying |= d_part_crc && d_part_crc[i]; ++n_used; }
		if (i >= K) want_missing_parity |= want[i] && !d_parts[i] && d_out && d_out[i];
	}
	const RecoverPlan pl = recover_plan(K, M, direct, available, want_missing_parity, verifying, d_chunk_out != nullptr, fs->recover);
	const lzgpu_recover_plan &o = pl.out;
	if (!o.fused) return LZGPU_NOT_HANDLED;
	const uint32_t e = o.lost_data_parts, G = o.G;
	RecoverParams p{};
	std::memset(p.slot_of_data, 0xff, sizeof(p.slot_of_data));
	for (int a = 0; a < K; ++a) {
		const int idx = pl.used[a];
		p.part_id[a] = static_cast<uint8_t>(idx);
		p.data_of_slot[a] = idx < K ? static_cast<uint8_t>(idx) : 0xff;
		if (idx < K) p.slot_of_data[idx] = static_cast<uint8_t>(a);
	}
	for (uint32_t x = 0; x < e; ++x) {
		p.erased_idx[x] = pl.erased_idx[x];
		p.par_slot[x] = pl.par_slot[x];
		p.par_row[x] = pl.par_row[x];
	}
	const uint32_t pb = (nb + K - 1) / K;
	for (uint32_t x = 0; x < e; ++x) {   // a part nothing is requested for is still solved (cheap), not stored
		const int j = p.erased_idx[x];
		void *dst = d_out ? d_out[j] : nullptr;
		p.out[x] = (want[j] || d_chunk_out) ? static_cast<uint8_t *>(dst) : nullptr;
	}
	p.image = static_cast<uint8_t *>(d_chunk_out);
	p.out_stride = part_stride;
	p.image_stride = chunk_out_stride;
	p.tables = ctx->d_crc_tables;
	p.first_bad = d_first_bad;
	p.n_chunks = n_chunks;
	p.nb = nb;
	p.pb = pb;
	p.K = K;
	p.G = G;
	p.units_per_chunk = (pb + G - 1) / G;
	const uint64_t total = static_cast<uint64_t>(p.units_per_chunk) * n_chunks;
	if (total > 0x7fffffffull) return LZGPU_NOT_HANDLED;
	p.total_units = static_cast<uint32_t>(total);
	p.e = e;
	p.n_stages = o.stages;
	std::memcpy(p.qmult, fs->qmult, sizeof(p.qmult));
	p.zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	for (int a = 0; a < K; ++a) p.stored[a] = d_part_crc ? static_cast<const uint32_t *>(d_part_crc[pl.used[a]]) : nullptr;
	// V[r][x] = (2^row_r)^(erased_x); W = V^-1
	uint8_t V[16], W[16];
	for (uint32_t r = 0; r < e; ++r) {
		const uint8_t gen = gf_pow2(p.par_row[r]);
		for (uint32_t x = 0; x < e; ++x) {
			uint8_t v = 1;
			for (int t = 0; t < p.erased_idx[x]; ++t) v = lz::gf_mul_host(v, gen);
			V[r * e + x] = v;
		}
	}
	if (!direct && gf_invert_matrix(V, W, static_cast<int>(e)) != 0) return LZGPU_NOT_HANDLED;  // generic path reports the singular case
	if (direct) {
		// rows of the reference's inverted k x k system for the erased data parts, over the k used parts in slot order
		uint8_t erased_flags[LZGPU_MAX_PARTS] = {0}, wanted[LZGPU_MAX_PARTS] = {0}, rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
		for (int i = 0; i < N; ++i) erased_flags[i] = 1;
		for (int a = 0; a < K; ++a) erased_flags[pl.used[a]] = 0;
		for (uint32_t x = 0; x < e; ++x) wanted[p.erased_idx[x]] = 1;
		bool singular = false;
		if (lz::rs_recovery_matrix(K, M, erased_flags, wanted, rows, &singular) != static_cast<int>(e)) return LZGPU_NOT_HANDLED;
		for (uint32_t x = 0; x < e; ++x)   // rs_recovery_matrix emits its rows in ascending part order = erased_idx order
			for (int a = 0; a < K; ++a) coef_planes_set(p.rw[x * 32 + a], rows[x * K + a]);
		std::memset(W, 0, sizeof(W));
	}
	for (uint32_t x = 0; x < e; ++x)
		for (uint32_t r = 0; r < e; ++r) {
			coef_planes_set(p.w[x * 4 + r], W[x * e + r]);
		}
	p.raid6_dbl = 0xffu;
	const bool k8 = K == 8 && (G == 8 || pl.geo == 2);
	if (e == 2 && p.par_row[0] == 0 && p.par_row[1] == 1 && !k8) {
		// RAID-6 shape on a runtime-k instantiation (see the kernel)
		set_raid6_pair(p.w, p.erased_idx[0], p.erased_idx[1]);
		if (o.solve == LZGPU_RECOVER_SOLVE_RAID6 && o.doublings >= 0) p.raid6_dbl = static_cast<uint32_t>(o.doublings);
	}
	// "rows 0, 1, .., e-1 in use" (the first e parity parts are the available ones — the common case): instantiations that
	// multiply row r by 2^r in one step
	bool consecutive = true;
	for (uint32_t r = 0; r < e; ++r) consecutive &= p.par_row[r] == r;
	p.elim3_dbl = 0xffu;
	uint8_t elim3[6] = {0};
	if (e == 3 && consecutive) {
		// three unknowns, parity rows 0, 1, 2: w[0..3] = alpha, beta, gamma, delta; w[4], w[5] = 2^a, 4^a when a > 3
		elim3_constants(p.erased_idx[0], p.erased_idx[1], p.erased_idx[2], elim3);
		for (int i = 0; i < 6; ++i) coef_planes_set(p.w[i], elim3[i]);
		if (o.solve == LZGPU_RECOVER_SOLVE_ELIM3 && o.doublings >= 0) p.elim3_dbl = static_cast<uint32_t>(o.doublings);
	}
	TmapArray maps;
	for (int a = 0; a < K; ++a)
		if (make_tensor_map(fs, &maps.m[a], d_parts[pl.used[a]], static_cast<uint64_t>(pb) * 4, n_chunks, part_stride, G * 4) != CUDA_SUCCESS)
			return LZGPU_NOT_HANDLED;
	if (verifying && !d_first_bad) return LZGPU_NOT_HANDLED;  // (callers that pass stored CRCs always pass the result word, initialised to ~0)
	// what the plan names is what launches
	const lzgpu_launch_geometry geo = launch_geo(o.kernel, o.threads, G, o.stages, o.gf_warps, o.smem_bytes);
	if (o.kernel == LZGPU_KERNEL_RECOVER_BS3) {
		// the six constants of the elimination (set above for the packed-word kernel) as 8 x 8 bit matrices of all-ones / zero words
		BsRecoverMasks mk;
		for (int i = 0; i < 6; ++i) bs_mask_set(mk.m[i], elim3[i]);
		for (const auto &k : kBsRecoverers)
			if (k.kt == o.kt) return launch(ctx, k.fn, geo, 1, p.total_units, st, maps, p, mk);
	} else {
		const bool first_e = o.rows == LZGPU_RECOVER_ROWS_FIRST_E;
		for (const RecoverKernelEntry &k : kRecoverers)
			if (k.kernel == o.kernel && k.e == e && k.kt == o.kt && k.first_e == first_e && k.wide == pl.wide)
				return launch(ctx, k.fn, geo, o.kernel == LZGPU_KERNEL_RECOVER_GEO1 ? 2 : 1, p.total_units, st, maps, p);
	}
	lz_set_error("recover: no instantiation for k = %u, e = %u", o.kt, o.lost_data_parts);
	return LZGPU_ERR_ARG;
}

// ---------------------------------------------------------------------------------------------------
// fused stripe check (check_kernel.cuh)
// ---------------------------------------------------------------------------------------------------
int lz_fused_check(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                   const void *const *d_part_crc, void *d_verdict, cudaStream_t st, unsigned long long *d_first_bad, bool map,
                   const uint8_t *elim, unsigned long long *d_failed) {
	FusedState *fs = ctx->fused;
	if (d_failed && !map) return LZGPU_ERR_ARG;  // (cannot happen: only the repair asks for the failing blocks, through the map)
	if (!fs || fs->disabled) return LZGPU_NOT_HANDLED;
	const int K = goal->k, M = goal->m;
	if (part_stride % 16) return LZGPU_NOT_HANDLED;
	// the geometry (check_plan, fused_plan.h): the checked parity rows, G and the stage ring
	uint8_t given[LZGPU_MAX_PARTS];
	for (int i = 0; i < K + M; ++i) given[i] = d_parts[i] ? 1 : 0;
	const CheckPlan pl = check_plan(K, M, lz::uses_cauchy(K, M), given);
	const lzgpu_check_plan &o = pl.out;
	if (!o.fused) return LZGPU_NOT_HANDLED;
	CheckParams p{};
	CheckLost lost{};
	const void *slot_ptr[kCheckMaxSlots];
	// the given data parts in slots 0 .. D-1, then the parity rows; a lost data part has no slot
	uint32_t D = 0;
	for (int a = 0; a < K; ++a) {
		if (!d_parts[a]) {
			lost.mask |= 1u << a;
			continue;
		}
		slot_ptr[D] = d_parts[a];
		p.part_id[D++] = static_cast<uint8_t>(a);
	}
	const uint32_t R = o.rows, G = o.G, n_stages = o.stages, NSLOT = D + R, E = K - D;
	if (E > 0 && (!map || !elim)) return LZGPU_ERR_ARG;  // (cannot happen: only the degraded map loses data parts)
	bool verifying = false;
	for (uint32_t r = 0; r < R; ++r) {
		slot_ptr[D + r] = d_parts[K + pl.row[r]];
		p.part_id[D + r] = static_cast<uint8_t>(K + pl.row[r]);
		p.row[r] = pl.row[r];
	}
	for (uint32_t i = 0; E > 0 && i < (R - E) * E; ++i) coef_planes_set(lost.elim[i], elim[i]);
	for (uint32_t a = 0; a < NSLOT; ++a) {
		p.stored[a] = d_part_crc ? static_cast<const uint32_t *>(d_part_crc[p.part_id[a]]) : nullptr;
		verifying |= p.stored[a] != nullptr;
	}
	if (verifying && !d_first_bad) return LZGPU_NOT_HANDLED;
	const uint32_t pb = (nb + K - 1) / K;
	p.tables = ctx->d_crc_tables;
	p.first_bad = d_first_bad;
	p.verdict = map ? nullptr : static_cast<int *>(d_verdict);
	p.n_chunks = n_chunks;
	p.pb = pb;
	p.K = K;
	p.G = G;
	p.units_per_chunk = (pb + G - 1) / G;
	const uint64_t total = static_cast<uint64_t>(p.units_per_chunk) * n_chunks;
	if (total > 0x7fffffffull) return LZGPU_NOT_HANDLED;
	p.total_units = static_cast<uint32_t>(total);
	p.n_stages = n_stages;
	std::memcpy(p.qmult, fs->qmult, sizeof(p.qmult));
	p.zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	CheckTmaps maps;
	for (uint32_t a = 0; a < NSLOT; ++a)
		if (make_tensor_map(fs, &maps.m[a], slot_ptr[a], static_cast<uint64_t>(pb) * 4, n_chunks, part_stride, G * 4) != CUDA_SUCCESS) return LZGPU_NOT_HANDLED;
	const lzgpu_launch_geometry geo = launch_geo(E > 0 ? LZGPU_KERNEL_CHECK_DEGRADED : LZGPU_KERNEL_CHECK, o.threads, G, n_stages, 0, o.smem_bytes);
	uint32_t *d_map = static_cast<uint32_t *>(d_verdict);
	const bool consecutive = o.consecutive != 0;
	if (E > 0) {
		for (const CheckDegradedKernels &k : kDegradedCheckers)
			if (k.e == E && k.r == R && k.consecutive == consecutive)
				return d_failed ? launch(ctx, k.repair, geo, 1, p.total_units, st, maps, p, d_map, lost, d_failed)
				                : launch(ctx, k.map, geo, 1, p.total_units, st, maps, p, d_map, lost);
	} else {
		for (const CheckKernels &k : kCheckers)
			if (k.r == R && k.consecutive == consecutive)
				return d_failed ? launch(ctx, k.repair, geo, 1, p.total_units, st, maps, p, d_map, d_failed)
				       : map    ? launch(ctx, k.map, geo, 1, p.total_units, st, maps, p, d_map)
				                : launch(ctx, k.check, geo, 1, p.total_units, st, maps, p);
	}
	// (cannot happen: check_plan only gives the (E, R, rows) the lists hold, see kCheckers)
	lz_set_error("check: no instantiation for e = %u, r = %u, consecutive = %d", E, R, consecutive ? 1 : 0);
	return LZGPU_ERR_ARG;
}

// ---------------------------------------------------------------------------------------------------
// fused slice conversion (convert_kernel.cuh)
// ---------------------------------------------------------------------------------------------------

// Source slice `src` (k of its parts available in d_parts, at most two data parts lost, the parity parts in use being its rows
// 0 .. e-1) -> every wanted part of the destination slice `dst` in d_out (nullptr = not wanted) + the destination slice's block
// CRCs in chunk order (d_crc: nb data blocks, then m x pbd parity blocks per chunk), one pass.  LZGPU_NOT_HANDLED = use the two-pass route.
int lz_fused_convert(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb, const void *const *d_parts,
                     size_t part_stride, const void *const *d_part_crc, void *const *d_out, size_t out_stride, void *d_crc, size_t crc_stride,
                     cudaStream_t st, unsigned long long *d_first_bad) {
	FusedState *fs = ctx->fused;
	bool verifying = false;
	if (!fs || fs->disabled || fs->convert_off) return LZGPU_NOT_HANDLED;
	const int Ks = src->k, Ms = src->m, Kd = dst->k, Md = dst->m;
	if (src->kind == LZGPU_KIND_STD || dst->kind == LZGPU_KIND_STD) return LZGPU_NOT_HANDLED;
	if ((part_stride % 16) || (out_stride % 16) || n_chunks == 0 || nb == 0) return LZGPU_NOT_HANDLED;
	// inputs: the first k available parts (ec_read_plan.h:126-133); geometry from the shared plan (fused_plan.h, unit-tested on the CPU)
	ConvertParams p{};
	uint8_t avail[LZGPU_MAX_PARTS] = {0};
	for (int i = 0; i < Ks + Ms; ++i) avail[i] = d_parts[i] ? 1 : 0;
	const ConvertPlan pl = convert_plan(Ks, Ms, lz::uses_cauchy(Ks, Ms), Kd, Md, lz::uses_cauchy(Kd, Md), avail, fs->max_smem);
	if (!pl.ok) return LZGPU_NOT_HANDLED;
	int used[LZGPU_MAX_DATA], n_used = 0;
	for (int i = 0; i < Ks + Ms && n_used < Ks; ++i)
		if (d_parts[i]) used[n_used++] = i;
	const uint32_t e = pl.e;
	for (int a = 0; a < Ks; ++a)
		if (used[a] < Ks) p.slot_present[used[a]] = 1;
	p.erased_idx[0] = pl.erased[0];
	p.erased_idx[1] = pl.erased[1];
	const uint32_t G = pl.G, T = pl.T, RR = pl.region_rows, n_stages = pl.n_stages;
	const uint32_t pbs = (nb + Ks - 1) / Ks, pbd = (nb + Kd - 1) / Kd;
	const uint32_t R = G * Kd;
	p.Kd = Kd; p.G = G; p.pbd = pbd; p.Ks = Ks; p.T = T; p.pbs = pbs; p.region_rows = RR;
	p.n_chunks = n_chunks; p.nb = nb; p.n_stages = n_stages;
	p.units_per_chunk = (nb + R - 1) / R;
	const uint64_t total = static_cast<uint64_t>(p.units_per_chunk) * n_chunks;
	if (total > 0x7fffffffull) return LZGPU_NOT_HANDLED;
	p.total_units = static_cast<uint32_t>(total);
	for (int j = 0; j < Kd; ++j) p.data_out[j] = static_cast<uint8_t *>(d_out[j]);
	for (int r = 0; r < Md; ++r) p.par_out[r] = static_cast<uint8_t *>(d_out[Kd + r]);
	p.part_out_stride = out_stride;
	p.crc = static_cast<uint32_t *>(d_crc);
	p.crc_stride = crc_stride;
	p.tables = ctx->d_crc_tables;
	p.first_bad = d_first_bad;
	std::memcpy(p.qmult, fs->qmult, sizeof(p.qmult));
	p.zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	TmapArray maps;
	uint32_t n_par_seen = 0;
	for (int a = 0; a < Ks; ++a) {
		const int idx = used[a];
		const uint32_t slot = idx < Ks ? static_cast<uint32_t>(idx) : static_cast<uint32_t>(Ks) + n_par_seen++;
		p.loaded_slot[a] = static_cast<uint8_t>(slot);
		p.part_id[slot] = static_cast<uint8_t>(idx);
		p.stored[slot] = d_part_crc ? static_cast<const uint32_t *>(d_part_crc[idx]) : nullptr;
		if (p.stored[slot]) verifying = true;
		if (reinterpret_cast<uintptr_t>(d_parts[idx]) % 16) return LZGPU_NOT_HANDLED;
		if (make_tensor_map(fs, &maps.m[a], d_parts[idx], static_cast<uint64_t>(pbs) * 4, n_chunks, part_stride, T * 4) != CUDA_SUCCESS) return LZGPU_NOT_HANDLED;
	}
	p.n_loaded = static_cast<uint32_t>(Ks);
	for (uint32_t bl = 0; bl < R; ++bl) {
		const uint32_t row0 = (bl % Ks) * RR + (bl / Ks) * 4;
		p.bl_entry[bl] = static_cast<uint16_t>(row0 * kStepBytes + ((row0 & 4) ? 64 : 0));
	}
	for (uint32_t x = 0; x < e; ++x) p.part_id[Ks + x] = static_cast<uint8_t>(Ks + x);
	if (verifying && !d_first_bad) return LZGPU_NOT_HANDLED;
	if (e == 2) set_raid6_pair(p.w, p.erased_idx[0], p.erased_idx[1]);
	p.dbl0 = (e == 2 && p.erased_idx[0] <= 4) ? p.erased_idx[0] : 0xffu;
	const uint32_t rebuild_warps = kConvertThreads / 32 - pl.n_workers;   // (0 without lost parts: every warp is a worker)
	ConvertKernel fn = nullptr;   // the compile-time destination k where the list holds it, else the runtime-k kernel
	for (const auto &k : kConverters)
		if (k.m == Md && k.e == e && (k.kd == Kd || (k.kd == 0 && !fn))) fn = k.fn;
	if (!fn) return LZGPU_NOT_HANDLED;
	return launch(ctx, fn, launch_geo(LZGPU_KERNEL_CONVERT, kConvertThreads, G, n_stages, rebuild_warps, pl.smem), 2, p.total_units, st, maps, p);
}

// ---------------------------------------------------------------------------------------------------
// one-pass encode for several slices (slices_kernel.cuh)
// ---------------------------------------------------------------------------------------------------

// Every slice of `goals` (xor/ec goals and at most the standard slice; the caller has checked the arguments) in one pass over the
// data: parity of slice i to d_parity[i], CRC arrays as lz_fused_encode writes them (standard slice: the nb data CRCs) to d_crc[i].
// LZGPU_NOT_HANDLED = the plan refuses the set, or the strides / alignment are not the kernel's: take the per-slice route.
int lz_fused_encode_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb, const void *d_data,
                           size_t chunk_stride, void *const *d_parity, const size_t *parity_stride, void *const *d_crc, const size_t *crc_stride,
                           cudaStream_t st) {
	FusedState *fs = ctx->fused;
	if (!fs || fs->disabled || n_chunks == 0 || nb == 0) return LZGPU_NOT_HANDLED;
	if ((chunk_stride % 16) || (reinterpret_cast<uintptr_t>(d_data) % 16)) return LZGPU_NOT_HANDLED;
	bool cauchy[kSlicesMax] = {false};
	for (uint32_t i = 0; i < n_slices; ++i) {
		if (slice_is_std(goals[i])) continue;
		cauchy[i] = lz::uses_cauchy(goals[i].k, goals[i].m);
		if ((parity_stride[i] % 16) || (reinterpret_cast<uintptr_t>(d_parity[i]) % 16)) return LZGPU_NOT_HANDLED;
	}
	const SlicesPlan pl = slices_plan(goals, cauchy, n_slices, n_chunks, nb);
	const lzgpu_slices_plan &o = pl.out;
	if (!o.fused) return LZGPU_NOT_HANDLED;
	SlicesParams p{};
	uint32_t gs = 0, prow4 = 0;
	for (uint32_t i = 0; i < n_slices; ++i) {
		const bool std_slice = slice_is_std(goals[i]);
		p.parity[i] = std_slice ? nullptr : static_cast<uint8_t *>(d_parity[i]);
		p.crc[i] = static_cast<uint32_t *>(d_crc[i]);
		p.parity_stride[i] = std_slice ? 0 : parity_stride[i];
		p.crc_stride[i] = crc_stride[i];
		p.k[i] = static_cast<uint32_t>(goals[i].k);
		p.m[i] = std_slice ? 0 : static_cast<uint32_t>(goals[i].m);
		p.pb[i] = std_slice ? 0 : (nb + p.k[i] - 1) / p.k[i];
		p.S[i] = pl.S[i];
		p.prow4[i] = prow4;
		if (p.m[i] > 1) prow4 += p.S[i] * (p.m[i] - 1);
		for (uint32_t s = 0; s < p.S[i]; ++s, ++gs) {
			p.gs_slice[gs] = static_cast<uint8_t>(i);
			p.gs_stripe[gs] = static_cast<uint8_t>(s);
		}
	}
	p.tables = ctx->d_crc_tables;
	p.n_slices = n_slices;
	p.n_stripes = gs;
	p.n_chunks = n_chunks;
	p.nb = nb;
	p.R = pl.R;
	p.prows = pl.prows;
	p.units_per_chunk = (nb + pl.R - 1) / pl.R;
	p.total_units = o.units;
	p.n_stages = o.stages;
	std::memcpy(p.qmult, fs->qmult, sizeof(p.qmult));
	p.zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	CUtensorMap map;
	const CUresult r = make_tensor_map(fs, &map, d_data, static_cast<uint64_t>(nb) * 4, n_chunks, chunk_stride, 4 * pl.R);
	if (r != CUDA_SUCCESS) {
		lz_set_error("cuTensorMapEncodeTiled failed with CUresult %d (rows/chunk %u, chunks %u, stride %zu, box rows %u)", static_cast<int>(r), nb * 4,
		             n_chunks, chunk_stride, 4 * pl.R);
		return LZGPU_ERR_CUDA;
	}
	for (const auto &k : kSlicers)
		if (k.m == pl.m)
			return launch(ctx, k.fn, launch_geo(LZGPU_KERNEL_ENCODE_SLICES, o.threads, o.G, o.stages, 0, o.smem_bytes), 1, p.total_units, st, map, p);
	return LZGPU_NOT_HANDLED;   // (cannot happen: the plan refuses m > 4, which only Cauchy goals have)
}

// ---------------------------------------------------------------------------------------------------
// recovery from the parts of every slice together (recover_slices_kernel.cuh)
// ---------------------------------------------------------------------------------------------------

// The kernel's tables for one stripe shape: what is read and staged, what is written, the CRC streams, the solve.  image_crc: the
// image blocks get CRC streams (the salvage form).  chk: the check form's checks of this shape (slices_check.h): each defining block
// staged at L + E + h, its prediction as the wanted-parity entry h (a further copy of position q: row kRsNone, stripe q), and the
// particular-solution rows instead of the solve's
static void rs_fill_shape(RsShape &o, const SliceLayout &lay, const SliceSolve &sv, const void *const *d_parts, const void *const *d_stored,
                          const uint8_t *want, void *const *d_out_crc, bool image, bool image_crc, const SliceChecks *chk = nullptr) {
	const uint32_t L = lay.L, E = sv.n_eq;
	std::memset(&o, 0, sizeof(o));
	uint64_t staged = 0;
	auto add_state = [&](uint8_t part, uint8_t s, uint8_t written) -> uint8_t {
		o.state[o.n_state] = RsEntry{part, s, written, static_cast<uint8_t>(written ? 0 : o.n_read)};   // a read block's: its read entry
		return static_cast<uint8_t>(o.n_state++);
	};
	for (uint32_t i = 0; i < lay.n_slices; ++i)
		for (uint32_t p = 0; p < lay.k[i] + lay.m[i]; ++p) {
			const uint32_t g = lay.base[i] + p;
			if (!d_parts[g]) continue;
			for (uint32_t s = 0; s < L / lay.k[i]; ++s) {
				if (!stripe_exists(lay, i, s, sv.valid)) continue;
				uint8_t slot = kRsNone;
				if (p < lay.k[i]) {
					const uint32_t q = s * lay.k[i] + p;
					if (q < sv.valid && !((staged >> q) & 1ull)) { slot = static_cast<uint8_t>(q); staged |= 1ull << q; }
				} else {
					for (uint32_t e = 0; e < E; ++e)
						if (sv.eq_slice[e] == i && sv.eq_row[e] == p - lay.k[i] && sv.eq_stripe[e] == s) slot = static_cast<uint8_t>(L + e);
				}
				if (chk && chk->check_of[g][s] >= 0) {
					const uint32_t h = static_cast<uint32_t>(chk->check_of[g][s]);
					slot = static_cast<uint8_t>(L + E + h);
					o.out_slice[h] = static_cast<uint8_t>(i);
					o.out_row[h] = p < lay.k[i] ? kRsNone : static_cast<uint8_t>(p - lay.k[i]);
					o.out_stripe[h] = static_cast<uint8_t>(p < lay.k[i] ? s * lay.k[i] + p : s);
				}
				const bool verify = d_stored && d_stored[g];
				if (slot == kRsNone && !verify) continue;   // neither used nor verified: not read
				const uint8_t st = verify ? add_state(static_cast<uint8_t>(g), static_cast<uint8_t>(s), 0) : kRsNone;   // names read entry n_read
				o.read[o.n_read++] = RsEntry{static_cast<uint8_t>(g), static_cast<uint8_t>(s), slot, st};
			}
		}
	for (uint32_t q = 0; q < L; ++q)
		if (!((staged >> q) & 1ull)) o.zero[o.n_zero++] = static_cast<uint8_t>(q);
	o.n_unknown = static_cast<uint16_t>(sv.n_unknown);
	o.n_eq = static_cast<uint16_t>(E);
	std::memcpy(o.unk_pos, sv.unk_pos, sizeof(o.unk_pos));
	std::memcpy(o.eq_slice, sv.eq_slice, sizeof(o.eq_slice));
	std::memcpy(o.eq_row, sv.eq_row, sizeof(o.eq_row));
	std::memcpy(o.eq_stripe, sv.eq_stripe, sizeof(o.eq_stripe));
	std::memcpy(o.rows, chk ? chk->prow : sv.rows, sizeof(o.rows));
	if (chk) o.n_out = static_cast<uint16_t>(chk->n_checks);
	for (uint32_t i = 0; i < lay.n_slices; ++i)
		for (uint32_t p = 0; p < lay.k[i] + lay.m[i]; ++p) {
			const uint32_t g = lay.base[i] + p;
			if (!want[g]) continue;
			for (uint32_t s = 0; s < L / lay.k[i]; ++s) {
				if (!stripe_exists(lay, i, s, sv.valid)) continue;
				uint8_t slot;
				if (p < lay.k[i]) {
					slot = static_cast<uint8_t>(s * lay.k[i] + p);
				} else {
					o.out_slice[o.n_out] = static_cast<uint8_t>(i);
					o.out_row[o.n_out] = static_cast<uint8_t>(p - lay.k[i]);
					o.out_stripe[o.n_out] = static_cast<uint8_t>(s);
					slot = static_cast<uint8_t>(L + E + o.n_out++);
				}
				const uint8_t st = d_out_crc && d_out_crc[g] ? add_state(static_cast<uint8_t>(g), static_cast<uint8_t>(s), 1) : kRsNone;
				o.write[o.n_write++] = RsEntry{static_cast<uint8_t>(g), static_cast<uint8_t>(s), slot, st};
			}
		}
	if (image)
		for (uint32_t q = 0; q < sv.valid; ++q)
			o.write[o.n_write++] = RsEntry{kRsNone, static_cast<uint8_t>(q), static_cast<uint8_t>(q), image_crc ? add_state(kRsNone, static_cast<uint8_t>(q), 1) : kRsNone};
}

// The salvage form's masks for one stripe shape, from the tables rs_fill_shape made of it: a known position depends on the read entry
// that staged it; a solved one on every equation its row uses (rows[x][e] != 0), i.e. on that equation's parity block and on the
// staged known positions of its slice stripe.  Status from the solve's masks.
static void rs_fill_salvage(RsSalvage &o, const RsShape &sh, const SliceLayout &lay, const SliceSolve &sv) {
	const uint32_t L = lay.L, E = sv.n_eq;
	std::memset(&o, 0, sizeof(o));
	int stager[kRsMaxL], eq_read[kRsMaxL];
	for (uint32_t q = 0; q < L; ++q) stager[q] = eq_read[q] = -1;
	for (uint32_t r = 0; r < sh.n_read; ++r) {
		const uint32_t slot = sh.read[r].slot;
		if (slot == kRsNone) continue;
		if (slot < L) stager[slot] = static_cast<int>(r);
		else eq_read[slot - L] = static_cast<int>(r);
	}
	auto depend = [&](uint32_t q, int r) {
		if (r >= 0) o.dep[q][r >> 5] |= 1u << (r & 31);
	};
	for (uint32_t q = 0; q < sv.valid; ++q) {
		const bool known = (sv.known >> q) & 1ull, determined = (sv.determined >> q) & 1ull;
		o.status[q] = known ? LZGPU_SALVAGE_KNOWN : determined ? LZGPU_SALVAGE_SOLVED : LZGPU_SALVAGE_HOLE;
		if (known) depend(q, stager[q]);
	}
	for (uint32_t x = 0; x < sv.n_unknown; ++x) {
		const uint32_t q = sv.unk_pos[x];
		for (uint32_t e = 0; e < E; ++e) {
			if (!sv.rows[x][e]) continue;
			const uint32_t i = sv.eq_slice[e], s = sv.eq_stripe[e];
			depend(q, eq_read[e]);
			for (uint32_t j = 0; j < lay.k[i]; ++j)
				if (s * lay.k[i] + j < sv.valid && ((sv.known >> (s * lay.k[i] + j)) & 1ull)) depend(q, stager[s * lay.k[i] + j]);
		}
	}
}

// part_stride, spc and every flat part's slice and pointer, alike in the parameters of the recovery, locate and correct kernels
template <class Params>
static void rs_fill_parts(Params &o, const SliceLayout &lay, const void *const *d_parts, const size_t *part_stride) {
	for (uint32_t i = 0; i < lay.n_slices; ++i) {
		o.part_stride[i] = part_stride[i];
		o.spc[i] = lay.L / lay.k[i];
		for (uint32_t g = lay.base[i]; g < lay.base[i] + lay.k[i] + lay.m[i]; ++g) {
			o.part_slice[g] = static_cast<uint8_t>(i);
			o.parts[g] = static_cast<uint8_t *>(const_cast<void *>(d_parts[g]));
		}
	}
}

// lzgpu_check_slices' locate pass, after the CHECK launch has written every entry to d_map: the tables of both shapes in a
// stream-ordered temporary, and one CTA per bad entry.  lzgpu_correct_slices, after the CORRECT launch (d_map a temporary, d_crc_failed
// its masks): the rows of P of both shapes after the annihilators, then correct_slices_kernel over every entry, into d.map's fix entries.
static int rs_locate(lzgpu_ctx *ctx, const RecoverSlicesCall &c, const SlicesBufs &d, uint32_t n_chunks, uint32_t nb, RsCheckEntry *d_map,
                     const unsigned long long *d_crc_failed, cudaStream_t st) {
	const SliceLayout &lay = c.lay;
	const SliceChecks *checks = c.checks;
	RsFixEntry *d_fix = c.mode == RsMode::CORRECT ? static_cast<RsFixEntry *>(d.map) : nullptr;
	const uint32_t n_cs = (nb + lay.L - 1) / lay.L, tail = nb % lay.L ? 1u : 0u;
	size_t rows = checks[0].ann.size() / kScMaxChecks + (tail ? checks[1].ann.size() / kScMaxChecks : 0);
	const size_t ann_rows = rows;
	if (d_fix) rows += checks[0].n_blocks + (tail ? checks[1].n_blocks : 0);
	std::vector<uint8_t> host(sizeof(RsLocate) + rows * kRsMaxOut, 0);
	RsLocate *loc = reinterpret_cast<RsLocate *>(host.data());
	uint8_t *ann = host.data() + sizeof(RsLocate);
	uint32_t row0 = 0;
	for (int t = 0; t < 2; ++t) {
		if (t == 0 ? nb < lay.L : !tail) continue;
		const SliceChecks &ck = checks[t];
		RsLocateShape &o = loc->shape[t];
		o.n_blocks = ck.n_blocks;
		o.n_checks = ck.n_checks;
		o.ann0 = row0;
		for (uint32_t b = 0; b < ck.n_blocks; ++b) {
			o.blk_part[b] = ck.blk_part[b];
			o.blk_s[b] = ck.blk_s[b];
			for (uint32_t h = 0; h < ck.n_checks; ++h) o.H[h][b] = ck.H[h * ck.n_blocks + b];
		}
		for (uint32_t g = 0; g < LZGPU_MAX_PARTS; ++g) {
			if (!((ck.parts >> g) & 1ull)) continue;
			o.cand_part[o.n_cand] = static_cast<uint8_t>(g);
			o.cand_first[o.n_cand] = static_cast<uint16_t>(ck.ann_first[g]);
			o.cand_first[++o.n_cand] = static_cast<uint16_t>(ck.ann_first[g + 1]);
		}
		std::memcpy(ann + static_cast<size_t>(row0) * kRsMaxOut, ck.ann.data(), ck.ann.size());
		row0 += static_cast<uint32_t>(ck.ann.size() / kScMaxChecks);
	}
	auto cp = std::make_unique<CorrectSlicesParams>();
	std::memset(cp.get(), 0, sizeof(CorrectSlicesParams));
	size_t smem = 0;
	for (uint32_t t = 0, prow = static_cast<uint32_t>(ann_rows); d_fix && t < 2; ++t) {
		if (t == 0 ? nb < lay.L : !tail) continue;
		const SliceChecks &ck = checks[t];
		RsCorrectShape &o = cp->shape[t];
		o.correctable = ck.correctable;
		o.prow0 = prow;
		uint32_t most = 0;
		for (uint32_t b = 0; b < ck.n_blocks; ++b) {
			const uint32_t g = ck.blk_part[b];
			if (!o.blk_count[g]) o.blk_first[g] = static_cast<uint8_t>(b);
			++o.blk_count[g];
			if ((ck.correctable >> g) & 1ull) most = std::max<uint32_t>(most, o.blk_count[g]);
			std::memcpy(ann + static_cast<size_t>(prow + b) * kRsMaxOut, &ck.pinv[static_cast<size_t>(b) * kScMaxChecks], kScMaxChecks);
		}
		prow += ck.n_blocks;
		smem = std::max(smem, rsc_smem_bytes(ck.n_checks, most));
	}
	TmpBuf d_loc(ctx, st);
	int rc;
	if ((rc = d_loc.alloc(host.size()))) return rc;
	CUDA_TRY(cudaMemcpyAsync(d_loc.p, host.data(), host.size(), cudaMemcpyHostToDevice, st));
	auto p = std::make_unique<LocateSlicesParams>();
	std::memset(p.get(), 0, sizeof(LocateSlicesParams));
	rs_fill_parts(*p, lay, d.parts, d.part_stride);
	p->map = d_map;
	p->loc = static_cast<const RsLocate *>(d_loc.p);
	p->n_entries = static_cast<unsigned long long>(n_chunks) * n_cs;
	p->n_cs = n_cs;
	p->tail = tail;
	uint64_t grid = std::min<uint64_t>(p->n_entries, static_cast<uint64_t>(ctx->sm_count) * 8);
	if (ctx->fused->grid_cap) grid = std::min<uint64_t>(grid, ctx->fused->grid_cap);
	locate_slices_kernel<<<static_cast<unsigned>(grid), kRslThreads, 0, st>>>(*p);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	if (!d_fix) return LZGPU_OK;
	rs_fill_parts(*cp, lay, d.parts, d.part_stride);
	std::memcpy(cp->pb, c.pb, sizeof(cp->pb));
	for (uint32_t g = 0; g < lay.n_parts; ++g) cp->new_crc[g] = d.new_crc ? static_cast<uint32_t *>(d.new_crc[g]) : nullptr;
	cp->map = d_map;
	cp->crc_failed = d_crc_failed;
	cp->fix = d_fix;
	cp->loc = p->loc;
	cp->tables = ctx->d_crc_tables;
	cp->n_entries = p->n_entries;
	cp->n_cs = n_cs;
	cp->tail = tail;
	cp->crc_off = lzgpu_crc_enabled() ? 0u : 1u;
	cp->zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	cp->run_mult = lz::crc_xpow_bytes(kRscRun);
	for (int i = 0; i < 5; ++i) cp->tree_mult[i] = lz::crc_xpow_bytes(2048ull << i);
	correct_slices_kernel<<<static_cast<unsigned>(grid), kRscThreads, smem, st>>>(*cp);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

int lz_recover_slices(lzgpu_ctx *ctx, const RecoverSlicesCall &c, const SlicesBufs &d, uint32_t n_chunks, uint32_t nb, cudaStream_t st,
                      unsigned long long *d_first_bad) {
	const SliceLayout &lay = c.lay;
	const RsGeometry &geo = c.geo;
	const RsMode mode = c.mode;
	const bool checks = mode == RsMode::CHECK || mode == RsMode::CORRECT;
	auto p = std::make_unique<RecoverSlicesParams>();
	std::memset(p.get(), 0, sizeof(RecoverSlicesParams));
	const bool crc_on = lzgpu_crc_enabled() != 0;
	rs_fill_parts(*p, lay, d.parts, d.part_stride);
	for (uint32_t i = 0; i < lay.n_slices; ++i) p->out_stride[i] = d.out_stride ? d.out_stride[i] : 0;
	for (uint32_t g = 0; g < lay.n_parts; ++g) {
		p->stored[g] = d.part_crc ? static_cast<const uint32_t *>(d.part_crc[g]) : nullptr;
		p->out[g] = d.want[g] ? static_cast<uint8_t *>(d.out[g]) : nullptr;
		p->out_crc[g] = d.want[g] && d.out_crc ? static_cast<uint32_t *>(d.out_crc[g]) : nullptr;
	}
	std::memcpy(p->k, lay.k, sizeof(p->k));
	std::memcpy(p->pb, c.pb, sizeof(p->pb));
	std::memcpy(p->gen, lay.gen, sizeof(p->gen));
	p->image = static_cast<uint8_t *>(d.image);
	p->image_stride = d.image_stride;
	p->tables = ctx->d_crc_tables;
	p->first_bad = d_first_bad;
	p->L = lay.L;
	p->G = geo.G;
	p->nb = nb;
	p->n_cs = (nb + lay.L - 1) / lay.L;
	p->tail = nb % lay.L ? 1u : 0u;
	p->units_per_chunk = (p->n_cs + geo.G - 1) / geo.G;
	p->total_units = p->units_per_chunk * n_chunks;
	p->n_slots = geo.slots;
	p->n_states_max = geo.states;
	p->crc_off = crc_on ? 0u : 1u;
	p->zconst = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
	for (int i = 0; i < 5; ++i) p->tree_mult[i] = lz::crc_xpow_bytes(2048ull << i);
	const bool verifying = d.part_crc != nullptr;
	if (verifying && !d_first_bad) return LZGPU_ERR_ARG;  // (cannot happen: the caller arms a ticket whenever it passes stored CRCs)
	p->image_crc = static_cast<uint32_t *>(d.image_crc);
	p->map = static_cast<uint8_t *>(d.map);
	TmpBuf d_tmp(ctx, st);   // CORRECT: the check's entries and the failing-part masks, before correct_slices_kernel writes d.map
	const unsigned long long n_entries = static_cast<unsigned long long>(n_chunks) * p->n_cs;
	if (mode == RsMode::CORRECT) {
		int rc;
		if ((rc = d_tmp.alloc(n_entries * (sizeof(RsCheckEntry) + sizeof(unsigned long long))))) return rc;
		p->map = static_cast<uint8_t *>(d_tmp.p);
		p->crc_failed = reinterpret_cast<unsigned long long *>(p->map + n_entries * sizeof(RsCheckEntry));
	}
	for (int t = 0; t < 2; ++t)
		if (t == 0 ? nb >= lay.L : p->tail != 0) {
			rs_fill_shape(p->shape[t], lay, c.shapes[t], d.parts, d.part_crc, d.want, d.out_crc, d.image != nullptr, d.image_crc != nullptr,
			              checks ? &c.checks[t] : nullptr);
			if (mode == RsMode::SALVAGE) rs_fill_salvage(p->salvage[t], p->shape[t], lay, c.shapes[t]);
		}
	static const int kKernelOf[] = {LZGPU_KERNEL_RECOVER_SLICES, LZGPU_KERNEL_SALVAGE_SLICES, LZGPU_KERNEL_CHECK_SLICES,
	                                LZGPU_KERNEL_CORRECT_SLICES};
	const lzgpu_launch_geometry g = launch_geo(kKernelOf[static_cast<int>(mode)], geo.threads, geo.G, geo.stages, 0, geo.smem);
	int rc = launch(ctx, kRecoverSlicers[static_cast<int>(mode)], g, 1, p->total_units, st, *p);
	if (rc || !checks) return rc;
	return rs_locate(ctx, c, d, n_chunks, nb, reinterpret_cast<RsCheckEntry *>(p->map), p->crc_failed, st);
}
