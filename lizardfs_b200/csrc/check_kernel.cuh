// check_kernel.cuh — fused stripe-consistency check (lzgpu_check_stripes): do the k data parts and the given parity parts of
// every stripe still form a codeword, and does every part block still match its stored CRC?  ONE pass over the parts.
//
// The syndrome of checked parity row r is  S_r = p_r ^ sum_j (2^r)^j d_j  (Vandermonde generator, galois_field_isal.cc:53-69;
// xorN is row 0 alone); a stripe is a codeword exactly when every S_r is zero.  Only the position of the first non-zero stripe of
// each chunk leaves this kernel: locate_kernel (kernels_generic.cuh) recomputes that stripe's syndromes to name a part.
//
// Data movement and roles follow fused_recover_kernel's 16-warp geometry (fused_kernel.cuh): a work unit is G stripes of one chunk,
// each of the 128 steps loads one TMA box [G*4 rows x 128 B] per slot (k data parts, then the checked parity parts) into a stage
// ring tracked by full / empty mbarriers, and the consumer warp whose arrival empties a stage refills it.
//   CRC role  thread t owns row t of the stage (slot t / 4G): a 16 KiB stream folded with the sparse multiple of P, compared with
//             the stored CRC of its block at the end of the unit; the first mismatch lowers first_bad.
//   GF role   item (stripe g, quarter q, 16-byte column): Horner over the k data columns per checked row, XOR the stored parity
//             column, OR-reduce.  A thread keeps the lowest non-zero stripe of its unit and lowers the chunk's verdict word once
//             (fused_check_kernel), or keeps the non-zero rows of each stripe for the stripe map (fused_check_map_kernel).
//
// Lost data parts (lzgpu_check_stripe_map_degraded, fused_check_degraded_kernel): E data positions L have no slot.  The inputs are the
// k - E given data parts and the first E given parity rows P_in, the spares the other given rows P_sp (ECReadPlan::recoverParts).
// The Horner pass still runs over all k positions (a lost one contributes its multiply step only), so S_r = p_r ^ sum_{j not in L}
// g_rj d_j for every given row, and the spare rows are checked by  T_i = S_sp_i ^ sum_x C_ix S_in_x  with C = G[P_sp, L] G[P_in, L]^-1
// (the host reads C off the spares' recovery rows: the coefficients of the input parity parts).  T_i is spare block sp_i minus its
// re-encoding from the k inputs, what the generic route compares; it costs (R - E) E gf_mac per packed word.
#pragma once
#include "fused_kernel.cuh"

namespace lzd {

// (kCheckThreads and the geometry: check_plan, fused_plan.h)
constexpr int kCheckMaxSlots = 36;  // k data parts + up to four parity rows (ec(32,3) is the widest Vandermonde goal)

struct CheckTmaps {
	CUtensorMap m[kCheckMaxSlots];
};

struct CheckParams {
	const uint32_t *stored[kCheckMaxSlots];  // stored CRCs of slot a (chunk c at + c*pb), nullptr = not verified
	const uint32_t *tables;
	unsigned long long *first_bad;           // stored-CRC mismatch: atomicMin of (c*64 + part)*1024 + block
	int *verdict;                            // lzgpu_stripe_verdict[n_chunks]: first_bad_stripe (word 3c) lowered by atomicMin
	uint32_t n_chunks, pb, K, G, units_per_chunk, total_units, n_stages;
	uint32_t qmult[4];
	uint32_t zconst;
	uint8_t row[4];                          // generator row of checked parity slot K + r
	uint8_t part_id[kCheckMaxSlots];         // slot -> part index (error reporting)
};

// fused_check_degraded_kernel's own parameter (CheckParams keeps its layout: the existing kernels' parameter offsets do not move)
struct CheckLost {
	uint32_t mask;                           // bit j: data position j has no slot
	CoefPlanes elim[4];                      // C[i][x] at elim[i * E + x]: spare row E + i, input row x
};

// R = checked parity rows; CONSEC: they are rows 0 .. R-1 (row r multiplies by 2^r in one step), else p.row[r] doublings.
// MAP = false: the per-chunk verdict word (lzgpu_check_stripes).  MAP = true (lzgpu_check_stripe_map): every stripe's bad_rows goes to
// map[2 (c pb + s)] and its suspect_part word is set to -1 (locate_map_kernel names the suspects of the bad ones).  The items of
// stripe g are items 32g .. 32g + 31, i.e. the 32 lanes of one warp in the same pass of the item loop, and that warp owns the stripe
// for the whole unit: each lane keeps its row bits in a nibble per pass (at most 2048 items, four passes), and at the end of the unit
// the warp OR-reduces each nibble and lane 0 stores the stripe's entry.  Units partition the stripes, so the map needs no memset and
// no atomics.  E lost data positions (MAP only): slots 0 .. K-E-1 hold the given data parts, slot K - E + r parity row r.
// FAILED (lzgpu_repair_stripes, MAP only): a block that fails its stored CRC also sets bit part in failed[c pb + s] (zeroed by the
// caller), so that every failing block of every stripe is known, not only the first of the batch.
template <int R, bool CONSEC, bool MAP, int E = 0, bool FAILED = false>
__device__ __forceinline__ void fused_check_body(const CheckTmaps &tmaps, const CheckParams &p, uint32_t *map, const CheckLost *lost = nullptr,
                                                 unsigned long long *failed = nullptr) {
	static_assert(!FAILED || MAP, "the failing blocks are recorded by the map form");
	static_assert(E == 0 || (MAP && E < R), "a lost data part needs a spare row, and only the map form has one");
	constexpr int W = 4;
	constexpr uint32_t CPI = 32 / W;
	extern __shared__ __align__(1024) uint8_t smem[];
	const uint32_t sbase = smem_u32(smem);
	const uint32_t K = p.K, G = p.G, NSLOT = K - E + R, n_stages = p.n_stages;
	const uint32_t RG = G * 4;                       // rows per slot region
	const uint32_t ROWS = NSLOT * RG;
	const uint32_t region_bytes = RG * kStepBytes;   // multiple of 1024 (G even)
	const uint32_t stage_bytes = ROWS * kStepBytes;
	const uint32_t a_full = sbase + n_stages * stage_bytes, a_empty = a_full + 8 * n_stages;

	const uint32_t tid = threadIdx.x, lane = tid & 31, cw = tid >> 5;
	const uint32_t n_items = 4 * CPI * G;
	const uint32_t n_gf_warps = (min(n_items, static_cast<uint32_t>(kCheckThreads)) + 31) / 32;
	const uint32_t n_stage_warps = max((ROWS + 31) / 32, n_gf_warps);
	const uint32_t my_units = blockIdx.x < p.total_units ? (p.total_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
	const uint32_t total_steps = my_units * kStepsPerUnit;

	auto issue_load = [&](uint32_t c, uint32_t gi, uint32_t step, uint32_t st) {
		mbar_expect_tx(a_full + 8 * st, stage_bytes);
		for (uint32_t a = 0; a < NSLOT; ++a)
			tma_load_3d(sbase + st * stage_bytes + a * region_bytes, &tmaps.m[a], static_cast<int>(step * kStepBytes),
			            static_cast<int>(gi * RG), static_cast<int>(c), a_full + 8 * st);
	};

	if (tid == 0) {
		for (uint32_t s = 0; s < n_stages; ++s) {
			mbar_init(a_full + 8 * s, 1);
			mbar_init(a_empty + 8 * s, n_stage_warps);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		if (total_steps)
			for (uint32_t s = 0; s < n_stages; ++s) issue_load(blockIdx.x / p.units_per_chunk, blockIdx.x % p.units_per_chunk, s, s);
	}
	__syncthreads();
	if (cw >= n_stage_warps) return;

	const bool has_stream = tid < ROWS;
	const uint32_t slot = tid / RG, rr = tid % RG;           // this thread's stream: slot `slot`, block rr/4, quarter rr%4
	const bool verify = has_stream && p.stored[has_stream ? slot : 0] != nullptr;
	const uint32_t row_addr0 = (sbase + tid * kStepBytes) ^ ((tid & 7) << 4);
	const bool warp_has_items = cw < n_gf_warps;

	uint32_t win[64];
	FoldAux aux;  // unused: the fold without the auxiliary sequence keeps the window next to the Horner accumulators
	uint32_t it = 0, st = 0, ph = 0;
	for (uint32_t unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
		const uint32_t c = unit / p.units_per_chunk, gi = unit % p.units_per_chunk;
		const uint32_t stripe0 = gi * G;
		const uint32_t next_unit = unit + gridDim.x;
		const uint32_t next_c = next_unit / p.units_per_chunk, next_gi = next_unit % p.units_per_chunk;
		uint32_t bad_stripe = 0xffffffffu;
		uint32_t map_bits = 0;  // MAP: nibble i = the row bits of this thread's item in pass i of the item loop
#pragma unroll
		for (int i = 0; i < 64; ++i) win[i] = 0;

		for (int step0 = 0; step0 < kStepsPerUnit; step0 += 2) {
#pragma unroll
			for (int sub = 0; sub < 2; ++sub) {
				const int step = step0 + sub;
				const uint32_t stage = sbase + st * stage_bytes;
				mbar_wait(a_full + 8 * st, ph);

				if (warp_has_items) {
					for (uint32_t item = tid; item < n_items; item += kCheckThreads) {
						const uint32_t col = item % CPI, q = (item / CPI) & 3, g = item / (4 * CPI);
						const uint32_t r0 = g * 4 + q;   // row inside every slot region; region bases are multiples of 8 rows
						const uint32_t a_item = (stage + r0 * kStepBytes) ^ ((col ^ (r0 & 7)) << 4);
						uint32_t acc[R][W];
#pragma unroll
						for (int r = 0; r < R; ++r)
#pragma unroll
							for (int w = 0; w < W; ++w) acc[r][w] = 0;
						uint32_t slot_j = K - E;  // E > 0: the slot of the next given data position is slot_j - 1
						for (int j = static_cast<int>(K) - 1; j >= 0; --j) {
							uint32_t v[W];
							if constexpr (E == 0) {
								lds_item<W>(a_item + j * region_bytes, v);
							} else if ((lost->mask >> j) & 1u) {
#pragma unroll
								for (int w = 0; w < W; ++w) v[w] = 0;  // the multiply step alone
							} else {
								lds_item<W>(a_item + --slot_j * region_bytes, v);
							}
#pragma unroll
							for (int r = 0; r < R; ++r) {
								const int fixed = CONSEC ? r : -1;
#pragma unroll
								for (int w = 0; w < W; ++w) {
									uint32_t a = acc[r][w];
									if (fixed == 0) a ^= v[w];
									else if (fixed == 1) a = gf_x2_add(a, v[w]);
									else if (fixed == 2) a = gf_x4_add(a, v[w]);
									else if (fixed == 3) a = gf_x8_add(a, v[w]);
									else {
										for (uint32_t t = 0; t < p.row[r]; ++t) a = gf_x2(a);
										a ^= v[w];
									}
									acc[r][w] = a;
								}
							}
						}
						if constexpr (MAP && E == 0) {
							uint32_t bits = 0;
#pragma unroll
							for (int r = 0; r < R; ++r) {
								uint32_t pv[W], d = 0;
								lds_item<W>(a_item + (K + r) * region_bytes, pv);
#pragma unroll
								for (int w = 0; w < W; ++w) d |= acc[r][w] ^ pv[w];
								if (d) bits |= 1u << (CONSEC ? r : p.row[r]);  // parity rows are 0..3 (m <= 4 on this route)
							}
							map_bits |= bits << (4 * (item / kCheckThreads));
						} else if constexpr (MAP) {
							// acc[r] becomes S_r; only the spare rows E .. R-1 get a bit
#pragma unroll
							for (int r = 0; r < R; ++r) {
								uint32_t pv[W];
								lds_item<W>(a_item + (K - E + r) * region_bytes, pv);
#pragma unroll
								for (int w = 0; w < W; ++w) acc[r][w] ^= pv[w];
							}
							// word by word, and the funnel-shift form of every product: the (E, R) = (2, 4) instantiation spills otherwise
							uint32_t d[R] = {};
#pragma unroll
							for (int w = 0; w < W; ++w)
#pragma unroll
								for (int i = E; i < R; ++i) {
									uint32_t t = acc[i][w];
#pragma unroll
									for (int x = 0; x < E; ++x) t = gf_mac<8>(t, acc[x][w], lost->elim[(i - E) * E + x]);
									d[i] |= t;
								}
							uint32_t bits = 0;
#pragma unroll
							for (int i = E; i < R; ++i)
								if (d[i]) bits |= 1u << (CONSEC ? i : p.row[i]);
							map_bits |= bits << (4 * (item / kCheckThreads));
						} else {
							uint32_t any = 0;
#pragma unroll
							for (int r = 0; r < R; ++r) {
								uint32_t pv[W];
								lds_item<W>(a_item + (K + r) * region_bytes, pv);
#pragma unroll
								for (int w = 0; w < W; ++w) any |= acc[r][w] ^ pv[w];
							}
							if (any) bad_stripe = min(bad_stripe, stripe0 + g);  // rows past the last stripe are zero-filled: never non-zero
						}
					}
				}

				if (verify) fold_step<64, false>(win, aux, sub * 32, row_addr0 + st * stage_bytes);
				__syncwarp();
				if (lane == 0 && mbar_arrive_is_last(a_empty + 8 * st) && it + n_stages < total_steps) {
					asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
					if (step + n_stages < kStepsPerUnit) issue_load(c, gi, step + n_stages, st);
					else issue_load(next_c, next_gi, step + n_stages - kStepsPerUnit, st);
				}
				++it;
				if (++st == n_stages) { st = 0; ph ^= 1; }
			}
		}

		if constexpr (MAP) {
			// every lane of a GF warp ran the same passes (n_items and the thread count are multiples of 32)
			if (warp_has_items)
				for (uint32_t item0 = cw * 32, i = 0; item0 < n_items; item0 += kCheckThreads, ++i) {
					const uint32_t bits = __reduce_or_sync(0xffffffffu, (map_bits >> (4 * i)) & 15u);
					const uint32_t s = stripe0 + item0 / 32;
					if (lane == 0 && s < p.pb) {
						uint32_t *e = map + 2ull * (static_cast<unsigned long long>(c) * p.pb + s);
						e[0] = bits;
						e[1] = 0xffffffffu;
					}
				}
		} else {
			if (bad_stripe != 0xffffffffu) atomicMin(p.verdict + 3ull * c, static_cast<int>(bad_stripe));
		}
		// unit epilogue: the block CRCs against the stored ones
		uint32_t lin = 0;
		if (verify) lin = crc_mulmod(fold_finish<64>(win, p.tables), p.qmult[rr & 3]);
		lin ^= __shfl_xor_sync(0xffffffffu, lin, 1);
		lin ^= __shfl_xor_sync(0xffffffffu, lin, 2);
		if (verify && (rr & 3) == 0) {
			const uint32_t s = stripe0 + (rr >> 2);
			if (s < p.pb) {
				const uint32_t want = __ldg(p.stored[slot] + static_cast<unsigned long long>(c) * p.pb + s);
				if ((lin ^ p.zconst) != want) {
					atomicMin(p.first_bad, (static_cast<unsigned long long>(c) * 64ull + p.part_id[slot]) * 1024ull + s);
					if constexpr (FAILED) atomicOr(failed + static_cast<unsigned long long>(c) * p.pb + s, 1ull << p.part_id[slot]);
				}
			}
		}
	}
}

template <int R, bool CONSEC>
__global__ void __launch_bounds__(kCheckThreads, 1)
fused_check_kernel(const __grid_constant__ CheckTmaps tmaps, const __grid_constant__ CheckParams p) {
	fused_check_body<R, CONSEC, false>(tmaps, p, nullptr);
}

// lzgpu_check_stripe_map: map = lzgpu_stripe_state[n_chunks * pb] as two words per entry
template <int R, bool CONSEC>
__global__ void __launch_bounds__(kCheckThreads, 1)
fused_check_map_kernel(const __grid_constant__ CheckTmaps tmaps, const __grid_constant__ CheckParams p, uint32_t *map) {
	fused_check_body<R, CONSEC, true>(tmaps, p, map);
}

// lzgpu_check_stripe_map_degraded: the map with E lost data parts (1 <= E < R), bad_rows bits for the spare rows only
template <int E, int R, bool CONSEC>
__global__ void __launch_bounds__(kCheckThreads, 1)
fused_check_degraded_kernel(const __grid_constant__ CheckTmaps tmaps, const __grid_constant__ CheckParams p, uint32_t *map,
                            const __grid_constant__ CheckLost lost) {
	fused_check_body<R, CONSEC, true, E>(tmaps, p, map, &lost);
}

// lzgpu_repair_stripes: the map kernels that also record every block that fails its stored CRC (failed[c * pb + s], bit part)
template <int R, bool CONSEC>
__global__ void __launch_bounds__(kCheckThreads, 1)
fused_check_repair_kernel(const __grid_constant__ CheckTmaps tmaps, const __grid_constant__ CheckParams p, uint32_t *map, unsigned long long *failed) {
	fused_check_body<R, CONSEC, true, 0, true>(tmaps, p, map, nullptr, failed);
}

template <int E, int R, bool CONSEC>
__global__ void __launch_bounds__(kCheckThreads, 1)
fused_check_repair_degraded_kernel(const __grid_constant__ CheckTmaps tmaps, const __grid_constant__ CheckParams p, uint32_t *map,
                                   const __grid_constant__ CheckLost lost, unsigned long long *failed) {
	fused_check_body<R, CONSEC, true, E, true>(tmaps, p, map, &lost, failed);
}

}  // namespace lzd
