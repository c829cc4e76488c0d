// convert_kernel.cuh — slice-type conversion in ONE pass over HBM: read k parts of the source slice, verify their stored
// CRCs, rebuild the lost data parts, and write every wanted part of the DESTINATION slice (data parts picked by the
// BlockConverter rule, parity parts recomputed) together with the CRC of each destination block.
//
// Reference work it replaces, per chunk (chunkserver replication of a part of another slice type):
//   SliceRecoveryPlanner::buildPlanFor -> kRecoverDataPart / kRecoverParityPart (src/chunkserver/slice_recovery_planner.h:102-119,
//   144-204): ChunkReadPlanner + ReadPlan::postProcessData (read k parts, mycrc32 of every received block, ECReadPlan::recoverParts
//   / XorReadPlan::postProcessRead), BlockConverter (slice_recovery_planner.h:41-64) for data parts, ECReadPlan::RecoverParity /
//   XorReadPlan::RecoverParity (ec_read_plan.h:38-76, xor_read_plan.h:39-62) for parity parts, then mycrc32 of every block that
//   is written (chunk_replicator.cc:186-192).
// The two-pass route (fused_recover_kernel -> chunk image -> SPLIT fused_stream_kernel) moves the chunk through HBM three more
// times than necessary; here a work unit is a run of R = G*Kd = T*Ks consecutive chunk blocks (G destination stripes = T source
// stripes), so both stripings are whole inside one unit and the image never exists.
//
// Shared-memory stage: [source slot a][source stripe t][quarter q] rows of 128 B, slot a = data part a for a < Ks (the regions of
// lost parts are not loaded: the REBUILD role fills them), slot Ks + x = the x-th parity part in use.  Slot regions are padded to
// a multiple of 8 rows (1024 B) so that every TMA box starts on a swizzle-pattern boundary.  Chunk block bl of the unit
// (bl = 0 .. R-1) is row (bl % Ks) * region_rows + (bl / Ks) * 4 + q.
//
// Warp roles (hand-offs are mbarriers; no CTA-wide sync inside the stream of steps):
//   REBUILD warps (only with lost parts: the warps the CRC rows do not need) do nothing else and run ahead of the workers by as many
//            stages as are loaded.  Item (source stripe t, quarter q, 16-byte column): syndromes by Horner over the surviving data
//            columns + the parity columns, RAID-6 elimination, rebuilt words stored into the lost slots' rows of the stage; arrive
//            `rfull`, release the stage.
//   WORKER warps, per 128-byte step, after `full` and `rfull`:
//     GF     item (destination stripe g, quarter q, column): walks the Kd blocks of the stripe (block -> stage offset from a table in
//            the kernel parameters), stores them part-major into the destination data parts, Horner-evaluates the destination parity
//            rows, stores them and stages rows 1.. for their CRC.
//     CRC    one row per thread: R*4 data rows (verified against the stored CRC when the row was read from a part, emitted as the
//            destination data part's CRC either way), E*T*4 source parity rows (verified only), G*(M-1)*4 staged destination
//            parity rows; the CRC of destination parity row 0 comes from linearity as in the encoder.
#pragma once
#include "fused_kernel.cuh"

namespace lzd {

// kConvertThreads (256) and kConvertNPST (4 staging stages) live in fused_plan.h next to convert_plan()

// mbar_wait for warps that mostly find the phase incomplete (the rebuild warps run ahead of the TMA loads): sleep between the polls so
// that the loop does not take issue slots from the worker warps of the same scheduler (without the sleep the polling loops were a
// large share of all executed instructions)
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t addr, uint32_t parity) {
	uint32_t done;
	for (;;) {
		asm volatile(
		    "{\n\t.reg .pred p;\n\t"
		    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
		    "selp.u32 %0, 1, 0, p;\n\t}"
		    : "=r"(done)
		    : "r"(addr), "r"(parity), "r"(0x989680u)
		    : "memory");
		if (done) break;
		__nanosleep(400);
	}
}

struct ConvertParams {
	// destination slice
	uint8_t *data_out[32];        // destination data part j (chunk c at + c*part_out_stride), nullptr = not wanted
	uint8_t *par_out[4];          // destination parity part r, nullptr = not wanted
	unsigned long long part_out_stride;
	uint32_t *crc;                // chunk-order CRC array of the destination slice: nb data blocks, then M x pbd parity blocks
	unsigned long long crc_stride;
	uint32_t Kd, G, pbd;          // destination data parts, destination stripes per unit, destination stripes per chunk
	// source slice
	uint32_t Ks, T, pbs;          // source data parts, source stripes per unit (G*Kd == T*Ks), source stripes per chunk
	uint32_t region_rows;         // rows per slot region in a stage: T*4 rounded up to a multiple of 8
	uint32_t n_loaded;            // tensor maps in use (one per part that is read)
	uint8_t loaded_slot[32];      // tensor map i -> slot
	uint16_t bl_entry[64];        // chunk block bl of a unit -> byte offset of its quarter-0 row in a stage, with the swizzle phase of that
	                              // row in bit 6: row0 = (bl % Ks) * region_rows + (bl / Ks) * 4, entry = row0 * 128 + (row0 & 4 ? 64 : 0);
	                              // the 16-byte column col of quarter q is at (stage + entry + q*128) ^ ((col ^ q) << 4)
	uint8_t slot_present[36];     // slot a < Ks: 1 = read from the part, 0 = lost (rebuilt)
	uint8_t erased_idx[4];        // data indices of the lost parts, ascending
	uint8_t part_id[36];          // slot -> source part index (error reporting)
	const uint32_t *stored[36];   // stored CRCs of the part in slot a (chunk c at + c*pbs) or nullptr = not verified
	unsigned long long *first_bad;  // atomicMin target: (c * 64 + part) * 1024 + block
	const uint32_t *tables;
	uint32_t n_chunks, nb, units_per_chunk, total_units, n_stages;
	uint32_t qmult[4];
	uint32_t zconst;
	uint32_t dbl0;                // E = 2: x0 when 2^x0 * S0 is cheaper as x0 doublings (x0 <= 4), else 0xff = multiply by w[0]
	CoefPlanes w[2];              // E = 2: planes of 2^x0 and of (2^x0 ^ 2^x1)^-1
};

// M = destination parity parts (1..3, Vandermonde rows 1, 2^j, 4^j), E = lost source data parts (0..2; the parity parts in use
// are source parity rows 0 .. E-1), KD = compile-time number of destination data parts (0 = p.Kd at run time): the walk over a
// destination stripe unrolls and its parameter loads become immediates (ec(3,2) destinations: 125 instead of 166 instructions per item)
template <int M, int E, int KD = 0>
__global__ void __launch_bounds__(kConvertThreads, 2)
fused_convert_kernel(const __grid_constant__ TmapArray tmaps, const __grid_constant__ ConvertParams p) {
	constexpr int NT = kConvertThreads, FW = 64, W = 4;
	constexpr uint32_t CPI = 32 / W;
	constexpr int PC = M - 1;
	extern __shared__ __align__(1024) uint8_t smem[];
	const uint32_t sbase = smem_u32(smem);
	const uint32_t Ks = p.Ks, Kd = KD ? KD : p.Kd, G = p.G, T = p.T, RR = p.region_rows, NST = p.n_stages;
	const uint32_t R = G * Kd;                                  // chunk blocks per unit
	const uint32_t stage_bytes = (Ks + E) * RR * kStepBytes;    // multiple of 1024
	const uint32_t box_bytes = T * 4 * kStepBytes;
	const uint32_t DROWS = R * 4, SPROWS = E * T * 4, PROWS = G * PC * 4;
	const uint32_t pstage_bytes = (PROWS * kStepBytes + 1023u) & ~1023u;
	const uint32_t pstage0 = sbase + NST * stage_bytes;
	const uint32_t misc = pstage0 + kConvertNPST * pstage_bytes;
	const uint32_t a_blk = misc;                                // s_blk[2][64]
	const uint32_t a_full = misc + 520, a_empty = a_full + 8 * NST, a_rfull = a_empty + 8 * NST, a_pfull = a_rfull + 8 * NST,
	               a_pempty = a_pfull + 8 * kConvertNPST;

	const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	// Warp roles.  WORKER warps (the first n_wk) own the CRC streams and the GF items; with lost parts the remaining warps are
	// REBUILD warps and do nothing else: they run ahead of the workers by as many stages as are loaded, so the workers find the
	// lost rows in place (`rfull`) when a stage's turn comes.  (Measured, runs 9 / 10: with the rebuild in front of — or inside — warps
	// that also carry GF items every step waited for it.)
	const uint32_t n_rows = DROWS + SPROWS + PROWS;
	const uint32_t n_wk = E ? (n_rows + 31) / 32 : NT / 32;        // the host guarantees n_wk < NT / 32 when E > 0
	const uint32_t n_wk_threads = n_wk * 32;
	const uint32_t n_rb_warps = NT / 32 - n_wk;
	const uint32_t n_items = 4 * CPI * G;
	const uint32_t n_gf_warps = min((n_items + 31) / 32, n_wk);
	const uint32_t n_rb_items = 4 * CPI * T;
	const uint32_t first_pwarp = (DROWS + SPROWS) / 32, last_pwarp = PROWS ? (n_rows - 1) / 32 : 0;

	const uint32_t my_units = blockIdx.x < p.total_units ? (p.total_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
	const uint32_t total_steps = my_units * kStepsPerUnit;

	// load of this CTA's step number `n` (unit blockIdx.x + (n / 128) * gridDim.x, step n % 128) into stage st: one box of T*4 rows per
	// part that is read
	auto issue_load = [&](uint32_t n, uint32_t st) {
		const uint32_t unit = blockIdx.x + (n / kStepsPerUnit) * gridDim.x, step = n % kStepsPerUnit;
		const uint32_t c = unit / p.units_per_chunk, ui = unit % p.units_per_chunk;
		mbar_expect_tx(a_full + 8 * st, p.n_loaded * box_bytes);
		for (uint32_t i = 0; i < p.n_loaded; ++i)
			tma_load_3d(sbase + st * stage_bytes + p.loaded_slot[i] * RR * kStepBytes, &tmaps.m[i], static_cast<int>(step * kStepBytes),
			            static_cast<int>(ui * T * 4), static_cast<int>(c), a_full + 8 * st);
	};
	// release stage st after step n; the arrival that completes the phase refills it with step n + NST
	auto release_stage = [&](uint32_t n, uint32_t st) {
		if (lane == 0 && mbar_arrive_is_last(a_empty + 8 * st) && n + NST < total_steps) {
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			issue_load(n + NST, st);
		}
	};

	if (tid == 0) {
		for (uint32_t s = 0; s < NST; ++s) {
			mbar_init(a_full + 8 * s, 1);
			mbar_init(a_empty + 8 * s, NT / 32);
			mbar_init(a_rfull + 8 * s, n_rb_warps ? n_rb_warps : 1);
		}
		for (int s = 0; s < kConvertNPST; ++s) {
			mbar_init(a_pfull + 8 * s, n_gf_warps * LZ_RING_ARRIVERS);
			mbar_init(a_pempty + 8 * s, (PROWS ? (last_pwarp - first_pwarp + 1) : 1) * LZ_RING_ARRIVERS);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		for (uint32_t g0 = 0; g0 < NST && g0 < total_steps; ++g0) issue_load(g0, g0);
	}
	__syncthreads();

	// REBUILD role for the stage at shared address `stage`: the lost source data parts of every source stripe of the unit
	auto rebuild_stage = [&](uint32_t stage, uint32_t rfull_bar) {
		for (uint32_t item = tid - n_wk_threads; item < n_rb_items; item += n_rb_warps * 32) {
			const uint32_t col = item % CPI, q = (item / CPI) & 3, t = item / (4 * CPI);
			const uint32_t r0 = t * 4 + q;      // row inside every slot region (regions start on multiples of 8 rows)
			const uint32_t a_item = ((stage + r0 * kStepBytes) ^ ((col ^ (r0 & 7)) << 4));
			uint32_t s0[W], s1[W];
#pragma unroll
			for (int w = 0; w < W; ++w) s0[w] = s1[w] = 0;
			for (int j = static_cast<int>(Ks) - 1; j >= 0; --j) {
				uint32_t v[W];
#pragma unroll
				for (int w = 0; w < W; ++w) v[w] = 0;
				if (p.slot_present[j]) lds_item<W>(a_item + j * RR * kStepBytes, v);
#pragma unroll
				for (int w = 0; w < W; ++w) {
					s0[w] ^= v[w];
					if (E == 2) s1[w] = gf_x2_add(s1[w], v[w]);
				}
			}
			{
				uint32_t v[W];
				lds_item<W>(a_item + Ks * RR * kStepBytes, v);
#pragma unroll
				for (int w = 0; w < W; ++w) s0[w] ^= v[w];
				if (E == 2) {
					lds_item<W>(a_item + (Ks + 1) * RR * kStepBytes, v);
#pragma unroll
					for (int w = 0; w < W; ++w) s1[w] ^= v[w];
				}
			}
			if (E == 2) {
				// S0 = d0 ^ d1, S1 = 2^x0 d0 ^ 2^x1 d1  ->  d1 = (S1 ^ 2^x0 S0) / (2^x0 ^ 2^x1), d0 = S0 ^ d1: the unique
				// solution, i.e. the bytes of the reference's inverted matrix (reed_solomon.h:229-281)
				uint32_t tt[W];
#pragma unroll
				for (int w = 0; w < W; ++w) tt[w] = s0[w];
				if (p.dbl0 != 0xffu) {
					for (uint32_t i = 0; i < p.dbl0; ++i)
#pragma unroll
						for (int w = 0; w < W; ++w) tt[w] = gf_x2_add(tt[w], 0u);
				} else {
#pragma unroll
					for (int w = 0; w < W; ++w) tt[w] = gf_mac<2>(0u, tt[w], p.w[0]);
				}
#pragma unroll
				for (int w = 0; w < W; ++w) {
					s1[w] = gf_mac<2>(0u, s1[w] ^ tt[w], p.w[1]);
					s0[w] ^= s1[w];
				}
				sts_item<W>(a_item + p.erased_idx[1] * RR * kStepBytes, s1);
			}
			sts_item<W>(a_item + p.erased_idx[0] * RR * kStepBytes, s0);
		}
		__syncwarp();
		if (lane == 0) mbar_arrive(rfull_bar);
	};

	if constexpr (E > 0) {
		if (warp >= n_wk) {
			// ===================== REBUILD warps =====================
			uint32_t st = 0, ph = 0;
			for (uint32_t n = 0; n < total_steps; ++n) {
				mbar_wait_relaxed(a_full + 8 * st, ph);   // these warps are ahead of the loads most of the time: poll slowly
				rebuild_stage(sbase + st * stage_bytes, a_rfull + 8 * st);   // (ends with __syncwarp: every lane's reads are done)
				release_stage(n, st);
				if (++st == NST) { st = 0; ph ^= 1; }
			}
			return;
		}
	}

	// ===================== WORKER warps: stream / item assignment =====================
	const bool is_data_row = tid < DROWS;
	const bool is_sp_row = E > 0 && tid >= DROWS && tid < DROWS + SPROWS;
	const bool is_parity_row = PC > 0 && tid >= DROWS + SPROWS && tid < n_rows;
	// data stream: chunk block bl of the unit, quarter q
	const uint32_t my_q = tid & 3;                              // DROWS and SPROWS are multiples of 4
	const uint32_t my_bl = tid >> 2;
	const uint32_t my_a = is_data_row ? my_bl % Ks : (is_sp_row ? Ks + (tid - DROWS) / (T * 4) : 0);
	const uint32_t my_t = is_data_row ? my_bl / Ks : (is_sp_row ? ((tid - DROWS) >> 2) % T : 0);
	const uint32_t prow = tid - DROWS - SPROWS;                 // staged destination parity row (g*PC + r')*4 + q
	const uint32_t my_row = is_parity_row ? prow : my_a * RR + my_t * 4 + my_q;
	const uint32_t row_addr0 = ((is_parity_row ? pstage0 : sbase) + my_row * kStepBytes) ^ ((my_row & 7) << 4);
	const uint32_t row_stride = is_parity_row ? pstage_bytes : stage_bytes;
	// a source parity row is only folded when its stored CRC is to be checked; data rows always (their CRC is an output)
	const bool has_stream = is_data_row || is_parity_row || (is_sp_row && p.stored[my_a] != nullptr);
	const bool warp_has_items = warp < n_gf_warps;
	const bool warp_has_prow = PROWS && warp >= first_pwarp && warp <= last_pwarp;
	// GF items of this thread: column and quarter are fixed (see the GF role)
	const uint32_t gf_col = tid % CPI, gf_q = (tid / CPI) & 3;
	const uint32_t gf_cx = (gf_col ^ gf_q) << 4, gf_qoff = gf_q * kStepBytes;
	const uint32_t gf_ip0 = (gf_q << 14) + gf_col * (4 * W);

	uint32_t win[FW];
	FoldAux aux;
	uint32_t it = 0, st = 0, ph = 0, pst = 0, pph = 0, unit_parity = 0;

	for (uint32_t unit = blockIdx.x; unit < p.total_units; unit += gridDim.x, unit_parity ^= 1) {
		const uint32_t c = unit / p.units_per_chunk, ui = unit % p.units_per_chunk;
		const uint32_t stripe0 = ui * G;                        // first destination stripe of the unit
		const unsigned long long c_off = static_cast<unsigned long long>(c) * p.part_out_stride;
#pragma unroll
		for (int i = 0; i < FW; ++i) win[i] = 0;
#pragma unroll
		for (int i = 0; i < 32; ++i) aux.y[i] = 0;

		for (int step0 = 0; step0 < kStepsPerUnit; step0 += FW / 32) {
#pragma unroll
			for (int sub_step = 0; sub_step < FW / 32; ++sub_step) {
				const int step = step0 + sub_step;
				const uint32_t stage = sbase + st * stage_bytes;
				const uint32_t pstage = pstage0 + pst * pstage_bytes;
				mbar_wait(a_full + 8 * st, ph);

				if constexpr (E > 0) mbar_wait(a_rfull + 8 * st, ph);   // the lost rows of this stage are in place

				// ---------------- GF role: destination stripes ----------------
				// item (stripe g, quarter q, 16-byte column col): col and q are the same for every item of a thread (the worker thread
				// count is a multiple of 32), g advances by the number of worker warps.  All addresses are "constant + table entry":
				// the swizzled offset of chunk block bl inside a stage comes from p.bl_entry (no division, no per-block address maths).
				if (warp_has_items) {
					if (PC > 0) mbar_wait(a_pempty + 8 * pst, pph ^ 1);
					const uint32_t pre = stage + gf_qoff;
					const unsigned long long off_step = c_off + gf_ip0 + static_cast<uint32_t>(step) * kStepBytes;
					for (uint32_t g = warp; g < G; g += n_wk) {
						uint32_t acc[M][W];
#pragma unroll
						for (int r = 0; r < M; ++r)
#pragma unroll
							for (int w = 0; w < W; ++w) acc[r][w] = 0;
						const uint32_t stripe = stripe0 + g;
						const bool live = stripe < p.pbd;
						const unsigned long long off = off_step + (static_cast<unsigned long long>(stripe) << 16);
						// chunk blocks of the stripe, walked downwards (Horner): bl = g*Kd + j
						uint32_t bl = g * Kd + Kd - 1;
#pragma unroll
						for (int j = static_cast<int>(Kd) - 1; j >= 0; --j, --bl) {
							uint32_t v[W];
							lds_item<W>((pre + p.bl_entry[bl]) ^ gf_cx, v);
							// BlockConverter (slice_recovery_planner.h:41-57): chunk block stripe*Kd + j is block `stripe` of data part j
							uint8_t *dp = p.data_out[j];
							if (dp && live) stg_item<W>(dp + off, v);
#pragma unroll
							for (int r = 0; r < M; ++r)
#pragma unroll
								for (int w = 0; w < W; ++w) {
									const uint32_t aa = acc[r][w], d = v[w];
									acc[r][w] = r == 0 ? (aa ^ d) : r == 1 ? gf_x2_add(aa, d) : gf_x4_add(aa, d);
								}
						}
						if (live) {
#pragma unroll
							for (int r = 0; r < M; ++r)
								if (p.par_out[r]) stg_item<W>(p.par_out[r] + off, acc[r]);
						}
#pragma unroll
						for (int r = 1; r < M; ++r) {
							// staged row (g*PC + r-1)*4 + q: its swizzle (row & 7) = 4*((g*PC + r-1) & 1) + q
							const uint32_t pr4 = g * PC + (r - 1);
							sts_item<W>(((pstage + pr4 * (4 * kStepBytes) + gf_qoff) ^ gf_cx) ^ ((pr4 & 1) << 6), acc[r]);
						}
					}
					if (PC > 0) {
						__syncwarp();
						if (LZ_RING_LANE(lane)) mbar_arrive(a_pfull + 8 * pst);
					}
				}

				// ---------------- CRC role ----------------
				if (PC > 0 && warp_has_prow) mbar_wait(a_pfull + 8 * pst, pph);
				if (has_stream) fold_step<FW, true>(win, aux, sub_step * 32, row_addr0 + (is_parity_row ? pst : st) * row_stride);
				__syncwarp();
				release_stage(it, st);
				if (PC > 0 && warp_has_prow && LZ_RING_LANE(lane)) mbar_arrive(a_pempty + 8 * pst);
				++it;
				if (++st == NST) { st = 0; ph ^= 1; }
				if (++pst == kConvertNPST) { pst = 0; pph ^= 1; }
			}
		}

		// ---------------- unit epilogue: streams -> block CRCs ----------------
		uint32_t lin = 0;
		if (has_stream) lin = crc_mulmod(fold_finish<FW>(win, p.tables), p.qmult[tid & 3]);
		lin ^= __shfl_xor_sync(0xffffffffu, lin, 1);
		lin ^= __shfl_xor_sync(0xffffffffu, lin, 2);
		const uint32_t blk = a_blk + unit_parity * 256;
		const uint32_t s_src = ui * T + my_t;                   // source stripe of a data / source parity stream
		if (is_data_row && my_q == 0) {
			asm volatile("st.shared.u32 [%0], %1;" ::"r"(blk + 4 * my_bl), "r"(lin) : "memory");
			const uint32_t b = ui * R + my_bl;                  // block index in the chunk
			const uint32_t have = lin ^ p.zconst;
			if (b < p.nb) p.crc[c * p.crc_stride + b] = have;
			if (p.slot_present[my_a] && p.stored[my_a] && s_src < p.pbs) {
				const uint32_t want = __ldg(p.stored[my_a] + static_cast<unsigned long long>(c) * p.pbs + s_src);
				if (have != want) atomicMin(p.first_bad, (static_cast<unsigned long long>(c) * 64ull + p.part_id[my_a]) * 1024ull + s_src);
			}
		}
		if (is_sp_row && my_q == 0 && p.stored[my_a] && s_src < p.pbs) {
			const uint32_t have = lin ^ p.zconst;
			const uint32_t want = __ldg(p.stored[my_a] + static_cast<unsigned long long>(c) * p.pbs + s_src);
			if (have != want) atomicMin(p.first_bad, (static_cast<unsigned long long>(c) * 64ull + p.part_id[my_a]) * 1024ull + s_src);
		}
		if (is_parity_row && (prow & 3) == 0) {
			constexpr uint32_t PCD = PC ? PC : 1;
			const uint32_t g = (prow >> 2) / PCD, r = 1 + (prow >> 2) % PCD;
			const uint32_t stripe = stripe0 + g;
			if (stripe < p.pbd) p.crc[c * p.crc_stride + p.nb + r * p.pbd + stripe] = lin ^ p.zconst;
		}
		// CRC of destination parity row 0 (plain XOR of the stripe): xor of the data blocks' linear CRCs (crc.h:29 mycrc32_xorblocks)
		asm volatile("bar.sync 1, %0;" ::"r"(n_wk_threads) : "memory");   // worker warps only
		if (tid < G) {
			uint32_t x = 0;
			for (uint32_t j = 0; j < Kd; ++j) {
				uint32_t tt;
				asm volatile("ld.shared.u32 %0, [%1];" : "=r"(tt) : "r"(blk + 4 * (tid * Kd + j)));
				x ^= tt;
			}
			const uint32_t stripe = stripe0 + tid;
			if (stripe < p.pbd) p.crc[c * p.crc_stride + p.nb + stripe] = x ^ p.zconst;
		}
	}
}

}  // namespace lzd
