// slices_kernel.cuh — encode a chunk for EVERY slice of its goal in one pass over the data: the parity parts of each xor/ec slice
// and the CRC of every data and parity block, each slice's arrays laid out as lzgpu_encode_chunks lays them out.
//
// Reference work it replaces, per chunk: ChunkWriter works on combined stripes of lcm(k_i) blocks and computes the parity of every
// slice from the same data blocks (src/mount/chunk_writer.cc:150-156, 494-545), plus mycrc32 of every block it writes.  Encoding
// slice by slice reads the chunk once per slice and folds the CRC of every data block once per slice.
//
// A work unit is G combined stripes of one chunk: R = G*L consecutive chunk blocks (L = lcm of the striped slices' k), i.e. 4R
// consecutive quarter-rows of the encoder's [chunk][row][16 KiB] tensor map, one TMA box per 128-byte step (rows past nb arrive as
// zeros, as the encoder's short last stripe).  The unit starts on a multiple of L, so stripe s of slice i is the blocks s*k_i ..
// s*k_i + k_i - 1 of the unit: contiguous stage rows, no block table.
//
// Roles (as fused_stream_kernel / fused_convert_kernel; hand-offs are mbarriers, no CTA-wide sync inside the stream of steps):
//   GF     item (slice i, stripe s of that slice, quarter q, column): Horner over the k_i blocks of the stripe (row r: acc = acc*2^r ^ d),
//          16- or 8-byte parity words stored part-major into parity[i] (stripes past pb_i are not stored), rows 1 .. m_i - 1 staged
//          for their CRC.  Every warp takes items; a stripe's items are whole warps, so m_i is uniform across a warp.
//   CRC    thread t < 4R: data row t, folded once, its block CRC stored into every slice's array; the next threads: the staged parity
//          rows.  Parity row 0 of every slice (its XOR) takes its CRC from linearity: the XOR of the stripe's data-block lin values,
//          so xor-only goal sets need no parity streams at all.
#pragma once
#include "fused_kernel.cuh"

namespace lzd {

struct SlicesParams {
	uint8_t *parity[kSlicesMax];                  // part-major parity of slice i (chunk c at + c*parity_stride[i]); nullptr: standard slice
	uint32_t *crc[kSlicesMax];                    // CRC array of slice i (chunk c at + c*crc_stride[i] elements)
	unsigned long long parity_stride[kSlicesMax], crc_stride[kSlicesMax];
	uint32_t k[kSlicesMax], m[kSlicesMax], pb[kSlicesMax];
	uint32_t S[kSlicesMax];                       // stripes of slice i per unit (R / k_i; 0 for a standard slice)
	uint32_t prow4[kSlicesMax];                   // first staged parity row of slice i, in units of 4 rows
	uint8_t gs_slice[kSlicesMaxStripes];          // stripe gs of the unit (all slices, in slice order) -> slice
	uint8_t gs_stripe[kSlicesMaxStripes];         //                                                    -> stripe of that slice in the unit
	const uint32_t *tables;
	uint32_t n_slices, n_stripes, n_chunks, nb, R, prows, units_per_chunk, total_units, n_stages;
	uint32_t qmult[4];
	uint32_t zconst;
};

// M = the largest m of the slices (1..4): the accumulator count; each stripe's rows stop at its own slice's m
template <int M>
__global__ void __launch_bounds__(kSlicesThreads, 1)
fused_slices_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ SlicesParams p) {
	constexpr int NT = kSlicesThreads, FW = 64, W = slices_item_words(M);
	constexpr uint32_t CPI = 32 / W, IPS = 4 * CPI;   // items per row step, per stripe and step
	extern __shared__ __align__(1024) uint8_t smem[];
	const uint32_t sbase = smem_u32(smem);
	const uint32_t R = p.R, NST = p.n_stages;
	const uint32_t DROWS = 4 * R, PROWS = M > 1 ? p.prows : 0;
	const uint32_t box_bytes = DROWS * kStepBytes;
	const uint32_t stage_bytes = (box_bytes + 1023u) & ~1023u;
	const uint32_t pstage_bytes = (PROWS * kStepBytes + 1023u) & ~1023u;
	const uint32_t pstage0 = sbase + NST * stage_bytes;
	const uint32_t misc = pstage0 + kSlicesNPST * pstage_bytes;
	const uint32_t a_blk = misc;                                // s_blk[2][64]
	const uint32_t a_full = misc + 520, a_empty = a_full + 8 * NST, a_pfull = a_empty + 8 * NST, a_pempty = a_pfull + 8 * kSlicesNPST;

	const uint32_t tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
	const uint32_t n_items = IPS * p.n_stripes;
	const uint32_t n_gf_warps = min((n_items + 31) / 32, static_cast<uint32_t>(NT / 32));
	const uint32_t first_pwarp = DROWS / 32, last_pwarp = PROWS ? (DROWS + PROWS - 1) / 32 : 0;

	const uint32_t my_units = blockIdx.x < p.total_units ? (p.total_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
	const uint32_t total_steps = my_units * kStepsPerUnit;

	// load of this CTA's step number `n` (unit blockIdx.x + (n / 128) * gridDim.x, step n % 128) into stage st
	auto issue_load = [&](uint32_t n, uint32_t st) {
		const uint32_t unit = blockIdx.x + (n / kStepsPerUnit) * gridDim.x, step = n % kStepsPerUnit;
		const uint32_t c = unit / p.units_per_chunk, ui = unit % p.units_per_chunk;
		mbar_expect_tx(a_full + 8 * st, box_bytes);
		tma_load_3d(sbase + st * stage_bytes, &tmap, static_cast<int>(step * kStepBytes), static_cast<int>(ui * DROWS), static_cast<int>(c),
		            a_full + 8 * st);
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
		}
		for (int s = 0; s < kSlicesNPST; ++s) {
			mbar_init(a_pfull + 8 * s, n_gf_warps * LZ_RING_ARRIVERS);
			mbar_init(a_pempty + 8 * s, (PROWS ? (last_pwarp - first_pwarp + 1) : 1) * LZ_RING_ARRIVERS);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		for (uint32_t g0 = 0; g0 < NST && g0 < total_steps; ++g0) issue_load(g0, g0);
	}
	__syncthreads();

	const bool is_data_row = tid < DROWS;
	const bool is_parity_row = tid >= DROWS && tid < DROWS + PROWS;
	const bool has_stream = is_data_row || is_parity_row;
	const uint32_t prow = tid - DROWS;                          // staged parity row (prow4[i] + s*(m_i - 1) + r - 1)*4 + q
	const uint32_t my_row = is_data_row ? tid : prow;
	const uint32_t row_addr0 = ((is_data_row ? sbase : pstage0) + my_row * kStepBytes) ^ ((my_row & 7) << 4);
	const uint32_t row_stride = is_data_row ? stage_bytes : pstage_bytes;
	const bool warp_has_items = warp < n_gf_warps;
	const bool warp_has_prow = PROWS && warp >= first_pwarp && warp <= last_pwarp;
	// GF items of this thread: column and quarter are fixed, the stripe advances by NT / IPS
	const uint32_t gf_col = tid % CPI, gf_q = (tid / CPI) & 3, gf_gs0 = tid / IPS;
	const uint32_t gf_c16 = (gf_col * W) >> 2, gf_sub = ((gf_col * W) & 3) << 2;   // 16-byte chunk of the row step, byte offset in it
	const uint32_t gf_ip0 = (gf_q << 14) + gf_col * (4 * W);

	uint32_t win[FW];
	FoldAux aux;
	uint32_t it = 0, st = 0, ph = 0, pst = 0, pph = 0, unit_parity = 0;

	for (uint32_t unit = blockIdx.x; unit < p.total_units; unit += gridDim.x, unit_parity ^= 1) {
		const uint32_t c = unit / p.units_per_chunk, ui = unit % p.units_per_chunk;
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

				// ---------------- GF role: every stripe of every slice ----------------
				if (warp_has_items) {
					if (PROWS) mbar_wait(a_pempty + 8 * pst, pph ^ 1);
					for (uint32_t gs = gf_gs0; gs < p.n_stripes; gs += NT / IPS) {
						const uint32_t i = p.gs_slice[gs], s = p.gs_stripe[gs];
						const uint32_t k = p.k[i], m = p.m[i];
						uint32_t acc[M][W];
#pragma unroll
						for (int r = 0; r < M; ++r)
#pragma unroll
							for (int w = 0; w < W; ++w) acc[r][w] = 0;
						// row (s*k + j)*4 + q of the stage: its swizzle (row & 7) = 4*((s*k + j) & 1) + q
						for (int j = static_cast<int>(k) - 1; j >= 0; --j) {
							const uint32_t row = (s * k + static_cast<uint32_t>(j)) * 4 + gf_q;
							uint32_t v[W];
							lds_item<W>(((stage + row * kStepBytes) ^ ((gf_c16 ^ (row & 7)) << 4)) + gf_sub, v);
#pragma unroll
							for (int r = 0; r < M; ++r) {
								if (r >= static_cast<int>(m)) break;
#pragma unroll
								for (int w = 0; w < W; ++w) {
									const uint32_t a = acc[r][w], d = v[w];
									acc[r][w] = r == 0 ? (a ^ d) : r == 1 ? gf_x2_add(a, d) : r == 2 ? gf_x4_add(a, d) : gf_x8_add(a, d);
								}
							}
						}
						const uint32_t stripe = ui * p.S[i] + s;
						if (stripe < p.pb[i]) {
							uint8_t *dst = p.parity[i] + c * p.parity_stride[i] + (static_cast<unsigned long long>(stripe) << 16) + gf_ip0 +
							               static_cast<uint32_t>(step) * kStepBytes;
							const unsigned long long part_bytes = static_cast<unsigned long long>(p.pb[i]) << 16;
#pragma unroll
							for (int r = 0; r < M; ++r)
								if (r < static_cast<int>(m)) stg_item<W>(dst + r * part_bytes, acc[r]);
						}
#pragma unroll
						for (int r = 1; r < M; ++r) {
							if (r >= static_cast<int>(m)) break;
							const uint32_t pr = (p.prow4[i] + s * (m - 1) + (r - 1)) * 4 + gf_q;
							sts_item<W>(((pstage + pr * kStepBytes) ^ ((gf_c16 ^ (pr & 7)) << 4)) + gf_sub, acc[r]);
						}
					}
					if (PROWS) {
						__syncwarp();
						if (LZ_RING_LANE(lane)) mbar_arrive(a_pfull + 8 * pst);
					}
				}

				// ---------------- CRC role ----------------
				if (warp_has_prow) mbar_wait(a_pfull + 8 * pst, pph);
				if (has_stream) fold_step<FW, true>(win, aux, sub_step * 32, row_addr0 + (is_parity_row ? pst : st) * row_stride);
				__syncwarp();
				release_stage(it, st);
				if (warp_has_prow && LZ_RING_LANE(lane)) mbar_arrive(a_pempty + 8 * pst);
				++it;
				if (++st == NST) { st = 0; ph ^= 1; }
				if (++pst == kSlicesNPST) { pst = 0; pph ^= 1; }
			}
		}

		// ---------------- unit epilogue: streams -> block CRCs ----------------
		uint32_t lin = 0;
		if (has_stream) lin = crc_mulmod(fold_finish<FW>(win, p.tables), p.qmult[tid & 3]);
		lin ^= __shfl_xor_sync(0xffffffffu, lin, 1);
		lin ^= __shfl_xor_sync(0xffffffffu, lin, 2);
		const uint32_t blk = a_blk + unit_parity * 256;
		if (is_data_row && (tid & 3) == 0) {
			const uint32_t bl = tid >> 2;                       // block of the unit
			asm volatile("st.shared.u32 [%0], %1;" ::"r"(blk + 4 * bl), "r"(lin) : "memory");
			const uint32_t b = ui * R + bl;                     // block of the chunk
			if (b < p.nb)
				for (uint32_t i = 0; i < p.n_slices; ++i) p.crc[i][c * p.crc_stride[i] + b] = lin ^ p.zconst;
		}
		if (is_parity_row && (prow & 3) == 0) {
			const uint32_t p4 = prow >> 2;
			for (uint32_t i = 0; i < p.n_slices; ++i) {
				const uint32_t m = p.m[i];
				if (m < 2 || p4 < p.prow4[i] || p4 >= p.prow4[i] + p.S[i] * (m - 1)) continue;
				const uint32_t s = (p4 - p.prow4[i]) / (m - 1), r = 1 + (p4 - p.prow4[i]) % (m - 1);
				const uint32_t stripe = ui * p.S[i] + s;
				if (stripe < p.pb[i]) p.crc[i][c * p.crc_stride[i] + p.nb + r * p.pb[i] + stripe] = lin ^ p.zconst;
			}
		}
		// CRC of parity row 0 of every stripe (plain XOR of its blocks): xor of the blocks' linear CRCs (crc.h:29 mycrc32_xorblocks)
		__syncthreads();
		for (uint32_t gs = tid; gs < p.n_stripes; gs += NT) {
			const uint32_t i = p.gs_slice[gs], s = p.gs_stripe[gs], k = p.k[i];
			uint32_t x = 0;
			for (uint32_t j = 0; j < k; ++j) {
				uint32_t t;
				asm volatile("ld.shared.u32 %0, [%1];" : "=r"(t) : "r"(blk + 4 * (s * k + j)));
				x ^= t;
			}
			const uint32_t stripe = ui * p.S[i] + s;
			if (stripe < p.pb[i]) p.crc[i][c * p.crc_stride[i] + p.nb + stripe] = x ^ p.zconst;
		}
	}
}

}  // namespace lzd
