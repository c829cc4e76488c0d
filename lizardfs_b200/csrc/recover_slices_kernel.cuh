// recover_slices_kernel.cuh — lzgpu_recover_slices: rebuild a chunk of a multi-slice goal from the surviving parts of ALL its slices
// together, in one pass over the given parts.
//
// Reference work it extends: ChunkCopiesCalculator::evalRedundancyLevel scores each slice on its own (a chunk is lost once every slice
// has fewer than k parts), and SliceRecoveryPlanner reads one source slice.  All slices store the same chunk bytes, so a data block
// lost in one slice may be held by another, or pinned down by the parity equations of several slices together (slices_solve.h).
//
// A work unit is G combined stripes of one chunk (L = lcm(k_i) chunk blocks each), so the unit's blocks of a given part of slice i
// are one contiguous run of G L / k_i part blocks.  For each combined stripe the CTA walks the 64 KiB block in 64 slabs: lane l of a
// warp owns bytes [2048 l, 2048 l + 2048) of every block and moves 32 of them per slab, so its CRC stream over a block is contiguous
// and the 32 lane streams merge once per block (the tree of crc_blocks_kernel).
//   load    warp w takes read entries w, w + 8, ...: every block of every given part in the stripe; its CRC is folded when the part
//           has stored CRCs, and it is staged when it is the first copy of a known position or a chosen equation's parity block
//   solve   thread t owns word t of every staged 1 KiB slab: the syndromes of the chosen equations, the unknowns by the host rows
//           (general GF products, as the DIRECT form of fused_recover_kernel), then the wanted parity blocks of every slice from the
//           completed combined stripe
//   store   warp w takes write entries: the wanted data and parity blocks (CRC folded when out_crc is given) and the image
// At the end of a combined stripe every CRC stream is merged; a read block is compared with its stored CRC (the smallest mismatch,
// (chunk * 64 + flat part) * 1024 + block, lowers the result word), a written block's CRC is stored.
#pragma once
#include <cstdint>

#include "device_math.cuh"
#include "slices_solve.h"

namespace lzd {

constexpr int kRsThreads = kRsThreadsPerCta;
constexpr uint32_t kRsMaxEntries = kRsEntryCap;   // read entries, write entries and CRC streams per combined stripe
constexpr uint32_t kRsMaxOut = kRsOutCap;         // wanted parity blocks per combined stripe
constexpr uint32_t kRsSlab = 1024;        // bytes of one block per slab: 32 lanes x 32 bytes
constexpr uint8_t kRsNone = 0xff;

struct RsEntry {
	uint8_t part;   // flat part (read / written); kRsNone: the image
	uint8_t s;      // stripe of the part's slice in the combined stripe; the image: the position
	uint8_t slot;   // staged slab slot: position q < L, L + e (equation e), L + E + w (wanted parity block w); kRsNone: not staged
	uint8_t state;  // CRC stream; kRsNone: none
};

struct RsShape {
	uint16_t n_read, n_write, n_state, n_zero, n_unknown, n_eq, n_out;
	RsEntry read[kRsMaxEntries], write[kRsMaxEntries];
	RsEntry state[kRsMaxEntries];   // stream z: part, s (slot: 1 = a written block, 0 = a read block)
	uint8_t zero[kRsMaxL];           // slots of positions not loaded (unknown, or past the chunk's end): cleared before the solve
	uint8_t unk_pos[kRsMaxL];
	uint8_t eq_slice[kRsMaxL], eq_row[kRsMaxL], eq_stripe[kRsMaxL];
	uint8_t out_slice[kRsMaxOut], out_row[kRsMaxOut], out_stripe[kRsMaxOut];
	uint8_t rows[kRsMaxL][kRsMaxL];
};

struct RecoverSlicesParams {
	const uint8_t *parts[LZGPU_MAX_PARTS];
	const uint32_t *stored[LZGPU_MAX_PARTS];   // nullptr: not verified
	uint8_t *out[LZGPU_MAX_PARTS];
	uint32_t *out_crc[LZGPU_MAX_PARTS];
	uint8_t *image;
	unsigned long long part_stride[kSlicesMax], out_stride[kSlicesMax], image_stride;
	uint32_t k[kSlicesMax], spc[kSlicesMax], pb[kSlicesMax];   // spc: stripes of slice i per combined stripe (L / k_i)
	uint8_t part_slice[LZGPU_MAX_PARTS];
	uint8_t gen[kSlicesMax][32][32];
	const uint32_t *tables;
	unsigned long long *first_bad;
	uint32_t L, G, nb, n_cs, units_per_chunk, total_units, tail, n_slots, n_states_max, crc_off, zconst;
	uint32_t tree_mult[5];
	RsShape shape[2];   // 0: a full combined stripe, 1: the chunk's last one when L does not divide nb
};

// c * v for the four bytes of v; c is uniform across the CTA
__device__ __forceinline__ uint32_t rs_gf_mul(uint32_t v, uint32_t c) {
	if (c <= 1) return c ? v : 0u;
	uint32_t r = 0;
#pragma unroll
	for (int b = 7; b >= 0; --b) {
		r = gf_x2(r);
		if ((c >> b) & 1u) r ^= v;
	}
	return r;
}

__global__ void __launch_bounds__(kRsThreads, 1) recover_slices_kernel(const __grid_constant__ RecoverSlicesParams p) {
	extern __shared__ __align__(1024) uint8_t smem[];
	uint32_t *s_tab = reinterpret_cast<uint32_t *>(smem);
	uint8_t *s_slab = smem + 4096;
	uint32_t *s_crc = reinterpret_cast<uint32_t *>(s_slab + static_cast<size_t>(p.n_slots) * kRsSlab);
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, NW = kRsThreads / 32;
	for (uint32_t i = tid; i < 1024; i += kRsThreads) s_tab[i] = p.tables[i];
	uint32_t *W = reinterpret_cast<uint32_t *>(s_slab);   // word t of slot z: W[z * 256 + t]
	const uint32_t L = p.L;

	for (uint32_t unit = blockIdx.x; unit < p.total_units; unit += gridDim.x) {
		const uint32_t c = unit / p.units_per_chunk, u = unit % p.units_per_chunk;
		for (uint32_t g = 0; g < p.G; ++g) {
			const uint32_t cs = u * p.G + g;
			if (cs >= p.n_cs) break;
			const RsShape &sh = p.shape[(p.tail && cs == p.n_cs - 1) ? 1 : 0];
			const uint32_t E = sh.n_eq;
			__syncthreads();   // the previous stripe's streams are merged
			for (uint32_t i = tid; i < sh.n_state * 32u; i += kRsThreads) s_crc[i] = 0;
			__syncthreads();
			for (uint32_t slab = 0; slab < 64; ++slab) {
				const uint32_t off = lane * 2048 + slab * 32;
				// ---------------- load ----------------
				for (uint32_t e = warp; e < sh.n_read; e += NW) {
					const RsEntry en = sh.read[e];
					const uint32_t i = p.part_slice[en.part];
					const unsigned long long blk = static_cast<unsigned long long>(cs) * p.spc[i] + en.s;
					const uint4 *src = reinterpret_cast<const uint4 *>(p.parts[en.part] + c * p.part_stride[i] + (blk << 16) + off);
					const uint4 a = ld_stream(src), b = ld_stream(src + 1);
					if (en.state != kRsNone && !p.crc_off) {
						uint32_t st = s_crc[en.state * 32 + lane];
						st = crc_step_word(st, a.x, s_tab); st = crc_step_word(st, a.y, s_tab);
						st = crc_step_word(st, a.z, s_tab); st = crc_step_word(st, a.w, s_tab);
						st = crc_step_word(st, b.x, s_tab); st = crc_step_word(st, b.y, s_tab);
						st = crc_step_word(st, b.z, s_tab); st = crc_step_word(st, b.w, s_tab);
						s_crc[en.state * 32 + lane] = st;
					}
					if (en.slot != kRsNone) {
						uint4 *dst = reinterpret_cast<uint4 *>(s_slab + en.slot * kRsSlab + lane * 32);
						dst[0] = a;
						dst[1] = b;
					}
				}
				__syncthreads();
				// ---------------- solve: word tid of every slot ----------------
				for (uint32_t z = 0; z < sh.n_zero; ++z) W[sh.zero[z] * 256u + tid] = 0;
				for (uint32_t e = 0; e < E; ++e) {
					const uint32_t i = sh.eq_slice[e], r = sh.eq_row[e], s = sh.eq_stripe[e], k = p.k[i];
					uint32_t syn = W[(L + e) * 256u + tid];
					for (uint32_t j = 0; j < k; ++j) syn ^= rs_gf_mul(W[(s * k + j) * 256u + tid], p.gen[i][r][j]);
					W[(L + e) * 256u + tid] = syn;
				}
				for (uint32_t x = 0; x < sh.n_unknown; ++x) {
					uint32_t acc = 0;
					for (uint32_t e = 0; e < E; ++e) acc ^= rs_gf_mul(W[(L + e) * 256u + tid], sh.rows[x][e]);
					W[sh.unk_pos[x] * 256u + tid] = acc;
				}
				for (uint32_t w = 0; w < sh.n_out; ++w) {
					const uint32_t i = sh.out_slice[w], r = sh.out_row[w], s = sh.out_stripe[w], k = p.k[i];
					uint32_t v = 0;
					for (uint32_t j = 0; j < k; ++j) v ^= rs_gf_mul(W[(s * k + j) * 256u + tid], p.gen[i][r][j]);
					W[(L + E + w) * 256u + tid] = v;
				}
				__syncthreads();
				// ---------------- store ----------------
				for (uint32_t e = warp; e < sh.n_write; e += NW) {
					const RsEntry en = sh.write[e];
					const uint4 *src = reinterpret_cast<const uint4 *>(s_slab + en.slot * kRsSlab + lane * 32);
					const uint4 a = src[0], b = src[1];
					uint8_t *dst;
					if (en.part == kRsNone) {
						dst = p.image + c * p.image_stride + (static_cast<unsigned long long>(cs * L + en.s) << 16) + off;
					} else {
						const uint32_t i = p.part_slice[en.part];
						const unsigned long long blk = static_cast<unsigned long long>(cs) * p.spc[i] + en.s;
						dst = p.out[en.part] + c * p.out_stride[i] + (blk << 16) + off;
					}
					st_stream(reinterpret_cast<uint4 *>(dst), a);
					st_stream(reinterpret_cast<uint4 *>(dst) + 1, b);
					if (en.state != kRsNone && !p.crc_off) {
						uint32_t st = s_crc[en.state * 32 + lane];
						st = crc_step_word(st, a.x, s_tab); st = crc_step_word(st, a.y, s_tab);
						st = crc_step_word(st, a.z, s_tab); st = crc_step_word(st, a.w, s_tab);
						st = crc_step_word(st, b.x, s_tab); st = crc_step_word(st, b.y, s_tab);
						st = crc_step_word(st, b.z, s_tab); st = crc_step_word(st, b.w, s_tab);
						s_crc[en.state * 32 + lane] = st;
					}
				}
				__syncthreads();
			}
			// ---------------- merge the lane streams of every block ----------------
			for (uint32_t z = warp; z < sh.n_state; z += NW) {
				uint32_t st = s_crc[z * 32 + lane];
#pragma unroll
				for (int i = 0; i < 5; ++i) {
					const uint32_t right = __shfl_down_sync(0xffffffffu, st, 1u << i);
					st = crc_mulmod(st, p.tree_mult[i]) ^ right;
				}
				if (lane != 0) continue;
				const RsEntry en = sh.state[z];
				const uint32_t i = p.part_slice[en.part];
				const unsigned long long blk = static_cast<unsigned long long>(cs) * p.spc[i] + en.s;
				const unsigned long long at = static_cast<unsigned long long>(c) * p.pb[i] + blk;
				const uint32_t crc = p.crc_off ? LZGPU_FAKE_CRC : (st ^ p.zconst);
				if (en.slot) {
					p.out_crc[en.part][at] = crc;
				} else if (p.stored[en.part][at] != crc) {
					atomicMin(p.first_bad, (static_cast<unsigned long long>(c) * 64ull + en.part) * 1024ull + blk);
				}
			}
		}
	}
}

}  // namespace lzd
