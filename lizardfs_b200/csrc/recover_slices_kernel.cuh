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
//
// The SALVAGE instantiation (lzgpu_salvage_slices) writes the image only, with a CRC stream per image block, whatever the given parts
// determine: an undetermined unknown has an all-zero solve row, so it comes out as zeros.  A read block that fails its stored CRC also
// sets its read entry's bit in a shared mask; after the merge every position whose value depends on a failing read entry (the host's
// dependency mask, RsSalvage) is withheld: the CTA zeroes its image block, which it stored earlier in the stripe, and gives it the CRC
// of zeros.  Then the stripe's status bytes are written to the map.
//
// The CHECK instantiation (lzgpu_check_slices) writes nothing but one map entry per combined stripe.  It stages the basis of
// slices_check.h (the first copy of each known position, the chosen equations' parity blocks) and every check's defining block (slot
// L + E + h), solves the unknowns by the particular-solution rows, and in the wanted-parity step re-encodes each check's prediction (a
// further copy of a known position: that position) and compares it with the defining block word by word.  Each thread ORs bit h into
// a 64-bit mask where they differ; the warps OR theirs into a shared word pair, and the stripe's entry is {mask, -1, 0}.
// locate_slices_kernel then names the suspect part of every entry whose mask is not zero.
//
// The CORRECT instantiation (lzgpu_correct_slices) is the CHECK one, writing its entries to a temporary map, plus one 64-bit mask per
// combined stripe: the parts with a read block that fails its stored CRC (the SALVAGE form's shared failing-read-entry mask, mapped to
// parts).  locate_slices_kernel names the suspects, and correct_slices_kernel applies the rule and rewrites the suspect's blocks.
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
	uint8_t state;  // CRC stream; kRsNone: none.  In a stream entry of a read block: that block's read entry
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

// lzgpu_salvage_slices, per stripe shape: bit r of dep[q] = the value of position q depends on read entry r (its staged copy, or a
// chosen equation's parity block or known position that its solve row uses); status[q] = LZGPU_SALVAGE_KNOWN / _SOLVED / _HOLE
constexpr uint32_t kRsMaskWords = kRsMaxEntries / 32;
struct RsSalvage {
	uint32_t dep[kRsMaxL][kRsMaskWords];
	uint8_t status[kRsMaxL];
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
	// the SALVAGE instantiation only: the image's block CRCs (nullptr: none) and status bytes, block c * nb + b, and the shapes' masks
	uint32_t *image_crc;
	uint8_t *map;
	RsSalvage salvage[2];
	// the CORRECT instantiation only: bit g of crc_failed[c * n_cs + cs] = a read block of part g fails its stored CRC
	unsigned long long *crc_failed;
};
static_assert(sizeof(RecoverSlicesParams) <= 32764, "recover_slices_kernel's parameter block must fit the 32764-byte kernel parameter limit");

// lzgpu_slices_check as the kernels write it
struct RsCheckEntry {
	unsigned long long bad_checks;
	int suspect_part;
	uint32_t zero;
};

// The per-stripe shared words of the SALVAGE instantiation: the failing read entries, then the withheld positions (CHECK: words 0
// and 1 are the stripe's bad_checks; CORRECT: the failing read entries, then bad_checks)
__device__ __forceinline__ uint32_t *rs_salvage_smem() {
	__shared__ uint32_t words[kRsMaskWords + 2];
	return words;
}

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

template <RsMode MODE>
__global__ void __launch_bounds__(kRsThreads, 1) recover_slices_kernel(const __grid_constant__ RecoverSlicesParams p) {
	constexpr bool SALVAGE = MODE == RsMode::SALVAGE, CORRECT = MODE == RsMode::CORRECT, CHECK = MODE == RsMode::CHECK || CORRECT;
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
			[[maybe_unused]] unsigned long long bad = 0;   // CHECK, CORRECT: the checks this thread has seen differ
			__syncthreads();   // the previous stripe's streams are merged
			for (uint32_t i = tid; i < sh.n_state * 32u; i += kRsThreads) s_crc[i] = 0;
			if constexpr (SALVAGE || CHECK)
				if (tid < kRsMaskWords + 2) rs_salvage_smem()[tid] = 0;
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
					if (CHECK && r == kRsNone) v = W[s * 256u + tid];   // a further copy of position s
					else
						for (uint32_t j = 0; j < k; ++j) v ^= rs_gf_mul(W[(s * k + j) * 256u + tid], p.gen[i][r][j]);
					if constexpr (CHECK) bad |= static_cast<unsigned long long>(v != W[(L + E + w) * 256u + tid]) << w;
					else W[(L + E + w) * 256u + tid] = v;
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
				if constexpr (SALVAGE) {
					if (en.part == kRsNone) {   // an image block; a withheld one is given the CRC of zeros below
						p.image_crc[static_cast<unsigned long long>(c) * p.nb + cs * L + en.s] = p.crc_off ? LZGPU_FAKE_CRC : (st ^ p.zconst);
						continue;
					}
				}
				const uint32_t i = p.part_slice[en.part];
				const unsigned long long blk = static_cast<unsigned long long>(cs) * p.spc[i] + en.s;
				const unsigned long long at = static_cast<unsigned long long>(c) * p.pb[i] + blk;
				const uint32_t crc = p.crc_off ? LZGPU_FAKE_CRC : (st ^ p.zconst);
				if (en.slot) {
					p.out_crc[en.part][at] = crc;
				} else if (p.stored[en.part][at] != crc) {
					atomicMin(p.first_bad, (static_cast<unsigned long long>(c) * 64ull + en.part) * 1024ull + blk);
					if constexpr (SALVAGE || CORRECT) atomicOr(&rs_salvage_smem()[en.state >> 5], 1u << (en.state & 31));
				}
			}
			if constexpr (CHECK) {
				// ---------------- the stripe's entry ----------------
				uint32_t *mask = rs_salvage_smem() + (CORRECT ? kRsMaskWords : 0);
				const uint32_t lo = __reduce_or_sync(0xffffffffu, static_cast<uint32_t>(bad)), hi = __reduce_or_sync(0xffffffffu, static_cast<uint32_t>(bad >> 32));
				if (lane == 0 && (lo | hi)) {
					atomicOr(&mask[0], lo);
					atomicOr(&mask[1], hi);
				}
				__syncthreads();
				if (tid == 0) {
					RsCheckEntry *en = reinterpret_cast<RsCheckEntry *>(p.map) + static_cast<unsigned long long>(c) * p.n_cs + cs;
					en->bad_checks = (static_cast<unsigned long long>(mask[1]) << 32) | mask[0];
					en->suspect_part = -1;
					en->zero = 0;
				}
				if constexpr (CORRECT) {
					if (warp == 0) {   // the failing read entries, mapped to parts
						const uint32_t *fail = rs_salvage_smem();
						unsigned long long parts = 0;
						for (uint32_t r = lane; r < sh.n_read; r += 32)
							if ((fail[r >> 5] >> (r & 31)) & 1u) parts |= 1ull << sh.read[r].part;
						const uint32_t plo = __reduce_or_sync(0xffffffffu, static_cast<uint32_t>(parts));
						const uint32_t phi = __reduce_or_sync(0xffffffffu, static_cast<uint32_t>(parts >> 32));
						if (lane == 0) p.crc_failed[static_cast<unsigned long long>(c) * p.n_cs + cs] = (static_cast<unsigned long long>(phi) << 32) | plo;
					}
				}
			}
			if constexpr (SALVAGE) {
				// ---------------- withhold what depends on a failing block, then the stripe's map bytes ----------------
				__syncthreads();
				uint32_t *fail = rs_salvage_smem(), *withheld = fail + kRsMaskWords;
				const RsSalvage &sv = p.salvage[(p.tail && cs == p.n_cs - 1) ? 1 : 0];
				const uint32_t valid = min(L, p.nb - cs * L);
				const unsigned long long b0 = static_cast<unsigned long long>(c) * p.nb + cs * L;
				if (tid < valid) {
					bool w = false;
#pragma unroll
					for (uint32_t i = 0; i < kRsMaskWords; ++i) w |= (fail[i] & sv.dep[tid][i]) != 0;
					p.map[b0 + tid] = w ? LZGPU_SALVAGE_WITHHELD : sv.status[tid];
					if (w) {
						if (p.image_crc) p.image_crc[b0 + tid] = p.crc_off ? LZGPU_FAKE_CRC : p.zconst;
						atomicOr(&withheld[tid >> 5], 1u << (tid & 31));
					}
				}
				__syncthreads();
				for (uint32_t q = 0; q < valid; ++q) {
					if (!((withheld[q >> 5] >> (q & 31)) & 1u)) continue;
					uint4 *dst = reinterpret_cast<uint4 *>(p.image + c * p.image_stride + (static_cast<unsigned long long>(cs * L + q) << 16));
					for (uint32_t i = tid; i < 65536u / 16u; i += kRsThreads) dst[i] = make_uint4(0, 0, 0, 0);
				}
			}
		}
	}
}

// lzgpu_check_slices' locate pass, per stripe shape (a device buffer: the dense rows and the annihilators exceed the parameter block).
// The given blocks of the shape, its check rows over them, and per candidate part (a given part with a block in the shape) its
// annihilator rows, kScMaxChecks bytes each, at rows[ann0 + first[c] ..] after the two shapes.
struct RsLocateShape {
	uint32_t n_blocks, n_checks, n_cand, ann0;
	uint8_t blk_part[kRsMaxEntries], blk_s[kRsMaxEntries];
	uint8_t cand_part[LZGPU_MAX_PARTS];
	uint16_t cand_first[LZGPU_MAX_PARTS + 1];
	uint8_t H[kRsMaxOut][kRsMaxEntries];
};
struct RsLocate {
	RsLocateShape shape[2];   // then the annihilator rows of both shapes
};
struct LocateSlicesParams {
	const uint8_t *parts[LZGPU_MAX_PARTS];
	unsigned long long part_stride[kSlicesMax];
	uint32_t spc[kSlicesMax];
	uint8_t part_slice[LZGPU_MAX_PARTS];
	RsCheckEntry *map;
	const RsLocate *loc;
	unsigned long long n_entries;
	uint32_t n_cs, tail;
};
constexpr int kRslThreads = 128;

// The syndrome words of word w of combined stripe cs of chunk c: S[h * stride] = sum over the shape's given blocks b of H[h][b] y_b
__device__ __forceinline__ void rs_syndrome_word(const RsLocateShape &sh, const uint8_t *const *parts, const unsigned long long *part_stride,
                                                 const uint32_t *spc, const uint8_t *part_slice, uint32_t c, uint32_t cs, uint32_t w,
                                                 uint32_t *S, uint32_t stride) {
	const uint32_t nc = sh.n_checks;
	for (uint32_t h = 0; h < nc; ++h) S[h * stride] = 0;
	for (uint32_t b = 0; b < sh.n_blocks; ++b) {
		const uint32_t g = sh.blk_part[b], i = part_slice[g];
		const unsigned long long blk = static_cast<unsigned long long>(cs) * spc[i] + sh.blk_s[b];
		const uint32_t v = reinterpret_cast<const uint32_t *>(parts[g] + c * part_stride[i] + (blk << 16))[w];
		for (uint32_t h = 0; h < nc; ++h) {
			const uint32_t coef = sh.H[h][b];
			if (coef) S[h * stride] ^= rs_gf_mul(v, coef);
		}
	}
}

// One CTA per bad entry (grid-stride over the map; a clean entry is skipped, its suspect is already -1).  Thread t owns words t,
// t + 128, ... of the stripe's blocks: it forms the syndrome words S_h = sum_b H[h][b] y_b, and where they are not all zero drops every
// candidate an annihilator row of which does not map them to zero (a 4-byte word: the test holds for each of its bytes).  The one
// candidate left is the suspect; none or several: -1.
__global__ void __launch_bounds__(kRslThreads) locate_slices_kernel(const __grid_constant__ LocateSlicesParams p) {
	__shared__ uint32_t S[kRsMaxOut][kRslThreads];
	__shared__ unsigned long long s_alive;
	const uint32_t tid = threadIdx.x;
	const uint8_t *ann = reinterpret_cast<const uint8_t *>(p.loc + 1);
	for (unsigned long long e = blockIdx.x; e < p.n_entries; e += gridDim.x) {
		if (p.map[e].bad_checks == 0) continue;
		const uint32_t c = static_cast<uint32_t>(e / p.n_cs), cs = static_cast<uint32_t>(e % p.n_cs);
		const RsLocateShape &sh = p.loc->shape[(p.tail && cs == p.n_cs - 1) ? 1 : 0];
		const uint32_t nc = sh.n_checks;
		if (tid == 0) s_alive = sh.n_cand >= 64 ? ~0ull : (1ull << sh.n_cand) - 1ull;
		__syncthreads();
		unsigned long long alive = s_alive;
		for (uint32_t w = tid; w < 65536u / 4u; w += kRslThreads) {
			rs_syndrome_word(sh, p.parts, p.part_stride, p.spc, p.part_slice, c, cs, w, &S[0][tid], kRslThreads);
			uint32_t any = 0;
			for (uint32_t h = 0; h < nc; ++h) any |= S[h][tid];
			if (!any) continue;
			for (unsigned long long left = alive; left; left &= left - 1) {
				const uint32_t ci = static_cast<uint32_t>(__ffsll(static_cast<long long>(left)) - 1);
				bool fits = true;
				for (uint32_t r = sh.cand_first[ci]; r < sh.cand_first[ci + 1] && fits; ++r) {
					const uint8_t *row = ann + static_cast<size_t>(sh.ann0 + r) * kRsMaxOut;
					uint32_t acc = 0;
					for (uint32_t h = 0; h < nc; ++h) acc ^= rs_gf_mul(S[h][tid], row[h]);
					fits = acc == 0;
				}
				if (!fits) alive &= ~(1ull << ci);
			}
		}
		atomicAnd(&s_alive, alive);
		__syncthreads();
		if (tid == 0) {
			const unsigned long long left = s_alive;
			p.map[e].suspect_part = left && !(left & (left - 1)) ? sh.cand_part[__ffsll(static_cast<long long>(left)) - 1] : -1;
		}
		__syncthreads();
	}
}

// lzgpu_slices_fix as correct_slices_kernel writes it
struct RsFixEntry {
	unsigned long long bad_checks;
	int suspect_part, status;
	unsigned long long crc_failed, changed;
};

// correct_slices_kernel's tables per stripe shape (the blocks and checks are the locate pass's RsLocateShape): the correctable parts,
// each part's run of blocks in the shape's list, and the row of P for block b of the list at rows[prow0 + b] (rows of kRsMaxOut bytes
// after the annihilators; zero for a part that is not correctable)
struct RsCorrectShape {
	unsigned long long correctable;
	uint32_t prow0;
	uint8_t blk_first[LZGPU_MAX_PARTS], blk_count[LZGPU_MAX_PARTS];
};
struct CorrectSlicesParams {
	uint8_t *parts[LZGPU_MAX_PARTS];
	uint32_t *new_crc[LZGPU_MAX_PARTS];   // nullptr: none
	unsigned long long part_stride[kSlicesMax];
	uint32_t spc[kSlicesMax], pb[kSlicesMax];
	uint8_t part_slice[LZGPU_MAX_PARTS];
	const RsCheckEntry *map;
	const unsigned long long *crc_failed;
	RsFixEntry *fix;
	const RsLocate *loc;
	const uint32_t *tables;
	unsigned long long n_entries;
	uint32_t n_cs, tail, crc_off, zconst, run_mult;   // run_mult: x^(8 * kRscRun) mod P
	uint32_t tree_mult[5];                            // x^(8 * 2048 * 2^i) mod P, as recover_slices_kernel's
	RsCorrectShape shape[2];
};
constexpr int kRscThreads = 128;
constexpr uint32_t kRscRun = 65536u / kRscThreads;   // bytes of each block per thread, contiguous
// dynamic shared memory: the CRC tables, the syndrome words [h][tid], the CRC streams of the suspect's blocks [j][tid]
constexpr size_t rsc_smem_bytes(uint32_t n_checks, uint32_t n_suspect_blocks) { return 4096 + (n_checks + n_suspect_blocks) * kRscThreads * 4ull; }

// One CTA per entry (grid-stride over the map), every fix entry written.  The rule: CLEAN without bad checks, UNEXPLAINED without a
// suspect g, CRC_CONFLICT when a part other than g has a failing block, UNDETERMINED when g is not correctable, else CORRECTED.  A
// corrected entry: thread t owns bytes [kRscRun t, kRscRun (t + 1)) of every block; per word it forms the syndromes (rs_syndrome_word),
// e_j = sum_h P[j][h] S_h for each block j of g, XORs e_j into the block in place and folds the word as written into block j's CRC
// stream.  The four streams of a lane's 2048 bytes are chained, then merged by the tree of crc_blocks_kernel.
__global__ void __launch_bounds__(kRscThreads) correct_slices_kernel(const __grid_constant__ CorrectSlicesParams p) {
	extern __shared__ __align__(16) uint32_t rsc_smem[];
	uint32_t *s_tab = rsc_smem, *S = rsc_smem + 1024;
	__shared__ uint32_t s_changed[2];
	const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	for (uint32_t i = tid; i < 1024; i += kRscThreads) s_tab[i] = p.tables[i];
	const uint8_t *rows = reinterpret_cast<const uint8_t *>(p.loc + 1);
	__syncthreads();
	for (unsigned long long e = blockIdx.x; e < p.n_entries; e += gridDim.x) {
		const RsCheckEntry en = p.map[e];
		const unsigned long long failed = p.crc_failed[e];
		const uint32_t c = static_cast<uint32_t>(e / p.n_cs), cs = static_cast<uint32_t>(e % p.n_cs), t = (p.tail && cs == p.n_cs - 1) ? 1 : 0;
		const RsLocateShape &sh = p.loc->shape[t];
		const RsCorrectShape &cor = p.shape[t];
		const int g = en.suspect_part;
		const int status = !en.bad_checks ? LZGPU_FIX_CLEAN
		                   : g < 0 ? LZGPU_FIX_UNEXPLAINED
		                   : (failed & ~(1ull << g)) ? LZGPU_FIX_CRC_CONFLICT
		                   : !((cor.correctable >> g) & 1ull) ? LZGPU_FIX_UNDETERMINED : LZGPU_FIX_CORRECTED;
		if (status != LZGPU_FIX_CORRECTED) {
			if (tid == 0) p.fix[e] = RsFixEntry{en.bad_checks, g, status, failed, 0ull};
			continue;
		}
		const uint32_t nc = sh.n_checks, b0 = cor.blk_first[g], nbk = cor.blk_count[g], i = p.part_slice[g];
		uint32_t *s_crc = S + nc * kRscThreads;
		uint8_t *base = p.parts[g] + c * p.part_stride[i] + ((static_cast<unsigned long long>(cs) * p.spc[i]) << 16);
		if (tid < 2) s_changed[tid] = 0;
		for (uint32_t j = 0; j < nbk; ++j) s_crc[j * kRscThreads + tid] = 0;
		unsigned long long changed = 0;
		for (uint32_t w = tid * (kRscRun / 4); w < (tid + 1) * (kRscRun / 4); ++w) {
			rs_syndrome_word(sh, reinterpret_cast<const uint8_t *const *>(p.parts), p.part_stride, p.spc, p.part_slice, c, cs, w, S + tid,
			                 kRscThreads);
			for (uint32_t j = 0; j < nbk; ++j) {
				const uint8_t *row = rows + static_cast<size_t>(cor.prow0 + b0 + j) * kRsMaxOut;
				uint32_t err = 0;
				for (uint32_t h = 0; h < nc; ++h) err ^= rs_gf_mul(S[h * kRscThreads + tid], row[h]);
				const uint32_t s = sh.blk_s[b0 + j];
				uint32_t *word = reinterpret_cast<uint32_t *>(base + (static_cast<unsigned long long>(s) << 16)) + w;
				uint32_t y = *word;
				if (err) {
					y ^= err;
					*word = y;
					changed |= 1ull << s;
				}
				if (!p.crc_off) s_crc[j * kRscThreads + tid] = crc_step_word(s_crc[j * kRscThreads + tid], y, s_tab);
			}
		}
		const uint32_t lo = __reduce_or_sync(0xffffffffu, static_cast<uint32_t>(changed)), hi = __reduce_or_sync(0xffffffffu, static_cast<uint32_t>(changed >> 32));
		__syncthreads();   // s_changed cleared, every stream complete
		if (lane == 0 && (lo | hi)) {
			atomicOr(&s_changed[0], lo);
			atomicOr(&s_changed[1], hi);
		}
		// ---------------- each block's CRC: lane l chains the runs of threads 4l .. 4l + 3, then the tree ----------------
		uint32_t *out = p.new_crc[g];
		for (uint32_t j = warp; out && j < nbk; j += kRscThreads / 32) {
			const uint32_t *sc = s_crc + j * kRscThreads + lane * 4;
			uint32_t st = sc[0];
			for (int r = 1; r < 4; ++r) st = crc_mulmod(st, p.run_mult) ^ sc[r];
#pragma unroll
			for (int l = 0; l < 5; ++l) {
				const uint32_t right = __shfl_down_sync(0xffffffffu, st, 1u << l);
				st = crc_mulmod(st, p.tree_mult[l]) ^ right;
			}
			if (lane == 0)
				out[static_cast<unsigned long long>(c) * p.pb[i] + static_cast<unsigned long long>(cs) * p.spc[i] + sh.blk_s[b0 + j]] =
				    p.crc_off ? LZGPU_FAKE_CRC : (st ^ p.zconst);
		}
		__syncthreads();
		if (tid == 0) p.fix[e] = RsFixEntry{en.bad_checks, g, status, failed, (static_cast<unsigned long long>(s_changed[1]) << 32) | s_changed[0]};
		__syncthreads();   // S, the streams and s_changed are free for the next entry
	}
}

}  // namespace lzd
