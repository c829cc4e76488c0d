// correct_kernel.cuh — lzgpu_correct_stripes: every stripe of the stripe map that names a suspect part gets that part's block
// rebuilt in place from k other blocks of the stripe, unless a given block other than the suspect's fails its stored CRC.
//
// One CTA (256 threads) per entry that has a suspect, grid-stride over the map; an entry without one only gets its status.  Thread t
// owns bytes [256t, 256t + 256) of every block of the stripe.  Each given block other than the suspect's is read once (16-byte
// loads): its CRC for the gate when it has a stored CRC, and its GF product with the suspect's coefficient when it is one of the k
// inputs (the first k given parts other than the suspect, ascending: the parts ECReadPlan::recoverParts picks when the suspect is
// unavailable).  The corrected bytes stay in registers until the gate has passed; then they are stored over the suspect's block and
// their CRC goes into the fix entry.  A CTA owns its stripe's blocks alone and the check pass has finished by stream order, so the
// in-place stores race with nothing.
//
// CRC of a block: thread t folds its 256 bytes with the slicing tables (crc_step_word), shifts the result by the bytes after its
// segment, x^(8 * 256 (255 - t)) (a multiplier computed once per CTA), and the CTA XOR-reduces: lin(block) = XOR_t lin(seg_t) *
// x^(8 * |bytes after seg_t|), one crc_mulmod per block and thread instead of the eight levels of cta_crc_tree.
#pragma once
#include "kernels_generic.cuh"
#include "lzgpu.h"
#include "repair_rows.h"
#include "decode_locate.h"

namespace lzd {

struct CorrectArgs {
	uint8_t *part[64];                 // part i of chunk 0; nullptr = not given
	const uint32_t *crc[64];           // stored CRCs of part i, [chunk * pb + block]; nullptr = none
	const uint32_t *map;               // the stripe map, two words per entry (bad_rows, suspect_part)
	lzgpu_stripe_fix *fix;             // one entry per map entry
	const uint32_t *tables;            // 4 * 256 slicing tables
	unsigned long long part_stride, n_entries;
	unsigned long long given;          // bit i: part i is given
	unsigned long long xor_row;        // bit i: every coefficient of suspect i's row is 1
	uint32_t n_parts, k, pb;
	int crc_disabled;                  // lzgpu_set_crc_enabled(0): stored CRCs are compared with the constant, blocks are not CRCed
	uint32_t pow2[32];                 // x^(8 * 2^i) mod P
	uint8_t coef[64][32];              // [suspect][input]: the suspect's block = sum_i coef * input block i
};

// one block of the stripe, thread t's 256 bytes: CRC (VERIFY) and, as input, acc ^= coef * v (MODE 1: coef 1; MODE 2: any coef)
template <bool VERIFY, int MODE>
__device__ __forceinline__ uint32_t correct_read(const uint8_t *blk, uint32_t (&acc)[64], const CoefPlanes &cp, const uint32_t *tab) {
	uint4 v[16];
	const uint4 *p = reinterpret_cast<const uint4 *>(blk) + threadIdx.x * 16;
#pragma unroll
	for (int i = 0; i < 16; ++i) v[i] = __ldg(p + i);
	uint32_t st = 0;
#pragma unroll
	for (int i = 0; i < 16; ++i) {
		const uint32_t w[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
#pragma unroll
		for (int j = 0; j < 4; ++j) {
			if constexpr (VERIFY) st = crc_step_word(st, w[j], tab);
			if constexpr (MODE == 1) acc[4 * i + j] ^= w[j];
			if constexpr (MODE == 2) acc[4 * i + j] = gf_mac(acc[4 * i + j], w[j], cp);
		}
	}
	return st;
}

// thread t's CRC state of its segment -> the block's linear CRC, XOR-reduced into s_out[warp] (the caller's barrier publishes it)
__device__ __forceinline__ void correct_crc_part(uint32_t st, uint32_t shift, uint32_t *s_out) {
	st = __reduce_xor_sync(0xffffffffu, crc_mulmod(st, shift));
	if ((threadIdx.x & 31) == 0) s_out[threadIdx.x >> 5] = st;
}

// the CRC of the 64 KiB block whose thread-t bytes are acc, in every thread (one barrier publishes s_out)
__device__ __forceinline__ uint32_t block_crc(const uint32_t (&acc)[64], const uint32_t *s_tab, uint32_t shift, uint32_t *s_out) {
	uint32_t st = 0;
#pragma unroll
	for (int i = 0; i < 64; ++i) st = crc_step_word(st, acc[i], s_tab);
	correct_crc_part(st, shift, s_out);
	__syncthreads();
	uint32_t crc = kCrcZeroBlock64K;
#pragma unroll
	for (int w = 0; w < 8; ++w) crc ^= s_out[w];
	return crc;
}

// thread t's 256 bytes of acc over its part of the block
__device__ __forceinline__ void block_store(uint8_t *blk, const uint32_t (&acc)[64]) {
	uint4 *dst = reinterpret_cast<uint4 *>(blk) + threadIdx.x * 16;
#pragma unroll
	for (int i = 0; i < 16; ++i) dst[i] = make_uint4(acc[4 * i], acc[4 * i + 1], acc[4 * i + 2], acc[4 * i + 3]);
}

// the per-CTA setup, on the first entry with work: the slicing tables, this thread's shift and (s_gf given) the GF tables
__device__ __forceinline__ void cta_setup(bool &ready, uint32_t &shift, uint32_t *s_tab, GfTables *s_gf, const uint32_t *tables,
                                          const uint32_t *pow2) {
	if (ready) return;
	const unsigned t = threadIdx.x;
	for (unsigned i = t; i < 1024; i += 256) s_tab[i] = tables[i];
	if (s_gf && t == 0) gf_tables_build(*s_gf);
	shift = crc_xpow_bytes_dev(256u * (255u - t), pow2);
	ready = true;
}

__global__ void __launch_bounds__(256) correct_map_kernel(const CorrectArgs a) {
	__shared__ uint32_t s_tab[1024];
	__shared__ CoefPlanes s_coef[32];
	__shared__ uint32_t s_lin[64][8];  // per part, per warp: the XOR of the warp's shifted segment CRCs
	__shared__ uint32_t s_out[8];
	const unsigned t = threadIdx.x;
	bool ready = false;
	uint32_t shift = 0;
	for (unsigned long long e = blockIdx.x; e < a.n_entries; e += gridDim.x) {
		const uint32_t bad_rows = a.map[2 * e];
		const int suspect = static_cast<int>(a.map[2 * e + 1]);
		if (bad_rows == 0 || suspect < 0) {
			if (t == 0) a.fix[e] = lzgpu_stripe_fix{bad_rows, suspect, bad_rows ? LZGPU_FIX_UNEXPLAINED : LZGPU_FIX_CLEAN, 0u};
			continue;
		}
		cta_setup(ready, shift, s_tab, nullptr, a.tables, a.pow2);
		if (t < a.k) coef_planes_set(s_coef[t], a.coef[suspect][t]);
		__syncthreads();
		const unsigned long long off = (e / a.pb) * a.part_stride + (e % a.pb) * 65536ull;
		const bool xor_row = (a.xor_row >> suspect) & 1ull;
		uint32_t acc[64];
#pragma unroll
		for (int i = 0; i < 64; ++i) acc[i] = 0;
		uint32_t used = 0;
		for (uint32_t p = 0; p < a.n_parts; ++p) {
			if (!((a.given >> p) & 1ull) || static_cast<int>(p) == suspect) continue;
			const bool input = used < a.k;
			const bool verify = a.crc[p] && !a.crc_disabled;
			const uint8_t *blk = a.part[p] + off;
			uint32_t st = 0;
			if (input && xor_row) st = verify ? correct_read<true, 1>(blk, acc, s_coef[0], s_tab) : correct_read<false, 1>(blk, acc, s_coef[0], s_tab);
			else if (input) st = verify ? correct_read<true, 2>(blk, acc, s_coef[used], s_tab) : correct_read<false, 2>(blk, acc, s_coef[used], s_tab);
			else if (verify) st = correct_read<true, 0>(blk, acc, s_coef[0], s_tab);
			if (verify) correct_crc_part(st, shift, s_lin[p]);
			used += input ? 1u : 0u;
		}
		__syncthreads();
		// the gate: thread p compares part p's stored CRC as the check does (the CRC-disabled mode: with the constant)
		bool fail = false;
		if (t < a.n_parts && ((a.given >> t) & 1ull) && static_cast<int>(t) != suspect && a.crc[t]) {
			const uint32_t stored = a.crc[t][e];  // e = chunk * pb + block
			if (a.crc_disabled) {
				fail = stored != LZGPU_FAKE_CRC;
			} else {
				uint32_t lin = 0;
#pragma unroll
				for (int w = 0; w < 8; ++w) lin ^= s_lin[t][w];
				fail = (lin ^ kCrcZeroBlock64K) != stored;
			}
		}
		const bool conflict = __syncthreads_or(fail);
		uint32_t crc = 0;
		if (!conflict) {
			block_store(a.part[suspect] + off, acc);
			crc = a.crc_disabled ? LZGPU_FAKE_CRC : block_crc(acc, s_tab, shift, s_out);
		}
		if (t == 0) a.fix[e] = lzgpu_stripe_fix{bad_rows, suspect, conflict ? LZGPU_FIX_CRC_CONFLICT : LZGPU_FIX_CORRECTED, crc};
		__syncthreads();  // s_coef, s_lin and s_out are re-used by the next entry
	}
}

// lzgpu_repair_stripes: the map entry and F = failed[e] (bit p: the block of part p fails its stored CRC, set by the check pass) give
// the set X of blocks to rebuild: {suspect} when F is empty (the correction's rule 1, without its gate: no block fails), F itself
// when the stripe is bad and |F| <= given - k (rule 3).  Every other entry only gets its status.  The inputs are the first k given
// parts outside X, ascending; the rows of X over them come from repair_rows (repair_rows.h) in shared memory.  One pass over the
// inputs per block of X (correct_read into 64 registers, then the CTA's CRC of the result): rule 3 stores nothing until every rebuilt
// block has matched its stored CRC, so the last block stays in registers and the others are computed again for the store (2|X| - 1
// passes, the later ones from L2).
struct RepairArgs {
	uint8_t *part[64];                 // part i of chunk 0; nullptr = not given
	const uint32_t *crc[64];           // stored CRCs of part i, [chunk * pb + block] (every given part has them)
	const uint32_t *map;               // the stripe map, two words per entry (bad_rows, suspect_part)
	const unsigned long long *failed;  // F per entry
	lzgpu_stripe_repair *fix;          // one entry per map entry
	const uint32_t *tables;            // 4 * 256 slicing tables
	unsigned long long part_stride, n_entries;
	unsigned long long given;          // bit i: part i is given
	uint32_t n_parts, k, pb;
	uint32_t pow2[32];                 // x^(8 * 2^i) mod P
	uint8_t gen[32 * 32];              // parity row r of the generator at gen[32 r]
};

// one block of X: thread t's 256 bytes of sum_j rows[j] * input j into acc (all-one rows by XOR), and the block's CRC in every thread
__device__ __forceinline__ uint32_t repair_block(const RepairArgs &a, unsigned long long off, const uint8_t *in, const uint8_t *row, uint32_t (&acc)[64],
                                                 CoefPlanes *s_coef, const uint32_t *s_tab, uint32_t shift, uint32_t *s_out) {
	const unsigned t = threadIdx.x;
	bool ones = true;
	for (uint32_t j = 0; j < a.k; ++j) ones &= row[j] == 1;
	if (t < a.k) coef_planes_set(s_coef[t], row[t]);
	__syncthreads();
#pragma unroll
	for (int i = 0; i < 64; ++i) acc[i] = 0;
	for (uint32_t j = 0; j < a.k; ++j) {
		const uint8_t *blk = a.part[in[j]] + off;
		if (ones) correct_read<false, 1>(blk, acc, s_coef[0], s_tab);
		else correct_read<false, 2>(blk, acc, s_coef[j], s_tab);
	}
	const uint32_t crc = block_crc(acc, s_tab, shift, s_out);
	__syncthreads();  // s_coef and s_out are re-used by the next block
	return crc;
}

struct CtaSync {
	__device__ void operator()() const { __syncthreads(); }
};

// The rule of one entry without its data (host and device): the status, and in *x the blocks to rebuild (0: the status is final).
// spare = given parts - k.  REBUILT and CORRECTED are provisional until the rebuilt blocks exist (rule 3: until their CRCs match).
LZ_HD inline int repair_rule(uint32_t bad_rows, int suspect, unsigned long long f, int spare, unsigned long long *x) {
	*x = 0;
	if (!f) {
		if (!bad_rows) return LZGPU_FIX_CLEAN;
		if (suspect < 0) return LZGPU_FIX_UNEXPLAINED;
		*x = 1ull << suspect;
		return LZGPU_FIX_CORRECTED;
	}
	if (!bad_rows) return LZGPU_FIX_CRC_ONLY;
	int n = 0;
	for (unsigned long long b = f; b; b &= b - 1) ++n;
	if (n > spare) return LZGPU_FIX_CRC_CONFLICT;
	*x = f;
	return LZGPU_FIX_REBUILT;
}

// the shared arrays of a rebuild (repair_rows' matrix and pivot, the inputs, the targets, their rows, the coefficient planes of one
// row and the CTA's CRC partials)
struct RebuildShared {
	CoefPlanes coef[32];
	uint8_t mat[32][64];
	uint8_t rows[32 * 32];
	uint8_t in[32], want[64];
	uint32_t pivot, out[8];
};

__global__ void __launch_bounds__(256) repair_map_kernel(const RepairArgs a) {
	__shared__ uint32_t s_tab[1024];
	__shared__ GfTables s_gf;
	__shared__ RebuildShared s;
	const unsigned t = threadIdx.x;
	const int spare = __popcll(a.given) - static_cast<int>(a.k);
	bool ready = false;
	uint32_t shift = 0;
	for (unsigned long long e = blockIdx.x; e < a.n_entries; e += gridDim.x) {
		const uint32_t bad_rows = a.map[2 * e];
		const int suspect = static_cast<int>(a.map[2 * e + 1]);
		const unsigned long long f = a.failed[e];
		unsigned long long x;
		int status = repair_rule(bad_rows, suspect, f, spare, &x);
		if (!x) {
			if (t == 0) a.fix[e] = lzgpu_stripe_repair{bad_rows, suspect, status, 0u, f};
			continue;
		}
		cta_setup(ready, shift, s_tab, &s_gf, a.tables, a.pow2);
		if (t == 0) {
			uint32_t ni = 0, nw = 0;
			for (uint32_t p = 0; p < a.n_parts; ++p) {
				if (!((a.given >> p) & 1ull)) continue;
				if ((x >> p) & 1ull) s.want[nw++] = static_cast<uint8_t>(p);
				else if (ni < a.k) s.in[ni++] = static_cast<uint8_t>(p);
			}
		}
		__syncthreads();
		const uint32_t nw = static_cast<uint32_t>(__popcll(x));
		const unsigned long long off = (e / a.pb) * a.part_stride + (e % a.pb) * 65536ull;
		uint32_t crc = 0;
		if (!repair_rows(a.k, a.gen, s.in, s.want, nw, s_gf, s.mat, &s.pivot, s.rows, t, 256u, CtaSync())) {
			status = f ? LZGPU_FIX_CRC_CONFLICT : LZGPU_FIX_UNEXPLAINED;  // a singular pattern: nothing rebuilt
		} else {
			uint32_t acc[64];
			bool match = true;
			for (uint32_t w = 0; w < nw && match; ++w) {
				crc = repair_block(a, off, s.in, s.rows + 32 * w, acc, s.coef, s_tab, shift, s.out);
				match = !f || crc == a.crc[s.want[w]][e];  // e = chunk * pb + block
			}
			if (!match) {
				status = LZGPU_FIX_CRC_CONFLICT;
			} else {
				block_store(a.part[s.want[nw - 1]] + off, acc);
				for (uint32_t w = 0; w + 1 < nw; ++w) {
					repair_block(a, off, s.in, s.rows + 32 * w, acc, s.coef, s_tab, shift, s.out);
					block_store(a.part[s.want[w]] + off, acc);
				}
			}
			if (f) crc = 0;  // REBUILT: the blocks match the CRCs the caller already has
		}
		if (t == 0) a.fix[e] = lzgpu_stripe_repair{bad_rows, suspect, status, status == LZGPU_FIX_CORRECTED ? crc : 0u, f};
		__syncthreads();  // s.in, s.want and s.rows are re-used by the next entry
	}
}

// lzgpu_decode_stripes: after repair_map_kernel has written every entry into a temporary, the entries it left UNEXPLAINED or
// CRC_CONFLICT are decoded up to the code's radius (decode_locate.h): with F = crc_failed and s = given - k, the code punctured by F
// (inputs: the first k given parts outside F; spares: the other given parts outside F) locates E, |E| <= 2 with 2 |E| + |F| <= s.
// Then X = F | E is rebuilt from the first k given parts outside X as repair_map_kernel rebuilds F, storing nothing until every block
// of F has matched its stored CRC.  Every other entry is copied with located = 0.
struct DecodeArgs {
	RepairArgs r;                     // the parts, CRCs, tables and generator of the repair (map, failed and fix unused)
	const lzgpu_stripe_repair *rep;   // the repair's entries
	lzgpu_stripe_decode *fix;         // one entry per repair entry
};

// Host and device: an entry of the repair that rule 2 of the decode can still serve (spare = given parts - k)
LZ_HD inline bool decode_eligible(int status, unsigned long long f, int spare) {
	int n = 0;
	for (unsigned long long b = f; b; b &= b - 1) ++n;
	if (status == LZGPU_FIX_UNEXPLAINED) return !f && spare >= 4;
	return status == LZGPU_FIX_CRC_CONFLICT && f && n + 2 <= spare;
}

__global__ void __launch_bounds__(256) decode_map_kernel(const DecodeArgs d) {
	const RepairArgs &a = d.r;
	__shared__ uint32_t s_tab[1024];
	__shared__ GfTables s_gf;
	__shared__ RebuildShared s;
	__shared__ uint8_t s_pt[64];
	__shared__ const uint8_t *s_blk[64];
	__shared__ LocateScratch s_loc;
	const unsigned t = threadIdx.x;
	const int spare = __popcll(a.given) - static_cast<int>(a.k);
	bool ready = false;
	uint32_t shift = 0;
	for (unsigned long long e = blockIdx.x; e < a.n_entries; e += gridDim.x) {
		const lzgpu_stripe_repair r = d.rep[e];
		const unsigned long long f = r.crc_failed;
		if (!decode_eligible(r.status, f, spare)) {
			if (t == 0) d.fix[e] = lzgpu_stripe_decode{r.bad_rows, r.suspect_part, r.status, r.crc, f, 0ull, {0u, 0u}};
			continue;
		}
		cta_setup(ready, shift, s_tab, &s_gf, a.tables, a.pow2);
		const unsigned long long off = (e / a.pb) * a.part_stride + (e % a.pb) * 65536ull;
		const unsigned long long kept = a.given & ~f;
		const uint32_t sp = static_cast<uint32_t>(__popcll(kept)) - a.k;
		if (t == 0) {  // the punctured code's columns: inputs, then spares
			uint32_t n = 0;
			for (uint32_t p = 0; p < a.n_parts; ++p)
				if ((kept >> p) & 1ull) {
					s_blk[n] = a.part[p] + off;
					s_pt[n++] = static_cast<uint8_t>(p);
				}
		}
		__syncthreads();
		int status = r.status;
		unsigned long long located = 0;
		uint32_t lcrc[2] = {0u, 0u};
		unsigned long long cols = 0;
		if (repair_rows(a.k, a.gen, s_pt, s_pt + a.k, sp, s_gf, s.mat, &s.pivot, s.rows, t, 256u, CtaSync()) &&
		    locate_errors(a.k, sp, s.rows, s_blk, 65536u, s_gf, s_loc, t, 256u, CtaSync(), &cols) > 0) {
			for (unsigned long long b = cols; b; b &= b - 1) located |= 1ull << s_pt[__ffsll(static_cast<long long>(b)) - 1];
			__syncthreads();  // every thread has read s_pt
			// X = F | E, F gated; E's CRCs go into the entry
			const unsigned long long x = f | located;
			if (t == 0) {
				uint32_t ni = 0, nw = 0;
				for (uint32_t p = 0; p < a.n_parts; ++p) {
					if (!((a.given >> p) & 1ull)) continue;
					if ((x >> p) & 1ull) s.want[nw++] = static_cast<uint8_t>(p);
					else if (ni < a.k) s.in[ni++] = static_cast<uint8_t>(p);
				}
			}
			__syncthreads();
			const uint32_t nw = static_cast<uint32_t>(__popcll(x));
			if (repair_rows(a.k, a.gen, s.in, s.want, nw, s_gf, s.mat, &s.pivot, s.rows, t, 256u, CtaSync())) {
				uint32_t acc[64];
				bool match = true;
				uint32_t nl = 0;
				for (uint32_t w = 0; w < nw && match; ++w) {
					const uint32_t crc = repair_block(a, off, s.in, s.rows + 32 * w, acc, s.coef, s_tab, shift, s.out);
					if ((f >> s.want[w]) & 1ull) match = crc == a.crc[s.want[w]][e];  // e = chunk * pb + block
					else if (nl++) lcrc[1] = crc;
					else lcrc[0] = crc;
				}
				if (match) {
					block_store(a.part[s.want[nw - 1]] + off, acc);
					for (uint32_t w = 0; w + 1 < nw; ++w) {
						repair_block(a, off, s.in, s.rows + 32 * w, acc, s.coef, s_tab, shift, s.out);
						block_store(a.part[s.want[w]] + off, acc);
					}
					status = LZGPU_FIX_DECODED;
				}
			}
		}
		if (status != LZGPU_FIX_DECODED) located = 0, lcrc[0] = lcrc[1] = 0;
		if (t == 0)
			d.fix[e] = lzgpu_stripe_decode{r.bad_rows, r.suspect_part, status, status == LZGPU_FIX_DECODED ? 0u : r.crc, f, located, {lcrc[0], lcrc[1]}};
		__syncthreads();  // s_pt, s_blk, s.in, s.want, s.rows and s_loc are re-used by the next entry
	}
}

}  // namespace lzd
