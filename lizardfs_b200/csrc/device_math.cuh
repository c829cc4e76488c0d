// device_math.cuh — device-side GF(2^8) and CRC-32 primitives shared by every kernel.
//
// GF(2^8) bytes are processed four at a time, packed in a 32-bit register ("packed word").
// CRC-32 is handled as its GF(2)-LINEAR part only:  lin(M) = M(x) * x^32 mod P  (reflected
// representation, P = 0xEDB88320, no initial complement, no final complement).  For a message
// of n bytes  mycrc32(0, M, n) = lin(M) xor mycrc32(0, 0^n, n);  the second term is a host
// constant (lz::crc_of_zeros) — e.g. 0xD7978EEB for a 64 KiB block
// (reference: src/common/crc.cc:54-56, crc.h:27-29 `mycrc32_xorblocks` is this very identity).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

// Parity / image stores: written once, never read back by the kernel — no L1 allocation.  (-DLZ_STG_CS: the streaming cache
// operator, -DLZ_STG_PLAIN: default write-back, for A/B runs.)
#if defined(LZ_STG_CS)
#define LZ_STG "st.global.cs"
#elif defined(LZ_STG_PLAIN)
#define LZ_STG "st.global"
#else
#define LZ_STG "st.global.L1::no_allocate"
#endif

namespace lzd {

constexpr uint32_t kCrcPoly = 0xEDB88320u;
constexpr uint32_t kCrcZeroBlock64K = 0xD7978EEBu;  // mycrc32(0, 65536 zero bytes); checked at ctx creation

// ---- GF(2^8) on packed words -----------------------------------------------------------------
// multiply each of the 4 bytes by 2 (x^8 = x^4+x^3+x^2+1, reference galois_coeff.h:30-32)
__device__ __forceinline__ uint32_t gf_x2(uint32_t v) {
	const uint32_t hi = v & 0x80808080u;
	// (hi >> 7) * 0x1d without the shift: hi * 0x1d is a multiple of 128, so the high half of
	// hi * (0x1d << 25) is exactly (hi * 0x1d) >> 7  (one IMAD.HI on the otherwise idle FMA pipe)
#ifndef LZ_X2_ON_FMA
	return ((v ^ hi) << 1) ^ __umulhi(hi, 0x3A000000u);
#else
	// diagnostics: (v - hi) * 2 = v*2 + hi*(-2), the byte-lane shift as two IMADs too.  Measured slower where gf_x2 is used
	// (rows 2, 3 of ec(8,4)) — the IMAD count then matches the LOP3 count and the FMA pipe binds.
	uint32_t dbl;
	asm("{\n\t.reg .u32 t;\n\tmul.lo.u32 t, %1, 2;\n\tmad.lo.u32 %0, %2, 0xFFFFFFFE, t;\n\t}" : "=r"(dbl) : "r"(v), "r"(hi));
	return dbl ^ __umulhi(hi, 0x3A000000u);
#endif
}

// acc*2 + d with the byte-lane doubling done on the FMA pipe: (v - hi)*2 = v*2 + hi*(-2) (two IMADs),
// leaving two LOP3 (mask, final 3-input XOR) on the ALU pipe, which is the busy one in the fused kernel
__device__ __forceinline__ uint32_t gf_x2_add(uint32_t v, uint32_t d) {
	const uint32_t hi = v & 0x80808080u;
#ifdef LZ_XTIME_SHALLOW
	// dependency depth 3 (two parallel masks -> shift | mulhi -> xor3) at the price of one more ALU op
	const uint32_t lo = v & 0x7F7F7F7Fu;
	return (lo << 1) ^ __umulhi(hi, 0x3A000000u) ^ d;
#else
	uint32_t dbl;
	asm("{\n\t.reg .u32 t;\n\tmul.lo.u32 t, %1, 2;\n\tmad.lo.u32 %0, %2, 0xFFFFFFFE, t;\n\t}" : "=r"(dbl) : "r"(v), "r"(hi));
	return dbl ^ __umulhi(hi, 0x3A000000u) ^ d;
#endif
}

// acc*4 + d and acc*8 + d in one step (generator rows 2 and 3: Horner with 4^j, 8^j).  The bits shifted out are reduced with
// x^8 = 0x1d, x^9 = 0x3a, x^10 = 0x74: one mask + one IMAD.HI each ((hi7 >> 7) * 0x3a = umulhi(hi7, 0x3a << 25), and so on —
// the constants come out as 0x74000000 for x4 and 0xE8000000 for x8); the lane shift is (v - hi) * 4 = v*4 + hi*(-4) on the FMA pipe.
// ALU ops per word: 5 (x4) and 6 (x8) instead of 6 and 10 for chained doublings, same number of FMA-pipe ops.
#ifndef LZ_CHAINED_DOUBLINGS
#ifndef LZ_X4_FUSED
// x4 as two chained doublings: 4 ALU + 6 FMA-pipe ops per word instead of the 5 + 4 of the one-step form below — one ALU op less
// where the ALU pipe binds and the FMA pipe idles (measured faster for ec(5,3) and ec(6,3), ec(8,4) unchanged).  -DLZ_X4_FUSED selects the one-step form.
__device__ __forceinline__ uint32_t gf_x4_add(uint32_t v, uint32_t d) { return gf_x2_add(gf_x2_add(v, 0u), d); }
#else
__device__ __forceinline__ uint32_t gf_x4_add(uint32_t v, uint32_t d) {
	const uint32_t hi = v & 0xC0C0C0C0u;
	uint32_t lo;
	asm("{\n\t.reg .u32 t;\n\tmul.lo.u32 t, %1, 4;\n\tmad.lo.u32 %0, %2, 0xFFFFFFFC, t;\n\t}" : "=r"(lo) : "r"(v), "r"(hi));
	const uint32_t r7 = __umulhi(v & 0x80808080u, 0x74000000u);  // bit 7 -> x^9  = 0x3a
	const uint32_t r6 = __umulhi(v & 0x40404040u, 0x74000000u);  // bit 6 -> x^8  = 0x1d
	return (lo ^ r7) ^ (r6 ^ d);
}
#endif
__device__ __forceinline__ uint32_t gf_x8_add(uint32_t v, uint32_t d) {
	const uint32_t hi = v & 0xE0E0E0E0u;
	uint32_t lo;
	asm("{\n\t.reg .u32 t;\n\tmul.lo.u32 t, %1, 8;\n\tmad.lo.u32 %0, %2, 0xFFFFFFF8, t;\n\t}" : "=r"(lo) : "r"(v), "r"(hi));
	const uint32_t r7 = __umulhi(v & 0x80808080u, 0xE8000000u);  // bit 7 -> x^10 = 0x74
	const uint32_t r6 = __umulhi(v & 0x40404040u, 0xE8000000u);  // bit 6 -> x^9  = 0x3a
	const uint32_t r5 = __umulhi(v & 0x20202020u, 0xE8000000u);  // bit 5 -> x^8  = 0x1d
	return (lo ^ r7 ^ r6) ^ (r5 ^ d);
}
#else
__device__ __forceinline__ uint32_t gf_x4_add(uint32_t v, uint32_t d) { return gf_x2_add(gf_x2(v), d); }
__device__ __forceinline__ uint32_t gf_x8_add(uint32_t v, uint32_t d) { return gf_x2_add(gf_x2(gf_x2(v)), d); }
#endif

// One coefficient c prepared for the bit-plane product  c*v = XOR_b ((v >> b) & 0x01010101) * (c * 2^b):  every partial product
// is a 0/1 byte times an 8-bit constant P_b = c*2^b (in GF(2^8)), so it stays inside its byte lane (no carries).
// The shift is folded into the multiplications so that the ALU pipe only sees the mask and the final XORs:
//   x = v & (0x01010101 << b)                      bit b of every byte, in place                      (1 LOP3)
//   (x >> b) * P_b = umulhi(x, lo[b]) + x * hi[b]  with  lo[b] = (P_b mod 2^b) << (32 - b),  hi[b] = P_b >> b
// — the low b bits of P_b come down through the high half of a 64-bit product, the high 8-b bits go up in place; the two
// results occupy disjoint bits of the lane, so the addend of IMAD.HI joins them (2 ops on the FMA pipe).
// Per packed word and coefficient: 8 LOP3 (masks) + 4 LOP3 (3-input XORs) on the ALU pipe and 15 IMAD/IMAD.HI on the FMA pipe;
// some bits may use a funnel shift instead (template parameter NS below) to level the two pipes.
struct CoefPlanes {
	uint32_t lo[8];     // lo[0] = 0
	uint32_t hi[8];     // hi[0] = c
	uint32_t plane[8];  // P_b itself, for the funnel-shift form
};

// host or device: fill the planes of coefficient c (x^8 = x^4+x^3+x^2+1, reference galois_coeff.h:30-32)
__host__ __device__ inline void coef_planes_set(CoefPlanes &out, uint32_t c) {
	uint32_t v = c & 0xffu;
	for (int b = 0; b < 8; ++b) {
		out.lo[b] = b ? ((v & ((1u << b) - 1u)) << (32 - b)) : 0u;
		out.hi[b] = v >> b;
		out.plane[b] = v;
		v = ((v << 1) ^ ((v & 0x80u) ? 0x1du : 0u)) & 0xffu;
	}
}

// NS = how many of the bits 7, 6, ... use the funnel-shift form  ((v >> b) & 0x01010101) * P_b  (2 ALU + 1 FMA op; mask and
// shift are shared by every coefficient applied to the same word) instead of the in-place form (1 ALU + 2 FMA).  With R
// coefficients per input word the ALU pipe sees 8 + NS + 4R ops and the FMA pipe R(15 - NS): callers pick NS so that the two
// pipes (both one warp instruction per two cycles) are level, counting what else the kernel puts on the ALU pipe.
template <int NS>
__device__ __forceinline__ uint32_t gf_mac_term(uint32_t v, const CoefPlanes &c, int b) {
	if (b == 0) return (v & 0x01010101u) * c.hi[0];
	if (b >= 8 - NS) return ((v >> b) & 0x01010101u) * c.plane[b];
	const uint32_t x = v & (0x01010101u << b);
	uint32_t up, r;
	asm("mul.lo.u32 %0, %1, %2;" : "=r"(up) : "r"(x), "r"(c.hi[b]));
	asm("mad.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(x), "r"(c.lo[b]), "r"(up));
	return r;
}

// acc ^= c * v for one packed word
template <int NS = 2>
__device__ __forceinline__ uint32_t gf_mac(uint32_t acc, uint32_t v, const CoefPlanes &c) {
#pragma unroll
	for (int b = 0; b < 8; b += 2) acc = acc ^ gf_mac_term<NS>(v, c, b) ^ gf_mac_term<NS>(v, c, b + 1);
	return acc;
}

// ---- CRC-32 linear part ------------------------------------------------------------------------
// a * b mod P in the reflected domain (bit 31 = x^0).  32 steps; used only O(1) times per block.
__device__ __forceinline__ uint32_t crc_mulmod(uint32_t a, uint32_t b) {
	uint32_t prod = 0;
#pragma unroll 8
	for (int i = 0; i < 32; ++i) {
		prod ^= (a & 0x80000000u) ? b : 0u;
		a <<= 1;
		b = (b >> 1) ^ ((b & 1u) ? kCrcPoly : 0u);
	}
	return prod;
}

// state <- (state + w) * x^32 : absorb one little-endian 32-bit word with the 4 slicing tables
// (tab[t][v] = v * x^(32+8t) style tables built by lz::crc_make_tables; tab points to 4*256 words)
__device__ __forceinline__ uint32_t crc_step_word(uint32_t state, uint32_t w, const uint32_t *tab) {
	const uint32_t v = state ^ w;
	return tab[768 + (v & 0xff)] ^ tab[512 + ((v >> 8) & 0xff)] ^ tab[256 + ((v >> 16) & 0xff)] ^ tab[v >> 24];
}

// same, tables in global memory (read-only path; used once per 16 KiB stream by the fused kernels)
__device__ __forceinline__ uint32_t crc_step_word_ldg(uint32_t state, uint32_t w, const uint32_t *tab) {
	const uint32_t v = state ^ w;
	return __ldg(tab + 768 + (v & 0xff)) ^ __ldg(tab + 512 + ((v >> 8) & 0xff)) ^ __ldg(tab + 256 + ((v >> 16) & 0xff)) ^ __ldg(tab + (v >> 24));
}

__device__ __forceinline__ uint32_t crc_step_byte(uint32_t state, uint32_t byte, const uint32_t *tab) {
	return tab[(state ^ byte) & 0xff] ^ (state >> 8);
}

__device__ __forceinline__ uint4 ld_stream(const uint4 *p) {  // streaming 16-byte load, no L1 allocation
	uint4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
	             : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
	             : "l"(p));
	return r;
}

__device__ __forceinline__ void st_stream(uint4 *p, const uint4 &v) {
	asm volatile(LZ_STG ".v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
	             "r"(v.w)
	             : "memory");
}

}  // namespace lzd
