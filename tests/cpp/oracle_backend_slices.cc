// oracle_backend_slices.cc — TEST-ONLY stand-in for lzgpu_encode_slices, linked next to oracle_backend.cc into the CPU build of
// test_stripe_batcher_slices.cc, so that the host logic of lzgpu::StripeBatcher over several slices runs without a GPU.  One
// lzo_encode_chunk per xor/ec slice; a standard slice gets the nb data-block CRCs.  Honours the failure injection of
// oracle_backend.cc.  Never part of the product.
#include <cstdint>
#include <cstring>

#include "lzgpu.h"
#include "../../oracle/lzoracle.h"

extern "C" {

extern int lzgpu_test_fail_next_encode;  // oracle_backend.cc: the next encode call fails

int lzgpu_encode_slices(lzgpu_ctx *, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len, const uint8_t *data,
                        size_t chunk_stride, uint8_t *const *parity, const size_t *parity_stride, uint32_t *const *crc, const size_t *crc_stride) {
	if (lzgpu_test_fail_next_encode) {
		lzgpu_test_fail_next_encode = 0;
		return LZGPU_ERR_CUDA;
	}
	const uint32_t B = LZGPU_BLOCK_SIZE, nb = (chunk_len + B - 1) / B;
	for (uint32_t i = 0; i < n_slices; ++i)
		for (uint32_t c = 0; c < n_chunks; ++c) {
			const uint8_t *chunk = data + c * chunk_stride;
			if (goals[i].kind != LZGPU_KIND_STD) {
				if (lzo_encode_chunk(goals[i].kind, goals[i].k, goals[i].m, chunk, chunk_len, parity[i] + c * parity_stride[i], crc[i] + c * crc_stride[i]))
					return LZGPU_ERR_ARG;
				continue;
			}
			for (uint32_t b = 0; b < nb; ++b) {  // a trailing partial block zero-extended
				const uint32_t len = b + 1 < nb ? B : chunk_len - b * B;
				crc[i][c * crc_stride[i] + b] = lzo_crc32_zeroexpanded(0, chunk + static_cast<size_t>(b) * B, len, B - len);
			}
		}
	return LZGPU_OK;
}

}  // extern "C"
