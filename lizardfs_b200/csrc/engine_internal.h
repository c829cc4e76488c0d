// engine_internal.h — private declarations shared by engine.cu and fused.cu
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <cstdint>
#include <mutex>
#include <utility>
#include <vector>

#include "lzgpu.h"

#define LZGPU_NOT_HANDLED 1  // internal: the fused path does not specialise this shape, use the generic kernels

void lz_set_error(const char *fmt, ...);

#define CUDA_TRY(expr)                                                                         \
	do {                                                                                       \
		cudaError_t e__ = (expr);                                                              \
		if (e__ != cudaSuccess) {                                                              \
			cudaGetLastError();                                                                \
			lz_set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(e__), __FILE__, __LINE__, \
			             cudaGetErrorString(e__));                                             \
			return LZGPU_ERR_CUDA;                                                             \
		}                                                                                      \
	} while (0)

constexpr size_t kHostTileBytes = size_t(128) << 20;  // staging tile of the host-pointer entry points
constexpr int kHostSlots = 3;                          // tiles in flight: H2D(t+1) | kernel(t) | D2H(t-1)
// Staging buffers of the HOST-pointer entry points (one set per pipeline slot; those calls hold ctx->mu).  The *_dev entry
// points never touch them: their temporaries come from the context's stream-ordered memory pool (TmpBuf below), so any
// number of threads may call *_dev functions on one context concurrently.
enum ScratchSlot {
	kScratchIn0 = 0, kScratchIn1, kScratchIn2, kScratchPar0, kScratchPar1, kScratchPar2, kScratchCrc0, kScratchCrc1, kScratchCrc2,
	kScratchOutCrc0, kScratchOutCrc1, kScratchOutCrc2,
	kScratchCount
};

struct ScratchBuf {
	void *ptr = nullptr;
	size_t size = 0;
};

struct FusedState;  // fused.cu

// per-context counters; updated from any thread
struct LzCounters {
	std::atomic<uint64_t> kernel_launches{0}, bytes_h2d{0}, bytes_d2h{0}, chunks_encoded{0}, chunks_recovered{0}, blocks_crc{0};
};

// A verification result slot: LZGPU_MAX_PARTS "first bad" words on the device and their pinned host mirror.  One slot per
// call that verifies stored CRCs (taken from a small pool, returned when the call has read its result), so concurrent calls
// never share a result word.
struct StatusSlot {
	unsigned long long *d = nullptr, *h = nullptr;
	cudaEvent_t copied = nullptr;  // recorded on the call's stream right after the copy of the words to h
	int index = -1;
};

// Owner of one verification in flight.  arm() takes a slot and sets its result words to ~0 on the call's stream; the kernels
// lower them to the first mismatch; publish_*() records how the words are encoded and copies them to the slot's pinned mirror
// on the same stream; take() decodes them once that stream has been synchronised (by the public *_dev call, by the host
// pipeline when it retires a tile, or by lzgpu_dev_sync in deferred mode) and returns the slot.  An armed owner that is
// destroyed without take() first waits for its stream, so a slot never goes back to the pool with work on it still queued.
class VerifyTicket {
public:
	VerifyTicket() = default;
	VerifyTicket(VerifyTicket &&o) noexcept { *this = std::move(o); }
	VerifyTicket &operator=(VerifyTicket &&o) noexcept;
	~VerifyTicket() { drop(); }
	bool armed() const { return slot_.index >= 0; }
	// takes a slot (the one already held, when armed) and enqueues the memset of its words to ~0 on `st`
	int arm(lzgpu_ctx *ctx, cudaStream_t st);
	unsigned long long *word(int i) const { return slot_.d + i; }  // device result word i (word(0) is nullptr when not armed)
	// fused route: one word (chunk*64 + part)*1024 + block
	int publish_fused() { return publish(true, 1, 0); }
	// one word per part (word i: part i), each chunk*blocks + block
	int publish_per_part(int n_words, uint32_t blocks) { return publish(false, n_words, blocks); }
	// after the stream has been synchronised: LZGPU_OK or LZGPU_ERR_CRC (+ first bad chunk / part / block); returns the slot
	int take(int64_t *bad);
	// waits for the stream, then take(); LZGPU_OK at once when nothing is armed
	int wait_take(int64_t *bad);
	// waits for the copy of the words (the slot's event), then take(): lzgpu_dev_sync collects a deferred verdict this way, since
	// the call that owns it may have been enqueued on another thread after the sync began, on a stream that may be gone by now
	int wait_copied_take(int64_t *bad);

private:
	int publish(bool fused, int n_words, uint32_t blocks);
	void drop();
	lzgpu_ctx *ctx_ = nullptr;
	cudaStream_t st_ = nullptr;
	StatusSlot slot_;
	bool fused_ = false;
	int n_words_ = 0;
	uint32_t blocks_ = 0;
};

// per-batch device timing (lzgpu_stats.batch_*): CUDA events recorded around the kernels of a batched call on its stream,
// resolved lazily (cudaEventQuery) when the statistics are read — the analogue of the reference's
// LOG_AVG_TILL_END_OF_SCOPE timers on this path (src/devtools/request_log.h:401-404, write_executor.cc:96)
struct TimingEntry {
	cudaEvent_t e0 = nullptr, e1 = nullptr;
	uint64_t bytes = 0;
	bool pending = false;
};
constexpr int kTimingRing = 64;

struct lzgpu_ctx {
	int device = 0;
	int sm_count = 0;
	cudaStream_t stream = nullptr;
	cudaStream_t slot_stream[kHostSlots] = {nullptr, nullptr, nullptr};
	uint32_t *d_crc_tables = nullptr;
	cudaMemPool_t pool = nullptr;            // stream-ordered temporaries of the *_dev entry points
	std::mutex slot_mu;                      // guards status_free / status_all
	std::vector<StatusSlot> status_all;
	std::vector<int> status_free;
	ScratchBuf scratch[kScratchCount];       // host-pointer entry points only (under mu)
	FusedState *fused = nullptr;
	LzCounters stats;
	std::mutex timing_mu;
	TimingEntry timing[kTimingRing];
	unsigned timing_next = 0;
	int timing_enabled = 1;
	int auto_register = 0;                   // LZGPU_AUTO_REGISTER: page-lock pageable caller buffers per host-pointer call
	uint64_t batches_timed = 0, batch_bytes_last = 0;
	double batch_ms_total = 0.0, batch_ms_last = 0.0, batch_bytes_total = 0.0;
	std::atomic<int> deferred_verify{0};     // lzgpu_ctx_set_deferred_verify: *_dev calls leave their verdict for lzgpu_dev_sync
	std::mutex pending_mu;
	std::vector<VerifyTicket> pending;       // verdicts not collected yet (deferred mode), in call order
	int64_t last_bad[3] = {-1, -1, -1};
	std::mutex mu;                           // serialises the host-pointer entry points (they share the staging slots)
};

int lz_scratch(lzgpu_ctx *ctx, int slot, size_t bytes, void **out);

// stream-ordered temporary: allocated from the context pool on `st`, released on `st` when the scope ends
struct TmpBuf {
	lzgpu_ctx *ctx;
	cudaStream_t st;
	void *p = nullptr;
	TmpBuf(lzgpu_ctx *c, cudaStream_t s) : ctx(c), st(s) {}
	TmpBuf(const TmpBuf &) = delete;
	TmpBuf &operator=(const TmpBuf &) = delete;
	~TmpBuf() {
		if (p) cudaFreeAsync(p, st);
	}
	int alloc(size_t bytes);
	void release() {
		if (p) cudaFreeAsync(p, st);
		p = nullptr;
	}
};

// scope guard for the batch timer: records the start event now and the end event + bytes at scope exit
struct BatchTimer {
	lzgpu_ctx *ctx;
	cudaStream_t st;
	int idx = -1;
	uint64_t bytes;
	BatchTimer(lzgpu_ctx *c, cudaStream_t s, uint64_t algorithmic_bytes);
	~BatchTimer();
};

// generic GF dot product descriptor (see kernels_generic.cuh DotArgs)
struct DotDesc {
	const uint8_t *src[32];
	uint8_t *const *dst;
	unsigned n_src, n_dst;
	unsigned long long total_units;
	unsigned long long src_chunk_stride, src_block_stride, dst_chunk_stride, dst_block_stride;
	unsigned units_per_block, blocks_per_chunk, valid_k, valid_nb;
};
int lz_gf_dot(lzgpu_ctx *ctx, const DotDesc &d, const uint8_t *coef, cudaStream_t st);
int lz_crc_blocks(lzgpu_ctx *ctx, const void *base, unsigned long long n_blocks, unsigned long long blocks_per_chunk,
                  unsigned long long chunk_stride, unsigned long long block_stride, uint32_t len, void *out,
                  unsigned long long out_chunk_stride, cudaStream_t st);

// fused TMA-streamed kernels (fused.cu).  Return LZGPU_NOT_HANDLED when the shape is not specialised.
int lz_fused_init(lzgpu_ctx *ctx);
void lz_fused_destroy(lzgpu_ctx *ctx);
int lz_fused_encode(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_data, size_t chunk_stride,
                    void *d_parity, size_t parity_stride, void *d_crc, size_t crc_stride, cudaStream_t st);
int lz_fused_encode_split(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_data, size_t chunk_stride,
                          void *const *d_out, size_t out_stride, void *d_crc, size_t crc_stride, cudaStream_t st);
// Fused degraded read (verify + rebuild erased data parts + chunk-order image).  When any part is verified,
// first-bad information is written to d_first_bad[0] encoded as (chunk*64 + part)*1024 + block (~0 = all good); the caller
// owns that word (a StatusSlot) and must pass it whenever d_part_crc is given.
int lz_fused_recover(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                     const void *const *d_part_crc, const uint8_t *want, void *const *d_out, void *d_chunk_out, size_t chunk_out_stride,
                     cudaStream_t st, unsigned long long *d_first_bad);
// Fused slice conversion (convert_kernel.cuh): k parts of the source slice -> every wanted part of the destination slice (d_out[i],
// nullptr = not wanted) + the destination slice's block CRCs in chunk order (nb data blocks, then m x pbd parity blocks per chunk),
// one pass; verification as in lz_fused_recover.  LZGPU_NOT_HANDLED = take the two-pass route.
int lz_fused_convert(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb, const void *const *d_parts,
                     size_t part_stride, const void *const *d_part_crc, void *const *d_out, size_t out_stride, void *d_crc, size_t crc_stride,
                     cudaStream_t st, unsigned long long *d_first_bad);
// Fused stripe check (check_kernel.cuh) of a Vandermonde / xorN goal: data parts d_parts[0..k-1] (all given), the non-NULL parity
// parts are the checked rows.  Lowers d_verdict's first_bad_stripe words (3 ints per chunk); stored-CRC mismatches as in lz_fused_recover.
// map: d_verdict is the stripe map instead (lzgpu_stripe_state[n_chunks * pb]); every entry gets its bad_rows and suspect_part = -1.
// A NULL data part (map only, lzgpu_check_stripe_map_degraded): elim = C[i][x], (R - E) x E, spare row E + i against input row x of
// the R given parity rows; bad_rows then has the bits of the spare rows only.  d_failed (map only, lzgpu_repair_stripes): one zeroed
// word per entry, in which every block that fails its stored CRC sets the bit of its part.
int lz_fused_check(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                   const void *const *d_part_crc, void *d_verdict, cudaStream_t st, unsigned long long *d_first_bad, bool map,
                   const uint8_t *elim, unsigned long long *d_failed = nullptr);
// One-pass encode for several slices (slices_kernel.cuh): parity of xor/ec slice i to d_parity[i], CRC arrays as lz_fused_encode
// writes them (the standard slice: nb data CRCs) to d_crc[i].  LZGPU_NOT_HANDLED = take the per-slice route.
int lz_fused_encode_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb, const void *d_data,
                           size_t chunk_stride, void *const *d_parity, const size_t *parity_stride, void *const *d_crc, const size_t *crc_stride,
                           cudaStream_t st);
// Recovery from the parts of every slice together (recover_slices_kernel.cuh): the one launch of lzgpu_recover_slices*, whose arguments,
// solve (shapes[0] a full combined stripe, shapes[1] the tail) and geometry the caller has checked.  d_first_bad: the armed result word
// whenever d_part_crc is given.
namespace lzd {
struct SliceLayout;
struct SliceSolve;
struct RsGeometry;
}  // namespace lzd
int lz_recover_slices(lzgpu_ctx *ctx, const lzd::SliceLayout &lay, const lzd::SliceSolve *shapes, const lzd::RsGeometry &geo, uint32_t n_chunks,
                      uint32_t nb, const void *const *d_parts, const size_t *part_stride, const void *const *d_part_crc, const uint8_t *want,
                      void *const *d_out, const size_t *out_stride, void *const *d_out_crc, void *d_image, size_t image_stride, cudaStream_t st,
                      unsigned long long *d_first_bad);
// CRC of 64 KiB blocks: block (c, b) at base + c*chunk_stride + b*65536, out[c*out_chunk_stride + b]
int lz_fused_crc(lzgpu_ctx *ctx, const void *base, unsigned long long n_blocks, unsigned long long blocks_per_chunk,
                 unsigned long long chunk_stride, void *out, unsigned long long out_chunk_stride, cudaStream_t st);
