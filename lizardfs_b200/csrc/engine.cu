// engine.cu — context management and the C ABI of liblzgpu.so (see include/lzgpu.h).
//
// Every data-path entry point ends in a CUDA kernel launch on the context's device; there is no
// CPU implementation of encode / recover / CRC in this library.  If CUDA is unusable the calls
// return LZGPU_ERR_NO_DEVICE / LZGPU_ERR_CUDA (or abort() for the void reference signatures).
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "engine_internal.h"
#include "host_math.h"
#include "correct_kernel.cuh"
#include "fused_plan.h"
#include "slices_check.h"
#include "kernels_generic.cuh"
#include "lzgpu.h"

using namespace lzd;

// ------------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------------
static thread_local char t_err[512] = "";

void lz_set_error(const char *fmt, ...) {
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(t_err, sizeof(t_err), fmt, ap);
	va_end(ap);
}

extern "C" const char *lzgpu_last_error(void) { return t_err; }

[[noreturn]] static void die(const char *what, int rc) {
	std::fprintf(stderr, "liblzgpu: FATAL: %s failed (status %d): %s\n", what, rc, t_err);
	std::abort();
}

// NVTX range around every batched entry point: the counterpart of the reference's TRACETHIS / LOG_AVG_TILL_END_OF_SCOPE
// scoped timers on this path (src/devtools/TracePrinter.h:132-146, request_log.h:401-415, e.g. write_executor.cc:96);
// visible in Nsight Systems / Compute, free when no tool is attached.
struct NvtxScope {
	explicit NvtxScope(const char *name) { nvtxRangePushA(name); }
	~NvtxScope() { nvtxRangePop(); }
};

// ------------------------------------------------------------------------------------------------
// context
// ------------------------------------------------------------------------------------------------
struct DeviceGuard {
	int prev = -1;
	explicit DeviceGuard(int dev) {
		cudaGetDevice(&prev);
		if (prev != dev) cudaSetDevice(dev);
		else prev = -1;
	}
	~DeviceGuard() {
		if (prev >= 0) cudaSetDevice(prev);
	}
};

// Pageable caller buffers: optional page-locking for the duration of one host-pointer call (LZGPU_AUTO_REGISTER=1).  Without
// it such buffers take the driver's pageable copy path; long-lived buffers are better registered once (lzgpu_host_register).
struct AutoPin {
	lzgpu_ctx *ctx;
	std::vector<void *> regs;
	explicit AutoPin(lzgpu_ctx *c) : ctx(c) {}
	AutoPin(const AutoPin &) = delete;
	AutoPin &operator=(const AutoPin &) = delete;
	void add(const void *p, size_t bytes);
	~AutoPin() {
		for (void *p : regs) cudaHostUnregister(p);
		if (!regs.empty()) cudaGetLastError();
	}
};

extern "C" int lzgpu_device_count(void) {
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) {
		cudaGetLastError();
		return 0;
	}
	return n;
}

extern "C" void lzgpu_ctx_destroy(lzgpu_ctx *ctx);

static int ctx_init_resources(lzgpu_ctx *ctx) {
	CUDA_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
	for (auto &s : ctx->slot_stream) CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
	uint32_t tabs[4][256];
	lz::crc_make_tables(tabs);
	CUDA_TRY(cudaMalloc(&ctx->d_crc_tables, sizeof(tabs)));
	CUDA_TRY(cudaMemcpy(ctx->d_crc_tables, tabs, sizeof(tabs), cudaMemcpyHostToDevice));
	{
		// stream-ordered pool for the temporaries of the *_dev entry points: kept (no trimming at synchronisation points), so a
		// steady stream of calls re-uses the same memory without touching the allocator
		cudaMemPoolProps props{};
		props.allocType = cudaMemAllocationTypePinned;
		props.handleTypes = cudaMemHandleTypeNone;
		props.location.type = cudaMemLocationTypeDevice;
		props.location.id = ctx->device;
		CUDA_TRY(cudaMemPoolCreate(&ctx->pool, &props));
		uint64_t keep = ~0ull;
		CUDA_TRY(cudaMemPoolSetAttribute(ctx->pool, cudaMemPoolAttrReleaseThreshold, &keep));
	}
	for (int i = 0; i < 8; ++i) {
		StatusSlot sl;
		CUDA_TRY(cudaMalloc(&sl.d, sizeof(unsigned long long) * LZGPU_MAX_PARTS));
		CUDA_TRY(cudaMallocHost(&sl.h, sizeof(unsigned long long) * LZGPU_MAX_PARTS));
		CUDA_TRY(cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming));
		sl.index = i;
		ctx->status_all.push_back(sl);
		ctx->status_free.push_back(i);
	}
	for (auto &t : ctx->timing) {
		CUDA_TRY(cudaEventCreate(&t.e0));
		CUDA_TRY(cudaEventCreate(&t.e1));
	}
	if (const char *e = std::getenv("LZGPU_TIMING")) ctx->timing_enabled = std::atoi(e);
	if (const char *e = std::getenv("LZGPU_AUTO_REGISTER")) ctx->auto_register = std::atoi(e);
	if (lz::crc_of_zeros(LZGPU_BLOCK_SIZE) != kCrcZeroBlock64K) {
		lz_set_error("internal: CRC constant self-check failed");
		return LZGPU_ERR_ARG;
	}
	return lz_fused_init(ctx);
}

extern "C" int lzgpu_ctx_create(int device, lzgpu_ctx **out) {
	if (!out) return LZGPU_ERR_ARG;
	*out = nullptr;
	int n = lzgpu_device_count();
	if (n <= 0) {
		lz_set_error("no CUDA device visible: liblzgpu has no CPU fallback");
		return LZGPU_ERR_NO_DEVICE;
	}
	if (device < 0 || device >= n) {
		lz_set_error("device %d out of range (0..%d)", device, n - 1);
		return LZGPU_ERR_ARG;
	}
	DeviceGuard g(device);
	cudaDeviceProp prop;
	CUDA_TRY(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9 || prop.minor != 0) {
		lz_set_error("device %d is sm_%d%d; this library only carries sm_90a code", device, prop.major, prop.minor);
		return LZGPU_ERR_NO_DEVICE;
	}
	auto *ctx = new lzgpu_ctx();
	ctx->device = device;
	ctx->sm_count = prop.multiProcessorCount;
	int rc = ctx_init_resources(ctx);
	if (rc != LZGPU_OK) {
		lzgpu_ctx_destroy(ctx);  // releases whatever was created before the failure
		return rc;
	}
	*out = ctx;
	return LZGPU_OK;
}

extern "C" void lzgpu_ctx_destroy(lzgpu_ctx *ctx) {
	if (!ctx) return;
	DeviceGuard g(ctx->device);
	cudaDeviceSynchronize();
	for (VerifyTicket &tk : ctx->pending) tk.take(nullptr);  // uncollected deferred verdicts: the device is idle, only the slots go back
	ctx->pending.clear();
	lz_fused_destroy(ctx);
	for (auto &b : ctx->scratch) if (b.ptr) cudaFree(b.ptr);
	if (ctx->d_crc_tables) cudaFree(ctx->d_crc_tables);
	for (auto &sl : ctx->status_all) {
		if (sl.d) cudaFree(sl.d);
		if (sl.h) cudaFreeHost(sl.h);
		if (sl.copied) cudaEventDestroy(sl.copied);
	}
	for (auto &t : ctx->timing) {
		if (t.e0) cudaEventDestroy(t.e0);
		if (t.e1) cudaEventDestroy(t.e1);
	}
	if (ctx->pool) cudaMemPoolDestroy(ctx->pool);
	for (auto &s : ctx->slot_stream) if (s) cudaStreamDestroy(s);
	if (ctx->stream) cudaStreamDestroy(ctx->stream);
	cudaGetLastError();
	delete ctx;
}

void AutoPin::add(const void *p, size_t bytes) {
	if (!ctx->auto_register || !p || !bytes) return;
	cudaPointerAttributes a{};
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return; }
	if (a.type != cudaMemoryTypeUnregistered) return;
	if (cudaHostRegister(const_cast<void *>(p), bytes, cudaHostRegisterDefault) == cudaSuccess) {
		regs.push_back(const_cast<void *>(p));
		static std::atomic<bool> said{false};
		if (!said.exchange(true)) std::fprintf(stderr, "liblzgpu: LZGPU_AUTO_REGISTER: page-locking pageable caller buffers per call\n");
	} else {
		cudaGetLastError();  // e.g. overlapping an existing registration: the copy falls back to the pageable path
	}
}

static std::mutex g_default_mu;
static lzgpu_ctx *g_default_ctx = nullptr;

extern "C" lzgpu_ctx *lzgpu_default_ctx(void) {
	std::lock_guard<std::mutex> lk(g_default_mu);
	if (!g_default_ctx) {
		int dev = 0;
		if (const char *e = std::getenv("LZGPU_DEVICE")) dev = std::atoi(e);
		int rc = lzgpu_ctx_create(dev, &g_default_ctx);
		if (rc != LZGPU_OK) return nullptr;
	}
	return g_default_ctx;
}

static lzgpu_ctx *need_default(const char *who) {
	lzgpu_ctx *c = lzgpu_default_ctx();
	if (!c) die(who, LZGPU_ERR_NO_DEVICE);
	return c;
}

// ---- per-batch device timing ------------------------------------------------------------------------------------
// completed entries of the event ring are folded into the totals (called with timing_mu held)
static void timing_collect(lzgpu_ctx *ctx, bool wait) {
	for (auto &t : ctx->timing) {
		if (!t.pending) continue;
		cudaError_t q = wait ? cudaEventSynchronize(t.e1) : cudaEventQuery(t.e1);
		if (q == cudaErrorNotReady) { cudaGetLastError(); continue; }
		float ms = 0.f;
		if (q == cudaSuccess && cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess) {
			ctx->batches_timed++;
			ctx->batch_ms_total += ms;
			ctx->batch_bytes_total += static_cast<double>(t.bytes);
			ctx->batch_ms_last = ms;
			ctx->batch_bytes_last = t.bytes;
		} else {
			cudaGetLastError();
		}
		t.pending = false;
	}
}

BatchTimer::BatchTimer(lzgpu_ctx *c, cudaStream_t s, uint64_t algorithmic_bytes) : ctx(c), st(s), bytes(algorithmic_bytes) {
	if (!ctx->timing_enabled) return;
	// events recorded into a stream that is being captured would become graph nodes of their own: a captured call is not timed
	cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
	if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap != cudaStreamCaptureStatusNone) { cudaGetLastError(); return; }
	std::lock_guard<std::mutex> lk(ctx->timing_mu);
	int i = static_cast<int>(ctx->timing_next % kTimingRing);
	if (ctx->timing[i].pending) {
		timing_collect(ctx, false);
		if (ctx->timing[i].pending) return;  // ring full of unfinished batches: this one goes untimed
	}
	ctx->timing_next++;
	if (cudaEventRecord(ctx->timing[i].e0, st) != cudaSuccess) { cudaGetLastError(); return; }
	idx = i;
}

BatchTimer::~BatchTimer() {
	if (idx < 0) return;
	std::lock_guard<std::mutex> lk(ctx->timing_mu);
	if (cudaEventRecord(ctx->timing[idx].e1, st) != cudaSuccess) { cudaGetLastError(); return; }
	ctx->timing[idx].bytes = bytes;
	ctx->timing[idx].pending = true;
}

extern "C" void lzgpu_get_stats(lzgpu_ctx *ctx, lzgpu_stats *out) {
	if (!ctx || !out) return;
	out->kernel_launches = ctx->stats.kernel_launches.load();
	out->bytes_h2d = ctx->stats.bytes_h2d.load();
	out->bytes_d2h = ctx->stats.bytes_d2h.load();
	out->chunks_encoded = ctx->stats.chunks_encoded.load();
	out->chunks_recovered = ctx->stats.chunks_recovered.load();
	out->blocks_crc = ctx->stats.blocks_crc.load();
	DeviceGuard g(ctx->device);
	std::lock_guard<std::mutex> lk(ctx->timing_mu);
	timing_collect(ctx, false);
	out->batches_timed = ctx->batches_timed;
	out->batch_ms_total = ctx->batch_ms_total;
	out->batch_ms_last = ctx->batch_ms_last;
	out->batch_bytes_last = ctx->batch_bytes_last;
	out->batch_gbps_last = ctx->batch_ms_last > 0.0 ? static_cast<double>(ctx->batch_bytes_last) / (ctx->batch_ms_last * 1e6) : 0.0;
	out->batch_gbps_mean = ctx->batch_ms_total > 0.0 ? ctx->batch_bytes_total / (ctx->batch_ms_total * 1e6) : 0.0;
}
extern "C" void lzgpu_reset_stats(lzgpu_ctx *ctx) {
	if (!ctx) return;
	ctx->stats.kernel_launches = 0; ctx->stats.bytes_h2d = 0; ctx->stats.bytes_d2h = 0;
	ctx->stats.chunks_encoded = 0; ctx->stats.chunks_recovered = 0; ctx->stats.blocks_crc = 0;
	DeviceGuard g(ctx->device);
	std::lock_guard<std::mutex> lk(ctx->timing_mu);
	timing_collect(ctx, true);
	ctx->batches_timed = 0; ctx->batch_ms_total = 0.0; ctx->batch_ms_last = 0.0; ctx->batch_bytes_last = 0; ctx->batch_bytes_total = 0.0;
}

// ---- temporaries and result slots of the *_dev entry points --------------------------------------------------------
int TmpBuf::alloc(size_t bytes) {
	cudaError_t e = cudaMallocFromPoolAsync(&p, bytes ? bytes : 16, ctx->pool, st);
	if (e != cudaSuccess) {
		cudaGetLastError();
		p = nullptr;
		lz_set_error("cudaMallocFromPoolAsync(%zu) failed: %s", bytes, cudaGetErrorString(e));
		return LZGPU_ERR_NOMEM;
	}
	return LZGPU_OK;
}

static int lz_status_acquire(lzgpu_ctx *ctx, StatusSlot *out) {
	std::lock_guard<std::mutex> lk(ctx->slot_mu);
	if (ctx->status_free.empty()) {
		StatusSlot sl;
		CUDA_TRY(cudaMalloc(&sl.d, sizeof(unsigned long long) * LZGPU_MAX_PARTS));
		CUDA_TRY(cudaMallocHost(&sl.h, sizeof(unsigned long long) * LZGPU_MAX_PARTS));
		CUDA_TRY(cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming));
		sl.index = static_cast<int>(ctx->status_all.size());
		ctx->status_all.push_back(sl);
		ctx->status_free.push_back(sl.index);
	}
	*out = ctx->status_all[ctx->status_free.back()];
	ctx->status_free.pop_back();
	return LZGPU_OK;
}

static void lz_status_release(lzgpu_ctx *ctx, const StatusSlot &s) {
	std::lock_guard<std::mutex> lk(ctx->slot_mu);
	ctx->status_free.push_back(s.index);
}

extern "C" int lzgpu_debug_status_slots(lzgpu_ctx *ctx, uint32_t *allocated, uint32_t *in_use) {
	if (!ctx || !allocated || !in_use) return LZGPU_ERR_ARG;
	std::lock_guard<std::mutex> lk(ctx->slot_mu);
	*allocated = static_cast<uint32_t>(ctx->status_all.size());
	*in_use = static_cast<uint32_t>(ctx->status_all.size() - ctx->status_free.size());
	return LZGPU_OK;
}

VerifyTicket &VerifyTicket::operator=(VerifyTicket &&o) noexcept {
	if (this != &o) {
		drop();
		ctx_ = o.ctx_; st_ = o.st_; slot_ = o.slot_; fused_ = o.fused_; n_words_ = o.n_words_; blocks_ = o.blocks_;
		o.slot_ = StatusSlot();
	}
	return *this;
}

int VerifyTicket::arm(lzgpu_ctx *ctx, cudaStream_t st) {
	if (!armed()) {
		int rc = lz_status_acquire(ctx, &slot_);
		if (rc) return rc;
		ctx_ = ctx;
	}
	st_ = st;
	CUDA_TRY(cudaMemsetAsync(slot_.d, 0xff, sizeof(unsigned long long) * LZGPU_MAX_PARTS, st));
	return LZGPU_OK;
}

int VerifyTicket::publish(bool fused, int n_words, uint32_t blocks) {
	fused_ = fused;
	n_words_ = n_words;
	blocks_ = blocks;
	CUDA_TRY(cudaMemcpyAsync(slot_.h, slot_.d, sizeof(unsigned long long) * n_words, cudaMemcpyDeviceToHost, st_));
	CUDA_TRY(cudaEventRecord(slot_.copied, st_));
	return LZGPU_OK;
}

int VerifyTicket::take(int64_t *bad) {
	if (!armed()) return LZGPU_OK;
	long long best_chunk = -1, best_part = -1, best_block = -1;
	if (fused_) {
		const unsigned long long v = slot_.h[0];
		if (v != ~0ull) {
			best_chunk = static_cast<long long>(v / (64ull * 1024ull));
			best_part = static_cast<long long>((v / 1024ull) % 64ull);
			best_block = static_cast<long long>(v % 1024ull);
		}
	} else {
		for (int i = 0; i < n_words_; ++i) {
			const unsigned long long v = slot_.h[i];
			if (v == ~0ull) continue;
			const long long c = static_cast<long long>(v / blocks_), b = static_cast<long long>(v % blocks_);
			if (best_chunk < 0 || c < best_chunk || (c == best_chunk && i < best_part)) { best_chunk = c; best_part = i; best_block = b; }
		}
	}
	lz_status_release(ctx_, slot_);
	slot_ = StatusSlot();
	if (best_chunk < 0) return LZGPU_OK;
	if (bad) { bad[0] = best_chunk; bad[1] = best_part; bad[2] = best_block; }
	lz_set_error("CRC mismatch: chunk %lld part %lld block %lld", best_chunk, best_part, best_block);
	return LZGPU_ERR_CRC;
}

int VerifyTicket::wait_take(int64_t *bad) {
	if (!armed()) return LZGPU_OK;
	cudaError_t e = cudaStreamSynchronize(st_);
	if (e != cudaSuccess) {
		cudaGetLastError();
		lz_set_error("CUDA error %s while waiting for the verification result", cudaGetErrorName(e));
		return LZGPU_ERR_CUDA;  // the slot goes back when the owner is destroyed
	}
	return take(bad);
}

int VerifyTicket::wait_copied_take(int64_t *bad) {
	if (!armed()) return LZGPU_OK;
	cudaError_t e = cudaEventSynchronize(slot_.copied);
	if (e != cudaSuccess) {
		cudaGetLastError();
		lz_set_error("CUDA error %s while waiting for the verification result", cudaGetErrorName(e));
		return LZGPU_ERR_CUDA;  // the slot goes back when the owner is destroyed
	}
	return take(bad);
}

void VerifyTicket::drop() {
	if (!armed()) return;
	cudaStreamSynchronize(st_);  // the memset, the compare kernels and the copy of the words must be done with the slot
	cudaGetLastError();
	lz_status_release(ctx_, slot_);
	slot_ = StatusSlot();
}

// staging buffers of the host-pointer entry points, grown on demand and kept (slot = purpose; callers hold ctx->mu)
int lz_scratch(lzgpu_ctx *ctx, int slot, size_t bytes, void **out) {
	auto &b = ctx->scratch[slot];
	if (b.size < bytes) {
		if (b.ptr) {
			CUDA_TRY(cudaDeviceSynchronize());
			CUDA_TRY(cudaFree(b.ptr));
			b.ptr = nullptr;
			b.size = 0;
		}
		size_t want = (bytes + (size_t(1) << 20) - 1) & ~((size_t(1) << 20) - 1);
		cudaError_t e = cudaMalloc(&b.ptr, want);
		if (e != cudaSuccess) {
			cudaGetLastError();
			lz_set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
			return LZGPU_ERR_NOMEM;
		}
		b.size = want;
	}
	*out = b.ptr;
	return LZGPU_OK;
}

// The tile pipeline of the host-pointer entry points: tile t of `tile` items (chunks or blocks) runs on slot t % n_slots, with
// that slot's stream and the caller's staging buffers for it, so the H2D copies of one tile overlap the kernels of the previous
// and the D2H copies of the one before.  stage(slot, first, count, stream, owner) enqueues one tile and arms `owner` when the
// tile verifies stored CRCs.  Stream order alone keeps a slot's staging buffers safe to re-use; a slot whose tile armed a
// verification is waited for and its verdict taken before the slot is re-used, and at the end every slot is retired oldest
// first, so the first CRC mismatch of the batch is the one reported (bad[0]: the chunk's index in the whole batch).  Every
// stream that was used is idle when the call returns, after an error too.  every_tile: a CRC mismatch does not stop the pipeline (the
// caller's other results are still wanted); the first one is reported once every tile has run.
template <class Stage>
static int run_tiles(lzgpu_ctx *ctx, size_t n_items, size_t tile, int n_slots, int64_t *bad, Stage &&stage, bool every_tile = false) {
	VerifyTicket tk[kHostSlots];
	size_t first[kHostSlots] = {};
	int crc_rc = LZGPU_OK;
	auto retire = [&](int s) {
		int64_t local[3];
		const int rc = tk[s].wait_take(local);
		if (rc == LZGPU_ERR_CRC && bad && !crc_rc) { bad[0] = local[0] + static_cast<int64_t>(first[s]); bad[1] = local[1]; bad[2] = local[2]; }
		if (rc == LZGPU_ERR_CRC && every_tile) {
			crc_rc = rc;
			return LZGPU_OK;
		}
		return rc;
	};
	int rc = LZGPU_OK;
	size_t t = 0;
	for (size_t i0 = 0; i0 < n_items && !rc; i0 += tile, ++t) {
		const int s = static_cast<int>(t % n_slots);
		if ((rc = retire(s))) break;
		first[s] = i0;
		rc = stage(s, i0, std::min(tile, n_items - i0), ctx->slot_stream[s], &tk[s]);
	}
	const int used = static_cast<int>(std::min<size_t>(t, n_slots));
	for (int i = 0; i < used && !rc; ++i) rc = retire(static_cast<int>((t + i) % used));
	for (int s = 0; s < used; ++s) {
		const cudaError_t e = cudaStreamSynchronize(ctx->slot_stream[s]);
		if (e != cudaSuccess && !rc) {
			lz_set_error("CUDA error %s in the host pipeline", cudaGetErrorName(e));
			rc = LZGPU_ERR_CUDA;
		}
	}
	cudaGetLastError();
	return rc ? rc : crc_rc;
}

// The given parts of a host-pointer call (parts[i] != NULL, each n_chunks x part_bytes at `stride`) and their stored CRCs (pb per
// chunk), staged tile by tile.  Device layout of a slot: the given parts packed, given part a at slot(s, a) (stride part_bytes); the
// input buffer is `width` parts wide, and the caller may put its own outputs in the slots after the given parts.
struct GivenParts {
	struct Tile {
		std::vector<const void *> dp, dc;  // per part: its staged copy / staged CRCs, nullptr when not given / without CRCs
		bool any_crc = false;
		const void *const *crcs() const { return any_crc ? dc.data() : nullptr; }
	};
	const uint8_t *const *parts;
	const uint32_t *const *crc;
	int n, n_given = 0;
	size_t stride, part_bytes;
	uint32_t pb, tile = 0;
	void *d_in[kHostSlots], *d_crc[kHostSlots];

	GivenParts(const uint8_t *const *p, const uint32_t *const *c, int n_parts, size_t part_stride, uint32_t blocks)
	    : parts(p), crc(c), n(n_parts), stride(part_stride), part_bytes(static_cast<size_t>(blocks) * LZGPU_BLOCK_SIZE), pb(blocks) {
		for (int i = 0; i < n; ++i) n_given += parts[i] ? 1 : 0;
	}
	// pins the given parts and takes the staging of n_slots slots of `tile_chunks` chunks
	int prepare(lzgpu_ctx *ctx, AutoPin &pin, uint32_t n_chunks, uint32_t tile_chunks, int n_slots, int width) {
		for (int i = 0; i < n; ++i)
			if (parts[i]) pin.add(parts[i], static_cast<size_t>(n_chunks - 1) * stride + part_bytes);
		tile = tile_chunks;
		int rc;
		for (int s = 0; s < n_slots; ++s)
			if ((rc = lz_scratch(ctx, kScratchIn0 + s, static_cast<size_t>(tile) * part_bytes * width, &d_in[s])) ||
			    (rc = lz_scratch(ctx, kScratchCrc0 + s, static_cast<size_t>(tile) * pb * 4 * std::max(n_given, 1), &d_crc[s])))
				return rc;
		return LZGPU_OK;
	}
	uint8_t *slot(int s, int a) const { return static_cast<uint8_t *>(d_in[s]) + static_cast<size_t>(a) * tile * part_bytes; }
	// copies chunks c0 .. c0 + nc - 1 of every given part and its stored CRCs to slot s
	int stage(lzgpu_ctx *ctx, int s, size_t c0, size_t nc, cudaStream_t st, Tile &t) const {
		t.dp.assign(n, nullptr);
		t.dc.assign(n, nullptr);
		for (int i = 0, a = 0; i < n; ++i) {
			if (!parts[i]) continue;
			uint8_t *dst = slot(s, a);
			CUDA_TRY(cudaMemcpy2DAsync(dst, part_bytes, parts[i] + c0 * stride, stride, part_bytes, nc, cudaMemcpyHostToDevice, st));
			ctx->stats.bytes_h2d += static_cast<uint64_t>(nc) * part_bytes;
			t.dp[i] = dst;
			if (crc && crc[i]) {
				uint8_t *cs = static_cast<uint8_t *>(d_crc[s]) + static_cast<size_t>(a) * tile * pb * 4;
				CUDA_TRY(cudaMemcpyAsync(cs, crc[i] + c0 * pb, nc * pb * 4, cudaMemcpyHostToDevice, st));
				t.dc[i] = cs;
				t.any_crc = true;
			}
			++a;
		}
		return LZGPU_OK;
	}
};

static int grid_for(const lzgpu_ctx *ctx, unsigned long long work_items, int threads, int ctas_per_sm) {
	unsigned long long need = (work_items + threads - 1) / threads;
	unsigned long long cap = static_cast<unsigned long long>(ctx->sm_count) * ctas_per_sm;
	return static_cast<int>(std::max<unsigned long long>(1, std::min(need, cap)));
}

// ------------------------------------------------------------------------------------------------
// device-level building blocks (all asynchronous on `st`)
// ------------------------------------------------------------------------------------------------
// the kernel arguments of dot-product pass r0 .. r0 + nd - 1; returns its dynamic shared memory
static size_t dot_pass_args(const DotDesc &d, const uint8_t *coef, unsigned r0, unsigned nd, DotArgs &a) {
	bool all_one = true;
	for (unsigned j = 0; j < d.n_src; ++j) a.src[j] = d.src[j];
	for (unsigned r = 0; r < nd; ++r) {
		a.dst[r] = d.dst[r0 + r];
		for (unsigned j = 0; j < d.n_src; ++j) {
			const uint8_t c = coef[(r0 + r) * d.n_src + j];
			all_one &= c == 1;
			a.coef[r * d.n_src + j] = c;  // the coefficients travel in the kernel parameters; the kernel expands them to planes
		}
	}
	a.total_units = d.total_units;
	a.src_chunk_stride = d.src_chunk_stride;
	a.src_block_stride = d.src_block_stride;
	a.dst_chunk_stride = d.dst_chunk_stride;
	a.dst_block_stride = d.dst_block_stride;
	a.units_per_block = d.units_per_block;
	a.blocks_per_chunk = d.blocks_per_chunk;
	a.n_src = d.n_src;
	a.n_dst = nd;
	a.valid_k = d.valid_k;
	a.valid_nb = d.valid_nb;
	a.pure_xor = all_one ? 1u : 0u;
	return sizeof(CoefPlanes) * nd * d.n_src;
}

// dst[r] = XOR_j coef[r][j] * src[j]  over the addressing described in DotDesc
int lz_gf_dot(lzgpu_ctx *ctx, const DotDesc &d, const uint8_t *coef /* n_dst x n_src */, cudaStream_t st) {
	if (d.n_src < 1 || d.n_src > kMaxSrc || d.n_dst < 1) return LZGPU_ERR_ARG;
	if (d.total_units == 0) return LZGPU_OK;
	for (unsigned r0 = 0; r0 < d.n_dst; r0 += kDotDests) {
		const unsigned nd = std::min<unsigned>(kDotDests, d.n_dst - r0);
		DotArgs a{};
		const size_t smem = dot_pass_args(d, coef, r0, nd, a);
		const int threads = 256;
		const int grid = grid_for(ctx, d.total_units, threads, 8);
		switch (nd) {
			case 1: gf_dot_kernel<1><<<grid, threads, smem, st>>>(a); break;
			case 2: gf_dot_kernel<2><<<grid, threads, smem, st>>>(a); break;
			case 3: gf_dot_kernel<3><<<grid, threads, smem, st>>>(a); break;
			default: gf_dot_kernel<4><<<grid, threads, smem, st>>>(a); break;
		}
		CUDA_TRY(cudaGetLastError());
		ctx->stats.kernel_launches++;
	}
	return LZGPU_OK;
}

// the same dot products compared with the stored rows d.dst[r] (read only): a 16-byte unit of chunk c, block s that differs lowers
// verdict[3c] to s (lzgpu_check_stripes, generic route; no parity-sized temporary).  map_rows (lzgpu_check_stripe_map): verdict is the
// stripe map, zeroed, and a differing dest r sets bit map_rows[r] in the bad_rows word of its block's entry.
static int lz_gf_check(lzgpu_ctx *ctx, const DotDesc &d, const uint8_t *coef, int *verdict, cudaStream_t st, const uint8_t *map_rows = nullptr) {
	for (unsigned r0 = 0; r0 < d.n_dst; r0 += kDotDests) {
		const unsigned nd = std::min<unsigned>(kDotDests, d.n_dst - r0);
		DotArgs a{};
		const size_t smem = dot_pass_args(d, coef, r0, nd, a);
		const int threads = 256;
		const int grid = grid_for(ctx, d.total_units, threads, 8);
		if (map_rows) {
			uint32_t rows = 0;
			for (unsigned r = 0; r < nd; ++r) rows |= static_cast<uint32_t>(map_rows[r0 + r]) << (8 * r);
			uint32_t *map = reinterpret_cast<uint32_t *>(verdict);
			switch (nd) {
				case 1: gf_check_map_kernel<1><<<grid, threads, smem, st>>>(a, map, rows); break;
				case 2: gf_check_map_kernel<2><<<grid, threads, smem, st>>>(a, map, rows); break;
				case 3: gf_check_map_kernel<3><<<grid, threads, smem, st>>>(a, map, rows); break;
				default: gf_check_map_kernel<4><<<grid, threads, smem, st>>>(a, map, rows); break;
			}
		} else switch (nd) {
			case 1: gf_check_kernel<1><<<grid, threads, smem, st>>>(a, verdict); break;
			case 2: gf_check_kernel<2><<<grid, threads, smem, st>>>(a, verdict); break;
			case 3: gf_check_kernel<3><<<grid, threads, smem, st>>>(a, verdict); break;
			default: gf_check_kernel<4><<<grid, threads, smem, st>>>(a, verdict); break;
		}
		CUDA_TRY(cudaGetLastError());
		ctx->stats.kernel_launches++;
	}
	return LZGPU_OK;
}

// out[c*out_chunk_stride + b] = mycrc32(0, block (c,b), len)
int lz_crc_blocks(lzgpu_ctx *ctx, const void *base, unsigned long long n_blocks, unsigned long long blocks_per_chunk,
                  unsigned long long chunk_stride, unsigned long long block_stride, uint32_t len, void *out,
                  unsigned long long out_chunk_stride, cudaStream_t st) {
	if (n_blocks == 0) return LZGPU_OK;
	if (len == 0 || (block_stride & 3) || (chunk_stride & 3) || (reinterpret_cast<uintptr_t>(base) & 3)) {
		lz_set_error("crc_blocks: len must be >= 1 and addresses 4-byte aligned");
		return LZGPU_ERR_ARG;
	}
	CrcArgs a{};
	a.base = static_cast<const uint8_t *>(base);
	a.out = static_cast<uint32_t *>(out);
	a.tables = ctx->d_crc_tables;
	a.n_blocks = n_blocks;
	a.blocks_per_chunk = blocks_per_chunk ? blocks_per_chunk : n_blocks;
	a.chunk_stride = chunk_stride;
	a.block_stride = block_stride;
	a.out_chunk_stride = out_chunk_stride;
	a.len = len;
	const unsigned n_words = len >> 2;
	a.wpl = std::max(1u, (n_words + 31) / 32);
	a.pad_words = 32 * a.wpl - n_words;
	uint32_t mult = lz::crc_xpow_bytes(4ull * a.wpl);
	for (int i = 0; i < 5; ++i) {
		a.tree_mult[i] = mult;
		mult = lz::crc_mulmod(mult, mult);
	}
	a.affine = lz::crc_of_zeros(len);
	const int threads = 256;
	const int grid = grid_for(ctx, n_blocks * 32ull, threads, 8);
	crc_blocks_kernel<<<grid, threads, 0, st>>>(a);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	ctx->stats.blocks_crc += n_blocks;
	return LZGPU_OK;
}

static int fill_crc(lzgpu_ctx *ctx, void *d_crc, size_t row_stride, size_t width, size_t rows, cudaStream_t st) {
	if (!width || !rows) return LZGPU_OK;
	fill_u32_2d_kernel<<<grid_for(ctx, width * rows, 256, 4), 256, 0, st>>>(static_cast<uint32_t *>(d_crc), row_stride, width, rows, LZGPU_FAKE_CRC);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

static int check_goal(const lzgpu_goal *g) {
	if (!lzgpu_goal_valid(g)) {
		lz_set_error("invalid goal");
		return LZGPU_ERR_ARG;
	}
	return LZGPU_OK;
}

// the context, goal and nb of a batched call (std_ok: the standard slice is a goal too, as in a conversion)
static int check_batch(const lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t nb, bool std_ok = false) {
	if (!ctx) return LZGPU_ERR_ARG;
	int rc = std_ok && slice_is_std(*goal) ? LZGPU_OK : check_goal(goal);
	if (rc) return rc;
	if (nb == 0 || nb > LZGPU_BLOCKS_IN_CHUNK) { lz_set_error("nb out of range"); return LZGPU_ERR_ARG; }
	return LZGPU_OK;
}

// Per-part pointer arrays of the recover / convert / split calls: every non-NULL buffer must be 16-byte aligned (the kernels load
// and store up to 16 bytes at a time, and a misaligned base makes the fused route's tensor maps fail), every non-NULL CRC array
// 4-byte aligned.  Checked before anything is enqueued.
static int check_part_ptrs(const char *call, const char *what, const void *const *p, int n, uintptr_t align) {
	if (!p) return LZGPU_OK;
	for (int i = 0; i < n; ++i)
		if (reinterpret_cast<uintptr_t>(p[i]) & (align - 1)) {
			lz_set_error("%s: %s[%d] is not %u-byte aligned", call, what, i, static_cast<unsigned>(align));
			return LZGPU_ERR_ARG;
		}
	return LZGPU_OK;
}

// parity coefficient rows of a goal: xorN is ec(N,1) (row of ones == plain XOR, chunk_writer.cc:373-381)
static void goal_parity_rows(const lzgpu_goal *g, uint8_t *rows /* m*k */) {
	uint8_t gen[LZGPU_MAX_PARTS * LZGPU_MAX_DATA];
	lz::rs_generator(g->k, g->m, gen);
	std::memcpy(rows, gen + g->k * g->k, static_cast<size_t>(g->m) * g->k);
}

// ------------------------------------------------------------------------------------------------
// batched encode: a chunk for one slice of its goal (lzgpu_encode_chunks*) or for several in one pass over the data
// (lzgpu_encode_slices*).  The one-goal calls are the one-slice case of the several-slice calls.
// ------------------------------------------------------------------------------------------------
// What slice g (a valid xor/ec goal, or the standard slice) holds of a chunk of nb blocks beside the data: m parity parts of pb
// blocks, none for the standard slice; so par_bytes of parity and n_crc block CRCs (nb data blocks, then m x pb parity blocks).
struct SliceShape {
	size_t m, pb, par_bytes, n_crc;
	SliceShape(const lzgpu_goal &g, size_t nb)
	    : m(slice_is_std(g) ? 0 : g.m), pb((nb + g.k - 1) / g.k), par_bytes(m * pb * LZGPU_BLOCK_SIZE), n_crc(nb + m * pb) {}
};

// SURVEY.md §8(d) over every slice, the data read once: read S, write each xor/ec slice's m*pb*B parity, write every slice's CRC array
static uint64_t slices_alg_bytes(const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len) {
	const uint64_t B = LZGPU_BLOCK_SIZE, nb = (chunk_len + B - 1) / B;
	uint64_t per_chunk = chunk_len;
	for (uint32_t i = 0; i < n_slices; ++i) {
		const SliceShape s(goals[i], nb);
		per_chunk += s.par_bytes + 4 * s.n_crc;
	}
	return n_chunks * per_chunk;
}

// The arguments of every encode call, checked before anything is enqueued and whatever n_chunks is.  dev: the device forms' rules (a
// chunk stride that holds whole blocks, since a trailing partial block is zero-extended in place; strides and buffers 16-byte
// aligned, because the kernels load and store 16 bytes at a time); else the host forms' (strides that hold the payload).
static int check_slices(const lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t chunk_len, const void *data, size_t chunk_stride,
                        const void *const *parity, const size_t *parity_stride, const void *const *crc, const size_t *crc_stride, bool dev) {
	if (!ctx || !goals || !data || !parity || !parity_stride || !crc || !crc_stride) return LZGPU_ERR_ARG;
	if (n_slices < 1 || n_slices > static_cast<uint32_t>(kSlicesMax)) { lz_set_error("encode: n_slices must be 1..%d", kSlicesMax); return LZGPU_ERR_ARG; }
	if (chunk_len == 0 || chunk_len > LZGPU_CHUNK_SIZE) { lz_set_error("chunk_len out of range"); return LZGPU_ERR_ARG; }
	const uint32_t B = LZGPU_BLOCK_SIZE, nb = (chunk_len + B - 1) / B;
	uint32_t n_striped = 0;
	for (uint32_t i = 0; i < n_slices; ++i) {
		const bool std_slice = slice_is_std(goals[i]);
		if (!std_slice && !lzgpu_goal_valid(&goals[i])) { lz_set_error("encode: goal %u is neither an xor/ec goal nor the standard slice", i); return LZGPU_ERR_ARG; }
		const SliceShape s(goals[i], nb);
		if (!crc[i] || (!std_slice && !parity[i])) { lz_set_error("encode: slice %u has no output buffer", i); return LZGPU_ERR_ARG; }
		if (crc_stride[i] < s.n_crc || (!std_slice && parity_stride[i] < s.par_bytes) ||
		    (dev && !std_slice && ((parity_stride[i] & 15) || (reinterpret_cast<uintptr_t>(parity[i]) & 15)))) {
			lz_set_error("encode: strides of slice %u too small or its parity buffer not 16-byte aligned", i);
			return LZGPU_ERR_ARG;
		}
		n_striped += std_slice ? 0 : 1;
	}
	if (n_striped == 0) { lz_set_error("encode: no xor/ec slice"); return LZGPU_ERR_ARG; }
	if (dev ? (chunk_stride < static_cast<size_t>(nb) * B || (chunk_stride & 15) || (reinterpret_cast<uintptr_t>(data) & 15)) : chunk_stride < chunk_len) {
		lz_set_error("encode: chunk stride too small or data not 16-byte aligned");
		return LZGPU_ERR_ARG;
	}
	return LZGPU_OK;
}

// One xor/ec slice of chunks of nb whole blocks: the fused route, else the generic one.  Nothing is checked, counted or filled here.
// slices_enqueue comes with the arguments check_slices took; convert_enqueue with a goal convert_check_args took, a chunk image whose
// stride and alignment it checked itself (or its own temporary) and parity / CRC temporaries it sized for this goal.
static int encode_enqueue(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_data, size_t chunk_stride,
                          void *d_parity, size_t parity_stride, void *d_crc, size_t crc_stride, cudaStream_t st) {
	int rc = lz_fused_encode(ctx, goal, n_chunks, nb, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, st);
	if (rc != LZGPU_NOT_HANDLED) return rc;
	// generic route: GF dot product over the chunk-order layout, then CRC of data and parity blocks
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const SliceShape s(*goal, nb);
	uint8_t rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
	goal_parity_rows(goal, rows);
	DotDesc d{};
	for (int j = 0; j < goal->k; ++j) d.src[j] = static_cast<const uint8_t *>(d_data) + static_cast<size_t>(j) * B;
	std::vector<uint8_t *> dst(goal->m);
	for (int r = 0; r < goal->m; ++r) dst[r] = static_cast<uint8_t *>(d_parity) + r * s.pb * B;
	d.dst = dst.data();
	d.n_src = goal->k;
	d.n_dst = goal->m;
	d.total_units = static_cast<unsigned long long>(n_chunks) * s.pb * (B / 16);
	d.src_chunk_stride = chunk_stride;
	d.src_block_stride = static_cast<unsigned long long>(goal->k) * B;
	d.dst_chunk_stride = parity_stride;
	d.dst_block_stride = B;
	d.units_per_block = B / 16;
	d.blocks_per_chunk = static_cast<unsigned>(s.pb);
	d.valid_k = goal->k;
	d.valid_nb = nb;
	if ((rc = lz_gf_dot(ctx, d, rows, st))) return rc;
	if ((rc = lz_crc_blocks(ctx, d_data, static_cast<unsigned long long>(n_chunks) * nb, nb, chunk_stride, B, B, d_crc, crc_stride, st))) return rc;
	return lz_crc_blocks(ctx, d_parity, n_chunks * s.m * s.pb, s.m * s.pb, parity_stride, B, B, static_cast<uint32_t *>(d_crc) + nb, crc_stride, st);
}

// One batch, once per call: the trailing partial block of every chunk zero-extended, then one pass over the data
// (lz_fused_encode_slices) or, where the plan refuses the set (a single xor/ec slice among the reasons), encode_enqueue per xor/ec
// slice.  Arguments checked by check_slices.
static int slices_enqueue(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len, const void *d_data,
                          size_t chunk_stride, void *const *d_parity, const size_t *parity_stride, void *const *d_crc, const size_t *crc_stride,
                          cudaStream_t st) {
	const uint32_t B = LZGPU_BLOCK_SIZE, nb = (chunk_len + B - 1) / B;
	// a trailing partial block is zero-extended to a whole block (the pad belongs to the stride)
	if (chunk_len % B) {
		CUDA_TRY(cudaMemset2DAsync(const_cast<uint8_t *>(static_cast<const uint8_t *>(d_data)) + chunk_len, chunk_stride, 0,
		                           static_cast<size_t>(nb) * B - chunk_len, n_chunks, st));
	}
	int rc = lz_fused_encode_slices(ctx, goals, n_slices, n_chunks, nb, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, st);
	int first = -1;   // the per-slice route ran: its first xor/ec slice (check_slices saw one)
	if (rc == LZGPU_NOT_HANDLED)
		for (uint32_t i = 0; i < n_slices; ++i) {
			if (slice_is_std(goals[i])) continue;
			if ((rc = encode_enqueue(ctx, &goals[i], n_chunks, nb, d_data, chunk_stride, d_parity[i], parity_stride[i], d_crc[i], crc_stride[i], st))) return rc;
			if (first < 0) first = static_cast<int>(i);
		}
	if (rc) return rc;
	ctx->stats.chunks_encoded += n_chunks;   // one count per chunk and call
	// The per-slice route computes nothing for a standard slice: its array is a copy of the first xor/ec slice's data CRCs (the same
	// bytes), or of the constant that stands there when CRCs are disabled.
	const bool per_slice = first >= 0;
	if (!lzgpu_crc_enabled())
		for (uint32_t i = 0; i < n_slices; ++i) {
			if (per_slice && slice_is_std(goals[i])) continue;
			if ((rc = fill_crc(ctx, d_crc[i], crc_stride[i], SliceShape(goals[i], nb).n_crc, n_chunks, st))) return rc;
		}
	for (uint32_t i = 0; per_slice && i < n_slices; ++i)
		if (slice_is_std(goals[i]))
			CUDA_TRY(cudaMemcpy2DAsync(d_crc[i], crc_stride[i] * 4, d_crc[first], crc_stride[first] * 4, static_cast<size_t>(nb) * 4, n_chunks,
			                           cudaMemcpyDeviceToDevice, st));
	return LZGPU_OK;
}

extern "C" int lzgpu_encode_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len,
                                        const void *d_data, size_t chunk_stride, void *const *d_parity, const size_t *parity_stride,
                                        void *const *d_crc, const size_t *crc_stride, void *stream) {
	NvtxScope nvtx_scope("lzgpu::encode_slices_dev");
	int rc = check_slices(ctx, goals, n_slices, chunk_len, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, true);
	if (rc || n_chunks == 0) return rc;
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	BatchTimer timer(ctx, st, slices_alg_bytes(goals, n_slices, n_chunks, chunk_len));
	return slices_enqueue(ctx, goals, n_slices, n_chunks, chunk_len, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, st);
}

// The one-slice case: the plan refuses a single slice, so encode_enqueue runs for it.  A standard goal has no xor/ec slice and is refused.
extern "C" int lzgpu_encode_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t chunk_len,
                                        const void *d_data, size_t chunk_stride, void *d_parity, size_t parity_stride,
                                        void *d_crc, size_t crc_stride, void *stream) {
	NvtxScope nvtx_scope("lzgpu::encode_chunks_dev");
	return lzgpu_encode_slices_dev(ctx, goal, 1, n_chunks, chunk_len, d_data, chunk_stride, &d_parity, &parity_stride, &d_crc, &crc_stride, stream);
}

extern "C" int lzgpu_encode_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len,
                                    const uint8_t *data, size_t chunk_stride, uint8_t *const *parity, const size_t *parity_stride,
                                    uint32_t *const *crc, const size_t *crc_stride) {
	NvtxScope nvtx_scope("lzgpu::encode_slices");
	int rc = check_slices(ctx, goals, n_slices, chunk_len, data, chunk_stride, reinterpret_cast<const void *const *>(parity), parity_stride,
	                      reinterpret_cast<const void *const *>(crc), crc_stride, false);
	if (rc || n_chunks == 0) return rc;
	const uint32_t B = LZGPU_BLOCK_SIZE, nb = (chunk_len + B - 1) / B;
	// device layout of a tile: the data dense; slice i's parity and CRCs dense too (the CRC stride rounded up to four words), at
	// par_off[i] / crc_off[i] per chunk of the tile
	size_t par_bytes[kSlicesMax] = {0}, n_crc[kSlicesMax] = {0}, d_crc_stride[kSlicesMax] = {0}, par_off[kSlicesMax] = {0}, crc_off[kSlicesMax] = {0};
	size_t par_total = 0, crc_total = 0;
	for (uint32_t i = 0; i < n_slices; ++i) {
		const SliceShape s(goals[i], nb);
		par_bytes[i] = s.par_bytes;
		n_crc[i] = s.n_crc;
		d_crc_stride[i] = (n_crc[i] + 3) & ~size_t(3);
		par_off[i] = par_total;
		crc_off[i] = crc_total;
		par_total += par_bytes[i];
		crc_total += d_crc_stride[i];
	}
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	AutoPin pin(ctx);
	pin.add(data, static_cast<size_t>(n_chunks - 1) * chunk_stride + chunk_len);
	for (uint32_t i = 0; i < n_slices; ++i) {
		if (par_bytes[i]) pin.add(parity[i], static_cast<size_t>(n_chunks - 1) * parity_stride[i] + par_bytes[i]);
		pin.add(crc[i], (static_cast<size_t>(n_chunks - 1) * crc_stride[i] + n_crc[i]) * 4);
	}
	const size_t d_chunk_stride = static_cast<size_t>(nb) * B;
	const uint32_t tile = std::max<uint32_t>(1, std::min<uint32_t>(n_chunks, kHostTileBytes / LZGPU_CHUNK_SIZE));
	void *d_in[kHostSlots], *d_par[kHostSlots], *d_c[kHostSlots];
	for (int s = 0; s < kHostSlots; ++s) {
		if ((rc = lz_scratch(ctx, kScratchIn0 + s, tile * d_chunk_stride, &d_in[s]))) return rc;
		if ((rc = lz_scratch(ctx, kScratchPar0 + s, tile * par_total, &d_par[s]))) return rc;
		if ((rc = lz_scratch(ctx, kScratchCrc0 + s, tile * crc_total * 4, &d_c[s]))) return rc;
	}
	return run_tiles(ctx, n_chunks, tile, kHostSlots, nullptr, [&](int s, size_t c0, size_t n, cudaStream_t st, VerifyTicket *) -> int {
		void *dp[kSlicesMax], *dc[kSlicesMax];
		for (uint32_t i = 0; i < n_slices; ++i) {
			dp[i] = static_cast<uint8_t *>(d_par[s]) + tile * par_off[i];
			dc[i] = static_cast<uint32_t *>(d_c[s]) + tile * crc_off[i];
		}
		CUDA_TRY(cudaMemcpy2DAsync(d_in[s], d_chunk_stride, data + c0 * chunk_stride, chunk_stride, chunk_len, n, cudaMemcpyHostToDevice, st));
		int rc = lzgpu_encode_slices_dev(ctx, goals, n_slices, static_cast<uint32_t>(n), chunk_len, d_in[s], d_chunk_stride, dp, par_bytes, dc,
		                                 d_crc_stride, st);
		if (rc) return rc;
		uint64_t d2h = 0;
		for (uint32_t i = 0; i < n_slices; ++i) {
			if (par_bytes[i])
				CUDA_TRY(cudaMemcpy2DAsync(parity[i] + c0 * parity_stride[i], parity_stride[i], dp[i], par_bytes[i], par_bytes[i], n, cudaMemcpyDeviceToHost, st));
			CUDA_TRY(cudaMemcpy2DAsync(crc[i] + c0 * crc_stride[i], crc_stride[i] * 4, dc[i], d_crc_stride[i] * 4, n_crc[i] * 4, n, cudaMemcpyDeviceToHost, st));
			d2h += par_bytes[i] + n_crc[i] * 4;
		}
		ctx->stats.bytes_h2d += static_cast<uint64_t>(n) * chunk_len;
		ctx->stats.bytes_d2h += static_cast<uint64_t>(n) * d2h;
		return LZGPU_OK;
	});
}

extern "C" int lzgpu_encode_chunks(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t chunk_len,
                                    const uint8_t *data, size_t chunk_stride, uint8_t *parity, size_t parity_stride,
                                    uint32_t *crc, size_t crc_stride) {
	NvtxScope nvtx_scope("lzgpu::encode_chunks");
	return lzgpu_encode_slices(ctx, goal, 1, n_chunks, chunk_len, data, chunk_stride, &parity, &parity_stride, &crc, &crc_stride);
}

// ------------------------------------------------------------------------------------------------
// batched recover
// ------------------------------------------------------------------------------------------------
static int crc_of_parts(lzgpu_ctx *ctx, const void *d_part, uint32_t n_chunks, uint32_t pb, size_t stride, void *d_out, cudaStream_t st) {
	const unsigned long long nblk = static_cast<unsigned long long>(n_chunks) * pb;
	int rc = lz_fused_crc(ctx, d_part, nblk, pb, stride, d_out, pb, st);
	if (rc == LZGPU_NOT_HANDLED) rc = lz_crc_blocks(ctx, d_part, nblk, pb, stride, LZGPU_BLOCK_SIZE, LZGPU_BLOCK_SIZE, d_out, pb, st);
	return rc;
}

// Checks the n_chunks x pb stored CRCs of one part against its blocks; the first mismatch (chunk*pb + block) lowers *d_word.
// d_tmp holds the computed CRCs.  With CRCs disabled a stored CRC is valid iff it is the constant, and the blocks are not read.
static int verify_part(lzgpu_ctx *ctx, const void *d_part, uint32_t n_chunks, uint32_t pb, size_t stride, const void *d_stored, void *d_tmp,
                       unsigned long long *d_word, cudaStream_t st) {
	const unsigned long long nblk = static_cast<unsigned long long>(n_chunks) * pb;
	if (!lzgpu_crc_enabled()) {
		crc_compare_const_kernel<<<grid_for(ctx, nblk, 256, 4), 256, 0, st>>>(static_cast<const uint32_t *>(d_stored), nblk, LZGPU_FAKE_CRC, 0, d_word);
	} else {
		int rc = crc_of_parts(ctx, d_part, n_chunks, pb, stride, d_tmp, st);
		if (rc) return rc;
		crc_compare_kernel<<<grid_for(ctx, nblk, 256, 4), 256, 0, st>>>(static_cast<const uint32_t *>(d_tmp), static_cast<const uint32_t *>(d_stored),
		                                                              nblk, kCrcZeroBlock64K, 0, 0, d_word);
	}
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

// The stored CRCs of the parts one enqueue reads: the first n_read given parts of d_parts[0 .. n-1] (the reference checks each block
// it receives, read_operation_executor.cc:257-269; a surplus part is never requested).  It decides whether they are verified, by which
// route, and how the ticket's words are encoded.  In the CRC-disabled build mode a stored CRC is valid iff it is the constant: begin()
// checks that before either route runs, and the kernels get no CRCs.  failed (lzgpu_repair_stripes, CRCs enabled): every failing block
// sets the bit of its part in its word of failed[n_chunks * pb] (zeroed here), and nothing else reports a mismatch: the result words
// are a stream-ordered temporary, no ticket is armed and nothing waits for the stream.
class InputCrcs {
public:
	InputCrcs(lzgpu_ctx *ctx, cudaStream_t st, VerifyTicket *tk, const void *const *d_parts, const void *const *d_part_crc, int n, int n_read,
	          uint32_t n_chunks, uint32_t pb, size_t stride, unsigned long long *failed = nullptr)
	    : ctx_(ctx), st_(st), tk_(tk), parts_(d_parts), crc_(d_part_crc), n_(n), n_chunks_(n_chunks), pb_(pb), stride_(stride), failed_(failed),
	      tmp_(ctx, st), words_(ctx, st) {
		for (int i = 0, used = 0; i < n && used < n_read; ++i)
			if (d_parts[i]) {
				++used;
				if (d_part_crc && d_part_crc[i]) read_ |= 1ull << i;
			}
	}
	bool any() const { return read_ != 0; }
	// arms the ticket when a part read has stored CRCs (in the CRC-disabled mode, also checks them)
	int begin() {
		if (failed_) {
			int rc = words_.alloc(sizeof(unsigned long long) * n_);
			if (rc) return rc;
			CUDA_TRY(cudaMemsetAsync(words_.p, 0xff, sizeof(unsigned long long) * n_, st_));
			CUDA_TRY(cudaMemsetAsync(failed_, 0, sizeof(unsigned long long) * n_chunks_ * pb_, st_));
			return LZGPU_OK;
		}
		if (!any()) return LZGPU_OK;
		int rc = tk_->arm(ctx_, st_);
		return (rc || lzgpu_crc_enabled()) ? rc : verify_each();
	}
	// the fused route's CRC array (nullptr: nothing left to verify) and its result word
	const void *const *for_kernels() const { return any() && lzgpu_crc_enabled() ? crc_ : nullptr; }
	unsigned long long *fused_word() const { return word(0); }
	unsigned long long *failed() const { return failed_; }
	// the generic route: every part read, part by part, before the kernels that read them
	int verify() {
		if (!for_kernels()) return LZGPU_OK;
		int rc = tmp_.alloc(static_cast<size_t>(n_chunks_) * pb_ * 4);
		return rc ? rc : verify_each();
	}
	// fused: the fused route ran with for_kernels()
	int publish(bool fused) {
		if (!any() || failed_) return LZGPU_OK;
		return fused && for_kernels() ? tk_->publish_fused() : tk_->publish_per_part(n_, pb_);
	}

private:
	unsigned long long *word(int i) const { return failed_ ? static_cast<unsigned long long *>(words_.p) + i : tk_->word(i); }
	int verify_each() {
		int rc;
		const unsigned long long nblk = static_cast<unsigned long long>(n_chunks_) * pb_;
		for (int i = 0; i < n_; ++i) {
			if (!((read_ >> i) & 1ull)) continue;
			if ((rc = verify_part(ctx_, parts_[i], n_chunks_, pb_, stride_, crc_[i], tmp_.p, word(i), st_))) return rc;
			if (!failed_) continue;
			crc_failed_kernel<<<grid_for(ctx_, nblk, 256, 4), 256, 0, st_>>>(static_cast<const uint32_t *>(tmp_.p), static_cast<const uint32_t *>(crc_[i]),
			                                                               nblk, 1ull << i, failed_);
			CUDA_TRY(cudaGetLastError());
			ctx_->stats.kernel_launches++;
		}
		return LZGPU_OK;
	}
	lzgpu_ctx *ctx_;
	cudaStream_t st_;
	VerifyTicket *tk_;
	const void *const *parts_;
	const void *const *crc_;
	int n_;
	uint32_t n_chunks_, pb_;
	size_t stride_;
	unsigned long long *failed_;
	unsigned long long read_ = 0;
	TmpBuf tmp_, words_;
};

// enqueue the whole degraded read on `st` without synchronising; *tk is armed when stored CRCs of the parts read are verified
static int recover_enqueue(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                           const void *const *d_part_crc, const uint8_t *want, void *const *d_out, void *d_chunk_out, size_t chunk_out_stride,
                           cudaStream_t st, VerifyTicket *tk) {
	const int k = goal->k, m = goal->m, n = k + m;
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const uint32_t pb = (nb + k - 1) / k;
	if (part_stride < static_cast<size_t>(pb) * B || (part_stride & 15)) { lz_set_error("recover: bad part_stride"); return LZGPU_ERR_ARG; }
	// validated before anything is enqueued: the fused route scatters the image straight from its stores
	if (d_chunk_out && (chunk_out_stride < static_cast<size_t>(nb) * B || (chunk_out_stride & 15))) {
		lz_set_error("recover: chunk_out_stride must cover nb blocks and be a multiple of 16");
		return LZGPU_ERR_ARG;
	}
	int rc;
	if ((rc = check_part_ptrs("recover", "parts", d_parts, n, 16)) || (rc = check_part_ptrs("recover", "out", d_out, n, 16)) ||
	    (rc = check_part_ptrs("recover", "part_crc", d_part_crc, n, 4)))
		return rc;
	if (reinterpret_cast<uintptr_t>(d_chunk_out) & 15) { lz_set_error("recover: chunk_out is not 16-byte aligned"); return LZGPU_ERR_ARG; }

	// ECReadPlan::recoverParts (ec_read_plan.h:126-133): the first k available parts are the inputs,
	// everything else counts as erased.
	uint8_t erased[LZGPU_MAX_PARTS] = {0}, wanted[LZGPU_MAX_PARTS] = {0};
	const uint8_t *src[LZGPU_MAX_DATA];
	int used = 0;
	for (int i = 0; i < n; ++i) {
		if (!d_parts[i] || used >= k) erased[i] = 1;
		else src[used++] = static_cast<const uint8_t *>(d_parts[i]);
	}
	if (used < k) { lz_set_error("recover: only %d of %d required parts available", used, k); return LZGPU_ERR_TOO_FEW_PARTS; }
	InputCrcs crcs(ctx, st, tk, d_parts, d_part_crc, n, k, n_chunks, pb, part_stride);
	if ((rc = crcs.begin())) return rc;

	// 0. fused route: verify + rebuild the erased data parts + chunk-order image in one pass over the inputs
	rc = lz_fused_recover(ctx, goal, n_chunks, nb, d_parts, part_stride, crcs.for_kernels(), want, d_out, d_chunk_out, chunk_out_stride, st,
	                      crcs.fused_word());
	if (rc != LZGPU_NOT_HANDLED) {
		if (rc) return rc;
		ctx->stats.chunks_recovered += n_chunks;
		return crcs.publish(true);
	}

	// 1. verify the stored CRC of every block of every part that is read
	if ((rc = crcs.verify())) return rc;

	// 2. rebuild the wanted parts
	std::vector<uint8_t *> dst;
	std::vector<void *> tmp_parts(n, nullptr);
	std::vector<std::unique_ptr<TmpBuf>> tmp_owned;
	for (int i = 0; i < n; ++i) {
		const bool need = (want[i] || (d_chunk_out && i < k)) && !d_parts[i];
		if (!need) continue;
		void *o = d_out ? d_out[i] : nullptr;
		if (!o) {
			if (!(d_chunk_out && i < k)) continue;  // not requested anywhere
			tmp_owned.emplace_back(new TmpBuf(ctx, st));
			if ((rc = tmp_owned.back()->alloc(static_cast<size_t>(n_chunks) * part_stride))) return rc;
			o = tmp_owned.back()->p;
			tmp_parts[i] = o;
		}
		wanted[i] = 1;
		dst.push_back(static_cast<uint8_t *>(o));
	}
	// parts that are available but unused (surplus) and wanted need no work: the caller already has them.
	if (!dst.empty()) {
		uint8_t rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
		bool singular = false;
		// parts marked erased only because they are surplus must not be "wanted"
		int nrows = lz::rs_recovery_matrix(k, m, erased, wanted, rows, &singular);
		if (nrows != static_cast<int>(dst.size())) {
			lz_set_error(singular ? "recover: decode matrix is singular" : "recover: bad erasure pattern");
			return LZGPU_ERR_ARG;
		}
		DotDesc d{};
		for (int j = 0; j < k; ++j) d.src[j] = src[j];
		d.dst = dst.data();
		d.n_src = k;
		d.n_dst = nrows;
		d.total_units = static_cast<unsigned long long>(n_chunks) * pb * (B / 16);
		d.src_chunk_stride = part_stride;
		d.src_block_stride = B;
		d.dst_chunk_stride = part_stride;
		d.dst_block_stride = B;
		d.units_per_block = B / 16;
		d.blocks_per_chunk = pb;
		if ((rc = lz_gf_dot(ctx, d, rows, st))) return rc;
	}

	// 3. optional chunk-order image (BlockConverter, chunk_read_planner.h:36-70)
	if (d_chunk_out) {
		GatherArgs ga{};
		for (int j = 0; j < k; ++j) {
			const void *p = d_parts[j] ? d_parts[j] : (d_out && d_out[j] ? d_out[j] : tmp_parts[j]);
			ga.part[j] = static_cast<const uint8_t *>(p);
		}
		ga.chunk_out = static_cast<uint8_t *>(d_chunk_out);
		ga.part_stride = part_stride;
		ga.chunk_out_stride = chunk_out_stride;
		ga.k = k;
		ga.nb = nb;
		ga.total_units = static_cast<unsigned long long>(n_chunks) * nb * (B / 16);
		parts_to_chunk_kernel<<<grid_for(ctx, ga.total_units, 256, 8), 256, 0, st>>>(ga);
		CUDA_TRY(cudaGetLastError());
		ctx->stats.kernel_launches++;
	}
	ctx->stats.chunks_recovered += n_chunks;
	return crcs.publish(false);
}

static int recover_check_args(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t nb, const void *parts, const uint8_t *want) {
	return !parts || !want ? LZGPU_ERR_ARG : check_batch(ctx, goal, nb);
}

static uint64_t recover_alg_bytes(const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *parts, const uint8_t *want,
                                  bool image, bool crcs) {
	// DESIGN.md §4.2: read k parts (+ their stored CRCs), write the rebuilt parts (+ the image)
	const uint64_t pb = (nb + goal->k - 1) / goal->k, B = LZGPU_BLOCK_SIZE;
	uint64_t out_parts = 0;
	for (int i = 0; i < goal->k + goal->m; ++i) out_parts += (!parts[i] && (want[i] || (image && i < goal->k))) ? 1 : 0;
	return n_chunks * (goal->k * pb * B + (crcs ? 4ull * goal->k * pb : 0) + out_parts * pb * B + (image ? static_cast<uint64_t>(nb) * B : 0));
}

// The frame of a *_dev call that may verify stored CRCs: enqueue(st, &tk) runs on the caller's stream (or the context's), timed as
// one batch of alg_bytes.  The verdict is collected by lzgpu_dev_sync in deferred mode, otherwise waited for and reported by the call
// itself (with or without `bad`) whenever stored CRCs were verified.
template <class Enqueue>
static int dev_call(lzgpu_ctx *ctx, void *stream, uint64_t alg_bytes, int64_t *bad, Enqueue &&enqueue) {
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	VerifyTicket tk;
	{
		BatchTimer timer(ctx, st, alg_bytes);
		if (int rc = enqueue(st, &tk)) return rc;
	}
	if (tk.armed() && ctx->deferred_verify.load()) {
		std::lock_guard<std::mutex> lk(ctx->pending_mu);
		ctx->pending.push_back(std::move(tk));
		return LZGPU_OK;
	}
	return tk.wait_take(bad);
}

extern "C" int lzgpu_recover_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                         const void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                                         const uint8_t *want, void *const *d_out, void *d_chunk_out, size_t chunk_out_stride,
                                         int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::recover_chunks_dev");
	int rc = recover_check_args(ctx, goal, nb, d_parts, want);
	if (rc || n_chunks == 0) return rc;
	return dev_call(ctx, stream, recover_alg_bytes(goal, n_chunks, nb, d_parts, want, d_chunk_out != nullptr, d_part_crc != nullptr), bad,
	                [&](cudaStream_t st, VerifyTicket *tk) {
		                return recover_enqueue(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, want, d_out, d_chunk_out, chunk_out_stride, st, tk);
	                });
}

extern "C" int lzgpu_recover_chunks(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                     const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                     const uint8_t *want, uint8_t *const *out, uint8_t *chunk_out, size_t chunk_out_stride,
                                     int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::recover_chunks");
	int rc = recover_check_args(ctx, goal, nb, parts, want);
	if (rc) return rc;
	if (n_chunks == 0) return LZGPU_OK;
	const int k = goal->k, n = goal->k + goal->m;
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const uint32_t pb = (nb + k - 1) / k;
	const size_t part_bytes = static_cast<size_t>(pb) * B;
	if (part_stride < part_bytes) { lz_set_error("recover: part_stride too small"); return LZGPU_ERR_ARG; }
	if (chunk_out && chunk_out_stride < static_cast<size_t>(nb) * B) { lz_set_error("recover: chunk_out_stride too small"); return LZGPU_ERR_ARG; }
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	AutoPin pin(ctx);
	for (int i = 0; i < n; ++i)
		if (!parts[i] && out && out[i] && want[i]) pin.add(out[i], static_cast<size_t>(n_chunks - 1) * part_stride + part_bytes);
	if (chunk_out) pin.add(chunk_out, static_cast<size_t>(n_chunks - 1) * chunk_out_stride + static_cast<size_t>(nb) * B);
	const uint32_t tile = static_cast<uint32_t>(std::max<size_t>(1, std::min<size_t>(n_chunks, (2 * kHostTileBytes) / (part_bytes * k))));
	void *d_img[kHostSlots] = {nullptr, nullptr, nullptr};
	const int n_slots = n_chunks > tile ? kHostSlots : 1;
	GivenParts in(parts, part_crc, n, part_stride, pb);
	if ((rc = in.prepare(ctx, pin, n_chunks, tile, n_slots, n))) return rc;  // n parts wide: the rebuilt parts follow the given ones
	for (int s = 0; s < n_slots; ++s)
		if (chunk_out && (rc = lz_scratch(ctx, kScratchPar0 + s, static_cast<size_t>(tile) * nb * B, &d_img[s]))) return rc;
	return run_tiles(ctx, n_chunks, tile, n_slots, bad, [&](int s, size_t c0, size_t nc, cudaStream_t st, VerifyTicket *tk) -> int {
		GivenParts::Tile t;
		int rc = in.stage(ctx, s, c0, nc, st, t);
		if (rc) return rc;
		std::vector<void *> dout(n, nullptr);
		for (int i = 0, a = in.n_given; i < n; ++i)
			if (!parts[i] && ((want[i] && out && out[i]) || (chunk_out && i < k))) dout[i] = in.slot(s, a++);
		{
			BatchTimer timer(ctx, st, recover_alg_bytes(goal, static_cast<uint32_t>(nc), nb, t.dp.data(), want, chunk_out != nullptr, t.any_crc));
			rc = recover_enqueue(ctx, goal, static_cast<uint32_t>(nc), nb, t.dp.data(), part_bytes, t.crcs(), want, dout.data(), d_img[s],
			                     static_cast<size_t>(nb) * B, st, tk);
		}
		if (rc) return rc;
		for (int i = 0; i < n; ++i) {
			if (dout[i] && out && out[i] && want[i] && !parts[i]) {
				CUDA_TRY(cudaMemcpy2DAsync(out[i] + c0 * part_stride, part_stride, dout[i], part_bytes, part_bytes, nc, cudaMemcpyDeviceToHost, st));
				ctx->stats.bytes_d2h += static_cast<uint64_t>(nc) * part_bytes;
			}
		}
		if (chunk_out) {
			CUDA_TRY(cudaMemcpy2DAsync(chunk_out + c0 * chunk_out_stride, chunk_out_stride, d_img[s], static_cast<size_t>(nb) * B,
			                           static_cast<size_t>(nb) * B, nc, cudaMemcpyDeviceToHost, st));
			ctx->stats.bytes_d2h += static_cast<uint64_t>(nc) * nb * B;
		}
		return LZGPU_OK;
	});
}

// ------------------------------------------------------------------------------------------------
// stripe check: do the parts of every stripe still form a codeword?
// ------------------------------------------------------------------------------------------------
// dev: device pointers, whose alignment the kernels need (the host variant stages into aligned buffers).  degraded: any part may be
// missing as long as k + 1 are given (the _degraded calls); otherwise every data part and one parity part are required.
static int check_args(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t nb, const void *const *parts, const void *const *part_crc,
                      const void *verdict, bool dev, bool degraded = false) {
	if (!parts || !verdict) return LZGPU_ERR_ARG;
	int rc = check_batch(ctx, goal, nb);
	if (rc) return rc;
	const int k = goal->k, n = goal->k + goal->m;
	int n_given = 0;
	bool any_parity = false;
	for (int i = 0; i < n; ++i) {
		if (i < k && !parts[i] && !degraded) { lz_set_error("check_stripes: data part %d is missing; every data part is required", i); return LZGPU_ERR_TOO_FEW_PARTS; }
		any_parity |= i >= k && parts[i];
		n_given += parts[i] ? 1 : 0;
	}
	if (degraded && n_given < k + 1) {
		lz_set_error("check_stripes: %d parts given; a degraded check needs k + 1 = %d (one beyond the inputs)", n_given, k + 1);
		return LZGPU_ERR_TOO_FEW_PARTS;
	}
	if (!any_parity) { lz_set_error("check_stripes: no parity part given, nothing to check"); return LZGPU_ERR_TOO_FEW_PARTS; }
	if (!dev) return LZGPU_OK;
	if ((rc = check_part_ptrs("check_stripes", "parts", parts, n, 16)) || (rc = check_part_ptrs("check_stripes", "part_crc", part_crc, n, 4))) return rc;
	if (reinterpret_cast<uintptr_t>(verdict) & 3) { lz_set_error("check_stripes: verdict is not 4-byte aligned"); return LZGPU_ERR_ARG; }
	return LZGPU_OK;
}

// enqueue the whole check on `st` (arguments validated by check_args); *tk is armed when stored CRCs are verified.  map: d_verdict is
// the stripe map (lzgpu_check_stripe_map) instead of the verdicts.  d_failed (map only, lzgpu_repair_stripes): the failing blocks of
// every stripe, one word per entry (InputCrcs), instead of the first mismatch on *tk.
static int check_enqueue(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                         const void *const *d_part_crc, void *d_verdict, cudaStream_t st, VerifyTicket *tk, bool map = false,
                         unsigned long long *d_failed = nullptr) {
	const int k = goal->k, m = goal->m, n = k + m;
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const uint32_t pb = (nb + k - 1) / k;
	if (part_stride < static_cast<size_t>(pb) * B || (part_stride & 15)) { lz_set_error("check_stripes: bad part_stride"); return LZGPU_ERR_ARG; }
	// The inputs are the first k given parts (ECReadPlan::recoverParts), the spares the given parts after them: always parity parts.
	// Each checked row is a spare against its recovery row over the inputs; with every data part given those are the data parts and
	// the generator's parity rows.  la.part[0 .. k-1] are the inputs, la.part[k + r] spare parity part r.
	LocateArgs la{};
	InputParts inputs{};
	uint8_t erased[LZGPU_MAX_PARTS] = {0}, spare[LZGPU_MAX_PARTS] = {0};
	int used = 0;
	for (int i = 0; i < n; ++i) {
		la.part[i] = static_cast<const uint8_t *>(d_parts[i]);
		if (!d_parts[i] || used >= k) erased[i] = 1;
		else inputs.part[used++] = static_cast<uint8_t>(i);
		spare[i] = erased[i] && d_parts[i];
	}
	const int lost = k - std::count_if(d_parts, d_parts + k, [](const void *p) { return p != nullptr; });
	uint8_t rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
	if (lost == 0) {
		goal_parity_rows(goal, rows);
	} else {
		bool singular = false;
		if (lz::rs_recovery_matrix(k, m, erased, spare, rows, &singular) < 1) {
			lz_set_error(singular ? "check_stripes: decode matrix is singular" : "check_stripes: bad erasure pattern");
			return LZGPU_ERR_ARG;
		}
		for (int j = 0; j < k; ++j) la.part[j] = static_cast<const uint8_t *>(d_parts[inputs.part[j]]);
	}
	for (int r = 0; r < m; ++r)
		if (spare[k + r]) {
			la.row[la.n_rows] = static_cast<uint8_t>(r);
			std::memcpy(la.coef + 32 * la.n_rows, rows + (lost ? la.n_rows : r) * k, k);  // recovery rows come in ascending part order
			++la.n_rows;
		}
	// the fused route's elimination C[i][x]: in spare i's recovery row, the coefficient of input parity part x (input k - lost + x);
	// that route takes at most three lost data parts (check_plan)
	uint8_t elim[LZGPU_MAX_PARITY * 3];
	if (lost > 0 && lost <= 3)
		for (uint32_t i = 0; i < la.n_rows; ++i)
			for (int x = 0; x < lost; ++x) elim[i * lost + x] = la.coef[32 * i + k - lost + x];

	InputCrcs crcs(ctx, st, tk, d_parts, d_part_crc, n, n, n_chunks, pb, part_stride, d_failed);  // every given part is read
	int rc = crcs.begin();
	if (rc) return rc;
	// first_bad_stripe of every chunk starts above any stripe; the check kernels lower it, locate_kernel writes the whole verdict.  The
	// fused map kernel writes every entry of the map; the generic route ORs into a zeroed one.
	const size_t map_bytes = static_cast<size_t>(n_chunks) * pb * sizeof(lzgpu_stripe_state);
	if (!map) CUDA_TRY(cudaMemsetAsync(d_verdict, 0x7f, static_cast<size_t>(n_chunks) * sizeof(lzgpu_stripe_verdict), st));

	rc = lz_fused_check(ctx, goal, n_chunks, nb, d_parts, part_stride, crcs.for_kernels(), d_verdict, st, crcs.fused_word(), map,
	                    lost ? elim : nullptr, crcs.failed());
	const bool fused = rc != LZGPU_NOT_HANDLED;
	if (fused && rc) return rc;
	if (!fused) {
		// generic route: stored CRCs part by part, then the parity rows recomputed from the data parts and compared per 16-byte unit
		if ((rc = crcs.verify())) return rc;
		uint8_t rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
		uint8_t *stored[LZGPU_MAX_PARITY];
		for (uint32_t i = 0; i < la.n_rows; ++i) {
			std::memcpy(rows + i * k, la.coef + 32 * i, k);
			stored[i] = const_cast<uint8_t *>(la.part[k + la.row[i]]);
		}
		DotDesc d{};
		for (int j = 0; j < k; ++j) d.src[j] = la.part[j];
		d.dst = stored;
		d.n_src = k;
		d.n_dst = la.n_rows;
		d.total_units = static_cast<unsigned long long>(n_chunks) * pb * (B / 16);
		d.src_chunk_stride = d.dst_chunk_stride = part_stride;
		d.src_block_stride = d.dst_block_stride = B;
		d.units_per_block = B / 16;
		d.blocks_per_chunk = pb;
		if (map) CUDA_TRY(cudaMemsetAsync(d_verdict, 0, map_bytes, st));
		if ((rc = lz_gf_check(ctx, d, rows, static_cast<int *>(d_verdict), st, map ? la.row : nullptr))) return rc;
	}
	la.verdict = static_cast<int *>(d_verdict);
	la.part_stride = part_stride;
	la.k = k;
	la.pb = pb;
	if (map) {
		const unsigned long long entries = static_cast<unsigned long long>(n_chunks) * pb;
		if (lost) locate_map_degraded_kernel<<<grid_for(ctx, entries * 256, 256, 8), 256, 0, st>>>(la, entries, inputs);
		else locate_map_kernel<<<grid_for(ctx, entries * 256, 256, 8), 256, 0, st>>>(la, entries);
	} else {
		locate_kernel<<<n_chunks, 256, 0, st>>>(la);
	}
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return crcs.publish(fused);
}

static uint64_t check_alg_bytes(const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *parts, const void *const *part_crc,
                                bool map = false) {
	// read every given part and its stored CRCs, write one verdict per chunk (the map: one state per stripe)
	const uint64_t pb = (nb + goal->k - 1) / goal->k, B = LZGPU_BLOCK_SIZE;
	uint64_t bytes = map ? pb * sizeof(lzgpu_stripe_state) : sizeof(lzgpu_stripe_verdict);
	for (int i = 0; i < goal->k + goal->m; ++i)
		if (parts[i]) bytes += pb * B + ((part_crc && part_crc[i]) ? 4 * pb : 0);
	return n_chunks * bytes;
}

static int check_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts, size_t part_stride,
                     const void *const *d_part_crc, void *d_out, int64_t *bad, void *stream, bool map, bool degraded = false) {
	int rc = check_args(ctx, goal, nb, d_parts, d_part_crc, d_out, true, degraded);
	if (rc || n_chunks == 0) return rc;
	return dev_call(ctx, stream, check_alg_bytes(goal, n_chunks, nb, d_parts, d_part_crc, map), bad, [&](cudaStream_t st, VerifyTicket *tk) {
		return check_enqueue(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_out, st, tk, map);
	});
}

extern "C" int lzgpu_check_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts,
                                       size_t part_stride, const void *const *d_part_crc, void *d_verdict, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::check_stripes_dev");
	return check_dev(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_verdict, bad, stream, false);
}

extern "C" int lzgpu_check_stripe_map_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *const *d_parts,
                                          size_t part_stride, const void *const *d_part_crc, void *d_map, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::check_stripe_map_dev");
	return check_dev(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map, bad, stream, true);
}

extern "C" int lzgpu_check_stripe_map_degraded_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                                   const void *const *d_parts, size_t part_stride, const void *const *d_part_crc, void *d_map,
                                                   int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::check_stripe_map_degraded_dev");
	return check_dev(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map, bad, stream, true, true);
}

// the host-pointer calls: out = lzgpu_stripe_verdict[n_chunks], or (map) lzgpu_stripe_state[n_chunks * pb]; failed (map only,
// lzgpu_repair_stripes): the failing blocks of every stripe, n_chunks * pb words, instead of the first mismatch
static int check_host(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *const *parts,
                      size_t part_stride, const uint32_t *const *part_crc, void *out, int64_t *bad, bool map, bool degraded = false,
                      uint64_t *failed = nullptr) {
	int rc = check_args(ctx, goal, nb, reinterpret_cast<const void *const *>(parts), nullptr, out, false, degraded);
	if (rc) return rc;
	if (n_chunks == 0) return LZGPU_OK;
	const int k = goal->k, n = goal->k + goal->m;
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const uint32_t pb = (nb + k - 1) / k;
	const size_t part_bytes = static_cast<size_t>(pb) * B;
	const size_t out_per_chunk = map ? pb * sizeof(lzgpu_stripe_state) : sizeof(lzgpu_stripe_verdict);
	const size_t failed_per_chunk = failed ? pb * sizeof(uint64_t) : 0;
	uint8_t *const out_bytes = static_cast<uint8_t *>(out);
	if (part_stride < part_bytes) { lz_set_error("check_stripes: part_stride too small"); return LZGPU_ERR_ARG; }
	GivenParts in(parts, part_crc, n, part_stride, pb);
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	AutoPin pin(ctx);
	pin.add(out, static_cast<size_t>(n_chunks) * out_per_chunk);
	if (failed) pin.add(failed, static_cast<size_t>(n_chunks) * failed_per_chunk);
	const uint32_t tile = static_cast<uint32_t>(std::max<size_t>(1, std::min<size_t>(n_chunks, (2 * kHostTileBytes) / (part_bytes * in.n_given))));
	void *d_ver[kHostSlots];
	const int n_slots = n_chunks > tile ? kHostSlots : 1;
	if ((rc = in.prepare(ctx, pin, n_chunks, tile, n_slots, in.n_given))) return rc;
	for (int s = 0; s < n_slots; ++s)
		if ((rc = lz_scratch(ctx, kScratchPar0 + s, static_cast<size_t>(tile) * (out_per_chunk + failed_per_chunk), &d_ver[s]))) return rc;
	// a stored-CRC mismatch does not stop the pipeline: every chunk gets its verdict (its map)
	rc = run_tiles(ctx, n_chunks, tile, n_slots, bad, [&](int s, size_t c0, size_t nc, cudaStream_t st, VerifyTicket *tk) -> int {
		GivenParts::Tile t;
		int rc = in.stage(ctx, s, c0, nc, st, t);
		if (rc) return rc;
		unsigned long long *d_failed = failed ? reinterpret_cast<unsigned long long *>(static_cast<uint8_t *>(d_ver[s]) + tile * out_per_chunk) : nullptr;
		{
			BatchTimer timer(ctx, st, check_alg_bytes(goal, static_cast<uint32_t>(nc), nb, t.dp.data(), t.crcs(), map));
			rc = check_enqueue(ctx, goal, static_cast<uint32_t>(nc), nb, t.dp.data(), part_bytes, t.crcs(), d_ver[s], st, tk, map, d_failed);
		}
		if (rc) return rc;
		CUDA_TRY(cudaMemcpyAsync(out_bytes + c0 * out_per_chunk, d_ver[s], nc * out_per_chunk, cudaMemcpyDeviceToHost, st));
		ctx->stats.bytes_d2h += nc * out_per_chunk;
		if (failed) {
			CUDA_TRY(cudaMemcpyAsync(failed + c0 * pb, d_failed, nc * failed_per_chunk, cudaMemcpyDeviceToHost, st));
			ctx->stats.bytes_d2h += nc * failed_per_chunk;
		}
		return LZGPU_OK;
	}, true);
	if (rc) return rc;
	if (map) {
		const lzgpu_stripe_state *e = static_cast<const lzgpu_stripe_state *>(out);
		for (size_t i = 0; i < static_cast<size_t>(n_chunks) * pb; ++i)
			if (e[i].bad_rows) {
				lz_set_error("check_stripe_map: chunk %zu stripe %zu is not a codeword", i / pb, i % pb);
				return LZGPU_ERR_INCONSISTENT;
			}
		return LZGPU_OK;
	}
	const lzgpu_stripe_verdict *verdict = static_cast<const lzgpu_stripe_verdict *>(out);
	for (uint32_t c = 0; c < n_chunks; ++c)
		if (verdict[c].first_bad_stripe >= 0) {
			lz_set_error("check_stripes: chunk %u stripe %d is not a codeword", c, verdict[c].first_bad_stripe);
			return LZGPU_ERR_INCONSISTENT;
		}
	return LZGPU_OK;
}

extern "C" int lzgpu_check_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *const *parts,
                                   size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_verdict *verdict, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::check_stripes");
	return check_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, verdict, bad, false);
}

extern "C" int lzgpu_check_stripe_map(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *const *parts,
                                      size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_state *map, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::check_stripe_map");
	return check_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, map, bad, true);
}

extern "C" int lzgpu_check_stripe_map_degraded(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                               const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                               lzgpu_stripe_state *map, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::check_stripe_map_degraded");
	return check_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, map, bad, true, true);
}

// ------------------------------------------------------------------------------------------------
// stripe correction: the stripe map, then every stripe that names a suspect rebuilt in place (correct_kernel.cuh)
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(lzgpu_stripe_fix) == 16 && sizeof(lzgpu_stripe_state) == 8, "fix and map entries as the kernels write them");

// part i and its stored CRCs into a.part[i] / a.crc[i] (nullptr: not given, no CRCs); returns the given mask, and its size in *n_given
template <class Args>
static unsigned long long fix_parts(Args &a, int n, void *const *parts, const void *const *part_crc, int *n_given = nullptr) {
	unsigned long long given = 0;
	for (int i = 0; i < n; ++i) {
		a.part[i] = static_cast<uint8_t *>(parts[i]);
		a.crc[i] = parts[i] && part_crc ? static_cast<const uint32_t *>(part_crc[i]) : nullptr;
		given |= parts[i] ? 1ull << i : 0ull;
	}
	if (n_given) *n_given = __builtin_popcountll(given);
	return given;
}

// the tail of the correction's and the repair's kernel arguments
template <class Args>
static void fix_tail(lzgpu_ctx *ctx, Args &a, unsigned long long n_entries, uint32_t pb, size_t part_stride) {
	a.tables = ctx->d_crc_tables;
	a.part_stride = part_stride;
	a.n_entries = n_entries;
	a.pb = pb;
	lz::crc_xpow2_table(a.pow2);
}

// The coefficient rows of every part that can be named (given, with k other given parts) for the parts given in `given`: the
// suspect's block from the first k given parts other than it, the inputs ECReadPlan::recoverParts picks when it is unavailable.
static int fix_table(const lzgpu_goal *goal, unsigned long long given, CorrectArgs &a) {
	const int k = goal->k, n = goal->k + goal->m;
	a.given = given;
	a.n_parts = n;
	a.k = k;
	for (int p = 0; p < n; ++p) {
		if (!((given >> p) & 1ull)) continue;
		uint8_t erased[LZGPU_MAX_PARTS] = {0}, wanted[LZGPU_MAX_PARTS] = {0}, row[LZGPU_MAX_DATA];
		int used = 0;
		for (int i = 0; i < n; ++i) {
			if (!((given >> i) & 1ull) || i == p || used >= k) erased[i] = 1;
			else ++used;
		}
		if (used < k) continue;  // never named: a suspect needs two checked rows, so k + 1 other given parts
		wanted[p] = 1;
		bool singular = false;
		if (lz::rs_recovery_matrix(k, goal->m, erased, wanted, row, &singular) != 1) {
			lz_set_error("correct_stripes: no recovery row for part %d%s", p, singular ? " (singular)" : "");
			return LZGPU_ERR_ARG;
		}
		bool ones = true;
		for (int j = 0; j < k; ++j) {
			a.coef[p][j] = row[j];
			ones &= row[j] == 1;
		}
		if (ones) a.xor_row |= 1ull << p;
	}
	return LZGPU_OK;
}

// correct_map_kernel over n_entries map entries (pb per chunk) on `st`; a carries the table (fix_table) and the part pointers.  The
// correction takes no F words (d_failed: unused).
static int fix_enqueue(lzgpu_ctx *ctx, CorrectArgs &a, unsigned long long n_entries, uint32_t pb, size_t part_stride, const void *d_map,
                       const void *d_failed, lzgpu_stripe_fix *d_fix, cudaStream_t st) {
	a.map = static_cast<const uint32_t *>(d_map);
	a.fix = d_fix;
	a.crc_disabled = lzgpu_crc_enabled() ? 0 : 1;
	fix_tail(ctx, a, n_entries, pb, part_stride);
	correct_map_kernel<<<grid_for(ctx, n_entries * 256, 256, 2), 256, 0, st>>>(a);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// stripe repair: the degraded map with every block that fails its stored CRC, then the correction's rule or those blocks rebuilt as
// erasures (repair_map_kernel, correct_kernel.cuh); stripe decode: the repair, then up to two located blocks beside the erasures
// where it gives up (decode_map_kernel)
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(lzgpu_stripe_repair) == 24 && alignof(lzgpu_stripe_repair) == 8, "repair entries as repair_map_kernel writes them");
static_assert(sizeof(lzgpu_stripe_decode) == 40 && alignof(lzgpu_stripe_decode) == 8 && offsetof(lzgpu_stripe_decode, located) == 24,
              "decode entries as decode_map_kernel writes them");

// the arguments of lzgpu_correct_stripes_degraded, and the repair's own refusals (before anything is enqueued); name: the call's
static int repair_args(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t nb, const void *const *parts, const void *const *part_crc, const void *fix,
                       bool dev, const char *name) {
	int rc = check_args(ctx, goal, nb, parts, part_crc, fix, dev, true);
	if (rc) return rc;
	if (!lzgpu_crc_enabled()) { lz_set_error("%s: CRCs are disabled, so nothing locates the blocks to rebuild", name); return LZGPU_ERR_ARG; }
	for (int i = 0; i < goal->k + goal->m; ++i)
		if (parts[i] && (!part_crc || !part_crc[i])) { lz_set_error("%s: part %d is given without stored CRCs", name, i); return LZGPU_ERR_ARG; }
	if (dev && (reinterpret_cast<uintptr_t>(fix) & 7)) { lz_set_error("%s: fix is not 8-byte aligned", name); return LZGPU_ERR_ARG; }
	return LZGPU_OK;
}

// the goal's part of the kernel arguments: the given parts and the generator's parity rows
static int fix_table(const lzgpu_goal *goal, unsigned long long given, RepairArgs &a) {
	uint8_t rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
	goal_parity_rows(goal, rows);
	for (int r = 0; r < goal->m; ++r) std::memcpy(a.gen + 32 * r, rows + r * goal->k, goal->k);
	a.given = given;
	a.n_parts = goal->k + goal->m;
	a.k = goal->k;
	return LZGPU_OK;
}

// repair_map_kernel over n_entries entries (pb per chunk) on `st`; a carries the table (fix_table) and the part and CRC pointers
static int fix_enqueue(lzgpu_ctx *ctx, RepairArgs &a, unsigned long long n_entries, uint32_t pb, size_t part_stride, const void *d_map,
                       const void *d_failed, lzgpu_stripe_repair *d_fix, cudaStream_t st) {
	a.map = static_cast<const uint32_t *>(d_map);
	a.failed = static_cast<const unsigned long long *>(d_failed);
	a.fix = d_fix;
	fix_tail(ctx, a, n_entries, pb, part_stride);
	repair_map_kernel<<<grid_for(ctx, n_entries * 256, 256, 2), 256, 0, st>>>(a);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

// lzgpu_decode_stripes: the repair into a stream-ordered temporary of repair entries, then decode_map_kernel over them
static int fix_enqueue(lzgpu_ctx *ctx, RepairArgs &a, unsigned long long n_entries, uint32_t pb, size_t part_stride, const void *d_map,
                       const void *d_failed, lzgpu_stripe_decode *d_fix, cudaStream_t st) {
	TmpBuf rep(ctx, st);
	int rc;
	if ((rc = rep.alloc(n_entries * sizeof(lzgpu_stripe_repair))) ||
	    (rc = fix_enqueue(ctx, a, n_entries, pb, part_stride, d_map, d_failed, static_cast<lzgpu_stripe_repair *>(rep.p), st)))
		return rc;
	const DecodeArgs d{a, static_cast<const lzgpu_stripe_repair *>(rep.p), d_fix};
	decode_map_kernel<<<grid_for(ctx, n_entries * 256, 256, 2), 256, 0, st>>>(d);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

// the blocks an entry says were written in place
static unsigned long long fix_written(const lzgpu_stripe_fix &f) { return f.status == LZGPU_FIX_CORRECTED ? 1ull << f.suspect_part : 0ull; }
static unsigned long long fix_written(const lzgpu_stripe_repair &f) {
	if (f.status == LZGPU_FIX_CORRECTED) return 1ull << f.suspect_part;
	return f.status == LZGPU_FIX_REBUILT ? f.crc_failed : 0ull;
}
static unsigned long long fix_written(const lzgpu_stripe_decode &f) {
	if (f.status == LZGPU_FIX_CORRECTED) return 1ull << f.suspect_part;
	return f.status == LZGPU_FIX_REBUILT || f.status == LZGPU_FIX_DECODED ? f.crc_failed | f.located : 0ull;
}

// The entry kind picks the kernel arguments, and whether the check's F words (the blocks that fail their stored CRCs) go with the map
template <class Fix>
using FixArgs = std::conditional_t<std::is_same_v<Fix, lzgpu_stripe_fix>, CorrectArgs, RepairArgs>;
template <class Fix>
constexpr bool kFixFailed = !std::is_same_v<Fix, lzgpu_stripe_fix>;

// the _dev call of the correction, the repair and the decode, after its argument check.  The repair's and the decode's check collects
// F words, so it never arms the ticket and the call never waits.
template <class Fix>
static int fix_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, void *const *d_parts, size_t part_stride,
                   const void *const *d_part_crc, void *d_fix, int64_t *bad, void *stream) {
	const uint32_t pb = (nb + goal->k - 1) / goal->k;
	const unsigned long long entries = static_cast<unsigned long long>(n_chunks) * pb;
	FixArgs<Fix> a{};
	int rc = fix_table(goal, fix_parts(a, goal->k + goal->m, d_parts, d_part_crc), a);
	if (rc) return rc;  // before anything is enqueued: no host work between check and correction
	// the map's bytes and one entry per stripe; the rewritten blocks are not counted (the host does not know them here)
	const uint64_t alg_bytes = check_alg_bytes(goal, n_chunks, nb, d_parts, d_part_crc, true) + entries * sizeof(Fix);
	return dev_call(ctx, stream, alg_bytes, bad, [&](cudaStream_t st, VerifyTicket *tk) {
		TmpBuf map(ctx, st), failed(ctx, st);  // the map kernels write 8-byte entries; the stripe kernels copy them into the fix entries
		int rc;
		if ((rc = map.alloc(entries * sizeof(lzgpu_stripe_state))) || (kFixFailed<Fix> && (rc = failed.alloc(entries * sizeof(uint64_t)))) ||
		    (rc = check_enqueue(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, map.p, st, tk, true,
		                        static_cast<unsigned long long *>(failed.p))))
			return rc;
		return fix_enqueue(ctx, a, entries, pb, part_stride, map.p, failed.p, static_cast<Fix *>(d_fix), st);
	});
}

extern "C" int lzgpu_correct_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, void *const *d_parts,
                                         size_t part_stride, const void *const *d_part_crc, void *d_fix, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::correct_stripes_dev");
	const int rc = check_args(ctx, goal, nb, d_parts, d_part_crc, d_fix, true);
	if (rc || n_chunks == 0) return rc;
	return fix_dev<lzgpu_stripe_fix>(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, bad, stream);
}

extern "C" int lzgpu_correct_stripes_degraded_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, void *const *d_parts,
                                                  size_t part_stride, const void *const *d_part_crc, void *d_fix, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::correct_stripes_degraded_dev");
	const int rc = check_args(ctx, goal, nb, d_parts, d_part_crc, d_fix, true, true);
	if (rc || n_chunks == 0) return rc;
	return fix_dev<lzgpu_stripe_fix>(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, bad, stream);
}

extern "C" int lzgpu_repair_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, void *const *d_parts,
                                        size_t part_stride, const void *const *d_part_crc, void *d_fix, void *stream) {
	NvtxScope nvtx_scope("lzgpu::repair_stripes_dev");
	const int rc = repair_args(ctx, goal, nb, d_parts, d_part_crc, d_fix, true, "repair_stripes");
	if (rc || n_chunks == 0) return rc;
	return fix_dev<lzgpu_stripe_repair>(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, nullptr, stream);
}

extern "C" int lzgpu_decode_stripes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, void *const *d_parts,
                                        size_t part_stride, const void *const *d_part_crc, void *d_fix, void *stream) {
	NvtxScope nvtx_scope("lzgpu::decode_stripes_dev");
	const int rc = repair_args(ctx, goal, nb, d_parts, d_part_crc, d_fix, true, "decode_stripes");
	if (rc || n_chunks == 0) return rc;
	return fix_dev<lzgpu_stripe_decode>(ctx, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, nullptr, stream);
}

// The host-pointer calls, phase 2: the stripes `todo` (map indices with work) gathered into one-stripe "chunks" (pb = 1: the parts
// are zero-padded, so a short last stripe has the same syndromes), tile by tile, through the kernels of the entry kind with the map
// entries (and F words) the check found; the entries go to fix[], the rewritten blocks back into the caller's parts.
template <class Fix>
static int fix_host_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t pb, uint8_t *const *parts, size_t part_stride,
                            const uint32_t *const *part_crc, const lzgpu_stripe_state *map, const uint64_t *failed,
                            const std::vector<size_t> &todo, Fix *fix) {
	const int n = goal->k + goal->m;
	const size_t B = LZGPU_BLOCK_SIZE;
	FixArgs<Fix> a{};
	int n_given;
	int rc = fix_table(goal, fix_parts(a, n, reinterpret_cast<void *const *>(parts), reinterpret_cast<const void *const *>(part_crc), &n_given), a);
	if (rc) return rc;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	const size_t tile = std::max<size_t>(1, std::min<size_t>(todo.size(), (2 * kHostTileBytes) / (B * n_given)));
	const size_t f_bytes = kFixFailed<Fix> ? sizeof(uint64_t) : 0;
	const size_t entry_bytes = sizeof(lzgpu_stripe_state) + f_bytes + sizeof(Fix);
	void *d_in, *d_crc, *d_entries;
	if ((rc = lz_scratch(ctx, kScratchIn0, tile * B * n, &d_in)) || (rc = lz_scratch(ctx, kScratchCrc0, tile * 4 * n, &d_crc)) ||
	    (rc = lz_scratch(ctx, kScratchPar0, tile * entry_bytes, &d_entries)))
		return rc;
	void *d_failed = d_entries;  // 8-byte words first: every part of d_entries stays 8-byte aligned
	void *d_fix = static_cast<uint8_t *>(d_entries) + tile * f_bytes;
	void *d_map = static_cast<uint8_t *>(d_fix) + tile * sizeof(Fix);
	for (int i = 0; i < n; ++i) {  // the staged copies: stripe j of part i at d_in + (tile i + j) B, its stored CRC at d_crc[tile i + j]
		if (a.part[i]) a.part[i] = static_cast<uint8_t *>(d_in) + tile * B * i;
		if (a.crc[i]) a.crc[i] = static_cast<const uint32_t *>(d_crc) + tile * i;
	}
	std::vector<uint32_t> h_crc(tile * n);
	std::vector<lzgpu_stripe_state> h_map(tile);
	std::vector<uint64_t> h_failed(kFixFailed<Fix> ? tile : 0);
	std::vector<Fix> h_fix(tile);
	cudaStream_t st = ctx->slot_stream[0];
	for (size_t t0 = 0; t0 < todo.size(); t0 += tile) {
		const size_t nt = std::min(tile, todo.size() - t0);
		for (size_t j = 0; j < nt; ++j) {
			const size_t e = todo[t0 + j], c = e / pb, s = e % pb;
			for (int i = 0; i < n; ++i) {
				if (!parts[i]) continue;
				CUDA_TRY(cudaMemcpyAsync(a.part[i] + j * B, parts[i] + c * part_stride + s * B, B, cudaMemcpyHostToDevice, st));
				if (a.crc[i]) h_crc[tile * i + j] = part_crc[i][e];
			}
			h_map[j] = map[e];
			if (kFixFailed<Fix>) h_failed[j] = failed[e];
		}
		ctx->stats.bytes_h2d += nt * n_given * B;
		CUDA_TRY(cudaMemcpyAsync(d_crc, h_crc.data(), tile * 4 * n, cudaMemcpyHostToDevice, st));
		CUDA_TRY(cudaMemcpyAsync(d_map, h_map.data(), nt * sizeof(lzgpu_stripe_state), cudaMemcpyHostToDevice, st));
		if (kFixFailed<Fix>) CUDA_TRY(cudaMemcpyAsync(d_failed, h_failed.data(), nt * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
		{
			BatchTimer timer(ctx, st, nt * (n_given * B + entry_bytes));
			if ((rc = fix_enqueue(ctx, a, nt, 1, B, d_map, d_failed, static_cast<Fix *>(d_fix), st))) return rc;
		}
		CUDA_TRY(cudaMemcpyAsync(h_fix.data(), d_fix, nt * sizeof(Fix), cudaMemcpyDeviceToHost, st));
		CUDA_TRY(cudaStreamSynchronize(st));
		for (size_t j = 0; j < nt; ++j) {
			const size_t e = todo[t0 + j], c = e / pb, s = e % pb;
			fix[e] = h_fix[j];
			for (unsigned long long written = fix_written(h_fix[j]); written; written &= written - 1) {
				const int p = __builtin_ctzll(written);
				CUDA_TRY(cudaMemcpyAsync(parts[p] + c * part_stride + s * B, a.part[p] + j * B, B, cudaMemcpyDeviceToHost, st));
				ctx->stats.bytes_d2h += B;
			}
		}
		CUDA_TRY(cudaStreamSynchronize(st));
	}
	return LZGPU_OK;
}

// The host-pointer calls: phase 1 maps the whole batch through the check's tile pipeline (with the F words for the repair and the
// decode), every entry gets repair_rule's status (F = 0 for the correction), and phase 2 stages the stripes with work (for the
// decode also the entries its rule 2 can still serve).  Returns the check's LZGPU_OK, LZGPU_ERR_CRC or LZGPU_ERR_INCONSISTENT, or
// the first other error.
template <class Fix>
static int fix_host(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts, size_t part_stride,
                    const uint32_t *const *part_crc, Fix *fix, int64_t *bad, bool degraded) {
	const uint32_t pb = goal && goal->k > 0 ? (nb + goal->k - 1) / goal->k : 0;
	const size_t entries = static_cast<size_t>(n_chunks) * pb;
	std::vector<lzgpu_stripe_state> map(std::max<size_t>(1, entries));
	std::vector<uint64_t> failed(kFixFailed<Fix> ? entries : 0);
	const int check_rc = check_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, map.data(), bad, true, degraded,
	                                kFixFailed<Fix> ? failed.data() : nullptr);
	if (check_rc != LZGPU_OK && check_rc != LZGPU_ERR_CRC && check_rc != LZGPU_ERR_INCONSISTENT) return check_rc;
	if (n_chunks == 0) return LZGPU_OK;
	int spare = -goal->k;
	for (int i = 0; i < goal->k + goal->m; ++i) spare += parts[i] ? 1 : 0;
	std::vector<size_t> todo;
	for (size_t e = 0; e < entries; ++e) {
		const uint64_t f = kFixFailed<Fix> ? failed[e] : 0;
		unsigned long long x;
		const int status = repair_rule(map[e].bad_rows, map[e].suspect_part, f, spare, &x);
		fix[e] = Fix{};
		fix[e].bad_rows = map[e].bad_rows;
		fix[e].suspect_part = map[e].suspect_part;
		fix[e].status = status;
		if constexpr (kFixFailed<Fix>) fix[e].crc_failed = f;
		if (x || (std::is_same_v<Fix, lzgpu_stripe_decode> && decode_eligible(status, f, spare))) todo.push_back(e);
	}
	// phase 2: only the stripes with work travel again
	int rc;
	if (!todo.empty() && (rc = fix_host_stripes(ctx, goal, pb, parts, part_stride, part_crc, map.data(), failed.data(), todo, fix))) return rc;
	return check_rc;
}

// LZGPU_ERR_INCONSISTENT with the first stripe left UNEXPLAINED ("<name>: chunk c stripe s is not a codeword and <why>"), else LZGPU_OK
template <class Fix>
static int fix_unexplained(const Fix *fix, size_t entries, uint32_t pb, const char *name, const char *why) {
	for (size_t e = 0; e < entries; ++e)
		if (fix[e].status == LZGPU_FIX_UNEXPLAINED) {
			lz_set_error("%s: chunk %zu stripe %zu is not a codeword and %s", name, e / pb, e % pb, why);
			return LZGPU_ERR_INCONSISTENT;
		}
	return LZGPU_OK;
}

static int correct_host(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts, size_t part_stride,
                        const uint32_t *const *part_crc, lzgpu_stripe_fix *fix, int64_t *bad, bool degraded) {
	if (!fix) return LZGPU_ERR_ARG;
	const int rc = fix_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, fix, bad, degraded);
	if (rc != LZGPU_OK && rc != LZGPU_ERR_INCONSISTENT) return rc;  // LZGPU_ERR_CRC: bad[0..2] and the message as the map set them
	if (n_chunks == 0) return LZGPU_OK;
	return fix_unexplained(fix, static_cast<size_t>(n_chunks) * ((nb + goal->k - 1) / goal->k), (nb + goal->k - 1) / goal->k,
	                       "correct_stripes", "no single part explains it");
}

extern "C" int lzgpu_correct_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                     size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_fix *fix, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::correct_stripes");
	return correct_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, fix, bad, false);
}

extern "C" int lzgpu_correct_stripes_degraded(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                              size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_fix *fix, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::correct_stripes_degraded");
	return correct_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, fix, bad, true);
}

// the repair's and the decode's host-pointer call: their refusals, then LZGPU_ERR_CRC for a block that still fails its stored CRC
template <class Fix>
static int repair_host(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts, size_t part_stride,
                       const uint32_t *const *part_crc, Fix *fix, const char *name, const char *why) {
	int rc = repair_args(ctx, goal, nb, reinterpret_cast<const void *const *>(parts), reinterpret_cast<const void *const *>(part_crc), fix, false, name);
	if (rc) return rc;
	if (n_chunks == 0) return LZGPU_OK;
	rc = fix_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, fix, nullptr, true);
	if (rc != LZGPU_OK && rc != LZGPU_ERR_INCONSISTENT) return rc;
	const uint32_t pb = (nb + goal->k - 1) / goal->k;
	const size_t entries = static_cast<size_t>(n_chunks) * pb;
	for (size_t e = 0; e < entries; ++e)
		if (fix[e].status == LZGPU_FIX_CRC_ONLY || fix[e].status == LZGPU_FIX_CRC_CONFLICT) {
			lz_set_error("%s: chunk %zu stripe %zu: a block still fails its stored CRC (status %d)", name, e / pb, e % pb, fix[e].status);
			return LZGPU_ERR_CRC;
		}
	return fix_unexplained(fix, entries, pb, name, why);
}

extern "C" int lzgpu_repair_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                    size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_repair *fix) {
	NvtxScope nvtx_scope("lzgpu::repair_stripes");
	return repair_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, fix, "repair_stripes", "no single part explains it");
}

extern "C" int lzgpu_decode_stripes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                    size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_decode *fix) {
	NvtxScope nvtx_scope("lzgpu::decode_stripes");
	return repair_host(ctx, goal, n_chunks, nb, parts, part_stride, part_crc, fix, "decode_stripes",
	                   "no set of parts within the code's radius explains it");
}

// ------------------------------------------------------------------------------------------------
// replication / slice-type conversion (SliceRecoveryPlanner, src/chunkserver/slice_recovery_planner.h:87-204)
// ------------------------------------------------------------------------------------------------
static bool same_goal(const lzgpu_goal *a, const lzgpu_goal *b) { return a->kind == b->kind && a->k == b->k && a->m == b->m; }

static int convert_check_args(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t nb, const void *parts, const uint8_t *want,
                              const void *out) {
	if (!ctx || !src || !dst || !parts || !want || !out) return LZGPU_ERR_ARG;
	if (!slice_is_std(*dst) && check_goal(dst)) return LZGPU_ERR_ARG;  // both goals before nb
	return check_batch(ctx, src, nb, true);
}

// The one-pass route of a slice conversion.  Handled (lz_fused_convert): sources on a Vandermonde generator with at most two data
// parts lost (their parity rows 0, 1 in use), destinations with up to three parity parts, at least one parity part wanted (data
// parts alone are BlockConverter picks, served by the degraded read + split).  LZGPU_OK: every wanted part is enqueued, *t_crc
// holds the destination slice's block CRCs in chunk order and *tk the pending verification; LZGPU_NOT_HANDLED: no part was written.
static int try_fused_convert(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb, const void *const *d_parts,
                             size_t part_stride, const void *const *d_part_crc, const uint8_t *want, void *const *d_out, size_t out_stride,
                             cudaStream_t st, VerifyTicket *tk, TmpBuf *t_crc, size_t *crc_stride_out) {
	const int ks = src->k, ns = src->k + src->m, kd = dst->k, nd = dst->k + dst->m;
	const uint32_t pbs = (nb + ks - 1) / ks, pbd = (nb + kd - 1) / kd;
	bool parity_wanted = false;
	int used = 0;
	for (int i = 0; i < ns; ++i) used += d_parts[i] ? 1 : 0;
	if (used < ks) return LZGPU_NOT_HANDLED;  // the two-pass route reports the error
	InputCrcs crcs(ctx, st, tk, d_parts, d_part_crc, ns, ks, n_chunks, pbs, part_stride);
	if (crcs.any() && !lzgpu_crc_enabled()) return LZGPU_NOT_HANDLED;  // the CRC-disabled build mode keeps its own checks
	for (int i = kd; i < nd; ++i) parity_wanted |= want[i] != 0;
	if (!parity_wanted) return LZGPU_NOT_HANDLED;
	int rc;
	{
		// the route is decided by pure host logic before anything is enqueued
		uint8_t avail[LZGPU_MAX_PARTS] = {0};
		for (int i = 0; i < ns; ++i) avail[i] = d_parts[i] ? 1 : 0;
		lzgpu_convert_plan plan;
		if (lzgpu_plan_convert(src, dst, avail, want, &plan) != LZGPU_OK || !plan.one_pass) return LZGPU_NOT_HANDLED;
	}
	const size_t crc_stride = (nb + static_cast<size_t>(dst->m) * pbd + 3) & ~size_t(3);
	if ((rc = t_crc->alloc(n_chunks * crc_stride * 4)) || (rc = crcs.begin())) return rc;
	void *outs[LZGPU_MAX_PARTS] = {nullptr};
	for (int i = 0; i < nd; ++i) outs[i] = want[i] ? d_out[i] : nullptr;
	rc = lz_fused_convert(ctx, src, dst, n_chunks, nb, d_parts, part_stride, crcs.for_kernels(), outs, out_stride, t_crc->p, crc_stride, st,
	                      crcs.fused_word());
	if (rc != LZGPU_OK) {
		// (a launch-time refusal — misaligned part pointers, a tensor map the driver rejects: rare)  The two-pass route re-arms the
		// slot it already holds
		t_crc->release();
		return rc;
	}
	if ((rc = crcs.publish(true))) return rc;
	*crc_stride_out = crc_stride;
	ctx->stats.chunks_recovered += n_chunks;
	ctx->stats.chunks_encoded += n_chunks;
	return LZGPU_OK;
}

static int convert_enqueue(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                           const void *const *d_parts, size_t part_stride, const void *const *d_part_crc, const uint8_t *want,
                           void *const *d_out, size_t out_stride, void *const *d_out_crc, cudaStream_t st, VerifyTicket *tk) {
	int rc;
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const int ks = src->k, kd = dst->k, nd = dst->k + dst->m;
	const uint32_t pbs = (nb + ks - 1) / ks, pbd = (nb + kd - 1) / kd;
	if (part_stride < static_cast<size_t>(pbs) * B || (part_stride & 15) || out_stride < static_cast<size_t>(pbd) * B || (out_stride & 15)) {
		lz_set_error("convert: strides too small or not multiples of 16");
		return LZGPU_ERR_ARG;
	}
	const int ns = src->k + src->m;
	if ((rc = check_part_ptrs("convert", "parts", d_parts, ns, 16)) || (rc = check_part_ptrs("convert", "out", d_out, nd, 16)) ||
	    (rc = check_part_ptrs("convert", "part_crc", d_part_crc, ns, 4)) || (rc = check_part_ptrs("convert", "out_crc", d_out_crc, nd, 4)))
		return rc;
	for (int i = 0; i < nd; ++i)
		if (want[i] && !d_out[i]) { lz_set_error("convert: wanted part %d has no output buffer", i); return LZGPU_ERR_ARG; }
	TmpBuf t_image(ctx, st), t_par(ctx, st), t_crc(ctx, st);
	void *d_encode_crc = nullptr;  // CRC array of the destination-slice encode, when that ran
	size_t encode_crc_stride = 0;

	if (same_goal(src, dst) && !slice_is_std(*src)) {
		// kReadDataPart (slice_recovery_planner.h:98-101): the part is read, or rebuilt from k parts of the same slice
		uint8_t need[LZGPU_MAX_PARTS] = {0};
		bool any = false;
		for (int i = 0; i < nd; ++i) {
			if (!want[i]) continue;
			if (d_parts[i]) {
				if (d_parts[i] != d_out[i])
					CUDA_TRY(cudaMemcpy2DAsync(d_out[i], out_stride, d_parts[i], part_stride, static_cast<size_t>(pbd) * B, n_chunks, cudaMemcpyDeviceToDevice, st));
			} else {
				need[i] = 1;
				any = true;
			}
		}
		if (any || d_part_crc) {
			if (any && out_stride != part_stride) { lz_set_error("convert: same-slice rebuild needs out_stride == part_stride"); return LZGPU_ERR_ARG; }
			if ((rc = recover_enqueue(ctx, src, n_chunks, nb, d_parts, part_stride, d_part_crc, need, d_out, nullptr, 0, st, tk))) return rc;
		}
	} else {
		// kRecoverDataPart / kRecoverParityPart (:102-119): chunk data first (ChunkReadPlanner), then BlockConverter or RecoverParity
		const uint8_t *image = nullptr;
		size_t image_stride = 0;
		bool converted = false;   // the one-pass route produced every wanted destination part
		void *direct_image = (slice_is_std(*dst) && want[0]) ? d_out[0] : nullptr;  // a standard destination IS the chunk image
		if (slice_is_std(*src)) {
			if (!d_parts[0]) { lz_set_error("convert: the standard chunk is not available"); return LZGPU_ERR_TOO_FEW_PARTS; }
			image = static_cast<const uint8_t *>(d_parts[0]);
			image_stride = part_stride;
			InputCrcs crcs(ctx, st, tk, d_parts, d_part_crc, 1, 1, n_chunks, nb, image_stride);
			if ((rc = crcs.begin()) || (rc = crcs.verify()) || (rc = crcs.publish(false))) return rc;
			if (direct_image && direct_image != image)
				CUDA_TRY(cudaMemcpy2DAsync(direct_image, out_stride, image, image_stride, static_cast<size_t>(nb) * B, n_chunks, cudaMemcpyDeviceToDevice, st));
		} else {
			// One pass (convert_kernel.cuh): source parts -> destination parts + their CRCs, no chunk image
			if (!slice_is_std(*dst)) {
				rc = try_fused_convert(ctx, src, dst, n_chunks, nb, d_parts, part_stride, d_part_crc, want, d_out, out_stride, st, tk, &t_crc, &encode_crc_stride);
				if (rc == LZGPU_OK) {
					converted = true;
					d_encode_crc = t_crc.p;
				} else if (rc != LZGPU_NOT_HANDLED) {
					return rc;
				}
			}
		}
		if (!slice_is_std(*src) && !converted) {
			void *d_img = direct_image;
			image_stride = direct_image ? out_stride : static_cast<size_t>(nb) * B;
			if (!d_img) {
				if ((rc = t_image.alloc(static_cast<size_t>(n_chunks) * image_stride))) return rc;
				d_img = t_image.p;
			}
			const uint8_t none_wanted[LZGPU_MAX_PARTS] = {0};
			if ((rc = recover_enqueue(ctx, src, n_chunks, nb, d_parts, part_stride, d_part_crc, none_wanted, nullptr, d_img, image_stride, st, tk)))
				return rc;
			image = static_cast<const uint8_t *>(d_img);
		}
		if (!slice_is_std(*dst) && !converted) {
			bool data_wanted = false, parity_wanted = false;
			void *dp[LZGPU_MAX_DATA] = {nullptr};
			for (int i = 0; i < nd; ++i) {
				if (!want[i]) continue;
				if (i < kd) { dp[i] = d_out[i]; data_wanted = true; }
				else parity_wanted = true;
			}
			// One pass over the image when a parity part is wanted: data part j, block s = chunk block s*k + j
			// (SliceRecoveryPlanner::BlockConverter, :41-57) and XorReadPlan::RecoverParity / ECReadPlan::RecoverParity
			// (xor_read_plan.h:39-62, ec_read_plan.h:38-76), every destination part stored straight into its buffer, block CRCs of
			// the whole destination slice as a by-product.  Algorithmic bytes: read the image once, write each wanted part once.
			bool fused_done = false;
			if (parity_wanted && image_stride >= static_cast<size_t>(nb) * B) {
				const size_t crc_stride = (nb + static_cast<size_t>(dst->m) * pbd + 3) & ~size_t(3);
				if ((rc = t_crc.alloc(n_chunks * crc_stride * 4))) return rc;
				void *outs[LZGPU_MAX_PARTS] = {nullptr};
				for (int i = 0; i < nd; ++i) outs[i] = want[i] ? d_out[i] : nullptr;
				rc = lz_fused_encode_split(ctx, dst, n_chunks, nb, image, image_stride, outs, out_stride, t_crc.p, crc_stride, st);
				if (rc == LZGPU_OK) {
					fused_done = true;
					d_encode_crc = t_crc.p;
					encode_crc_stride = crc_stride;
					ctx->stats.chunks_encoded += n_chunks;
				} else if (rc != LZGPU_NOT_HANDLED) {
					return rc;
				}
			}
			if (!fused_done) {
				if (data_wanted && (rc = lzgpu_split_chunks_dev(ctx, dst, n_chunks, nb, image, image_stride, dp, out_stride, st))) return rc;
				if (parity_wanted) {
					const size_t par_stride = static_cast<size_t>(dst->m) * pbd * B, crc_stride = (nb + static_cast<size_t>(dst->m) * pbd + 3) & ~size_t(3);
					if ((rc = t_par.alloc(n_chunks * par_stride)) || (!t_crc.p && (rc = t_crc.alloc(n_chunks * crc_stride * 4)))) return rc;
					if ((rc = encode_enqueue(ctx, dst, n_chunks, nb, image, image_stride, t_par.p, par_stride, t_crc.p, crc_stride, st))) return rc;
					ctx->stats.chunks_encoded += n_chunks;
					d_encode_crc = t_crc.p;
					encode_crc_stride = crc_stride;
					for (int r = 0; r < dst->m; ++r)
						if (want[kd + r])
							CUDA_TRY(cudaMemcpy2DAsync(d_out[kd + r], out_stride, static_cast<uint8_t *>(t_par.p) + static_cast<size_t>(r) * pbd * B, par_stride,
							                           static_cast<size_t>(pbd) * B, n_chunks, cudaMemcpyDeviceToDevice, st));
				}
			}
		}
	}
	// ChunkReplicator::replicate computes mycrc32 of every rebuilt block (chunk_replicator.cc:186-192)
	if (d_out_crc && !lzgpu_crc_enabled()) {
		for (int i = 0; i < nd; ++i)
			if (want[i] && d_out_crc[i] && (rc = fill_crc(ctx, d_out_crc[i], pbd, pbd, n_chunks, st))) return rc;
	} else if (d_out_crc) {
		if (d_encode_crc) {
			// the encode pass that produced the parity already checksummed every data and parity block of the destination slice
			CrcPartsArgs a{};
			bool any = false;
			for (int i = 0; i < nd; ++i)
				if (want[i] && d_out_crc[i]) { a.out[i] = static_cast<uint32_t *>(d_out_crc[i]); any = true; }
			if (any) {
				a.crc = static_cast<const uint32_t *>(d_encode_crc);
				a.crc_stride = encode_crc_stride;
				a.k = kd; a.m = dst->m; a.nb = nb; a.pb = pbd; a.zero_crc = kCrcZeroBlock64K;
				a.total = static_cast<unsigned long long>(n_chunks) * nd * pbd;
				crc_to_parts_kernel<<<grid_for(ctx, a.total, 256, 4), 256, 0, st>>>(a);
				CUDA_TRY(cudaGetLastError());
				ctx->stats.kernel_launches++;
			}
		} else {
			for (int i = 0; i < nd; ++i)
				if (want[i] && d_out_crc[i] && (rc = crc_of_parts(ctx, d_out[i], n_chunks, pbd, out_stride, d_out_crc[i], st))) return rc;
		}
	}
	return LZGPU_OK;
}

static uint64_t convert_alg_bytes(const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb, const uint8_t *want, bool crcs) {
	// DESIGN.md §4.5: read k source parts once (+ stored CRCs), write the wanted destination parts once (+ their CRCs)
	const uint64_t B = LZGPU_BLOCK_SIZE, pbs = (nb + src->k - 1) / src->k, pbd = (nb + dst->k - 1) / dst->k;
	uint64_t n_out = 0;
	for (int i = 0; i < dst->k + dst->m; ++i) n_out += want[i] ? 1 : 0;
	return n_chunks * (src->k * pbs * (B + (crcs ? 4 : 0)) + n_out * pbd * (B + 4));
}

extern "C" int lzgpu_convert_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                                         const void *const *d_parts, size_t part_stride, const void *const *d_part_crc,
                                         const uint8_t *want, void *const *d_out, size_t out_stride, void *const *d_out_crc,
                                         int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::convert_chunks_dev");
	int rc = convert_check_args(ctx, src, dst, nb, d_parts, want, d_out);
	if (rc || n_chunks == 0) return rc;
	if (bad) bad[0] = bad[1] = bad[2] = -1;
	return dev_call(ctx, stream, convert_alg_bytes(src, dst, n_chunks, nb, want, d_part_crc != nullptr), bad, [&](cudaStream_t st, VerifyTicket *tk) {
		return convert_enqueue(ctx, src, dst, n_chunks, nb, d_parts, part_stride, d_part_crc, want, d_out, out_stride, d_out_crc, st, tk);
	});
}

extern "C" int lzgpu_convert_chunks(lzgpu_ctx *ctx, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                                     const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc, const uint8_t *want,
                                     uint8_t *const *out, size_t out_stride, uint32_t *const *out_crc, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::convert_chunks");
	int rc = convert_check_args(ctx, src, dst, nb, parts, want, out);
	if (rc) return rc;
	if (n_chunks == 0) return LZGPU_OK;
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const int ns = src->k + src->m, nd = dst->k + dst->m;
	const uint32_t pbs = (nb + src->k - 1) / src->k, pbd = (nb + dst->k - 1) / dst->k;
	const size_t sbytes = static_cast<size_t>(pbs) * B, dbytes = static_cast<size_t>(pbd) * B;
	if (part_stride < sbytes || out_stride < dbytes) { lz_set_error("convert: strides too small"); return LZGPU_ERR_ARG; }
	GivenParts in(parts, part_crc, ns, part_stride, pbs);
	int n_out = 0;
	for (int i = 0; i < nd; ++i) {
		if (want[i] && !out[i]) { lz_set_error("convert: wanted part %d has no output buffer", i); return LZGPU_ERR_ARG; }
		n_out += want[i] != 0;
	}
	if (n_out == 0) return LZGPU_OK;
	if (bad) bad[0] = bad[1] = bad[2] = -1;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	AutoPin pin(ctx);
	for (int i = 0; i < nd; ++i)
		if (want[i]) pin.add(out[i], static_cast<size_t>(n_chunks - 1) * out_stride + dbytes);
	// a same-slice rebuild writes into buffers shaped like the inputs
	const int n_in = std::max(in.n_given, 1);
	const size_t per_chunk = sbytes * n_in + dbytes * n_out;
	const uint32_t tile = static_cast<uint32_t>(std::max<size_t>(1, std::min<size_t>(n_chunks, (2 * kHostTileBytes) / per_chunk)));
	const int n_slots = n_chunks > tile ? kHostSlots : 1;
	void *d_o[kHostSlots], *d_co[kHostSlots];
	if ((rc = in.prepare(ctx, pin, n_chunks, tile, n_slots, n_in))) return rc;
	for (int s = 0; s < n_slots; ++s) {
		if ((rc = lz_scratch(ctx, kScratchPar0 + s, tile * dbytes * n_out, &d_o[s]))) return rc;
		if ((rc = lz_scratch(ctx, kScratchOutCrc0 + s, static_cast<size_t>(tile) * pbd * 4 * n_out, &d_co[s]))) return rc;
	}
	return run_tiles(ctx, n_chunks, tile, n_slots, bad, [&](int s, size_t c0, size_t nc, cudaStream_t st, VerifyTicket *tk) -> int {
		GivenParts::Tile t;
		int rc = in.stage(ctx, s, c0, nc, st, t);
		if (rc) return rc;
		std::vector<void *> dout(nd, nullptr), dcrc(nd, nullptr);
		for (int i = 0, a = 0; i < nd; ++i) {
			if (!want[i]) continue;
			dout[i] = static_cast<uint8_t *>(d_o[s]) + static_cast<size_t>(a) * tile * dbytes;
			if (out_crc && out_crc[i]) dcrc[i] = static_cast<uint8_t *>(d_co[s]) + static_cast<size_t>(a) * tile * pbd * 4;
			++a;
		}
		{
			BatchTimer timer(ctx, st, convert_alg_bytes(src, dst, static_cast<uint32_t>(nc), nb, want, t.any_crc));
			rc = convert_enqueue(ctx, src, dst, static_cast<uint32_t>(nc), nb, t.dp.data(), sbytes, t.crcs(), want, dout.data(), dbytes,
			                     out_crc ? dcrc.data() : nullptr, st, tk);
		}
		if (rc) return rc;
		for (int i = 0; i < nd; ++i) {
			if (!want[i]) continue;
			CUDA_TRY(cudaMemcpy2DAsync(out[i] + c0 * out_stride, out_stride, dout[i], dbytes, dbytes, nc, cudaMemcpyDeviceToHost, st));
			ctx->stats.bytes_d2h += static_cast<uint64_t>(nc) * dbytes;
			if (dcrc[i]) CUDA_TRY(cudaMemcpyAsync(out_crc[i] + c0 * pbd, dcrc[i], nc * pbd * 4, cudaMemcpyDeviceToHost, st));
		}
		return LZGPU_OK;
	});
}

// ------------------------------------------------------------------------------------------------
// recovery from the parts of every slice of a goal together (lzgpu_recover_slices*)
// ------------------------------------------------------------------------------------------------
static const char *const kSlicesFn[] = {"recover_slices", "salvage_slices", "check_slices", "correct_slices"};   // by lzd::RsMode

// the salvage, check and correction want no part
static const uint8_t kWantNone[LZGPU_MAX_PARTS] = {0};

// The arguments of the four calls (c.mode: the recovery, salvage, check or correction) in the buffers b, checked before anything is
// enqueued and whatever n_chunks is; they fill the rest of c.  dev: the device form's alignment rules (16-byte buffers and strides,
// 4-byte CRC arrays, an 8-byte aligned map).  LZGPU_ERR_TOO_FEW_PARTS when a block the recovery must write is not determined (the
// salvage writes what is determined, holes are not refused), when no part is given to the other three, and when no shape of the
// batch has a check for the check and correction.  The salvage requires the image and the map, the check the map, the correction
// the fix entries (b.map); more than 64 checks in a shape is LZGPU_ERR_ARG.
static int recover_slices_args(const lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t nb, const SlicesBufs &b, bool dev,
                               RecoverSlicesCall &c) {
	if (!ctx || !b.parts || !b.part_stride || !b.want) return LZGPU_ERR_ARG;
	const bool salvage = c.mode == lzd::RsMode::SALVAGE, correct = c.mode == lzd::RsMode::CORRECT;
	const bool check = correct || c.mode == lzd::RsMode::CHECK;
	const char *fn = kSlicesFn[static_cast<int>(c.mode)];
	if (salvage && (!b.image || !b.map)) { lz_set_error("salvage_slices: the image and the map are required"); return LZGPU_ERR_ARG; }
	if (check && !b.map) { lz_set_error("%s: the %s is required", fn, correct ? "fix" : "map"); return LZGPU_ERR_ARG; }
	const char *why = nullptr;
	if (lzd::slice_layout(goals, n_slices, c.lay, &why)) { lz_set_error("%s: %s", fn, why); return LZGPU_ERR_ARG; }
	if (nb == 0 || nb > LZGPU_BLOCKS_IN_CHUNK) { lz_set_error("nb out of range"); return LZGPU_ERR_ARG; }
	const lzd::SliceLayout &lay = c.lay;
	const size_t B = LZGPU_BLOCK_SIZE;
	uint8_t given[LZGPU_MAX_PARTS] = {0};
	for (uint32_t i = 0; i < lay.n_slices; ++i) {
		c.pb[i] = (nb + lay.k[i] - 1) / lay.k[i];
		const size_t bytes = static_cast<size_t>(c.pb[i]) * B;
		for (uint32_t g = lay.base[i]; g < lay.base[i] + lay.k[i] + lay.m[i]; ++g) {
			given[g] = b.parts[g] != nullptr;
			if (given[g] && (b.part_stride[i] < bytes || (dev && (b.part_stride[i] & 15)))) {
				lz_set_error("%s: part_stride[%u] too small or not a multiple of 16", fn, i);
				return LZGPU_ERR_ARG;
			}
			if (!b.want[g]) continue;
			if (given[g]) { lz_set_error("recover_slices: part %u is given and wanted", g); return LZGPU_ERR_ARG; }
			if (!b.out || !b.out[g] || !b.out_stride) { lz_set_error("recover_slices: wanted part %u has no output buffer", g); return LZGPU_ERR_ARG; }
			if (b.out_stride[i] < bytes || (dev && (b.out_stride[i] & 15))) {
				lz_set_error("recover_slices: out_stride[%u] too small or not a multiple of 16", i);
				return LZGPU_ERR_ARG;
			}
		}
	}
	if (b.image && (b.image_stride < static_cast<size_t>(nb) * B || (dev && (b.image_stride & 15)))) {
		lz_set_error(salvage ? "salvage_slices: image_stride must cover nb blocks (and be a multiple of 16)"
		                     : "recover_slices: chunk_out_stride must cover nb blocks (and be a multiple of 16)");
		return LZGPU_ERR_ARG;
	}
	const int n = static_cast<int>(lay.n_parts);
	int rc;
	if (dev) {
		if ((rc = check_part_ptrs(fn, "parts", b.parts, n, 16)) || (rc = check_part_ptrs(fn, "out", b.out, n, 16)) ||
		    (rc = check_part_ptrs(fn, "part_crc", b.part_crc, n, 4)) || (rc = check_part_ptrs(fn, "out_crc", b.out_crc, n, 4)))
			return rc;
		if (reinterpret_cast<uintptr_t>(b.image) & 15) { lz_set_error("%s: %s is not 16-byte aligned", fn, salvage ? "image" : "chunk_out"); return LZGPU_ERR_ARG; }
		if (reinterpret_cast<uintptr_t>(b.image_crc) & 3) { lz_set_error("salvage_slices: image_crc is not 4-byte aligned"); return LZGPU_ERR_ARG; }
	}
	if (c.mode != lzd::RsMode::RECOVER) {
		bool any = false;
		for (uint32_t g = 0; g < lay.n_parts; ++g) any |= b.parts[g] != nullptr;
		if (!any) { lz_set_error("%s: no part is given", fn); return LZGPU_ERR_TOO_FEW_PARTS; }
	}
	const uint32_t tail = nb % lay.L;
	lzd::slice_shapes(lay, given, nb, c.mode, c);
	for (int t = 0; t < 2 && check; ++t) {
		if (t == 0 ? nb < lay.L : tail == 0) continue;   // a shape no chunk of the call has
		if (c.checks[t].n_checks > lzd::kScMaxChecks) {
			lz_set_error("%s: the %s combined stripe has %u checks, more than 64", fn, t ? "last" : "full", c.checks[t].n_checks);
			return LZGPU_ERR_ARG;
		}
	}
	if (check && (nb < lay.L || !c.checks[0].n_checks) && (!tail || !c.checks[1].n_checks)) {
		lz_set_error("%s: no combined stripe of the batch has a check", fn);
		return LZGPU_ERR_TOO_FEW_PARTS;
	}
	for (int t = 0; t < 2 && c.mode == lzd::RsMode::RECOVER; ++t) {
		if (t == 0 ? nb < lay.L : tail == 0) continue;
		const lzd::SliceSolve &sv = c.shapes[t];
		const uint64_t lost = lzd::slice_needed(lay, b.want, b.image != nullptr, sv.valid) & ~sv.determined;
		if (lost) {
			lz_set_error("recover_slices: positions %#llx of the %s combined stripe are not determined by the given parts",
			             static_cast<unsigned long long>(lost), t ? "last" : "full");
			return LZGPU_ERR_TOO_FEW_PARTS;
		}
	}
	if (!c.geo.ok) {
		lz_set_error("%s: a combined stripe has more blocks than the kernel stages (%u slots, %u CRC streams)", fn, c.geo.slots, c.geo.states);
		return LZGPU_ERR_ARG;
	}
	if (correct && (rc = check_part_ptrs(fn, "new_crc", b.new_crc, n, 4))) return rc;
	if (dev && check && (reinterpret_cast<uintptr_t>(b.map) & 7)) { lz_set_error("%s: %s is not 8-byte aligned", fn, correct ? "fix" : "map"); return LZGPU_ERR_ARG; }
	return LZGPU_OK;
}

// DESIGN.md §4.8: read the given parts (+ their stored CRCs), write the wanted parts (+ their CRCs) and the image (+ the salvage's
// image CRCs and map, or the check's or correction's entries)
static uint64_t recover_slices_alg_bytes(const RecoverSlicesCall &c, uint32_t n_chunks, uint32_t nb, const SlicesBufs &d) {
	const uint64_t B = LZGPU_BLOCK_SIZE;
	uint64_t per_chunk = d.image ? static_cast<uint64_t>(nb) * B : 0;
	if (c.mode == lzd::RsMode::SALVAGE) per_chunk += static_cast<uint64_t>(nb) * (d.image_crc ? 5 : 1);
	if (c.mode == lzd::RsMode::CHECK || c.mode == lzd::RsMode::CORRECT) per_chunk += (nb + c.lay.L - 1) / c.lay.L * c.entry_bytes();
	for (uint32_t i = 0; i < c.lay.n_slices; ++i)
		for (uint32_t g = c.lay.base[i]; g < c.lay.base[i] + c.lay.k[i] + c.lay.m[i]; ++g) {
			if (d.parts[g]) per_chunk += c.pb[i] * (B + (d.part_crc ? 4 : 0));
			if (d.want[g]) per_chunk += c.pb[i] * (B + (d.out_crc ? 4 : 0));
		}
	return n_chunks * per_chunk;
}

// bad[0..3] = chunk, slice, part of the slice, block from the ticket's chunk, flat part, block
static void recover_slices_bad(const lzd::SliceLayout &lay, const int64_t *b3, int64_t *bad) {
	if (!bad || b3[1] < 0) return;
	const int i = lay.slice_of(static_cast<uint32_t>(b3[1]));
	bad[0] = b3[0];
	bad[1] = i;
	bad[2] = b3[1] - lay.base[i];
	bad[3] = b3[2];
}

// one launch on the device buffers d; *tk is armed when a given part has stored CRCs (the kernel compares them with the constant
// while CRCs are disabled)
static int recover_slices_enqueue(lzgpu_ctx *ctx, const RecoverSlicesCall &c, uint32_t n_chunks, uint32_t nb, const SlicesBufs &d,
                                  cudaStream_t st, VerifyTicket *tk) {
	bool verifying = false;
	for (uint32_t g = 0; g < c.lay.n_parts; ++g) verifying |= d.parts[g] && d.part_crc && d.part_crc[g];
	int rc;
	if (verifying && (rc = tk->arm(ctx, st))) return rc;
	SlicesBufs k = d;
	if (!verifying) k.part_crc = nullptr;
	if ((rc = lz_recover_slices(ctx, c, k, n_chunks, nb, st, verifying ? tk->word(0) : nullptr))) return rc;
	if (c.mode == lzd::RsMode::RECOVER || c.mode == lzd::RsMode::SALVAGE) ctx->stats.chunks_recovered += n_chunks;
	return verifying ? tk->publish_fused() : LZGPU_OK;
}

// The device form of the four calls: the argument check, then one launch on the caller's stream
static int recover_slices_dev(lzgpu_ctx *ctx, lzd::RsMode mode, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                              const SlicesBufs &d, int64_t *bad, void *stream) {
	auto c = std::make_unique<RecoverSlicesCall>();
	c->mode = mode;
	int rc = recover_slices_args(ctx, goals, n_slices, nb, d, true, *c);
	if (rc || n_chunks == 0) return rc;
	if (bad) bad[0] = bad[1] = bad[2] = bad[3] = -1;
	int64_t b3[3] = {-1, -1, -1};
	rc = dev_call(ctx, stream, recover_slices_alg_bytes(*c, n_chunks, nb, d), b3,
	              [&](cudaStream_t st, VerifyTicket *tk) { return recover_slices_enqueue(ctx, *c, n_chunks, nb, d, st, tk); });
	if (rc == LZGPU_ERR_CRC) recover_slices_bad(c->lay, b3, bad);
	return rc;
}

extern "C" int lzgpu_recover_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                         const void *const *d_parts, const size_t *part_stride, const void *const *d_part_crc,
                                         const uint8_t *want, void *const *d_out, const size_t *out_stride, void *const *d_out_crc,
                                         void *d_chunk_out, size_t chunk_out_stride, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::recover_slices_dev");
	return recover_slices_dev(ctx, lzd::RsMode::RECOVER, goals, n_slices, n_chunks, nb,
	                          {d_parts, part_stride, d_part_crc, want, d_out, out_stride, d_out_crc, d_chunk_out, chunk_out_stride}, bad, stream);
}

extern "C" int lzgpu_salvage_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                         const void *const *d_parts, const size_t *part_stride, const void *const *d_part_crc, void *d_image,
                                         size_t image_stride, void *d_image_crc, void *d_map, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::salvage_slices_dev");
	SlicesBufs d{d_parts, part_stride, d_part_crc, kWantNone};
	d.image = d_image, d.image_stride = image_stride, d.image_crc = d_image_crc, d.map = d_map;
	return recover_slices_dev(ctx, lzd::RsMode::SALVAGE, goals, n_slices, n_chunks, nb, d, bad, stream);
}

extern "C" int lzgpu_check_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                       const void *const *d_parts, const size_t *part_stride, const void *const *d_part_crc, void *d_map,
                                       int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::check_slices_dev");
	SlicesBufs d{d_parts, part_stride, d_part_crc, kWantNone};
	d.map = d_map;
	return recover_slices_dev(ctx, lzd::RsMode::CHECK, goals, n_slices, n_chunks, nb, d, bad, stream);
}

extern "C" int lzgpu_correct_slices_dev(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                         void *const *d_parts, const size_t *part_stride, const void *const *d_part_crc, void *const *d_new_crc,
                                         void *d_fix, int64_t *bad, void *stream) {
	NvtxScope nvtx_scope("lzgpu::correct_slices_dev");
	SlicesBufs d{d_parts, part_stride, d_part_crc, kWantNone};
	d.map = d_fix, d.new_crc = d_new_crc;
	return recover_slices_dev(ctx, lzd::RsMode::CORRECT, goals, n_slices, n_chunks, nb, d, bad, stream);
}

// The host form of the four calls: the argument check, then the given parts (+ stored CRCs) staged tile by tile, the wanted parts
// (+ CRCs), the image and the salvage's image CRCs and map (or the check's entries) copied back.  The salvage, check and correction
// run every tile past a CRC mismatch, so that their outputs are complete.  The correction corrects the staged tile and copies back its
// fix entries, and then, for each corrected entry, only the suspect's rewritten blocks and their new CRCs (new_crc).  The check and
// correction return LZGPU_ERR_INCONSISTENT when an entry is left bad.
static int recover_slices_host(lzgpu_ctx *ctx, lzd::RsMode mode, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                               const SlicesBufs &h, int64_t *bad) {
	auto cp = std::make_unique<RecoverSlicesCall>();
	cp->mode = mode;
	int rc = recover_slices_args(ctx, goals, n_slices, nb, h, false, *cp);
	if (rc || n_chunks == 0) return rc;
	const RecoverSlicesCall &c = *cp;
	const bool check = mode == lzd::RsMode::CHECK || mode == lzd::RsMode::CORRECT;
	const auto parts = reinterpret_cast<const uint8_t *const *>(h.parts);
	const auto part_crc = reinterpret_cast<const uint32_t *const *>(h.part_crc);
	const auto out = reinterpret_cast<uint8_t *const *>(h.out);
	const auto out_crc = reinterpret_cast<uint32_t *const *>(h.out_crc);
	const auto new_crc = reinterpret_cast<uint32_t *const *>(h.new_crc);
	const auto chunk_out = static_cast<uint8_t *>(h.image), map = static_cast<uint8_t *>(h.map);
	const auto image_crc = static_cast<uint32_t *>(h.image_crc);
	const uint8_t *want = h.want;
	if (bad) bad[0] = bad[1] = bad[2] = bad[3] = -1;
	const lzd::SliceLayout &lay = c.lay;
	const uint32_t n = lay.n_parts;
	const size_t B = LZGPU_BLOCK_SIZE;
	// device layout of a tile: every given part, then every wanted part, then the image and the map, each dense (tile chunks of pb_i
	// blocks, nb blocks, nb bytes); the stored and the computed CRCs likewise, the image CRCs last
	size_t off[LZGPU_MAX_PARTS] = {0}, crc_off[LZGPU_MAX_PARTS] = {0}, bytes[LZGPU_MAX_PARTS] = {0}, per_chunk = 0, crc_words = 0;
	size_t new_crc_off[LZGPU_MAX_PARTS] = {0};
	size_t dstride[kSlicesMax] = {0};
	for (uint32_t g = 0; g < n; ++g) {
		const int i = lay.slice_of(g);
		dstride[i] = static_cast<size_t>(c.pb[i]) * B;
		if (!parts[g] && !want[g]) continue;
		bytes[g] = dstride[i];
		off[g] = per_chunk;
		per_chunk += bytes[g];
		if ((parts[g] && part_crc && part_crc[g]) || (want[g] && out_crc && out_crc[g])) {
			crc_off[g] = crc_words;
			crc_words += c.pb[i];
		}
		if (parts[g] && new_crc && new_crc[g]) {
			new_crc_off[g] = crc_words;
			crc_words += c.pb[i];
		}
	}
	const size_t img_off = per_chunk, img_bytes = chunk_out ? static_cast<size_t>(nb) * B : 0;
	per_chunk += img_bytes;
	const size_t map_off = per_chunk, img_crc_off = crc_words;
	const uint32_t n_cs = (nb + lay.L - 1) / lay.L;
	const size_t map_bytes = !map ? 0 : check ? n_cs * c.entry_bytes() : nb;
	per_chunk += map_bytes;
	if (image_crc) crc_words += nb;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard dg(ctx->device);
	AutoPin pin(ctx);
	for (uint32_t g = 0; g < n; ++g) {
		const int i = lay.slice_of(g);
		if (parts[g]) pin.add(parts[g], static_cast<size_t>(n_chunks - 1) * h.part_stride[i] + bytes[g]);
		if (want[g]) pin.add(out[g], static_cast<size_t>(n_chunks - 1) * h.out_stride[i] + bytes[g]);
	}
	if (chunk_out) pin.add(chunk_out, static_cast<size_t>(n_chunks - 1) * h.image_stride + img_bytes);
	if (image_crc) pin.add(image_crc, static_cast<size_t>(n_chunks) * nb * 4);
	if (map) pin.add(map, static_cast<size_t>(n_chunks) * map_bytes);
	const uint32_t tile = static_cast<uint32_t>(std::max<size_t>(1, std::min<size_t>(n_chunks, (2 * kHostTileBytes) / std::max<size_t>(per_chunk, 1))));
	const int n_slots = n_chunks > tile ? kHostSlots : 1;
	void *d_in[kHostSlots], *d_crc[kHostSlots];
	for (int s = 0; s < n_slots; ++s)
		if ((rc = lz_scratch(ctx, kScratchIn0 + s, tile * per_chunk, &d_in[s])) ||
		    (rc = lz_scratch(ctx, kScratchCrc0 + s, tile * std::max<size_t>(crc_words, 1) * 4, &d_crc[s])))
			return rc;
	int64_t b3[3] = {-1, -1, -1};
	rc = run_tiles(ctx, n_chunks, tile, n_slots, b3, [&](int s, size_t c0, size_t nc, cudaStream_t st, VerifyTicket *tk) -> int {
		void *dp[LZGPU_MAX_PARTS] = {nullptr}, *dpc[LZGPU_MAX_PARTS] = {nullptr}, *dout[LZGPU_MAX_PARTS] = {nullptr}, *docrc[LZGPU_MAX_PARTS] = {nullptr};
		void *dncrc[LZGPU_MAX_PARTS] = {nullptr};
		bool any_crc = false;
		for (uint32_t g = 0; g < n; ++g) {
			const int i = lay.slice_of(g);
			uint8_t *buf = static_cast<uint8_t *>(d_in[s]) + tile * off[g];
			uint32_t *cbuf = static_cast<uint32_t *>(d_crc[s]) + tile * crc_off[g];
			if (parts[g]) {
				CUDA_TRY(cudaMemcpy2DAsync(buf, bytes[g], parts[g] + c0 * h.part_stride[i], h.part_stride[i], bytes[g], nc, cudaMemcpyHostToDevice, st));
				ctx->stats.bytes_h2d += nc * bytes[g];
				dp[g] = buf;
				if (part_crc && part_crc[g]) {
					CUDA_TRY(cudaMemcpyAsync(cbuf, part_crc[g] + c0 * c.pb[i], nc * c.pb[i] * 4, cudaMemcpyHostToDevice, st));
					dpc[g] = cbuf;
					any_crc = true;
				}
				if (new_crc && new_crc[g]) dncrc[g] = static_cast<uint32_t *>(d_crc[s]) + tile * new_crc_off[g];
			} else if (want[g]) {
				dout[g] = buf;
				if (out_crc && out_crc[g]) docrc[g] = cbuf;
			}
		}
		const SlicesBufs d{dp, dstride, any_crc ? dpc : nullptr, want, dout, dstride, out_crc ? docrc : nullptr,
		                   chunk_out ? static_cast<uint8_t *>(d_in[s]) + tile * img_off : nullptr, img_bytes,
		                   image_crc ? static_cast<uint32_t *>(d_crc[s]) + tile * img_crc_off : nullptr,
		                   map ? static_cast<uint8_t *>(d_in[s]) + tile * map_off : nullptr, dncrc};
		int rc;
		{
			BatchTimer timer(ctx, st, recover_slices_alg_bytes(c, static_cast<uint32_t>(nc), nb, d));
			rc = recover_slices_enqueue(ctx, c, static_cast<uint32_t>(nc), nb, d, st, tk);
		}
		if (rc) return rc;
		for (uint32_t g = 0; g < n; ++g) {
			if (!want[g]) continue;
			const int i = lay.slice_of(g);
			CUDA_TRY(cudaMemcpy2DAsync(out[g] + c0 * h.out_stride[i], h.out_stride[i], dout[g], bytes[g], bytes[g], nc, cudaMemcpyDeviceToHost, st));
			ctx->stats.bytes_d2h += nc * bytes[g];
			if (docrc[g]) CUDA_TRY(cudaMemcpyAsync(out_crc[g] + c0 * c.pb[i], docrc[g], nc * c.pb[i] * 4, cudaMemcpyDeviceToHost, st));
		}
		if (chunk_out) {
			CUDA_TRY(cudaMemcpy2DAsync(chunk_out + c0 * h.image_stride, h.image_stride, d.image, img_bytes, img_bytes, nc, cudaMemcpyDeviceToHost, st));
			ctx->stats.bytes_d2h += nc * img_bytes;
		}
		if (map) {
			CUDA_TRY(cudaMemcpyAsync(map + c0 * map_bytes, d.map, nc * map_bytes, cudaMemcpyDeviceToHost, st));
			ctx->stats.bytes_d2h += nc * map_bytes;
		}
		if (image_crc) CUDA_TRY(cudaMemcpyAsync(image_crc + c0 * nb, d.image_crc, nc * nb * 4, cudaMemcpyDeviceToHost, st));
		if (mode != lzd::RsMode::CORRECT) return LZGPU_OK;
		// the corrected entries' rewritten blocks, a run of consecutive part blocks at a time, and their new CRCs
		CUDA_TRY(cudaStreamSynchronize(st));
		const lzgpu_slices_fix *fix = reinterpret_cast<const lzgpu_slices_fix *>(map) + c0 * n_cs;
		for (size_t e = 0; e < nc * n_cs; ++e) {
			if (fix[e].status != LZGPU_FIX_CORRECTED) continue;
			const size_t cc = e / n_cs, cs = e % n_cs;
			const lzd::SliceChecks &ck = c.checks[(nb % lay.L) && cs == n_cs - 1 ? 1 : 0];
			const uint32_t g = static_cast<uint32_t>(fix[e].suspect_part);
			const int i = lay.slice_of(g);
			const size_t spc = lay.L / lay.k[i];
			for (uint32_t b = 0; b < ck.n_blocks;) {
				if (ck.blk_part[b] != g) { ++b; continue; }
				uint32_t run = 1;
				while (b + run < ck.n_blocks && ck.blk_part[b + run] == g && ck.blk_s[b + run] == ck.blk_s[b] + run) ++run;
				const size_t blk = cs * spc + ck.blk_s[b];
				CUDA_TRY(cudaMemcpyAsync(const_cast<uint8_t *>(parts[g]) + (c0 + cc) * h.part_stride[i] + blk * B,
				                         static_cast<const uint8_t *>(dp[g]) + cc * bytes[g] + blk * B, run * B, cudaMemcpyDeviceToHost, st));
				ctx->stats.bytes_d2h += run * B;
				if (dncrc[g])
					CUDA_TRY(cudaMemcpyAsync(new_crc[g] + (c0 + cc) * c.pb[i] + blk, static_cast<const uint32_t *>(dncrc[g]) + cc * c.pb[i] + blk,
					                         run * 4, cudaMemcpyDeviceToHost, st));
				b += run;
			}
		}
		return LZGPU_OK;
	}, mode != lzd::RsMode::RECOVER);
	if (rc == LZGPU_ERR_CRC) recover_slices_bad(lay, b3, bad);
	if (rc || !check) return rc;
	const auto *entries = reinterpret_cast<const lzgpu_slices_check *>(map);
	const auto *fix = reinterpret_cast<const lzgpu_slices_fix *>(map);
	for (size_t e = 0; e < static_cast<size_t>(n_chunks) * n_cs; ++e)
		if (mode == lzd::RsMode::CHECK ? entries[e].bad_checks != 0
		                               : fix[e].status == LZGPU_FIX_UNEXPLAINED || fix[e].status == LZGPU_FIX_UNDETERMINED)
			return LZGPU_ERR_INCONSISTENT;
	return LZGPU_OK;
}

extern "C" int lzgpu_recover_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                     const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc, const uint8_t *want,
                                     uint8_t *const *out, const size_t *out_stride, uint32_t *const *out_crc, uint8_t *chunk_out,
                                     size_t chunk_out_stride, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::recover_slices");
	return recover_slices_host(ctx, lzd::RsMode::RECOVER, goals, n_slices, n_chunks, nb,
	                           {reinterpret_cast<const void *const *>(parts), part_stride, reinterpret_cast<const void *const *>(part_crc), want,
	                            reinterpret_cast<void *const *>(out), out_stride, reinterpret_cast<void *const *>(out_crc), chunk_out, chunk_out_stride},
	                           bad);
}

extern "C" int lzgpu_salvage_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                     const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc, uint8_t *image,
                                     size_t image_stride, uint32_t *image_crc, uint8_t *map, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::salvage_slices");
	SlicesBufs h{reinterpret_cast<const void *const *>(parts), part_stride, reinterpret_cast<const void *const *>(part_crc), kWantNone};
	h.image = image, h.image_stride = image_stride, h.image_crc = image_crc, h.map = map;
	return recover_slices_host(ctx, lzd::RsMode::SALVAGE, goals, n_slices, n_chunks, nb, h, bad);
}

extern "C" int lzgpu_check_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                   const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                                   lzgpu_slices_check *map, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::check_slices");
	SlicesBufs h{reinterpret_cast<const void *const *>(parts), part_stride, reinterpret_cast<const void *const *>(part_crc), kWantNone};
	h.map = map;
	return recover_slices_host(ctx, lzd::RsMode::CHECK, goals, n_slices, n_chunks, nb, h, bad);
}

extern "C" int lzgpu_correct_slices(lzgpu_ctx *ctx, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                     uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc, uint32_t *const *new_crc,
                                     lzgpu_slices_fix *fix, int64_t *bad) {
	NvtxScope nvtx_scope("lzgpu::correct_slices");
	SlicesBufs h{reinterpret_cast<const void *const *>(parts), part_stride, reinterpret_cast<const void *const *>(part_crc), kWantNone};
	h.map = fix, h.new_crc = reinterpret_cast<void *const *>(new_crc);
	return recover_slices_host(ctx, lzd::RsMode::CORRECT, goals, n_slices, n_chunks, nb, h, bad);
}

// ------------------------------------------------------------------------------------------------
// wire-format producer: LIZ_CLTOCS_WRITE_DATA prefixes from the CRC array
// ------------------------------------------------------------------------------------------------
extern "C" int lzgpu_write_data_prefixes_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_crc,
                                              size_t crc_stride, const void *d_chunk_ids, uint32_t write_id_base, void *d_out, void *stream) {
	if (!d_crc || !d_chunk_ids || !d_out) return LZGPU_ERR_ARG;
	int rc = check_batch(ctx, goal, nb);
	if (rc) return rc;
	const uint32_t k = goal->k, m = goal->m, pb = (nb + k - 1) / k;
	if (crc_stride < nb + static_cast<size_t>(m) * pb) { lz_set_error("prefixes: crc_stride too small"); return LZGPU_ERR_ARG; }
	if (n_chunks == 0) return LZGPU_OK;
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	PrefixArgs a{};
	a.crc = static_cast<const uint32_t *>(d_crc);
	a.chunk_ids = static_cast<const unsigned long long *>(d_chunk_ids);
	a.out = static_cast<uint8_t *>(d_out);
	a.crc_stride = crc_stride;
	a.k = k; a.m = m; a.nb = nb; a.pb = pb;
	a.write_id_base = write_id_base;
	a.total = static_cast<unsigned long long>(n_chunks) * (k + m) * pb;
	write_prefix_kernel<<<grid_for(ctx, a.total, 256, 4), 256, 0, st>>>(a);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

extern "C" int lzgpu_write_data_prefixes(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint32_t *crc,
                                          size_t crc_stride, const uint64_t *chunk_ids, uint32_t write_id_base, uint8_t *out) {
	if (!crc || !chunk_ids || !out) return LZGPU_ERR_ARG;
	int rc = check_batch(ctx, goal, nb);
	if (rc || n_chunks == 0) return rc;
	const uint32_t k = goal->k, m = goal->m, pb = (nb + k - 1) / k;
	const size_t n_crc = nb + static_cast<size_t>(m) * pb;
	if (crc_stride < n_crc) { lz_set_error("prefixes: crc_stride too small"); return LZGPU_ERR_ARG; }
	const size_t out_bytes = static_cast<size_t>(n_chunks) * (k + m) * pb * LZGPU_WRITE_PREFIX_SIZE;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	cudaStream_t st = ctx->stream;
	void *d_crc = nullptr, *d_ids = nullptr, *d_out = nullptr;
	if ((rc = lz_scratch(ctx, kScratchCrc0, static_cast<size_t>(n_chunks) * n_crc * 4, &d_crc))) return rc;
	if ((rc = lz_scratch(ctx, kScratchCrc0 + 1, static_cast<size_t>(n_chunks) * 8, &d_ids))) return rc;
	if ((rc = lz_scratch(ctx, kScratchPar0, out_bytes, &d_out))) return rc;
	CUDA_TRY(cudaMemcpy2DAsync(d_crc, n_crc * 4, crc, crc_stride * 4, n_crc * 4, n_chunks, cudaMemcpyHostToDevice, st));
	CUDA_TRY(cudaMemcpyAsync(d_ids, chunk_ids, static_cast<size_t>(n_chunks) * 8, cudaMemcpyHostToDevice, st));
	if ((rc = lzgpu_write_data_prefixes_dev(ctx, goal, n_chunks, nb, d_crc, n_crc, d_ids, write_id_base, d_out, st))) return rc;
	CUDA_TRY(cudaMemcpyAsync(out, d_out, out_bytes, cudaMemcpyDeviceToHost, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	return LZGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// chunk order -> part-major data parts
// ------------------------------------------------------------------------------------------------
extern "C" int lzgpu_split_chunks_dev(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const void *d_data,
                                       size_t chunk_stride, void *const *d_parts, size_t part_stride, void *stream) {
	if (!d_data || !d_parts) return LZGPU_ERR_ARG;
	int rc = check_batch(ctx, goal, nb);
	if (rc) return rc;
	const uint32_t B = LZGPU_BLOCK_SIZE, k = goal->k, pb = (nb + k - 1) / k;
	if (chunk_stride < static_cast<size_t>(nb) * B || part_stride < static_cast<size_t>(pb) * B || (chunk_stride & 15) || (part_stride & 15)) {
		lz_set_error("split: bad strides");
		return LZGPU_ERR_ARG;
	}
	if (reinterpret_cast<uintptr_t>(d_data) & 15) { lz_set_error("split: data is not 16-byte aligned"); return LZGPU_ERR_ARG; }
	if ((rc = check_part_ptrs("split", "parts", d_parts, static_cast<int>(k), 16))) return rc;
	if (n_chunks == 0) return LZGPU_OK;
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	SplitArgs a{};
	a.chunk = static_cast<const uint8_t *>(d_data);
	for (uint32_t j = 0; j < k; ++j) a.part[j] = static_cast<uint8_t *>(d_parts[j]);
	a.chunk_stride = chunk_stride;
	a.part_stride = part_stride;
	a.k = k;
	a.nb = nb;
	a.pb = pb;
	a.total_units = static_cast<unsigned long long>(n_chunks) * k * pb * (B / 16);
	chunk_to_parts_kernel<<<grid_for(ctx, a.total_units, 256, 8), 256, 0, st>>>(a);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

extern "C" int lzgpu_split_chunks(lzgpu_ctx *ctx, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *data,
                                   size_t chunk_stride, uint8_t *const *parts, size_t part_stride) {
	if (!data || !parts) return LZGPU_ERR_ARG;
	int rc = check_batch(ctx, goal, nb);
	if (rc || n_chunks == 0) return rc;
	const uint32_t B = LZGPU_BLOCK_SIZE, k = goal->k, pb = (nb + k - 1) / k;
	const size_t chunk_bytes = static_cast<size_t>(nb) * B, part_bytes = static_cast<size_t>(pb) * B;
	if (chunk_stride < chunk_bytes || part_stride < part_bytes) { lz_set_error("split: strides smaller than the payload"); return LZGPU_ERR_ARG; }
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	cudaStream_t st = ctx->stream;
	void *d_in = nullptr, *d_out = nullptr;
	if ((rc = lz_scratch(ctx, kScratchIn0, static_cast<size_t>(n_chunks) * chunk_bytes, &d_in))) return rc;
	if ((rc = lz_scratch(ctx, kScratchPar0, static_cast<size_t>(n_chunks) * part_bytes * k, &d_out))) return rc;
	CUDA_TRY(cudaMemcpy2DAsync(d_in, chunk_bytes, data, chunk_stride, chunk_bytes, n_chunks, cudaMemcpyHostToDevice, st));
	std::vector<void *> dp(k, nullptr);
	for (uint32_t j = 0; j < k; ++j)
		if (parts[j]) dp[j] = static_cast<uint8_t *>(d_out) + static_cast<size_t>(j) * n_chunks * part_bytes;
	if ((rc = lzgpu_split_chunks_dev(ctx, goal, n_chunks, nb, d_in, chunk_bytes, dp.data(), part_bytes, st))) return rc;
	for (uint32_t j = 0; j < k; ++j)
		if (parts[j]) CUDA_TRY(cudaMemcpy2DAsync(parts[j], part_stride, dp[j], part_bytes, part_bytes, n_chunks, cudaMemcpyDeviceToHost, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	ctx->stats.bytes_h2d += static_cast<uint64_t>(n_chunks) * chunk_bytes;
	return LZGPU_OK;
}

// ------------------------------------------------------------------------------------------------
// CRC of block arrays / scrub
// ------------------------------------------------------------------------------------------------
extern "C" int lzgpu_crc_blocks_dev(lzgpu_ctx *ctx, const void *d_data, size_t n_blocks, uint32_t block_len, size_t block_stride,
                                     void *d_crc_out, void *stream) {
	NvtxScope nvtx_scope("lzgpu::crc_blocks_dev");
	if (!ctx || !d_data || !d_crc_out) return LZGPU_ERR_ARG;
	if (block_len == 0 || block_len > LZGPU_BLOCK_SIZE || block_stride < block_len) { lz_set_error("crc_blocks: bad block_len/stride"); return LZGPU_ERR_ARG; }
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	if (!lzgpu_crc_enabled()) return fill_crc(ctx, d_crc_out, n_blocks, n_blocks, 1, st);
	if (block_len == LZGPU_BLOCK_SIZE && block_stride == LZGPU_BLOCK_SIZE) {
		int rc = lz_fused_crc(ctx, d_data, n_blocks, n_blocks, 0, d_crc_out, 0, st);
		if (rc != LZGPU_NOT_HANDLED) return rc;
	}
	return lz_crc_blocks(ctx, d_data, n_blocks, n_blocks, 0, block_stride, block_len, d_crc_out, 0, st);
}

extern "C" int lzgpu_crc_blocks(lzgpu_ctx *ctx, const uint8_t *data, size_t n_blocks, uint32_t block_len, size_t block_stride,
                                 uint32_t *crc_out) {
	NvtxScope nvtx_scope("lzgpu::crc_blocks");
	if (!ctx || !data || !crc_out) return LZGPU_ERR_ARG;
	if (block_len == 0 || block_len > LZGPU_BLOCK_SIZE || block_stride < block_len) { lz_set_error("crc_blocks: bad block_len/stride"); return LZGPU_ERR_ARG; }
	if (n_blocks == 0) return LZGPU_OK;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	const size_t dstride = (static_cast<size_t>(block_len) + 15) & ~size_t(15);
	const size_t per_tile = std::max<size_t>(1, kHostTileBytes / dstride);
	int rc;
	void *d_in[2], *d_c[2];
	for (int s = 0; s < 2; ++s) {
		if ((rc = lz_scratch(ctx, kScratchIn0 + s, std::min(per_tile, n_blocks) * dstride, &d_in[s]))) return rc;
		if ((rc = lz_scratch(ctx, kScratchCrc0 + s, std::min(per_tile, n_blocks) * 4, &d_c[s]))) return rc;
	}
	return run_tiles(ctx, n_blocks, per_tile, 2, nullptr, [&](int s, size_t b0, size_t n, cudaStream_t st, VerifyTicket *) -> int {
		CUDA_TRY(cudaMemcpy2DAsync(d_in[s], dstride, data + b0 * block_stride, block_stride, block_len, n, cudaMemcpyHostToDevice, st));
		int rc = lzgpu_crc_blocks_dev(ctx, d_in[s], n, block_len, dstride, d_c[s], st);
		if (rc) return rc;
		CUDA_TRY(cudaMemcpyAsync(crc_out + b0, d_c[s], n * 4, cudaMemcpyDeviceToHost, st));
		ctx->stats.bytes_h2d += n * block_len;
		ctx->stats.bytes_d2h += n * 4;
		return LZGPU_OK;
	});
}

static int verify_common(lzgpu_ctx *ctx, const uint8_t *h_data, size_t n_blocks, uint32_t block_len, size_t h_stride, size_t h_offset,
                         const uint32_t *h_stored, size_t stored_stride_bytes, int big_endian, int sparse_rule, int64_t *first_bad) {
	if (first_bad) *first_bad = -1;
	if (n_blocks == 0) return LZGPU_OK;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	cudaStream_t st = ctx->stream;
	const size_t dstride = (static_cast<size_t>(block_len) + 15) & ~size_t(15);
	// bounded staging: tiles of at most 1 GiB of block data, processed in order so the FIRST mismatch is reported
	const size_t per_tile = std::max<size_t>(1, (size_t(1) << 30) / dstride);
	const size_t tile_blocks = std::min(per_tile, n_blocks);
	void *d_in, *d_c, *d_s;
	int rc;
	if ((rc = lz_scratch(ctx, kScratchIn0, tile_blocks * dstride, &d_in))) return rc;
	if ((rc = lz_scratch(ctx, kScratchCrc0, tile_blocks * 4, &d_c))) return rc;
	if ((rc = lz_scratch(ctx, kScratchCrc0 + 1, tile_blocks * 4, &d_s))) return rc;
	VerifyTicket tk;  // one result word per tile: its first mismatching block, read back as block b of a single n-block "chunk"
	for (size_t b0 = 0; b0 < n_blocks; b0 += tile_blocks) {
		const size_t n = std::min(tile_blocks, n_blocks - b0);
		// cudaMemcpyDefault: the source may be host memory or (unified addressing) a device buffer, e.g. chunk files read straight
		// into device memory; either way the blocks land densely and 16-byte aligned in the staging tile the fused CRC kernel reads
		CUDA_TRY(cudaMemcpy2DAsync(d_in, dstride, h_data + h_offset + b0 * h_stride, h_stride, block_len, n, cudaMemcpyDefault, st));
		CUDA_TRY(cudaMemcpy2DAsync(d_s, 4, reinterpret_cast<const uint8_t *>(h_stored) + b0 * stored_stride_bytes, stored_stride_bytes, 4, n,
		                           cudaMemcpyDefault, st));
		if ((rc = tk.arm(ctx, st))) return rc;
		const int crc_off = lzgpu_crc_enabled() ? 0 : 1;
		if (crc_off && !sparse_rule) {
			crc_compare_const_kernel<<<grid_for(ctx, n, 256, 4), 256, 0, st>>>(static_cast<const uint32_t *>(d_s), n, LZGPU_FAKE_CRC, big_endian, tk.word(0));
			CUDA_TRY(cudaGetLastError());
			ctx->stats.kernel_launches++;
		} else {
			// (with CRCs disabled and the sparse rule on, the real CRCs are still needed to find the all-zero candidates)
			rc = LZGPU_NOT_HANDLED;
			if (block_len == LZGPU_BLOCK_SIZE && dstride == LZGPU_BLOCK_SIZE) rc = lz_fused_crc(ctx, d_in, n, n, 0, d_c, 0, st);
			if (rc == LZGPU_NOT_HANDLED) rc = lz_crc_blocks(ctx, d_in, n, n, 0, dstride, block_len, d_c, 0, st);
			if (rc) return rc;
			crc_compare_kernel<<<grid_for(ctx, n, 256, 4), 256, 0, st>>>(static_cast<const uint32_t *>(d_c), static_cast<const uint32_t *>(d_s), n,
			                                                            lz::crc_of_zeros(block_len), sparse_rule, big_endian, tk.word(0), crc_off);
			CUDA_TRY(cudaGetLastError());
			ctx->stats.kernel_launches++;
		}
		if (sparse_rule) {
			// holes accepted on their CRC are re-read and must really be all zero (crc.cc:235-243)
			const unsigned grid = static_cast<unsigned>(std::min<size_t>(n, static_cast<size_t>(ctx->sm_count) * 8));
			sparse_confirm_kernel<<<grid, 256, 0, st>>>(static_cast<const uint8_t *>(d_in), dstride, block_len, static_cast<const uint32_t *>(d_c),
			                                            static_cast<const uint32_t *>(d_s), n, lz::crc_of_zeros(block_len), tk.word(0));
			CUDA_TRY(cudaGetLastError());
			ctx->stats.kernel_launches++;
		}
		int64_t at[3];
		if ((rc = tk.publish_per_part(1, static_cast<uint32_t>(n)))) return rc;
		rc = tk.wait_take(at);
		if (rc && rc != LZGPU_ERR_CRC) return rc;
		ctx->stats.bytes_h2d += n * (block_len + 4ull);
		if (rc) {
			const unsigned long long bad = b0 + static_cast<unsigned long long>(at[2]);
			if (first_bad) *first_bad = static_cast<int64_t>(bad);
			lz_set_error("CRC mismatch in block %llu", bad);
			return LZGPU_ERR_CRC;
		}
	}
	return LZGPU_OK;
}

extern "C" int lzgpu_verify_blocks(lzgpu_ctx *ctx, const uint8_t *data, size_t n_blocks, uint32_t block_len, size_t block_stride,
                                    const uint32_t *stored_crc, int sparse_rule, int64_t *first_bad) {
	if (!ctx || !data || !stored_crc) return LZGPU_ERR_ARG;
	if (block_len == 0 || block_len > LZGPU_BLOCK_SIZE || block_stride < block_len) return LZGPU_ERR_ARG;
	return verify_common(ctx, data, n_blocks, block_len, block_stride, 0, stored_crc, 4, 0, sparse_rule, first_bad);
}

extern "C" int lzgpu_verify_interleaved(lzgpu_ctx *ctx, const uint8_t *records, size_t n_blocks, int64_t *first_bad) {
	if (!ctx || !records) return LZGPU_ERR_ARG;
	const size_t rec = 4 + LZGPU_BLOCK_SIZE;  // chunk.h:40 kDiskBlockSize
	return verify_common(ctx, records, n_blocks, LZGPU_BLOCK_SIZE, rec, 4, reinterpret_cast<const uint32_t *>(records), rec, 1, 1, first_bad);
}

// MooseFS chunk-file format (chunk.cc:126-190): 1 KiB signature block, then the table of big-endian block CRCs, then
// (for xor/ec parts: after padding to a 4 KiB disk block) the data blocks.  The reader of this format does not apply the
// sparse-block rule (hddspacemgr.cc:1746-1764).
extern "C" size_t lzgpu_moosefs_header_size(int data_parts) {
	if (data_parts < 1 || data_parts > LZGPU_MAX_DATA) return 0;
	const size_t max_blocks = (LZGPU_BLOCKS_IN_CHUNK + data_parts - 1) / data_parts;  // Chunk::maxBlocksInFile, chunk.cc:74-77
	const size_t required = 1024 + 4 * max_blocks;                                       // kMaxSignatureBlockSize + crc table
	return data_parts == 1 ? required : (required + 4095) / 4096 * 4096;                 // chunk.cc:169-181
}

extern "C" int lzgpu_verify_moosefs(lzgpu_ctx *ctx, int data_parts, const uint8_t *file_image, size_t n_blocks, int64_t *first_bad) {
	if (!ctx || !file_image) return LZGPU_ERR_ARG;
	const size_t hdr = lzgpu_moosefs_header_size(data_parts);
	if (!hdr || n_blocks > (LZGPU_BLOCKS_IN_CHUNK + data_parts - 1) / data_parts) return LZGPU_ERR_ARG;
	return verify_common(ctx, file_image, n_blocks, LZGPU_BLOCK_SIZE, LZGPU_BLOCK_SIZE, hdr, reinterpret_cast<const uint32_t *>(file_image + 1024), 4, 1, 0,
	                     first_bad);
}

// ------------------------------------------------------------------------------------------------
// chunkserver block writes (hdd_write, hddspacemgr.cc:1898-2008), batched
// ------------------------------------------------------------------------------------------------
static_assert(sizeof(BlockWrite) == sizeof(lzgpu_block_write) && offsetof(BlockWrite, status) == offsetof(lzgpu_block_write, status) &&
                  offsetof(BlockWrite, payload_off) == offsetof(lzgpu_block_write, payload_off),
              "device and ABI write descriptors must match");

extern "C" int lzgpu_write_blocks_dev(lzgpu_ctx *ctx, void *d_blocks, void *d_stored_crc, const void *d_payload, void *d_writes, uint32_t n_writes,
                                       int sparse_rule, void *stream) {
	NvtxScope nvtx_scope("lzgpu::write_blocks_dev");
	if (!ctx || !d_blocks || !d_stored_crc || !d_writes || (reinterpret_cast<uintptr_t>(d_blocks) & 15)) return LZGPU_ERR_ARG;
	if (!lzgpu_crc_enabled()) { lz_set_error("write_blocks: not available while CRCs are disabled (lzgpu_set_crc_enabled)"); return LZGPU_ERR_ARG; }
	if (n_writes == 0) return LZGPU_OK;
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	BlockWriteArgs a{};
	a.blocks = static_cast<uint8_t *>(d_blocks);
	a.stored_crc = static_cast<uint32_t *>(d_stored_crc);
	a.payload = static_cast<const uint8_t *>(d_payload);
	a.writes = static_cast<BlockWrite *>(d_writes);
	a.tables = ctx->d_crc_tables;
	lz::crc_xpow2_table(a.pow2);
	a.n_writes = n_writes;
	a.sparse_rule = sparse_rule;
	const unsigned grid = std::min<unsigned>(n_writes, static_cast<unsigned>(ctx->sm_count) * 8);
	block_write_kernel<<<grid, 256, 0, st>>>(a);
	CUDA_TRY(cudaGetLastError());
	ctx->stats.kernel_launches++;
	return LZGPU_OK;
}

extern "C" int lzgpu_write_blocks(lzgpu_ctx *ctx, uint8_t *blocks, uint32_t *stored_crc, size_t n_blocks, const uint8_t *payload, size_t payload_bytes,
                                   lzgpu_block_write *writes, uint32_t n_writes, int sparse_rule) {
	NvtxScope nvtx_scope("lzgpu::write_blocks");
	if (!ctx || !blocks || !stored_crc || !writes || (!payload && payload_bytes)) return LZGPU_ERR_ARG;
	if (n_writes == 0) return LZGPU_OK;
	const size_t B = LZGPU_BLOCK_SIZE;
	{
		// one write per block and call: the requests of a batch are independent, like the jobs of different chunks
		std::vector<uint32_t> seen(n_writes);
		for (uint32_t i = 0; i < n_writes; ++i) {
			if (writes[i].block >= n_blocks) { lz_set_error("write %u: block %u out of range", i, writes[i].block); return LZGPU_ERR_ARG; }
			if (writes[i].size <= B && writes[i].payload_off + writes[i].size > payload_bytes) { lz_set_error("write %u: payload out of range", i); return LZGPU_ERR_ARG; }
			seen[i] = writes[i].block;
		}
		std::sort(seen.begin(), seen.end());
		if (std::adjacent_find(seen.begin(), seen.end()) != seen.end()) { lz_set_error("write_blocks: two writes to the same block in one call"); return LZGPU_ERR_ARG; }
	}
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint32_t tile = std::min<uint32_t>(n_writes, 8192);
	void *d_blk, *d_crc, *d_pay, *d_wr;
	int rc;
	if ((rc = lz_scratch(ctx, kScratchIn0, tile * B, &d_blk))) return rc;
	if ((rc = lz_scratch(ctx, kScratchCrc0, tile * 4, &d_crc))) return rc;
	if ((rc = lz_scratch(ctx, kScratchPar0, std::max<size_t>(payload_bytes, 16), &d_pay))) return rc;
	if ((rc = lz_scratch(ctx, kScratchCrc0 + 1, tile * sizeof(lzgpu_block_write), &d_wr))) return rc;
	if (payload_bytes) CUDA_TRY(cudaMemcpyAsync(d_pay, payload, payload_bytes, cudaMemcpyHostToDevice, st));
	ctx->stats.bytes_h2d += payload_bytes;
	int first_error = LZGPU_OK;
	std::vector<lzgpu_block_write> local(tile);
	std::vector<uint32_t> crcs(tile);
	for (uint32_t w0 = 0; w0 < n_writes; w0 += tile) {
		const uint32_t n = std::min(tile, n_writes - w0);
		for (uint32_t i = 0; i < n; ++i) {
			const lzgpu_block_write &w = writes[w0 + i];
			local[i] = w;
			local[i].block = i;  // staged densely: slot i holds the block this write touches
			local[i].status = 0;
			crcs[i] = stored_crc[w.block];
			const bool partial = !(w.offset == 0 && w.size == B);
			if (w.exists && partial) {
				CUDA_TRY(cudaMemcpyAsync(static_cast<uint8_t *>(d_blk) + i * B, blocks + w.block * B, B, cudaMemcpyHostToDevice, st));
				ctx->stats.bytes_h2d += B;
			} else {
				local[i].exists = 0;  // a whole-block write never reads the stored block (hddspacemgr.cc:1920-1940)
			}
		}
		CUDA_TRY(cudaMemcpyAsync(d_crc, crcs.data(), n * 4, cudaMemcpyHostToDevice, st));
		CUDA_TRY(cudaMemcpyAsync(d_wr, local.data(), n * sizeof(lzgpu_block_write), cudaMemcpyHostToDevice, st));
		if ((rc = lzgpu_write_blocks_dev(ctx, d_blk, d_crc, d_pay, d_wr, n, sparse_rule, st))) return rc;
		CUDA_TRY(cudaMemcpyAsync(local.data(), d_wr, n * sizeof(lzgpu_block_write), cudaMemcpyDeviceToHost, st));
		CUDA_TRY(cudaMemcpyAsync(crcs.data(), d_crc, n * 4, cudaMemcpyDeviceToHost, st));
		CUDA_TRY(cudaStreamSynchronize(st));
		ctx->stats.bytes_d2h += n * (4 + sizeof(lzgpu_block_write));
		for (uint32_t i = 0; i < n; ++i) {
			lzgpu_block_write &w = writes[w0 + i];
			w.status = local[i].status;
			if (w.status != LZGPU_OK) {
				if (first_error == LZGPU_OK) {
					first_error = w.status;
					lz_set_error(w.status == LZGPU_ERR_CRC ? "write %u: payload CRC mismatch" : w.status == LZGPU_ERR_DAMAGED ? "write %u: stored block fails its CRC" : "write %u: bad offset/size", w0 + i);
				}
				continue;
			}
			// the caller's copy of the block is patched on the host: the bytes are the payload it already holds
			uint8_t *blk = blocks + w.block * B;
			if (!w.exists) std::memset(blk, 0, B);
			std::memcpy(blk + w.offset, payload + w.payload_off, w.size);
			stored_crc[w.block] = crcs[i];
		}
	}
	return first_error;
}

// ------------------------------------------------------------------------------------------------
// reference-shaped single calls (default context)
// ------------------------------------------------------------------------------------------------
// fragments -> device (dense, each padded to a 256-byte multiple), dot product, results back
static int fragments_dot(lzgpu_ctx *ctx, size_t len, int n_src, const uint8_t *const *src, int n_dst, uint8_t *const *dst,
                         const uint8_t *coef) {
	if (len == 0 || n_dst == 0) return LZGPU_OK;
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	cudaStream_t st = ctx->stream;
	const size_t stride = (len + 255) & ~size_t(255);
	void *d_buf;
	int rc;
	if ((rc = lz_scratch(ctx, kScratchIn0, stride * (n_src + n_dst), &d_buf))) return rc;
	uint8_t *base = static_cast<uint8_t *>(d_buf);
	DotDesc d{};
	std::vector<uint8_t *> dd(n_dst);
	for (int j = 0; j < n_src; ++j) {
		CUDA_TRY(cudaMemcpyAsync(base + stride * j, src[j], len, cudaMemcpyHostToDevice, st));
		d.src[j] = base + stride * j;
	}
	for (int r = 0; r < n_dst; ++r) dd[r] = base + stride * (n_src + r);
	d.dst = dd.data();
	d.n_src = n_src;
	d.n_dst = n_dst;
	d.units_per_block = static_cast<unsigned>((len + 15) / 16);
	d.blocks_per_chunk = 1;
	d.total_units = d.units_per_block;
	if ((rc = lz_gf_dot(ctx, d, coef, st))) return rc;
	for (int r = 0; r < n_dst; ++r) CUDA_TRY(cudaMemcpyAsync(dst[r], dd[r], len, cudaMemcpyDeviceToHost, st));
	CUDA_TRY(cudaStreamSynchronize(st));
	ctx->stats.bytes_h2d += len * n_src;
	ctx->stats.bytes_d2h += len * n_dst;
	return LZGPU_OK;
}

extern "C" void ec_encode_data(int len, int srcs, int dests, unsigned char *v, unsigned char **src, unsigned char **dest) {
	if (len <= 0 || dests <= 0) return;
	if (srcs < 1 || srcs > kMaxSrc || dests > LZGPU_MAX_PARTS || !v || !src || !dest) {
		lz_set_error("ec_encode_data: bad arguments (srcs=%d dests=%d)", srcs, dests);
		die("ec_encode_data", LZGPU_ERR_ARG);
	}
	lzgpu_ctx *ctx = need_default("ec_encode_data");
	// the coefficient of a 32-byte ISA-L table is its entry for the low nibble 1 (c*1)
	std::vector<uint8_t> coef(static_cast<size_t>(srcs) * dests);
	for (int i = 0; i < srcs * dests; ++i) coef[i] = v[32 * static_cast<size_t>(i) + 1];
	int rc = fragments_dot(ctx, static_cast<size_t>(len), srcs, src, dests, dest, coef.data());
	if (rc) die("ec_encode_data", rc);
}

extern "C" int lzgpu_rs_recover(int k, int m, const uint8_t *const *in, const uint8_t *erased, uint8_t *const *out, size_t size) {
	if (!in || !erased || !out) return LZGPU_ERR_ARG;
	if (k < 1 || k > LZGPU_MAX_DATA || m < 1 || m > LZGPU_MAX_PARITY) return LZGPU_ERR_ARG;
	lzgpu_ctx *ctx = lzgpu_default_ctx();
	if (!ctx) return LZGPU_ERR_NO_DEVICE;
	uint8_t wanted[LZGPU_MAX_PARTS] = {0}, rows[LZGPU_MAX_PARITY * LZGPU_MAX_DATA], reduced[LZGPU_MAX_PARITY * LZGPU_MAX_DATA];
	std::vector<uint8_t *> dst;
	for (int i = 0; i < k + m; ++i)
		if (erased[i] && out[i]) { wanted[i] = 1; dst.push_back(out[i]); }
	bool singular = false;
	int nrows = lz::rs_recovery_matrix(k, m, erased, wanted, rows, &singular);
	if (nrows < 0) { lz_set_error(singular ? "rs_recover: singular decode matrix" : "rs_recover: exactly m parts must be erased"); return LZGPU_ERR_ARG; }
	if (nrows == 0 || size == 0) return LZGPU_OK;
	// NULL inputs are all-zero parts: drop their columns (reed_solomon.h:104-110,202-209)
	std::vector<const uint8_t *> srcs;
	int col = 0, kept = 0;
	uint8_t keep[LZGPU_MAX_DATA];
	for (int i = 0; i < k + m; ++i) {
		if (erased[i]) continue;
		keep[col++] = in[i] != nullptr;
		if (in[i]) srcs.push_back(in[i]);
	}
	kept = static_cast<int>(srcs.size());
	if (kept == 0) {  // every input is zero: so is every output
		for (auto *p : dst) std::memset(p, 0, size);
		return LZGPU_OK;
	}
	for (int r = 0; r < nrows; ++r) {
		int c2 = 0;
		for (int c = 0; c < k; ++c)
			if (keep[c]) reduced[r * kept + c2++] = rows[r * k + c];
	}
	return fragments_dot(ctx, size, kept, srcs.data(), nrows, dst.data(), reduced);
}

extern "C" int lzgpu_rs_encode(int k, int m, const uint8_t *const *data, uint8_t *const *parity, size_t size) {
	if (!data || !parity) return LZGPU_ERR_ARG;
	if (k < 1 || k > LZGPU_MAX_DATA || m < 1 || m > LZGPU_MAX_PARITY) return LZGPU_ERR_ARG;
	const uint8_t *in[LZGPU_MAX_PARTS] = {nullptr};
	uint8_t *out[LZGPU_MAX_PARTS] = {nullptr};
	uint8_t erased[LZGPU_MAX_PARTS] = {0};
	for (int i = 0; i < k; ++i) in[i] = data[i];
	for (int r = 0; r < m; ++r) {
		if (!parity[r]) return LZGPU_ERR_ARG;  // reed_solomon.h:148
		erased[k + r] = 1;
		out[k + r] = parity[r];
	}
	return lzgpu_rs_recover(k, m, in, erased, out, size);
}

extern "C" void lzgpu_block_xor(uint8_t *dest, const uint8_t *source, size_t size) {
	if (size == 0) return;
	lzgpu_ctx *ctx = need_default("blockXor");
	std::lock_guard<std::mutex> lk(ctx->mu);
	DeviceGuard g(ctx->device);
	cudaStream_t st = ctx->stream;
	const size_t stride = (size + 255) & ~size_t(255);
	void *d_buf;
	int rc = lz_scratch(ctx, kScratchIn0, 2 * stride, &d_buf);
	if (rc) die("blockXor", rc);
	uint8_t *d0 = static_cast<uint8_t *>(d_buf), *d1 = d0 + stride;
	bool ok = cudaMemcpyAsync(d0, dest, size, cudaMemcpyHostToDevice, st) == cudaSuccess &&
	          cudaMemcpyAsync(d1, source, size, cudaMemcpyHostToDevice, st) == cudaSuccess;
	if (ok) {
		xor_inplace_kernel<<<grid_for(ctx, size / 16 + 16, 256, 8), 256, 0, st>>>(d0, d1, size / 16, static_cast<unsigned>(size % 16));
		ctx->stats.kernel_launches++;
		ok = cudaGetLastError() == cudaSuccess && cudaMemcpyAsync(dest, d0, size, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
		     cudaStreamSynchronize(st) == cudaSuccess;
	}
	if (!ok) {
		lz_set_error("CUDA: %s", cudaGetErrorString(cudaGetLastError()));
		die("blockXor", LZGPU_ERR_CUDA);
	}
}

extern "C" uint32_t lzgpu_mycrc32(uint32_t crc, const uint8_t *block, uint32_t leng) {
	if (!lzgpu_crc_enabled()) return LZGPU_FAKE_CRC;  // crc.cc:30-32
	if (leng == 0) return crc;
	lzgpu_ctx *ctx = need_default("mycrc32");
	// split into 64 KiB pieces (one warp each), then fold the pieces together with the
	// concatenation identity on the host
	const uint32_t B = LZGPU_BLOCK_SIZE;
	const size_t full = leng / B;
	const uint32_t tail = leng % B;
	std::vector<uint32_t> piece(full + 1);
	int rc = LZGPU_OK;
	if (full) rc = lzgpu_crc_blocks(ctx, block, full, B, B, piece.data());
	if (!rc && tail) rc = lzgpu_crc_blocks(ctx, block + full * B, 1, tail, tail, piece.data() + full);
	if (rc) die("mycrc32", rc);
	uint32_t acc = crc;
	for (size_t i = 0; i < full; ++i) acc = lz::crc_combine(acc, piece[i], B);
	if (tail) acc = lz::crc_combine(acc, piece[full], tail);
	return acc;
}

extern "C" void lzgpu_mycrc32_init(void) { (void)need_default("mycrc32_init"); }

extern "C" uint32_t lzgpu_mycrc32_zeroexpanded(uint32_t crc, const uint8_t *block, uint32_t leng, uint32_t zeros) {
	return lzgpu_mycrc32_zeroblock(lzgpu_mycrc32(crc, block, leng), zeros);
}

// crc.cc:235-243: a stored CRC of 0 on an all-zero block becomes the CRC of 64 KiB of zeros.  The block lives in
// host memory and the test is a plain zero scan (the reference uses memcmp), so it stays on the host; the batched
// equivalent on the GPU is the sparse_rule of lzgpu_verify_blocks / lzgpu_verify_interleaved.
extern "C" void lzgpu_recompute_crc_if_block_empty(const uint8_t *block, uint32_t *crc) {
	if (!block || !crc || *crc != 0) return;
	for (uint32_t i = 0; i < LZGPU_BLOCK_SIZE; ++i)
		if (block[i]) return;
	*crc = lz::crc_of_zeros(LZGPU_BLOCK_SIZE);
}

// ------------------------------------------------------------------------------------------------
// synthetic data + raw device helpers
// ------------------------------------------------------------------------------------------------
extern "C" int lzgpu_fill_chunks_dev(lzgpu_ctx *ctx, void *d_data, uint32_t n_chunks, size_t chunk_len, size_t chunk_stride, uint64_t seed,
                                      uint64_t first_chunk_index, void *stream) {
	if (!ctx || !d_data || (chunk_len & 7) || (chunk_stride & 7) || (reinterpret_cast<uintptr_t>(d_data) & 7)) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
	const unsigned long long wpc = chunk_len / 8, total = wpc * n_chunks;
	if (!total) return LZGPU_OK;
	fill_chunks_kernel<<<grid_for(ctx, total, 256, 8), 256, 0, st>>>(static_cast<uint8_t *>(d_data), chunk_stride, wpc, total, seed, first_chunk_index);
	CUDA_TRY(cudaGetLastError());
	return LZGPU_OK;
}

extern "C" int lzgpu_dev_alloc(lzgpu_ctx *ctx, size_t bytes, void **d_ptr) {
	if (!ctx || !d_ptr) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	cudaError_t e = cudaMalloc(d_ptr, bytes);
	if (e != cudaSuccess) { cudaGetLastError(); lz_set_error("cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e)); return LZGPU_ERR_NOMEM; }
	return LZGPU_OK;
}
extern "C" int lzgpu_dev_free(lzgpu_ctx *ctx, void *d_ptr) {
	if (!ctx) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	CUDA_TRY(cudaFree(d_ptr));
	return LZGPU_OK;
}
extern "C" int lzgpu_host_alloc(lzgpu_ctx *ctx, size_t bytes, void **h_ptr) {
	if (!ctx || !h_ptr) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	cudaError_t e = cudaHostAlloc(h_ptr, bytes, cudaHostAllocPortable);
	if (e != cudaSuccess) { cudaGetLastError(); lz_set_error("cudaHostAlloc(%zu): %s", bytes, cudaGetErrorString(e)); return LZGPU_ERR_NOMEM; }
	return LZGPU_OK;
}
extern "C" int lzgpu_host_free(lzgpu_ctx *ctx, void *h_ptr) {
	if (!ctx) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	CUDA_TRY(cudaFreeHost(h_ptr));
	return LZGPU_OK;
}
extern "C" int lzgpu_host_register(lzgpu_ctx *ctx, void *h_ptr, size_t bytes) {
	if (!ctx || !h_ptr || !bytes) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	cudaError_t e = cudaHostRegister(h_ptr, bytes, cudaHostRegisterPortable);
	if (e != cudaSuccess) { cudaGetLastError(); lz_set_error("cudaHostRegister(%zu): %s", bytes, cudaGetErrorString(e)); return LZGPU_ERR_CUDA; }
	return LZGPU_OK;
}
extern "C" int lzgpu_host_unregister(lzgpu_ctx *ctx, void *h_ptr) {
	if (!ctx || !h_ptr) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	CUDA_TRY(cudaHostUnregister(h_ptr));
	return LZGPU_OK;
}
extern "C" int lzgpu_dev_upload(lzgpu_ctx *ctx, void *d_dst, const void *h_src, size_t bytes) {
	if (!ctx) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	CUDA_TRY(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	return LZGPU_OK;
}
extern "C" int lzgpu_dev_download(lzgpu_ctx *ctx, void *h_dst, const void *d_src, size_t bytes) {
	if (!ctx) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	CUDA_TRY(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
	CUDA_TRY(cudaStreamSynchronize(ctx->stream));
	return LZGPU_OK;
}
extern "C" int lzgpu_ctx_set_deferred_verify(lzgpu_ctx *ctx, int enabled) {
	if (!ctx) return LZGPU_ERR_ARG;
	ctx->deferred_verify.store(enabled ? 1 : 0);
	return LZGPU_OK;
}
extern "C" int lzgpu_last_bad(lzgpu_ctx *ctx, int64_t *bad) {
	if (!ctx || !bad) return LZGPU_ERR_ARG;
	std::lock_guard<std::mutex> lk(ctx->pending_mu);
	bad[0] = ctx->last_bad[0]; bad[1] = ctx->last_bad[1]; bad[2] = ctx->last_bad[2];
	return LZGPU_OK;
}
extern "C" int lzgpu_dev_sync(lzgpu_ctx *ctx) {
	if (!ctx) return LZGPU_ERR_ARG;
	DeviceGuard g(ctx->device);
	CUDA_TRY(cudaDeviceSynchronize());
	// Deferred verdicts, in call order: the first mismatch is the one reported, every slot is returned.  Another thread may have
	// enqueued a deferred call and pushed its ticket after the device synchronisation began, so an idle device says nothing about
	// that call: each verdict is read only once its own result copy has completed.
	std::vector<VerifyTicket> mine;
	{
		std::lock_guard<std::mutex> lk(ctx->pending_mu);
		mine.swap(ctx->pending);
	}
	int rc = LZGPU_OK;
	int64_t first[3] = {-1, -1, -1};
	for (VerifyTicket &tk : mine) {
		int64_t bad[3] = {-1, -1, -1};
		const int r = tk.wait_copied_take(bad);
		if (r != LZGPU_OK && rc == LZGPU_OK) {
			rc = r;
			first[0] = bad[0]; first[1] = bad[1]; first[2] = bad[2];
		}
	}
	mine.clear();  // a ticket a CUDA error left armed waits for its stream here and returns its slot
	if (rc != LZGPU_OK) {
		std::lock_guard<std::mutex> lk(ctx->pending_mu);
		ctx->last_bad[0] = first[0]; ctx->last_bad[1] = first[1]; ctx->last_bad[2] = first[2];
	}
	return rc;
}
