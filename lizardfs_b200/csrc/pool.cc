// pool.cc — lzgpu_pool: ONE process driving several GPUs (include/lzgpu.h "device pool").
//
// The reference's callers are multi-threaded inside one process — ten write workers in the mount
// (src/mount/lizard_client.h:77, src/mount/writedata.cc:645), the chunkserver's background job pool — so the multi-GPU
// form of this engine that a drop-in needs is a pool of per-device contexts inside that process, not one process per GPU.
// Chunks are independent: a batch is cut into one contiguous run of chunks per device ("batch b -> device b", the static
// round-robin of chunk batches of BASELINE.json's north_star with a batch = ceil(n / devices) chunks); each run goes through
// the device's own 3-slot H2D | kernel | D2H pipeline on a worker thread that stays bound to that device.  No collective,
// no peer copy: the only cross-device state is the error code.
#include <cuda_runtime.h>

#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "engine_internal.h"
#include "lzgpu.h"
#include "slices_solve.h"

namespace {

struct Worker {
	lzgpu_ctx *ctx = nullptr;
	std::thread th;
	std::mutex mu;
	std::condition_variable cv;
	std::deque<std::function<void()>> q;
	bool stop = false;

	void loop() {
		cudaSetDevice(ctx->device);
		for (;;) {
			std::function<void()> job;
			{
				std::unique_lock<std::mutex> lk(mu);
				cv.wait(lk, [&] { return stop || !q.empty(); });
				if (q.empty()) return;
				job = std::move(q.front());
				q.pop_front();
			}
			job();
		}
	}
	void post(std::function<void()> f) {
		{
			std::lock_guard<std::mutex> lk(mu);
			q.push_back(std::move(f));
		}
		cv.notify_one();
	}
};

// completion latch of one pool call
struct Latch {
	std::mutex mu;
	std::condition_variable cv;
	int pending = 0;
	void done() {
		std::lock_guard<std::mutex> lk(mu);
		if (--pending == 0) cv.notify_all();
	}
	void wait() {
		std::unique_lock<std::mutex> lk(mu);
		cv.wait(lk, [&] { return pending == 0; });
	}
};

}  // namespace

struct lzgpu_pool {
	std::vector<Worker *> workers;
};

extern "C" void lzgpu_pool_destroy(lzgpu_pool *pool) {
	if (!pool) return;
	for (Worker *w : pool->workers) {
		if (w->th.joinable()) {
			{
				std::lock_guard<std::mutex> lk(w->mu);
				w->stop = true;
			}
			w->cv.notify_one();
			w->th.join();
		}
		lzgpu_ctx_destroy(w->ctx);
		delete w;
	}
	delete pool;
}

extern "C" int lzgpu_pool_create_list(const int *devices, int n_devices, lzgpu_pool **out) {
	if (!out || !devices || n_devices < 1 || n_devices > 64) return LZGPU_ERR_ARG;
	*out = nullptr;
	auto *pool = new lzgpu_pool();
	for (int i = 0; i < n_devices; ++i) {
		auto *w = new Worker();
		int rc = lzgpu_ctx_create(devices[i], &w->ctx);
		if (rc != LZGPU_OK) {
			delete w;
			lzgpu_pool_destroy(pool);
			return rc;
		}
		pool->workers.push_back(w);
		w->th = std::thread([w] { w->loop(); });
	}
	*out = pool;
	return LZGPU_OK;
}

extern "C" int lzgpu_pool_create(uint64_t device_mask, lzgpu_pool **out) {
	if (!out) return LZGPU_ERR_ARG;
	*out = nullptr;
	const int n = lzgpu_device_count();
	if (n <= 0) {
		lz_set_error("no CUDA device visible: liblzgpu has no CPU fallback");
		return LZGPU_ERR_NO_DEVICE;
	}
	std::vector<int> devs;
	for (int d = 0; d < n && d < 64; ++d)
		if (device_mask == 0 || (device_mask >> d) & 1) devs.push_back(d);
	if (devs.empty()) {
		lz_set_error("device mask 0x%llx selects none of the %d visible devices", static_cast<unsigned long long>(device_mask), n);
		return LZGPU_ERR_ARG;
	}
	return lzgpu_pool_create_list(devs.data(), static_cast<int>(devs.size()), out);
}

extern "C" int lzgpu_pool_size(const lzgpu_pool *pool) { return pool ? static_cast<int>(pool->workers.size()) : 0; }

extern "C" lzgpu_ctx *lzgpu_pool_ctx(lzgpu_pool *pool, int i) {
	if (!pool || i < 0 || i >= static_cast<int>(pool->workers.size())) return nullptr;
	return pool->workers[i]->ctx;
}

// which run of chunks device slot i of G takes: [first, first + count)
extern "C" void lzgpu_pool_share(uint32_t n_chunks, int n_devices, int i, uint32_t *first, uint32_t *count) {
	const uint32_t per = n_devices > 0 ? (n_chunks + n_devices - 1) / n_devices : n_chunks;
	const uint32_t f = std::min<uint64_t>(static_cast<uint64_t>(per) * i, n_chunks);
	if (first) *first = f;
	if (count) *count = std::min<uint32_t>(per, n_chunks - f);
}

// the codes and error texts of the shares of one pool call, by device slot
struct Shares {
	std::vector<int> rc;
	std::vector<std::string> err;
	int report(int i) const {  // slot i's code, with its text as the calling thread's lzgpu_last_error
		lz_set_error("device slot %d: %s", i, err[i].c_str());
		return rc[i];
	}
};

// run fn(worker index, first chunk, chunk count) on every device that gets a share and wait for all of them; an empty batch goes to
// slot 0 with a count of 0 (the calls that return early for one never get here)
static Shares pool_each(lzgpu_pool *pool, uint32_t n_chunks, const std::function<int(int, uint32_t, uint32_t)> &fn) {
	const int G = static_cast<int>(pool->workers.size());
	Shares sh{std::vector<int>(G, LZGPU_OK), std::vector<std::string>(G)};
	Latch latch;
	for (int i = 0; i < G; ++i) {
		uint32_t first, count;
		lzgpu_pool_share(n_chunks, G, i, &first, &count);
		if (count || (n_chunks == 0 && i == 0)) latch.pending++;
	}
	for (int i = 0; i < G; ++i) {
		uint32_t first, count;
		lzgpu_pool_share(n_chunks, G, i, &first, &count);
		if (!count && !(n_chunks == 0 && i == 0)) continue;
		pool->workers[i]->post([&, i, first, count] {
			sh.rc[i] = fn(i, first, count);
			if (sh.rc[i] != LZGPU_OK) sh.err[i] = lzgpu_last_error();  // thread-local text of the worker
			latch.done();
		});
	}
	latch.wait();
	return sh;
}

// pool_each, and the first error by device order wins
static int pool_run(lzgpu_pool *pool, uint32_t n_chunks, const std::function<int(int, uint32_t, uint32_t)> &fn) {
	const Shares sh = pool_each(pool, n_chunks, fn);
	for (size_t i = 0; i < sh.rc.size(); ++i)
		if (sh.rc[i] != LZGPU_OK) return sh.report(static_cast<int>(i));
	return LZGPU_OK;
}

extern "C" int lzgpu_pool_encode_chunks(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t chunk_len, const uint8_t *data,
                                         size_t chunk_stride, uint8_t *parity, size_t parity_stride, uint32_t *crc, size_t crc_stride) {
	if (!parity || !crc) return LZGPU_ERR_ARG;   // (refused for an empty batch too, which no context would see)
	return lzgpu_pool_encode_slices(pool, goal, 1, n_chunks, chunk_len, data, chunk_stride, &parity, &parity_stride, &crc, &crc_stride);
}

extern "C" int lzgpu_pool_encode_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t chunk_len,
                                         const uint8_t *data, size_t chunk_stride, uint8_t *const *parity, const size_t *parity_stride,
                                         uint32_t *const *crc, const size_t *crc_stride) {
	if (!pool || !goals || !data || !parity || !parity_stride || !crc || !crc_stride || n_slices < 1 || n_slices > 4) return LZGPU_ERR_ARG;
	if (n_chunks == 0) return LZGPU_OK;
	return pool_run(pool, n_chunks, [&](int i, uint32_t first, uint32_t count) {
		uint8_t *p[4] = {nullptr, nullptr, nullptr, nullptr};
		uint32_t *c[4] = {nullptr, nullptr, nullptr, nullptr};
		for (uint32_t s = 0; s < n_slices; ++s) {
			if (parity[s]) p[s] = parity[s] + static_cast<size_t>(first) * parity_stride[s];
			if (crc[s]) c[s] = crc[s] + static_cast<size_t>(first) * crc_stride[s];
		}
		return lzgpu_encode_slices(pool->workers[i]->ctx, goals, n_slices, count, chunk_len, data + static_cast<size_t>(first) * chunk_stride, chunk_stride,
		                           p, parity_stride, c, crc_stride);
	});
}

extern "C" int lzgpu_pool_recover_chunks(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *const *parts,
                                          size_t part_stride, const uint32_t *const *part_crc, const uint8_t *want, uint8_t *const *out,
                                          uint8_t *chunk_out, size_t chunk_out_stride, int64_t *bad) {
	if (!pool || !goal || !parts || !want) return LZGPU_ERR_ARG;
	if (goal->k < 1 || goal->k > LZGPU_MAX_DATA || goal->m < 0 || goal->m > LZGPU_MAX_PARITY) return LZGPU_ERR_ARG;
	if (n_chunks == 0) return LZGPU_OK;
	const int G = static_cast<int>(pool->workers.size()), n = goal->k + goal->m;
	const uint32_t pb = (nb + goal->k - 1) / goal->k;
	std::vector<int64_t> bads(static_cast<size_t>(G) * 3, -1);
	int rc = pool_run(pool, n_chunks, [&](int i, uint32_t first, uint32_t count) {
		std::vector<const uint8_t *> p(n, nullptr);
		std::vector<const uint32_t *> pc(n, nullptr);
		std::vector<uint8_t *> o(n, nullptr);
		for (int j = 0; j < n; ++j) {
			if (parts[j]) p[j] = parts[j] + static_cast<size_t>(first) * part_stride;
			if (part_crc && part_crc[j]) pc[j] = part_crc[j] + static_cast<size_t>(first) * pb;
			if (out && out[j]) o[j] = out[j] + static_cast<size_t>(first) * part_stride;
		}
		int r = lzgpu_recover_chunks(pool->workers[i]->ctx, goal, count, nb, p.data(), part_stride, part_crc ? pc.data() : nullptr, want,
		                             out ? o.data() : nullptr, chunk_out ? chunk_out + static_cast<size_t>(first) * chunk_out_stride : nullptr,
		                             chunk_out_stride, &bads[static_cast<size_t>(i) * 3]);
		if (r == LZGPU_ERR_CRC && bads[static_cast<size_t>(i) * 3] >= 0) bads[static_cast<size_t>(i) * 3] += first;
		return r;
	});
	if (rc == LZGPU_ERR_CRC && bad) {
		// lowest chunk index over the devices that reported a mismatch (shares are ascending runs of chunks)
		for (int i = 0; i < G; ++i)
			if (bads[static_cast<size_t>(i) * 3] >= 0) {
				std::memcpy(bad, &bads[static_cast<size_t>(i) * 3], 3 * sizeof(int64_t));
				break;
			}
	}
	return rc;
}

// Slice-type conversion (replication) over the devices of the pool: same arguments as lzgpu_convert_chunks, chunks dealt in runs
extern "C" int lzgpu_pool_convert_chunks(lzgpu_pool *pool, const lzgpu_goal *src, const lzgpu_goal *dst, uint32_t n_chunks, uint32_t nb,
                                          const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc, const uint8_t *want,
                                          uint8_t *const *out, size_t out_stride, uint32_t *const *out_crc, int64_t *bad) {
	if (!pool || !src || !dst || !parts || !want || !out) return LZGPU_ERR_ARG;
	if (src->k < 1 || src->k > LZGPU_MAX_DATA || src->m < 0 || src->m > LZGPU_MAX_PARITY || dst->k < 1 || dst->k > LZGPU_MAX_DATA || dst->m < 0 ||
	    dst->m > LZGPU_MAX_PARITY)
		return LZGPU_ERR_ARG;
	if (n_chunks == 0) return LZGPU_OK;
	const int G = static_cast<int>(pool->workers.size()), ns = src->k + src->m, nd = dst->k + dst->m;
	// blocks per chunk of a source / destination part (a standard slice has the single part 0 = the chunk itself)
	const uint32_t pbs = src->kind == LZGPU_KIND_STD ? nb : (nb + src->k - 1) / src->k, pbd = dst->kind == LZGPU_KIND_STD ? nb : (nb + dst->k - 1) / dst->k;
	std::vector<int64_t> bads(static_cast<size_t>(G) * 3, -1);
	int rc = pool_run(pool, n_chunks, [&](int i, uint32_t first, uint32_t count) {
		std::vector<const uint8_t *> p(ns, nullptr);
		std::vector<const uint32_t *> pc(ns, nullptr);
		std::vector<uint8_t *> o(nd, nullptr);
		std::vector<uint32_t *> oc(nd, nullptr);
		for (int j = 0; j < ns; ++j) {
			if (parts[j]) p[j] = parts[j] + static_cast<size_t>(first) * part_stride;
			if (part_crc && part_crc[j]) pc[j] = part_crc[j] + static_cast<size_t>(first) * pbs;
		}
		for (int j = 0; j < nd; ++j) {
			if (out[j]) o[j] = out[j] + static_cast<size_t>(first) * out_stride;
			if (out_crc && out_crc[j]) oc[j] = out_crc[j] + static_cast<size_t>(first) * pbd;
		}
		int r = lzgpu_convert_chunks(pool->workers[i]->ctx, src, dst, count, nb, p.data(), part_stride, part_crc ? pc.data() : nullptr, want, o.data(),
		                             out_stride, out_crc ? oc.data() : nullptr, &bads[static_cast<size_t>(i) * 3]);
		if (r == LZGPU_ERR_CRC && bads[static_cast<size_t>(i) * 3] >= 0) bads[static_cast<size_t>(i) * 3] += first;
		return r;
	});
	if (rc == LZGPU_ERR_CRC && bad) {
		for (int i = 0; i < G; ++i)
			if (bads[static_cast<size_t>(i) * 3] >= 0) {
				std::memcpy(bad, &bads[static_cast<size_t>(i) * 3], 3 * sizeof(int64_t));
				break;
			}
	}
	return rc;
}

extern "C" int lzgpu_pool_crc_blocks(lzgpu_pool *pool, const uint8_t *data, size_t n_blocks, uint32_t block_len, size_t block_stride,
                                      uint32_t *crc_out) {
	if (!pool || !data || !crc_out) return LZGPU_ERR_ARG;
	if (n_blocks == 0) return LZGPU_OK;
	if (n_blocks > 0xffffffffull) return LZGPU_ERR_ARG;
	return pool_run(pool, static_cast<uint32_t>(n_blocks), [&](int i, uint32_t first, uint32_t count) {
		return lzgpu_crc_blocks(pool->workers[i]->ctx, data + static_cast<size_t>(first) * block_stride, count, block_len, block_stride, crc_out + first);
	});
}

// ------------------------------------------------------------------------------------------------
// the chunkserver's stripe check, repair and decode and its block scrub over the pool (include/lzgpu.h "device pool")
// ------------------------------------------------------------------------------------------------
constexpr int64_t kUnset = INT64_MIN;  // a share's bad[0] before its call: the call wrote nothing there

// Run call(ctx, first, count, local_bad) on every share, every one to the end, and merge: a hard error (anything but LZGPU_OK,
// LZGPU_ERR_CRC and LZGPU_ERR_INCONSISTENT) wins by device slot, else LZGPU_ERR_CRC if any share returned it, else
// LZGPU_ERR_INCONSISTENT if any did, else LZGPU_OK: the precedence of the per-context calls.  bad[0 .. width-1] comes from the lowest
// slot that reported a position, with its first chunk (block) added to bad[0]: shares are ascending runs, so that is the position
// one context reports for the whole batch.  With none, the -1 a share wrote, or nothing when no share wrote (a refusal).
template <class Call>
static int pool_merged(lzgpu_pool *pool, uint32_t n_chunks, int64_t *bad, int width, Call &&call) {
	const int G = static_cast<int>(pool->workers.size());
	std::vector<int64_t> bads(static_cast<size_t>(G) * width, kUnset);
	const Shares sh = pool_each(pool, n_chunks, [&](int i, uint32_t first, uint32_t count) {
		return call(pool->workers[i]->ctx, first, count, bad ? &bads[static_cast<size_t>(i) * width] : nullptr);
	});
	if (bad) {
		auto at = [&](int i) { return bads[static_cast<size_t>(i) * width]; };
		int from = -1;
		for (int i = G - 1; i >= 0; --i)
			if (at(i) != kUnset) from = i;  // the lowest slot that wrote
		for (int i = G - 1; i >= 0; --i)
			if (at(i) >= 0) from = i;       // the lowest slot that reported a position
		if (from >= 0) {
			uint32_t first;
			lzgpu_pool_share(n_chunks, G, from, &first, nullptr);
			std::memcpy(bad, &bads[static_cast<size_t>(from) * width], width * sizeof(int64_t));
			if (bad[0] >= 0) bad[0] += first;
		}
	}
	for (int i = 0; i < G; ++i)
		if (sh.rc[i] != LZGPU_OK && sh.rc[i] != LZGPU_ERR_CRC && sh.rc[i] != LZGPU_ERR_INCONSISTENT) return sh.report(i);
	for (int code : {LZGPU_ERR_CRC, LZGPU_ERR_INCONSISTENT})
		for (int i = 0; i < G; ++i)
			if (sh.rc[i] == code) return sh.report(i);
	return LZGPU_OK;
}

// The part-batch calls: each share gets the part pointers moved by first * part_stride, the stored-CRC arrays by first * pb and `out`
// by first entries (per_stripe: first * pb).  Without parts, or with a goal or nb the per-context call refuses, the caller's arrays go
// through unmoved and every share refuses identically.
template <class P, class Out, class Call>
static int pool_part_batch(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, P *const *parts, size_t part_stride,
                           const uint32_t *const *part_crc, Out *out, bool per_stripe, int64_t *bad, Call &&call) {
	if (!pool) return LZGPU_ERR_ARG;
	const bool shaped = parts && lzgpu_goal_valid(goal) && nb >= 1 && nb <= LZGPU_BLOCKS_IN_CHUNK;
	const int n = shaped ? goal->k + goal->m : 0;
	const size_t pb = shaped ? (nb + goal->k - 1) / goal->k : 0;
	return pool_merged(pool, n_chunks, bad, 3, [&](lzgpu_ctx *ctx, uint32_t first, uint32_t count, int64_t *b) {
		P *p[LZGPU_MAX_PARTS];
		const uint32_t *c[LZGPU_MAX_PARTS];
		for (int j = 0; j < n; ++j) {
			p[j] = parts[j] ? parts[j] + first * part_stride : nullptr;
			c[j] = part_crc && part_crc[j] ? part_crc[j] + first * pb : nullptr;
		}
		return call(ctx, count, shaped ? p : parts, shaped && part_crc ? c : part_crc, out ? out + first * (per_stripe ? pb : 1) : nullptr, b);
	});
}

extern "C" int lzgpu_pool_check_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *const *parts,
                                         size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_verdict *verdict, int64_t *bad) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, verdict, false, bad,
	                       [&](lzgpu_ctx *ctx, uint32_t count, const uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_verdict *o, int64_t *b) {
		return lzgpu_check_stripes(ctx, goal, count, nb, p, part_stride, c, o, b);
	});
}

extern "C" int lzgpu_pool_check_stripe_map(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, const uint8_t *const *parts,
                                            size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_state *map, int64_t *bad) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, map, true, bad,
	                       [&](lzgpu_ctx *ctx, uint32_t count, const uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_state *o, int64_t *b) {
		return lzgpu_check_stripe_map(ctx, goal, count, nb, p, part_stride, c, o, b);
	});
}

extern "C" int lzgpu_pool_correct_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                           size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_fix *fix, int64_t *bad) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, fix, true, bad,
	                       [&](lzgpu_ctx *ctx, uint32_t count, uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_fix *o, int64_t *b) {
		return lzgpu_correct_stripes(ctx, goal, count, nb, p, part_stride, c, o, b);
	});
}

extern "C" int lzgpu_pool_check_stripe_map_degraded(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb,
                                                     const uint8_t *const *parts, size_t part_stride, const uint32_t *const *part_crc,
                                                     lzgpu_stripe_state *map, int64_t *bad) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, map, true, bad,
	                       [&](lzgpu_ctx *ctx, uint32_t count, const uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_state *o, int64_t *b) {
		return lzgpu_check_stripe_map_degraded(ctx, goal, count, nb, p, part_stride, c, o, b);
	});
}

extern "C" int lzgpu_pool_correct_stripes_degraded(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                                    size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_fix *fix, int64_t *bad) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, fix, true, bad,
	                       [&](lzgpu_ctx *ctx, uint32_t count, uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_fix *o, int64_t *b) {
		return lzgpu_correct_stripes_degraded(ctx, goal, count, nb, p, part_stride, c, o, b);
	});
}

extern "C" int lzgpu_pool_repair_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                          size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_repair *fix) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, fix, true, nullptr,
	                       [&](lzgpu_ctx *ctx, uint32_t count, uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_repair *o, int64_t *) {
		return lzgpu_repair_stripes(ctx, goal, count, nb, p, part_stride, c, o);
	});
}

extern "C" int lzgpu_pool_decode_stripes(lzgpu_pool *pool, const lzgpu_goal *goal, uint32_t n_chunks, uint32_t nb, uint8_t *const *parts,
                                          size_t part_stride, const uint32_t *const *part_crc, lzgpu_stripe_decode *fix) {
	return pool_part_batch(pool, goal, n_chunks, nb, parts, part_stride, part_crc, fix, true, nullptr,
	                       [&](lzgpu_ctx *ctx, uint32_t count, uint8_t *const *p, const uint32_t *const *c, lzgpu_stripe_decode *o, int64_t *) {
		return lzgpu_decode_stripes(ctx, goal, count, nb, p, part_stride, c, o);
	});
}

// One share of a multi-slice call: its first chunk, and shift(a, buf, step), the per-flat-part array a with part g moved by first *
// step[i] for its slice i (step NULL: not moved) in buf, or a itself when a is NULL or the per-context call refuses (not shaped)
struct SlicesShare {
	const lzd::SliceLayout &lay;
	bool shaped;
	uint32_t first;
	const size_t *pb;   // blocks per part of each slice
	size_t n_cs;        // combined stripes per chunk
	template <class T>
	T *const *shift(T *const *a, T **buf, const size_t *step) const {
		if (!shaped || !a) return a;
		for (uint32_t g = 0; g < lay.n_parts; ++g) buf[g] = a[g] ? a[g] + (step ? first * step[lay.slice_of(g)] : 0) : nullptr;
		return buf;
	}
};

// The multi-slice calls (lzgpu_recover_slices, _salvage_, _check_, _correct_) over the pool: each share gets slice i's part pointers
// moved by first * part_stride[i] and its stored-CRC arrays by first * pb_i (the flat layout of lzd::slice_layout); call(ctx, share,
// count, parts, part_crc, bad) moves the call's own arrays.  The codes and bad[0..3] are merged by pool_merged (a hard error, then
// LZGPU_ERR_CRC, then LZGPU_ERR_INCONSISTENT; bad from the lowest share).  With goals, nb or pointer arrays the per-context call
// refuses, the caller's arrays go through unmoved and every share refuses alike.
template <class P, class Call>
static int pool_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb, P *const *parts,
                       const size_t *part_stride, const uint32_t *const *part_crc, int64_t *bad, Call &&call) {
	if (!pool) return LZGPU_ERR_ARG;
	lzd::SliceLayout lay;
	const char *why = nullptr;
	const bool shaped = parts && part_stride && nb >= 1 && nb <= LZGPU_BLOCKS_IN_CHUNK && lzd::slice_layout(goals, n_slices, lay, &why) == LZGPU_OK;
	size_t pb[lzd::kSlicesMax] = {0};
	for (uint32_t i = 0; shaped && i < lay.n_slices; ++i) pb[i] = (nb + lay.k[i] - 1) / lay.k[i];
	const size_t n_cs = shaped ? (nb + lay.L - 1) / lay.L : 0;
	return pool_merged(pool, n_chunks, bad, 4, [&](lzgpu_ctx *ctx, uint32_t first, uint32_t count, int64_t *b) {
		const SlicesShare sh{lay, shaped, first, pb, n_cs};
		P *p[LZGPU_MAX_PARTS];
		const uint32_t *c[LZGPU_MAX_PARTS];
		return call(ctx, sh, count, sh.shift(parts, p, part_stride), sh.shift(part_crc, c, pb), b);
	});
}

// the image moves by first * chunk_out_stride, the wanted parts by first * out_stride[i] and their CRCs by first * pb_i
extern "C" int lzgpu_pool_recover_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                          const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                                          const uint8_t *want, uint8_t *const *out, const size_t *out_stride, uint32_t *const *out_crc,
                                          uint8_t *chunk_out, size_t chunk_out_stride, int64_t *bad) {
	return pool_slices(pool, goals, n_slices, n_chunks, nb, parts, part_stride, part_crc, bad,
	                   [&](lzgpu_ctx *ctx, const SlicesShare &sh, uint32_t count, const uint8_t *const *p, const uint32_t *const *c, int64_t *b) {
		uint8_t *o[LZGPU_MAX_PARTS];
		uint32_t *oc[LZGPU_MAX_PARTS];
		// without out_stride a wanted part is refused by every share, and an unwanted one is not touched
		return lzgpu_recover_slices(ctx, goals, n_slices, count, nb, p, part_stride, c, want, sh.shift(out, o, out_stride), out_stride,
		                            sh.shift(out_crc, oc, sh.pb), chunk_out ? chunk_out + sh.first * chunk_out_stride : nullptr,
		                            chunk_out_stride, b);
	});
}

// the image moves by first * image_stride, its CRCs and the map by first * nb
extern "C" int lzgpu_pool_salvage_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                          const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                                          uint8_t *image, size_t image_stride, uint32_t *image_crc, uint8_t *map, int64_t *bad) {
	return pool_slices(pool, goals, n_slices, n_chunks, nb, parts, part_stride, part_crc, bad,
	                   [&](lzgpu_ctx *ctx, const SlicesShare &sh, uint32_t count, const uint8_t *const *p, const uint32_t *const *c, int64_t *b) {
		const size_t at = static_cast<size_t>(sh.first) * nb;
		return lzgpu_salvage_slices(ctx, goals, n_slices, count, nb, p, part_stride, c, image ? image + sh.first * image_stride : nullptr,
		                            image_stride, image_crc ? image_crc + at : nullptr, map ? map + at : nullptr, b);
	});
}

// the map moves by first * n_cs
extern "C" int lzgpu_pool_check_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                        const uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                                        lzgpu_slices_check *map, int64_t *bad) {
	return pool_slices(pool, goals, n_slices, n_chunks, nb, parts, part_stride, part_crc, bad,
	                   [&](lzgpu_ctx *ctx, const SlicesShare &sh, uint32_t count, const uint8_t *const *p, const uint32_t *const *c, int64_t *b) {
		return lzgpu_check_slices(ctx, goals, n_slices, count, nb, p, part_stride, c, map && sh.shaped ? map + sh.first * sh.n_cs : map, b);
	});
}

// the new CRCs move by first * pb_i, the fix entries by first * n_cs
extern "C" int lzgpu_pool_correct_slices(lzgpu_pool *pool, const lzgpu_goal *goals, uint32_t n_slices, uint32_t n_chunks, uint32_t nb,
                                          uint8_t *const *parts, const size_t *part_stride, const uint32_t *const *part_crc,
                                          uint32_t *const *new_crc, lzgpu_slices_fix *fix, int64_t *bad) {
	return pool_slices(pool, goals, n_slices, n_chunks, nb, parts, part_stride, part_crc, bad,
	                   [&](lzgpu_ctx *ctx, const SlicesShare &sh, uint32_t count, uint8_t *const *p, const uint32_t *const *c, int64_t *b) {
		uint32_t *nc[LZGPU_MAX_PARTS];
		return lzgpu_correct_slices(ctx, goals, n_slices, count, nb, p, part_stride, c, sh.shift(new_crc, nc, sh.pb),
		                            fix && sh.shaped ? fix + sh.first * sh.n_cs : fix, b);
	});
}

// The scrub calls of a context also take device memory of its device; one device's memory cannot go to another device's context,
// so the pool refuses it before any share runs.  Asked on slot 0's device, so that no other device gets a context.
static int host_memory_only(lzgpu_pool *pool, const char *name, const void *a, const void *b) {
	int prev = 0;
	cudaGetDevice(&prev);
	cudaSetDevice(pool->workers[0]->ctx->device);
	bool device = false;
	for (const void *p : {a, b}) {
		cudaPointerAttributes attr;
		if (p && cudaPointerGetAttributes(&attr, p) == cudaSuccess) device |= attr.type == cudaMemoryTypeDevice;
	}
	cudaGetLastError();
	cudaSetDevice(prev);
	if (!device) return LZGPU_OK;
	lz_set_error("%s: device memory given; a pool scrubs host memory only", name);
	return LZGPU_ERR_ARG;
}

extern "C" int lzgpu_pool_verify_blocks(lzgpu_pool *pool, const uint8_t *data, size_t n_blocks, uint32_t block_len, size_t block_stride,
                                         const uint32_t *stored_crc, int sparse_rule, int64_t *first_bad) {
	if (!pool || n_blocks > 0xffffffffull) return LZGPU_ERR_ARG;
	const int rc = host_memory_only(pool, "pool_verify_blocks", data, stored_crc);
	if (rc) return rc;
	return pool_merged(pool, static_cast<uint32_t>(n_blocks), first_bad, 1, [&](lzgpu_ctx *ctx, uint32_t first, uint32_t count, int64_t *b) {
		return lzgpu_verify_blocks(ctx, data ? data + first * block_stride : nullptr, count, block_len, block_stride,
		                           stored_crc ? stored_crc + first : nullptr, sparse_rule, b);
	});
}

extern "C" int lzgpu_pool_verify_interleaved(lzgpu_pool *pool, const uint8_t *records, size_t n_blocks, int64_t *first_bad) {
	if (!pool || n_blocks > 0xffffffffull) return LZGPU_ERR_ARG;
	const int rc = host_memory_only(pool, "pool_verify_interleaved", records, nullptr);
	if (rc) return rc;
	return pool_merged(pool, static_cast<uint32_t>(n_blocks), first_bad, 1, [&](lzgpu_ctx *ctx, uint32_t first, uint32_t count, int64_t *b) {
		return lzgpu_verify_interleaved(ctx, records ? records + first * (4 + size_t(LZGPU_BLOCK_SIZE)) : nullptr, count, b);
	});
}

extern "C" void lzgpu_pool_get_stats(lzgpu_pool *pool, lzgpu_stats *out) {
	if (!pool || !out) return;
	std::memset(out, 0, sizeof(*out));
	double bytes_total = 0.0;
	for (Worker *w : pool->workers) {
		lzgpu_stats s;
		lzgpu_get_stats(w->ctx, &s);
		out->kernel_launches += s.kernel_launches;
		out->bytes_h2d += s.bytes_h2d;
		out->bytes_d2h += s.bytes_d2h;
		out->chunks_encoded += s.chunks_encoded;
		out->chunks_recovered += s.chunks_recovered;
		out->blocks_crc += s.blocks_crc;
		out->batches_timed += s.batches_timed;
		out->batch_ms_total += s.batch_ms_total;
		bytes_total += s.batch_gbps_mean * s.batch_ms_total * 1e6;
		if (s.batch_ms_last > 0.0) {
			out->batch_ms_last = s.batch_ms_last;
			out->batch_bytes_last = s.batch_bytes_last;
			out->batch_gbps_last = s.batch_gbps_last;
		}
	}
	// devices run concurrently: the mean rate of the pool is per-device mean x devices only if they overlap fully, so report
	// bytes / summed device time (a per-device mean) and leave aggregation over wall time to the caller
	out->batch_gbps_mean = out->batch_ms_total > 0.0 ? bytes_total / (out->batch_ms_total * 1e6) : 0.0;
}
