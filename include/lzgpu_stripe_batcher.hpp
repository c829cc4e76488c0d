// lzgpu_stripe_batcher.hpp — the mount's write path, batched (SURVEY.md §8 f4).
//
// The reference's ChunkWriter (src/mount/chunk_writer.cc) turns every combined stripe of the write journal into one
// "operation": startOperation (:475-547) completes the stripe (fillStripe, :437-466: blocks that were not written
// are READ from the chunkservers), computes each parity block with computeParityBlock (:365-401, one ReedSolomon
// object and one pass over the k data blocks per parity block) and hands every block to
// WriteExecutor::addDataPacket (src/common/write_executor.cc:91-107), which CRCs it (mycrc32, :97) and serialises
// the LIZ_CLTOCS_WRITE_DATA prefix (src/protocol/cltocs.h:116-137).
//
// StripeBatcher keeps the same unit — the combined stripe of L = lcm(k_i) blocks over every slice of the goal (a standard slice
// counts k = 1, :150-156) — and the same contract — a stripe is encoded only when all of its blocks are present, blocks that were
// read back are not sent again — but collects the complete stripes of any number of chunks in page-locked memory and encodes them
// in ONE GPU call: parity of every part of every slice, CRC of every data and parity block, and the 38-byte packet
// prefixes come back together; the sink receives exactly what addDataPacket would have been given for each part type (:488-545),
// plus the CRC and the finished prefix, so sending is a pointer hand-off.
//
// A goal of one xor/ec slice (L = k) passes its stripes to lzgpu_encode_chunks as k-block mini chunks, the flat-unit path of the
// one-slice encoder.  A goal of several slices (up to four: "std + xor2 + xor3", "ec(3,2) + ec(8,2)") passes them to
// lzgpu_encode_slices packed end to end into pseudo-chunks of up to
// 1024 blocks: L is a multiple of every k_i, so a run of s combined stripes is a valid chunk of s L blocks whose slice-i stripe t is
// slice stripe t % (L / k_i) of combined stripe t / (L / k_i), with that stripe's parity and CRCs byte for byte.  The one-pass kernel
// then plans the geometry of a whole chunk; one combined stripe per chunk would give it units of L blocks, which run slower than one
// call per slice (DESIGN.md §5).  Goals with L > 64 blocks (more than the 64-bit slot masks and the one-pass kernel take, e.g.
// "xor5 + ec(7,2) + xor9") are refused: batch their whole chunks through lzgpu_encode_slices instead.
//
// Sub-block operations (WriteCacheBlock::from / to, src/mount/write_cache_block.cc:64-68; startOperation takes block_from /
// block_to / block_size from the first block of the stripe and gives the parity blocks the same range,
// chunk_writer.cc:479-481,522-529) are batched as well: a stripe whose blocks cover [from, to) is staged as whole 64 KiB blocks
// that are zero outside the range.  GF(2^8) parity is byte-wise, so the whole-block parity is the range's parity inside
// [from, to) and zero outside; the CRC of the `to - from` bytes that travel comes from the whole-block CRC through the
// concatenation identity run backwards (lzgpu_mycrc32_subrange, host scalar).  The sink then receives offset = from,
// size = to - from, data = block + from and a prefix carrying that offset and size — what addDataPacket(writeId, block,
// from, size, data) is given in the reference.  The per-call path (computeParityBlock below) remains for callers that want a
// single stripe encoded at once.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "lzgpu.h"

namespace lzgpu {

// what WriteExecutor::addDataPacket receives (write id, block of the PART, offset 0, size 64 KiB, data), plus the results
struct PartBlock {
	uint64_t chunk_id;
	int slice;                 // index into the batcher's list of slices (0 for a one-goal batcher)
	int part;                  // this API's numbering within that slice: data 0..k-1, parity k..k+m-1; lzgpu_chunk_part_id(&slices[slice],
	                           // part) names the part type of an xor/ec slice, a standard slice has the one part 0
	uint32_t block;            // block index inside the part = slice stripe index (blockIndex / data_part_count, chunk_writer.cc:541)
	uint32_t write_id;
	uint32_t offset, size;     // byte range inside the block: 0 / 64 KiB for whole blocks, from / to - from for a sub-block stripe
	const uint8_t *data;       // `size` bytes (the block's bytes from `offset` on), valid until the next flush()/addBlock()
	uint32_t crc;              // mycrc32(0, data, size)
	const uint8_t *prefix;     // LZGPU_WRITE_PREFIX_SIZE bytes, ready to send in front of `data`
};

// ChunkWriter::computeParityBlock (src/mount/chunk_writer.cc:365-401) with the reference's arguments — the per-call path for
// what the batcher does not take (sub-block ranges: `size` < 64 KiB at the same offset in every block).  data_blocks[offset + i]
// is block i of the stripe, nullptr = a block that does not exist (zeros, :377,:396).  xorN: memcpy + blockXor == the all-ones row.
inline void computeParityBlock(const lzgpu_goal &goal, int parity_index, uint8_t *parity_block, const std::vector<uint8_t *> &data_blocks,
                               int offset, int size) {
	const uint8_t *in[LZGPU_MAX_PARTS] = {nullptr};
	uint8_t erased[LZGPU_MAX_PARTS] = {0};
	uint8_t *out[LZGPU_MAX_PARTS] = {nullptr};
	for (int i = 0; i < goal.k; ++i) in[i] = data_blocks[offset + i];
	for (int i = 0; i < goal.m; ++i) erased[goal.k + i] = 1;  // rs.recover with every parity part erased, one output (:386-400)
	out[goal.k + parity_index] = parity_block;
	if (lzgpu_rs_recover(goal.k, goal.m, in, erased, out, static_cast<size_t>(size)) != LZGPU_OK)
		throw std::runtime_error(std::string("computeParityBlock: ") + lzgpu_last_error());
}

class StripeBatcher {
public:
	typedef std::function<void(const PartBlock &)> Sink;

	// A goal of one xor/ec slice.
	StripeBatcher(lzgpu_ctx *ctx, const lzgpu_goal &goal, uint32_t max_stripes) { init(ctx, &goal, 1, max_stripes); }

	// A goal of 1..4 slices, each an xor/ec goal or the standard slice {LZGPU_KIND_STD, 1, 0}, at least one xor/ec, no slice type twice
	// (the reference writes every part type through one executor and chains the copies, chunk_writer.cc:140-147), and a combined
	// stripe of at most 64 blocks.  Anything else throws std::invalid_argument.  max_stripes: combined stripes buffered at once.
	// (A template only so that lzgpu_encode_slices is referenced where this constructor is used: a program that batches one-goal
	// stripes alone links against the entry points it always did.)
	template <class Goal, class = typename std::enable_if<std::is_same<Goal, lzgpu_goal>::value>::type>
	StripeBatcher(lzgpu_ctx *ctx, const Goal *slices, uint32_t n_slices, uint32_t max_stripes) : encode_slices_(lzgpu_encode_slices) {
		init(ctx, slices, n_slices, max_stripes);
	}
	~StripeBatcher() {
		lzgpu_host_free(ctx_, data_);
		for (uint32_t i = 0; i < n_slices_; ++i) {
			lzgpu_host_free(ctx_, parity_[i]);
			lzgpu_host_free(ctx_, crc_[i]);
		}
	}
	StripeBatcher(const StripeBatcher &) = delete;
	StripeBatcher &operator=(const StripeBatcher &) = delete;


	// ChunkWriter::addOperation for a whole block.  `read_back` marks a block fetched to complete a stripe
	// (WriteCacheBlock::kReadBlock): it takes part in the parity but is not handed to the sink (chunk_writer.cc:503-508).
	// A second write of the same block replaces the first.  Returns false when no stripe slot is free (flush first).
	bool addBlock(uint64_t chunk_id, uint32_t block_index, const uint8_t *data, bool read_back = false) {
		return addBlockRange(chunk_id, block_index, 0, LZGPU_BLOCK_SIZE, data, read_back);
	}

	// ChunkWriter::addOperation for bytes [from, to) of a block (`data` points at byte `from`).  Every block of a stripe must
	// carry the same range (the reference builds an operation from journal positions of one range, Operation::isExpandPossible):
	// a different range for a buffered stripe throws.
	bool addBlockRange(uint64_t chunk_id, uint32_t block_index, uint32_t from, uint32_t to, const uint8_t *data, bool read_back = false) {
		if (block_index >= LZGPU_BLOCKS_IN_CHUNK || !data || from >= to || to > LZGPU_BLOCK_SIZE)
			throw std::invalid_argument("StripeBatcher::addBlock: bad block or range");
		const Key key(chunk_id, block_index / L_);
		auto it = index_.find(key);
		if (it == index_.end()) {
			if (slots_.size() == capacity_) return false;
			Slot s;
			s.chunk_id = chunk_id;
			s.stripe = block_index / L_;
			// blocks past the end of the chunk do not exist: the last stripe of a chunk is complete without them
			// (range_end, chunk_writer.cc:449), and they enter the parity as zeros
			s.expected = std::min<uint32_t>(L_, LZGPU_BLOCKS_IN_CHUNK - s.stripe * L_);
			s.from = from;
			s.to = to;
			std::memset(slot_data(slots_.size()) + static_cast<size_t>(s.expected) * LZGPU_BLOCK_SIZE, 0,
			            static_cast<size_t>(L_ - s.expected) * LZGPU_BLOCK_SIZE);
			it = index_.emplace(key, static_cast<uint32_t>(slots_.size())).first;
			slots_.push_back(s);
		}
		Slot &s = slots_[it->second];
		if (s.from != from || s.to != to) throw std::invalid_argument("StripeBatcher::addBlock: the blocks of a stripe must cover the same byte range");
		const uint32_t j = block_index % L_;
		uint8_t *dst = slot_data(it->second) + static_cast<size_t>(j) * LZGPU_BLOCK_SIZE;
		if (from) std::memset(dst, 0, from);  // staged as a whole block that is zero outside the range
		std::memcpy(dst + from, data, to - from);
		if (to < LZGPU_BLOCK_SIZE) std::memset(dst + to, 0, LZGPU_BLOCK_SIZE - to);
		s.present |= 1ull << j;
		if (read_back) s.read_back |= 1ull << j;
		else s.read_back &= ~(1ull << j);
		return true;
	}

	// (chunk id, chunk block index) of every block still missing from a buffered stripe — what fillStripe would read
	std::vector<std::pair<uint64_t, uint32_t>> missingBlocks() const {
		std::vector<std::pair<uint64_t, uint32_t>> r;
		for (const Slot &s : slots_)
			for (uint32_t j = 0; j < s.expected; ++j)
				if (!(s.present >> j & 1)) r.emplace_back(s.chunk_id, s.stripe * L_ + j);
		return r;
	}

	size_t bufferedStripes() const { return slots_.size(); }

	// Encodes every COMPLETE stripe in one GPU call and hands its blocks to `sink`; incomplete stripes stay buffered.
	// Per stripe the sink gets, slice by slice and part by part, the blocks of ChunkWriter::startOperation: data part j of a slice
	// with k data parts every written block with blockIndex % k == j, a parity part one block per slice stripe whose first block
	// exists (:510-520).  Write ids are allocated consecutively from first_write_id (ChunkWriter::allocateId).  Returns the
	// number of stripes encoded; throws std::runtime_error on an engine failure (there is no CPU fallback).
	size_t flush(uint32_t first_write_id, const Sink &sink) {
		const size_t B = LZGPU_BLOCK_SIZE, stripe_bytes = L_ * B;
		// complete stripes to the front (stable for the incomplete ones)
		size_t n = 0;
		for (size_t i = 0; i < slots_.size(); ++i) {
			if (!complete(slots_[i])) continue;
			if (i != n) swap_slots(i, n);
			++n;
		}
		// the slots moved: the (chunk, stripe) -> slot map is rebuilt BEFORE anything can throw, so a failed encode leaves the
		// batcher consistent and a retry copies into the right stripe
		rebuild_index();
		if (n == 0) return 0;
		// q pseudo-chunks of s stripes: the incomplete stripes step aside for the zero padding stripes of the last one
		const Packing pk = packed(n);
		const size_t staged = pk.stripes(), rest = slots_.size() - n;
		if (staged != n) {
			std::memmove(slot_data(staged), slot_data(n), rest * stripe_bytes);
			std::memset(slot_data(n), 0, (staged - n) * stripe_bytes);
		}
		const uint32_t chunk_len = static_cast<uint32_t>(pk.s * stripe_bytes);
		uint8_t *parity[4];
		uint32_t *crc[4];
		size_t parity_stride[4], crc_stride[4];
		for (uint32_t i = 0; i < n_slices_; ++i) {
			const size_t pb = pk.s * (L_ / slices_[i].k);
			parity[i] = parity_[i];
			parity_stride[i] = slice_m(i) * pb * B;
			crc[i] = crc_[i];
			crc_stride[i] = pk.s * L_ + slice_m(i) * pb;
		}
		// one slice: n k-block chunks through the one-goal call (the one-slice case of lzgpu_encode_slices, same bytes)
		int rc = n_slices_ == 1 ? lzgpu_encode_chunks(ctx_, slices_, static_cast<uint32_t>(pk.q), chunk_len, data_, chunk_len, parity[0],
		                                               parity_stride[0], crc[0], crc_stride[0])
		                        : encode_slices_(ctx_, slices_, n_slices_, static_cast<uint32_t>(pk.q), chunk_len, data_, chunk_len, parity,
		                                         parity_stride, crc, crc_stride);
		if (staged != n) std::memmove(slot_data(n), slot_data(staged), rest * stripe_bytes);
		if (rc != LZGPU_OK) throw std::runtime_error(std::string("StripeBatcher::flush: ") + lzgpu_last_error());
		uint32_t write_id = first_write_id;
		uint8_t *px = prefix_.data();
		for (size_t g = 0; g < n; ++g) {
			const Slot &st = slots_[g];
			const size_t p = g / pk.s, c = g % pk.s;  // pseudo-chunk, stripe inside it
			for (uint32_t i = 0; i < n_slices_; ++i) {
				const int k = slices_[i].k, m = static_cast<int>(slice_m(i));
				const uint32_t per = L_ / k;
				const size_t pb = pk.s * per;
				const uint32_t *crc_c = crc[i] + p * crc_stride[i];
				for (int part = 0; part < k + m; ++part)
					for (uint32_t t = 0; t < per; ++t) {
						const uint32_t j = t * k + (part < k ? part : 0);  // data block of the combined stripe (a parity block's first)
						if (j >= st.expected || (part < k && (st.read_back >> j & 1))) continue;
						const size_t row = part < k ? c * L_ + j : pk.s * L_ + (part - k) * pb + c * per + t;  // in the CRC layout
						PartBlock pb_out;
						pb_out.chunk_id = st.chunk_id;
						pb_out.slice = static_cast<int>(i);
						pb_out.part = part;
						pb_out.block = st.stripe * per + t;
						pb_out.write_id = write_id++;
						pb_out.offset = st.from;
						pb_out.size = st.to - st.from;
						pb_out.data = (part < k ? slot_data(g) + j * B : parity[i] + p * parity_stride[i] + (row - pk.s * L_) * B) + st.from;
						// whole-block CRCs from the encoder
						pb_out.crc = (st.from == 0 && st.to == B) ? crc_c[row] : lzgpu_mycrc32_subrange(crc_c[row], st.from, st.to);
						write_prefix(px, st.chunk_id, pb_out.write_id, static_cast<uint16_t>(pb_out.block), pb_out.offset, pb_out.size, pb_out.crc);
						pb_out.prefix = px;
						px += LZGPU_WRITE_PREFIX_SIZE;
						sink(pb_out);
					}
			}
		}
		// drop the encoded stripes, keep the rest (moved to the front)
		std::vector<Slot> rest_slots(slots_.begin() + n, slots_.end());
		std::memmove(slot_data(0), slot_data(n), rest * stripe_bytes);
		slots_.swap(rest_slots);
		rebuild_index();
		return n;
	}

private:
	void init(lzgpu_ctx *ctx, const lzgpu_goal *slices, uint32_t n_slices, uint32_t max_stripes) {
		ctx_ = ctx;
		n_slices_ = n_slices;
		capacity_ = max_stripes;
		if (!ctx || !slices || n_slices < 1 || n_slices > 4 || max_stripes == 0) throw std::invalid_argument("StripeBatcher: bad arguments");
		uint32_t L = 1;
		bool any_striped = false;
		for (uint32_t i = 0; i < n_slices; ++i) {
			const lzgpu_goal &g = slices[i];
			const bool std_slice = g.kind == LZGPU_KIND_STD && g.k == 1 && g.m == 0;
			if (!std_slice && !lzgpu_goal_valid(&g)) throw std::invalid_argument("StripeBatcher: a slice is neither an xor/ec goal nor the standard slice");
			for (uint32_t j = 0; j < i; ++j)
				if (slices[j].kind == g.kind && slices[j].k == g.k && slices[j].m == g.m) throw std::invalid_argument("StripeBatcher: a slice type is repeated");
			any_striped |= !std_slice;
			slices_[i] = g;
			uint32_t a = L, b = static_cast<uint32_t>(g.k);
			while (b) { const uint32_t t = a % b; a = b; b = t; }
			L = L / a * static_cast<uint32_t>(g.k);
		}
		if (!any_striped) throw std::invalid_argument("StripeBatcher: no xor/ec slice");
		if (L > 64) throw std::invalid_argument("StripeBatcher: the combined stripe is longer than 64 blocks; encode whole chunks with lzgpu_encode_slices");
		L_ = L;
		// One slice passes one k-block chunk per stripe: the one-slice encoder's flat mode already runs a batch of such chunks as one
		// run of stripes across chunks.  The one-pass kernel of several slices has no such mode, so they pack up to 1024 / L stripes
		// into each chunk.
		per_chunk_ = n_slices == 1 ? 1 : LZGPU_BLOCKS_IN_CHUNK / L_;
		size_t padding = 0;  // the most padding stripes a flush of at most capacity_ stripes adds
		for (size_t n = 1; n <= capacity_; ++n) padding = std::max(padding, packed(n).stripes() - n);
		const size_t staged = capacity_ + padding, B = LZGPU_BLOCK_SIZE;
		alloc(reinterpret_cast<void **>(&data_), staged * L_ * B);
		size_t sink_blocks = 0;  // per combined stripe
		for (uint32_t i = 0; i < n_slices_; ++i) {
			const size_t m = slice_m(i), per = L_ / slices_[i].k;
			if (m) alloc(reinterpret_cast<void **>(&parity_[i]), staged * per * m * B);
			alloc(reinterpret_cast<void **>(&crc_[i]), staged * (L_ + per * m) * sizeof(uint32_t));
			sink_blocks += L_ + per * m;
		}
		prefix_.resize(static_cast<size_t>(capacity_) * sink_blocks * LZGPU_WRITE_PREFIX_SIZE);
		slots_.reserve(capacity_);
	}

	typedef std::pair<uint64_t, uint32_t> Key;  // (chunk id, combined stripe)
	struct Slot {
		uint64_t chunk_id = 0;
		uint32_t stripe = 0, expected = 0;
		uint32_t from = 0, to = LZGPU_BLOCK_SIZE;  // byte range every block of the stripe covers
		uint64_t present = 0, read_back = 0;  // bit j = block j of the combined stripe (L <= 64)
	};
	// A flush of n stripes passes q pseudo-chunks of s stripes: q = ceil(n / per_chunk_), s = ceil(n / q); the last q s - n < q
	// stripes are zero padding whose outputs are dropped.
	struct Packing {
		size_t q, s;
		size_t stripes() const { return q * s; }
	};
	Packing packed(size_t n) const {
		const size_t q = (n + per_chunk_ - 1) / per_chunk_;
		return Packing{q, (n + q - 1) / q};
	}

	void rebuild_index() {
		index_.clear();
		for (size_t i = 0; i < slots_.size(); ++i) index_.emplace(Key(slots_[i].chunk_id, slots_[i].stripe), static_cast<uint32_t>(i));
	}

	void alloc(void **p, size_t bytes) {
		if (lzgpu_host_alloc(ctx_, bytes, p) != LZGPU_OK) throw std::runtime_error(std::string("StripeBatcher: ") + lzgpu_last_error());
	}
	size_t slice_m(uint32_t i) const { return slices_[i].kind == LZGPU_KIND_STD ? 0 : static_cast<size_t>(slices_[i].m); }
	uint8_t *slot_data(size_t i) { return data_ + i * static_cast<size_t>(L_) * LZGPU_BLOCK_SIZE; }
	bool complete(const Slot &s) const { return s.present == (s.expected == 64 ? ~0ull : (1ull << s.expected) - 1); }
	void swap_slots(size_t a, size_t b) {
		const size_t bytes = static_cast<size_t>(L_) * LZGPU_BLOCK_SIZE;
		scratch_.resize(bytes);
		std::memcpy(scratch_.data(), slot_data(a), bytes);
		std::memcpy(slot_data(a), slot_data(b), bytes);
		std::memcpy(slot_data(b), scratch_.data(), bytes);
		std::swap(slots_[a], slots_[b]);
	}
	// cltocs::writeData::serializePrefix (src/protocol/cltocs.h:116-137): header (type 1212, length 30 + size), version 0,
	// chunkId, writeId, block, offset, size, crc — big-endian
	static void write_prefix(uint8_t *p, uint64_t chunk_id, uint32_t write_id, uint16_t block, uint32_t offset, uint32_t size, uint32_t crc) {
		auto be = [&p](uint64_t v, int bytes) {
			for (int i = bytes - 1; i >= 0; --i) *p++ = static_cast<uint8_t>(v >> (8 * i));
		};
		be(1212, 4); be(30u + size, 4); be(0, 4); be(chunk_id, 8); be(write_id, 4); be(block, 2); be(offset, 4);
		be(size, 4); be(crc, 4);
	}

	lzgpu_ctx *ctx_ = nullptr;
	lzgpu_goal slices_[4] = {};
	uint32_t n_slices_ = 0;
	uint32_t L_ = 0;                  // blocks per combined stripe
	uint32_t capacity_ = 0;
	decltype(&lzgpu_encode_slices) encode_slices_ = nullptr;  // set by the constructor that takes a list of slices
	size_t per_chunk_ = 1;            // most stripes per pseudo-chunk
	uint8_t *data_ = nullptr, *parity_[4] = {nullptr, nullptr, nullptr, nullptr};
	uint32_t *crc_[4] = {nullptr, nullptr, nullptr, nullptr};
	std::vector<uint8_t> prefix_, scratch_;
	std::vector<Slot> slots_;
	std::map<Key, uint32_t> index_;
};

}  // namespace lzgpu
