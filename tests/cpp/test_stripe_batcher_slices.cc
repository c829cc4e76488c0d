// Test of lzgpu::StripeBatcher (include/lzgpu_stripe_batcher.hpp) over goals of several slices: a slot is one combined stripe of
// L = lcm(k_i) blocks, a flush is one lzgpu_encode_slices call over pseudo-chunks of packed stripes, and the sink must receive
// exactly the blocks ChunkWriter::startOperation hands to addDataPacket (src/mount/chunk_writer.cc:475-547) for every part type of
// every slice.  The set of (slice, part, block) is computed here from that contract, independently of the batcher; every block is
// checked against the CPU oracle (oracle/lzoracle.h, linked by this test only): the slice stripe encoded as a k-block mini chunk,
// mycrc32 of the bytes sent, the serialized packet prefix.  Built twice: against liblzgpu.so (with the launch and geometry checks of
// the one-pass kernel) and, with LZ_TEST_CPU_BACKEND, against tests/cpp/oracle_backend.cc.  Exit code 0 = all passed.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <random>
#include <set>
#include <stdexcept>
#include <string>
#include <tuple>
#include <vector>

#include "lzgpu_stripe_batcher.hpp"
#include "../../oracle/lzoracle.h"

static int failures = 0;
#define EXPECT(cond)                                                        \
	do {                                                                    \
		if (!(cond)) {                                                      \
			std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); \
			++failures;                                                     \
		}                                                                   \
	} while (0)

static const uint32_t B = LZGPU_BLOCK_SIZE, NB = LZGPU_BLOCKS_IN_CHUNK;

struct GoalSet {
	std::string name;
	std::vector<lzgpu_goal> g;
	uint32_t L = 1;
};

static GoalSet goal_set(const std::vector<const char *> &names) {
	GoalSet s;
	for (const char *n : names) {
		lzgpu_goal g;
		EXPECT(lzgpu_goal_parse(n, &g) == LZGPU_OK);
		s.g.push_back(g);
		s.name += (s.name.empty() ? "" : "+") + std::string(n);
		uint32_t a = s.L, b = static_cast<uint32_t>(g.k);
		while (b) { const uint32_t t = a % b; a = b; b = t; }
		s.L = s.L / a * static_cast<uint32_t>(g.k);
	}
	return s;
}

typedef std::pair<uint64_t, uint32_t> BlockKey;  // (chunk, chunk block) or (chunk, combined stripe)

// what the batcher was given, as it stages it: whole blocks, zero outside the stripe's range
struct Store {
	std::map<BlockKey, std::vector<uint8_t>> blocks;
	std::set<BlockKey> read_back;
	std::map<BlockKey, std::pair<uint32_t, uint32_t>> range;  // per combined stripe
};

struct Seen {
	lzgpu::PartBlock pb;
	std::vector<uint8_t> data, prefix;
};

static void random_bytes(std::mt19937_64 &rng, uint8_t *p, size_t n) {
	for (size_t i = 0; i < n; i += 8) {
		const uint64_t v = rng();
		std::memcpy(p + i, &v, std::min<size_t>(8, n - i));
	}
}

// one block of the journal: bytes [from, to) of `payload` go to the batcher, the store keeps the whole staged block
static bool put(lzgpu::StripeBatcher &b, Store &st, const GoalSet &gs, uint64_t chunk, uint32_t block, const std::vector<uint8_t> &payload,
                bool read_back = false, uint32_t from = 0, uint32_t to = B) {
	const bool ok = from == 0 && to == B ? b.addBlock(chunk, block, payload.data(), read_back)
	                                     : b.addBlockRange(chunk, block, from, to, payload.data(), read_back);
	if (!ok) return false;
	std::vector<uint8_t> whole(B, 0);
	std::memcpy(whole.data() + from, payload.data(), to - from);
	st.blocks[{chunk, block}] = whole;
	if (read_back) st.read_back.insert({chunk, block});
	else st.read_back.erase({chunk, block});
	st.range[{chunk, block / gs.L}] = {from, to};
	return true;
}

static std::vector<uint8_t> random_block(std::mt19937_64 &rng, size_t n = B) {
	std::vector<uint8_t> v(n);
	random_bytes(rng, v.data(), n);
	return v;
}

typedef std::tuple<uint64_t, int, int, uint32_t> PartKey;  // chunk, slice, part, block of the part

// The blocks ChunkWriter::startOperation sends for combined stripe `cs` of `chunk` (chunk_writer.cc:488-545), derived here from the
// contract: data part j of a slice with k data parts gets every journal block with blockIndex % k == j that is not a read-back block,
// at part block blockIndex / k; a parity part gets one block per slice stripe i whose first block i k exists after fillStripe
// (i k < range_end = min(L, 1024 - first_block)), at part block (first_block + i k) / k.
static void expected_parts(const GoalSet &gs, const Store &st, uint64_t chunk, uint32_t cs, std::set<PartKey> &out) {
	const uint32_t first = cs * gs.L, range_end = std::min(gs.L, NB - first);
	for (size_t i = 0; i < gs.g.size(); ++i) {
		const lzgpu_goal &g = gs.g[i];
		const uint32_t k = static_cast<uint32_t>(g.k), m = g.kind == LZGPU_KIND_STD ? 0 : static_cast<uint32_t>(g.m);
		for (uint32_t b = first; b < first + gs.L; ++b)
			if (st.blocks.count({chunk, b}) && !st.read_back.count({chunk, b})) out.insert(PartKey(chunk, static_cast<int>(i), static_cast<int>(b % k), b / k));
		for (uint32_t s = 0; s < gs.L / k; ++s)
			if (s * k < range_end)
				for (uint32_t r = 0; r < m; ++r) out.insert(PartKey(chunk, static_cast<int>(i), static_cast<int>(k + r), (first + s * k) / k));
	}
}

// the oracle's view of one slice stripe: a k-block mini chunk (absent blocks zero) encoded by lzo_encode_chunk
struct MiniStripe {
	std::vector<uint8_t> data, parity;
	std::vector<uint32_t> crc;
};

static const MiniStripe &mini(std::map<PartKey, MiniStripe> &cache, const GoalSet &gs, const Store &st, uint64_t chunk, int slice, uint32_t t) {
	const PartKey key(chunk, slice, 0, t);
	auto it = cache.find(key);
	if (it != cache.end()) return it->second;
	const lzgpu_goal &g = gs.g[slice];
	MiniStripe ms;
	ms.data.assign(static_cast<size_t>(g.k) * B, 0);
	for (int j = 0; j < g.k; ++j) {
		auto b = st.blocks.find({chunk, t * g.k + j});
		if (b != st.blocks.end()) std::memcpy(&ms.data[static_cast<size_t>(j) * B], b->second.data(), B);
	}
	if (g.kind == LZGPU_KIND_STD) {
		ms.crc.push_back(lzo_crc32(0, ms.data.data(), B));
	} else {
		ms.parity.resize(static_cast<size_t>(g.m) * B);
		ms.crc.resize(g.k + g.m);
		EXPECT(lzo_encode_chunk(g.kind, g.k, g.m, ms.data.data(), ms.data.size(), ms.parity.data(), ms.crc.data()) == 0);
	}
	return cache.emplace(key, std::move(ms)).first->second;
}

// everything one flush handed to the sink, against the contract and the oracle
static void check_flush(const GoalSet &gs, const Store &st, const std::set<BlockKey> &stripes, const std::vector<Seen> &seen, uint32_t first_id) {
	std::set<PartKey> want;
	for (const BlockKey &s : stripes) expected_parts(gs, st, s.first, s.second, want);
	std::set<PartKey> got;
	std::map<PartKey, MiniStripe> cache;
	for (size_t n = 0; n < seen.size(); ++n) {
		const lzgpu::PartBlock &pb = seen[n].pb;
		EXPECT(pb.write_id == first_id + n);  // consecutive in sink order
		const PartKey key(pb.chunk_id, pb.slice, pb.part, pb.block);
		EXPECT(got.insert(key).second);
		EXPECT(pb.slice >= 0 && pb.slice < static_cast<int>(gs.g.size()));
		if (!want.count(key) || pb.slice < 0 || pb.slice >= static_cast<int>(gs.g.size())) continue;
		const lzgpu_goal &g = gs.g[pb.slice];
		const MiniStripe &ms = mini(cache, gs, st, pb.chunk_id, pb.slice, pb.block);
		const uint8_t *whole = pb.part < g.k ? &ms.data[static_cast<size_t>(pb.part) * B] : &ms.parity[static_cast<size_t>(pb.part - g.k) * B];
		const std::pair<uint32_t, uint32_t> r = st.range.at({pb.chunk_id, pb.block * g.k / gs.L});
		const uint32_t size = r.second - r.first;
		EXPECT(pb.offset == r.first && pb.size == size);
		EXPECT(seen[n].data.size() == size && std::memcmp(seen[n].data.data(), whole + r.first, size) == 0);
		EXPECT(pb.crc == lzo_crc32(0, whole + r.first, size));
		if (size == B) EXPECT(pb.crc == ms.crc[pb.part]);
		uint8_t prefix[LZO_WRITE_PREFIX_SIZE];
		lzo_write_data_prefix(prefix, pb.chunk_id, pb.write_id, static_cast<uint16_t>(pb.block), r.first, size, pb.crc);
		EXPECT(std::memcmp(seen[n].prefix.data(), prefix, sizeof(prefix)) == 0);
	}
	EXPECT(got == want);
	if (got != want) std::fprintf(stderr, "  %s: sink got %zu blocks, the contract gives %zu\n", gs.name.c_str(), got.size(), want.size());
}

struct Recorder {
	std::vector<Seen> seen;
	lzgpu::StripeBatcher::Sink sink() {
		return [this](const lzgpu::PartBlock &pb) {
			seen.push_back(Seen{pb, std::vector<uint8_t>(pb.data, pb.data + pb.size),
			                    std::vector<uint8_t>(pb.prefix, pb.prefix + LZGPU_WRITE_PREFIX_SIZE)});
		};
	}
};

// the pseudo-chunks a flush of n stripes passes, by the batcher's rule (one slice: n chunks of one stripe)
static void packing(const GoalSet &gs, size_t n, size_t &q, size_t &s) {
	const size_t per = gs.g.size() == 1 ? 1 : NB / gs.L;
	q = (n + per - 1) / per;
	s = (n + q - 1) / q;
}

static int plan_refusal(const GoalSet &gs, size_t n, lzgpu_slices_plan &pl) {
	size_t q, s;
	packing(gs, n, q, s);
	EXPECT(lzgpu_plan_encode_slices(gs.g.data(), static_cast<uint32_t>(gs.g.size()), static_cast<uint32_t>(q), static_cast<uint32_t>(s * gs.L), &pl) ==
	       LZGPU_OK);
	return pl.refusal;
}

// flushes and, on the GPU, checks that a fused flush of at most two pseudo-chunks (one staging tile) is one launch of the one-pass
// kernel at the geometry the planner gives the packed batch — the geometry of a whole chunk, not of one combined stripe
static size_t flush_checked(lzgpu::StripeBatcher &b, const GoalSet &gs, uint32_t first_id, Recorder &rec, size_t expect_n) {
#ifndef LZ_TEST_CPU_BACKEND
	lzgpu_stats before;
	lzgpu_get_stats(lzgpu_default_ctx(), &before);
#endif
	const size_t n = b.flush(first_id, rec.sink());
	EXPECT(n == expect_n);
#ifndef LZ_TEST_CPU_BACKEND
	lzgpu_slices_plan pl;
	size_t q, s;
	packing(gs, n, q, s);
	if (n && plan_refusal(gs, n, pl) == LZGPU_SLICES_FUSED && q <= 2) {
		lzgpu_stats after;
		lzgpu_get_stats(lzgpu_default_ctx(), &after);
		EXPECT(after.kernel_launches - before.kernel_launches == 1);
		lzgpu_launch_geometry geo;
		EXPECT(lzgpu_debug_last_geometry(lzgpu_default_ctx(), &geo) == LZGPU_OK);
		EXPECT(geo.kernel == LZGPU_KERNEL_ENCODE_SLICES);
		EXPECT(geo.G == pl.G);
	}
#endif
	return n;
}

// blocks of several chunks in random order: whole stripes, a read-back block, the last combined stripe of a full chunk, a rewritten
// block, a stripe held back until its last block arrives; then a full batcher
static void test_journal(const GoalSet &gs, unsigned seed) {
	std::mt19937_64 rng(seed);
	const uint32_t L = gs.L;
	lzgpu::StripeBatcher batcher(lzgpu_default_ctx(), gs.g.data(), static_cast<uint32_t>(gs.g.size()), 24);
	Store st;
	struct Item { uint64_t chunk; uint32_t block; bool read_back; };
	std::vector<Item> items;
	const uint64_t A = 0x1122334455667788ull;
	const uint32_t last = (NB - 1) / L;
	for (uint32_t s : {0u, 1u, 5u})
		for (uint32_t j = 0; j < L; ++j) items.push_back({A, s * L + j, s == 5 && (j == 0 || j == L / 2 + 1)});
	for (uint32_t b = last * L; b < NB; ++b) items.push_back({42, b, false});
	for (uint32_t j = 0; j < L; ++j) items.push_back({7, 3 * L + j, false});
	std::shuffle(items.begin(), items.end(), rng);
	const uint32_t held = 2 * L + L - 1;
	for (uint32_t j = 0; j + 1 < L; ++j) items.push_back({9, 2 * L + j, false});
	for (const Item &it : items) {
		std::vector<uint8_t> blk = random_block(rng);
		if (it.chunk == 42 && it.block == NB - 1) std::fill(blk.begin(), blk.end(), 0);
		EXPECT(put(batcher, st, gs, it.chunk, it.block, blk, it.read_back));
	}
	EXPECT(put(batcher, st, gs, 7, 3 * L + 1, std::vector<uint8_t>(B, 0x5a)));  // written again: replaces the first write
	const auto missing = batcher.missingBlocks();
	EXPECT(missing.size() == 1 && missing[0].first == 9 && missing[0].second == held);
	EXPECT(batcher.bufferedStripes() == 6);

	Recorder rec;
	EXPECT(flush_checked(batcher, gs, 1000, rec, 5) == 5);
	EXPECT(batcher.bufferedStripes() == 1);
	check_flush(gs, st, {{A, 0}, {A, 1}, {A, 5}, {42, last}, {7, 3}}, rec.seen, 1000);

	rec.seen.clear();
	EXPECT(put(batcher, st, gs, 9, held, random_block(rng)));
	EXPECT(batcher.missingBlocks().empty());
	EXPECT(flush_checked(batcher, gs, 5, rec, 1) == 1);
	EXPECT(batcher.bufferedStripes() == 0);
	check_flush(gs, st, {{9, 2}}, rec.seen, 5);
	EXPECT(batcher.flush(0, rec.sink()) == 0);

	// capacity: the 25th distinct stripe is refused until a flush; a block of a buffered stripe still goes in
	std::vector<uint8_t> blk(B, 1);
	for (uint32_t s = 0; s < 24; ++s) EXPECT(batcher.addBlock(100 + s, 0, blk.data()));
	EXPECT(!batcher.addBlock(999, 0, blk.data()));
	EXPECT(batcher.addBlock(100, L - 1, blk.data()));
	std::printf("journal %s: ok\n", gs.name.c_str());
}

// sub-block stripes: every block of a stripe carries [from, to), the parity blocks too; batched with whole-block stripes, the tail
// stripe of the chunk among them
static void test_sub_block(const GoalSet &gs, unsigned seed) {
	std::mt19937_64 rng(seed);
	const uint32_t L = gs.L, last = (NB - 1) / L;
	lzgpu::StripeBatcher batcher(lzgpu_default_ctx(), gs.g.data(), static_cast<uint32_t>(gs.g.size()), 8);
	Store st;
	struct Range { uint32_t stripe, from, to; };
	const Range ranges[] = {{0, 0, B}, {1, 0, 4096}, {2, 4096, B}, {3, 100, 101}, {4, 12345, 54321}, {last, 65535, B}};
	std::set<BlockKey> stripes;
	for (const Range &r : ranges) {
		for (uint32_t b = r.stripe * L; b < std::min((r.stripe + 1) * L, NB); ++b)
			EXPECT(put(batcher, st, gs, 77, b, random_block(rng, r.to - r.from), false, r.from, r.to));
		stripes.insert({77, r.stripe});
	}
	bool threw = false;
	try {
		std::vector<uint8_t> x(10);
		batcher.addBlockRange(77, L, 0, 10, x.data());
	} catch (const std::invalid_argument &) { threw = true; }
	EXPECT(threw);
	Recorder rec;
	EXPECT(flush_checked(batcher, gs, 9, rec, 6) == 6);
	check_flush(gs, st, stripes, rec.seen, 9);
	std::printf("sub-block stripes %s: ok\n", gs.name.c_str());
}

// more complete stripes than one pseudo-chunk holds (q >= 2, with zero padding), an incomplete stripe buffered in front of them
// that has to step aside for the padding and keep its data
static void test_packing(const GoalSet &gs, size_t n, unsigned seed) {
	std::mt19937_64 rng(seed);
	const uint32_t L = gs.L;
	size_t q, s;
	packing(gs, n, q, s);
	EXPECT(q >= 2 && q * s > n);
	lzgpu::StripeBatcher batcher(lzgpu_default_ctx(), gs.g.data(), static_cast<uint32_t>(gs.g.size()), static_cast<uint32_t>(n + 1));
	Store st;
	for (uint32_t j = 0; j + 1 < L; ++j) EXPECT(put(batcher, st, gs, 5, j, random_block(rng)));
	std::set<BlockKey> stripes;
	for (size_t g = 0; g < n; ++g) {
		const uint64_t chunk = 1000 + g / 7;
		const uint32_t cs = static_cast<uint32_t>(g % 7) * 3;
		for (uint32_t j = 0; j < L; ++j) EXPECT(put(batcher, st, gs, chunk, cs * L + j, random_block(rng)));
		stripes.insert({chunk, cs});
	}
	Recorder rec;
	EXPECT(flush_checked(batcher, gs, 0, rec, n) == n);
	check_flush(gs, st, stripes, rec.seen, 0);
	rec.seen.clear();
	EXPECT(batcher.bufferedStripes() == 1);
	EXPECT(put(batcher, st, gs, 5, L - 1, random_block(rng)));
	EXPECT(flush_checked(batcher, gs, 77, rec, 1) == 1);
	check_flush(gs, st, {{5, 0}}, rec.seen, 77);
	std::printf("packing %s, %zu stripes as %zu x %zu: ok\n", gs.name.c_str(), n, q, s);
}

// a one-slice list gives what the one-goal constructor gives
static void test_one_slice_list(const char *text, unsigned seed) {
	lzgpu_goal goal;
	EXPECT(lzgpu_goal_parse(text, &goal) == LZGPU_OK);
	lzgpu::StripeBatcher one(lzgpu_default_ctx(), goal, 16), list(lzgpu_default_ctx(), &goal, 1, 16);
	std::mt19937_64 rng(seed);
	for (uint32_t b = 0; b < 3u * goal.k; ++b) {
		const std::vector<uint8_t> blk = random_block(rng);
		EXPECT(one.addBlock(3, b, blk.data(), b == 1) && list.addBlock(3, b, blk.data(), b == 1));
	}
	const uint32_t tail = (NB - 1) / goal.k * goal.k;
	for (uint32_t b = tail; b < NB; ++b) {
		const std::vector<uint8_t> blk = random_block(rng, 1000);
		EXPECT(one.addBlockRange(4, b, 10, 1010, blk.data()) && list.addBlockRange(4, b, 10, 1010, blk.data()));
	}
	Recorder a, b;
	EXPECT(one.flush(50, a.sink()) == 4 && list.flush(50, b.sink()) == 4);
	EXPECT(a.seen.size() == b.seen.size());
	for (size_t i = 0; i < std::min(a.seen.size(), b.seen.size()); ++i) {
		const lzgpu::PartBlock &x = a.seen[i].pb, &y = b.seen[i].pb;
		EXPECT(x.chunk_id == y.chunk_id && x.slice == 0 && y.slice == 0 && x.part == y.part && x.block == y.block && x.write_id == y.write_id &&
		       x.offset == y.offset && x.size == y.size && x.crc == y.crc);
		EXPECT(a.seen[i].data == b.seen[i].data && a.seen[i].prefix == b.seen[i].prefix);
	}
	std::printf("one-slice list %s: ok\n", text);
}

static bool refused(const std::vector<const char *> &names) {
	std::vector<lzgpu_goal> g;
	for (const char *n : names) {
		lzgpu_goal x;
		EXPECT(lzgpu_goal_parse(n, &x) == LZGPU_OK);
		g.push_back(x);
	}
	try {
		lzgpu::StripeBatcher b(lzgpu_default_ctx(), g.data(), static_cast<uint32_t>(g.size()), 4);
	} catch (const std::invalid_argument &) { return true; }
	return false;
}

static void test_refusals() {
	EXPECT(refused({"xor2", "xor2"}));                   // repeated slice type
	EXPECT(refused({"std", "std", "xor3"}));
	EXPECT(refused({"xor9", "ec(8,2)"}));               // L = 72
	EXPECT(refused({"xor5", "ec(7,2)", "xor9"}));       // L = 315
	EXPECT(refused({"std"}));                           // no xor/ec slice
	EXPECT(refused({"xor2", "xor3", "xor4", "xor5", "std"}));  // five slices
	EXPECT(refused({}));
	const lzgpu_goal bad{LZGPU_KIND_XOR, 1, 1};
	bool threw = false;
	try {
		lzgpu::StripeBatcher b(lzgpu_default_ctx(), &bad, 1, 4);
	} catch (const std::invalid_argument &) { threw = true; }
	EXPECT(threw);
	EXPECT(!refused({"xor2", "xor3", "xor4", "xor5"}));  // L = 60
	EXPECT(!refused({"ec(32,2)"}));
	std::printf("refusals: ok\n");
}

#ifdef LZ_TEST_CPU_BACKEND
extern "C" int lzgpu_test_fail_next_encode;  // oracle_backend.cc: makes the next encode call fail
// a failed flush leaves the batcher consistent: the stripe map follows the reordered slots, and the incomplete stripe that stepped
// aside for the padding is back with its data, so the retry delivers every stripe with its own bytes
static void test_failed_flush(const GoalSet &gs) {
	std::mt19937_64 rng(17);
	const uint32_t L = gs.L;
	const size_t n = NB / L + 2;  // two pseudo-chunks with one padding stripe
	size_t q, s;
	packing(gs, n, q, s);
	EXPECT(q == 2 && q * s == n + 1);
	lzgpu::StripeBatcher batcher(lzgpu_default_ctx(), gs.g.data(), static_cast<uint32_t>(gs.g.size()), static_cast<uint32_t>(n + 1));
	Store st;
	for (uint32_t j = 0; j + 1 < L; ++j) EXPECT(put(batcher, st, gs, 1, j, random_block(rng)));
	std::set<BlockKey> stripes{{1, 0}};
	for (size_t g = 0; g < n; ++g) {
		for (uint32_t j = 0; j < L; ++j) EXPECT(put(batcher, st, gs, 2 + g, 4 * L + j, random_block(rng)));
		stripes.insert({2 + g, 4});
	}
	lzgpu_test_fail_next_encode = 1;
	bool threw = false;
	try {
		batcher.flush(0, [](const lzgpu::PartBlock &) {});
	} catch (const std::runtime_error &) { threw = true; }
	EXPECT(threw);
	EXPECT(batcher.bufferedStripes() == n + 1);
	EXPECT(put(batcher, st, gs, 1, L - 1, random_block(rng)));
	Recorder rec;
	EXPECT(batcher.flush(3, rec.sink()) == n + 1);
	check_flush(gs, st, stripes, rec.seen, 3);
	std::printf("failed flush %s: ok\n", gs.name.c_str());
}
#endif

int main() {
	if (!lzgpu_default_ctx()) {
		std::fprintf(stderr, "no GPU context: %s\n", lzgpu_last_error());
		return 2;
	}
	struct Case { std::vector<const char *> names; int refusal; };
	const Case cases[] = {
	    {{"std", "xor2", "xor3"}, LZGPU_SLICES_FUSED},          // L 6
	    {{"ec(3,2)", "ec(8,2)"}, LZGPU_SLICES_FUSED},           // L 24
	    {{"xor2", "ec(8,4)"}, LZGPU_SLICES_FUSED},              // L 8, m 4
	    {{"ec(5,3)", "xor2"}, LZGPU_SLICES_FUSED},              // L 10, tail of 4
	    {{"xor2", "xor3", "xor4", "xor5"}, LZGPU_SLICES_FUSED}, // L 60
	    {{"std", "ec(8,2)"}, LZGPU_SLICES_REFUSED_SINGLE},
	    {{"ec(4,2)", "ec(4,5)"}, LZGPU_SLICES_REFUSED_CAUCHY},
	};
	unsigned seed = 1;
	for (const Case &c : cases) {
		const GoalSet gs = goal_set(c.names);
		lzgpu_slices_plan pl;
		EXPECT(plan_refusal(gs, 5, pl) == c.refusal);
		test_journal(gs, seed++);
		test_sub_block(gs, seed++);
	}
	test_packing(goal_set({"ec(3,2)", "ec(8,2)"}), 43, 101);     // 2 x 22, one padding stripe
	test_packing(goal_set({"std", "xor2", "xor3"}), 171, 102);   // 2 x 86, one padding stripe
	test_packing(goal_set({"ec(4,2)", "ec(4,5)"}), 257, 103);    // the per-slice route, 2 x 129
	test_one_slice_list("ec(5,3)", 7);
	test_one_slice_list("xor3", 8);
	test_refusals();
#ifdef LZ_TEST_CPU_BACKEND
	test_failed_flush(goal_set({"xor2", "xor3", "xor4", "xor5"}));
#endif
	if (failures) {
		std::fprintf(stderr, "%d failure(s)\n", failures);
		return 1;
	}
	std::printf("stripe batcher over several slices: all tests passed\n");
	return 0;
}
