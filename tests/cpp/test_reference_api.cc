// C++ restatement of the reference's unit tests for the hot path, linked against liblzgpu.so through the
// reference-named interfaces: ReedSolomon<32,32> (include/lzgpu_reed_solomon.hpp), mycrc32 /
// mycrc32_combine / blockXor with C++ linkage (lizardfs_b200/csrc/compat_cxx.cc) and the ISA-L names.
// Mirrors src/common/reed_solomon_unittest.cc:136-199, crc_unittest.cc:27-63, block_xor_unittest.cc:24-35.
// Exit code 0 = all passed.  Needs an H100 (run by tests/test_gpu_cpp.py).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "lzgpu_reed_solomon.hpp"

uint32_t mycrc32(uint32_t crc, const uint8_t *block, uint32_t leng);
uint32_t mycrc32_combine(uint32_t crc1, uint32_t crc2, uint32_t leng2);
void mycrc32_init(void);
void blockXor(uint8_t *dest, const uint8_t *source, size_t size);
#define mycrc32_zeroblock(crc, zeros) mycrc32_combine((crc) ^ 0xFFFFFFFF, 0xFFFFFFFF, (zeros))

static int failures = 0;
#define EXPECT(cond)                                                        \
	do {                                                                    \
		if (!(cond)) {                                                      \
			std::fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); \
			++failures;                                                     \
		}                                                                   \
	} while (0)

typedef ReedSolomon<32, 32> RS;

static void fill(std::vector<uint8_t> &v, unsigned seed) {
	uint64_t s = 0x9E3779B97F4A7C15ull * (seed + 1);
	for (auto &b : v) {
		s ^= s << 13; s ^= s >> 7; s ^= s << 17;
		b = static_cast<uint8_t>(s >> 24);
	}
}

static void test_recovery(int k, int m, std::vector<int> erase, bool with_zero_parts) {
	const size_t size = 64 * 1024;
	std::vector<std::vector<uint8_t>> parts(k + m, std::vector<uint8_t>(size));
	RS::ConstFragmentMap in{{0}};
	RS::FragmentMap par{{0}};
	for (int i = 0; i < k; ++i) {
		if (with_zero_parts && i % 3 == 0) std::fill(parts[i].begin(), parts[i].end(), 0);
		else fill(parts[i], i);
		in[i] = (with_zero_parts && i % 3 == 0) ? nullptr : parts[i].data();  // NULL = all-zero part
	}
	for (int i = 0; i < m; ++i) par[i] = parts[k + i].data();
	RS rs(k, m);
	rs.encode(in, par, size);

	RS::ErasedMap erased;
	RS::ConstFragmentMap avail{{0}};
	RS::FragmentMap out{{0}};
	std::vector<std::vector<uint8_t>> rec(k + m, std::vector<uint8_t>(size, 0xAA));
	for (int e : erase) erased.set(e);
	for (int i = 0; i < k + m; ++i) {
		if (erased[i]) out[i] = rec[i].data();
		else avail[i] = (i < k) ? in[i] : parts[i].data();
	}
	rs.recover(avail, erased, out, size);
	for (int e : erase) EXPECT(std::memcmp(rec[e].data(), parts[e].data(), size) == 0);
}

int main() {
	mycrc32_init();
	// crc_unittest.cc:27-41
	std::vector<std::pair<std::string, uint32_t>> kat{{"a", 0xE8B7BE43}, {"aa", 0x78A19D7}, {"aaaa", 0xAD98E545},
	                                                  {"aaaaaaaa", 0xBF848046}, {std::string(16, 'a'), 0xCFD668D5},
	                                                  {std::string(32, 'a'), 0xCAB11777}, {std::string(64, 'a'), 0x89B46555}};
	for (auto &p : kat) EXPECT(mycrc32(0, reinterpret_cast<const uint8_t *>(p.first.data()), p.first.size()) == p.second);
	// crc_unittest.cc:43-46
	std::vector<uint8_t> zeros(LZGPU_BLOCK_SIZE);
	EXPECT(mycrc32(0, zeros.data(), LZGPU_BLOCK_SIZE) == mycrc32_zeroblock(0, LZGPU_BLOCK_SIZE));
	// crc_unittest.cc:48-63
	std::vector<uint8_t> data(LZGPU_BLOCK_SIZE);
	for (size_t i = 0; i < data.size(); ++i) data[i] = static_cast<uint8_t>(i);
	const uint32_t crc = mycrc32(0, data.data(), data.size());
	for (size_t length = 2; length < LZGPU_BLOCK_SIZE; length *= 2)
		for (int off : {-1, 0, 1}) {
			const uint32_t n = static_cast<uint32_t>(length + off);
			const uint32_t c1 = mycrc32(0, data.data(), data.size() - n);
			const uint32_t c2 = mycrc32(0, data.data() + data.size() - n, n);
			EXPECT(mycrc32_combine(c1, c2, n) == crc);
		}
	// block_xor_unittest.cc:24-35 (plus a value check)
	std::vector<uint8_t> a(LZGPU_BLOCK_SIZE + 64), b(LZGPU_BLOCK_SIZE + 64), want;
	fill(a, 100); fill(b, 101);
	for (int oa : {0, 1, 7, 16})
		for (int ob : {0, 3, 16}) {
			std::vector<uint8_t> d(a.begin() + oa, a.begin() + oa + LZGPU_BLOCK_SIZE);
			want = d;
			for (size_t i = 0; i < want.size(); ++i) want[i] ^= b[ob + i];
			blockXor(d.data(), b.data() + ob, LZGPU_BLOCK_SIZE);
			EXPECT(d == want);
		}
	// reed_solomon_unittest.cc:136-166 and :168-199
	test_recovery(4, 2, {0, 2}, false);
	test_recovery(4, 2, {0, 5}, false);
	test_recovery(4, 2, {4, 5}, false);
	test_recovery(8, 2, {1, 4}, true);
	test_recovery(32, 32, {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 32, 33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47}, false);
	if (failures) {
		std::fprintf(stderr, "%d check(s) failed\n", failures);
		return 1;
	}
	std::printf("reference-API C++ tests passed\n");
	return 0;
}
