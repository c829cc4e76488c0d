// gtest.h — a few dozen lines standing in for <gtest/gtest.h> (googletest is not in this image) so that the REFERENCE'S OWN
// unit-test sources (src/common/*_unittest.cc, compiled where they lie under /root/reference) build unmodified against
// liblzgpu.so: oracle/Makefile target _ref/test_link_substitution.  Only what those files use: TEST, EXPECT_/ASSERT_ EQ, NE,
// TRUE, FALSE, GE, NO_THROW with optional `<< message`.  main() is in tests/cpp/link_substitution_main.cc.
#pragma once
#include <functional>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

namespace testing {

struct TestCase {
	std::string suite, name;
	std::function<void()> body;
};
inline std::vector<TestCase> &registry() {
	static std::vector<TestCase> r;
	return r;
}
inline int &failures() {
	static int f = 0;
	return f;
}
struct Registrar {
	Registrar(const char *s, const char *n, std::function<void()> b) { registry().push_back(TestCase{s, n, std::move(b)}); }
};

// collects the optional streamed message and reports on destruction
struct Reporter {
	bool failed;
	std::ostringstream msg;
	Reporter(bool f, const char *file, int line, const char *expr) : failed(f) {
		if (failed) msg << file << ":" << line << ": Failure: " << expr << " ";
	}
	~Reporter() {
		if (failed) {
			std::cerr << msg.str() << "\n";
			++failures();
		}
	}
	template <typename T>
	Reporter &operator<<(const T &v) {
		if (failed) msg << v;
		return *this;
	}
};
struct FatalVoid {  // lets ASSERT_* `return` from a void test body after the message has been streamed
	void operator=(const Reporter &) const {}
};

class Test {};

}  // namespace testing

#define TEST(suite, name)                                                                                  \
	static void lz_test_##suite##_##name();                                                                 \
	static ::testing::Registrar lz_reg_##suite##_##name(#suite, #name, lz_test_##suite##_##name);           \
	static void lz_test_##suite##_##name()

#define LZ_EXPECT_(cond, text) ::testing::Reporter(!(cond), __FILE__, __LINE__, text)
#define LZ_ASSERT_(cond, text) \
	if (cond) {                \
	} else                     \
		return ::testing::FatalVoid() = ::testing::Reporter(true, __FILE__, __LINE__, text)

#define EXPECT_TRUE(c) LZ_EXPECT_(static_cast<bool>(c), "EXPECT_TRUE(" #c ")")
#define EXPECT_FALSE(c) LZ_EXPECT_(!static_cast<bool>(c), "EXPECT_FALSE(" #c ")")
#define EXPECT_EQ(a, b) LZ_EXPECT_((a) == (b), "EXPECT_EQ(" #a ", " #b ")")
#define EXPECT_NE(a, b) LZ_EXPECT_((a) != (b), "EXPECT_NE(" #a ", " #b ")")
#define EXPECT_GE(a, b) LZ_EXPECT_((a) >= (b), "EXPECT_GE(" #a ", " #b ")")
#define EXPECT_LE(a, b) LZ_EXPECT_((a) <= (b), "EXPECT_LE(" #a ", " #b ")")
#define ASSERT_TRUE(c) LZ_ASSERT_(static_cast<bool>(c), "ASSERT_TRUE(" #c ")")
#define ASSERT_FALSE(c) LZ_ASSERT_(!static_cast<bool>(c), "ASSERT_FALSE(" #c ")")
#define ASSERT_EQ(a, b) LZ_ASSERT_((a) == (b), "ASSERT_EQ(" #a ", " #b ")")
#define ASSERT_NE(a, b) LZ_ASSERT_((a) != (b), "ASSERT_NE(" #a ", " #b ")")
#define ASSERT_NO_THROW(stmt)                                                                                \
	do {                                                                                                     \
		try {                                                                                                \
			stmt;                                                                                            \
		} catch (...) {                                                                                      \
			::testing::Reporter(true, __FILE__, __LINE__, "ASSERT_NO_THROW(" #stmt ")");                      \
			return;                                                                                          \
		}                                                                                                    \
	} while (0)
#define EXPECT_NO_THROW(stmt) ASSERT_NO_THROW(stmt)
#define SCOPED_TRACE(msg) ((void)0)
