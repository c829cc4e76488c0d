# builds tests/cpp/test_stripe_batcher_slices.cc twice (make -f slices.mk, from this directory): against the in-tree liblzgpu.so with
# the CPU oracle as the checker, and against the oracle backend (oracle_backend.cc + oracle_backend_slices.cc + the real host_math.cc)
# for the tests that run without a GPU
CXX ?= g++
ROOT := $(abspath ../..)
RPATH := -Wl,-rpath,'$$ORIGIN/../../../lizardfs_b200' -Wl,-rpath,'$$ORIGIN/../../../oracle'
HDRS := $(ROOT)/include/lzgpu_stripe_batcher.hpp $(ROOT)/include/lzgpu.h
CPU_BACKEND := oracle_backend.cc oracle_backend_slices.cc $(ROOT)/lizardfs_b200/csrc/host_math.cc
all: build/test_stripe_batcher_slices build/test_stripe_batcher_slices_cpu
build/test_stripe_batcher_slices: test_stripe_batcher_slices.cc $(HDRS) $(ROOT)/oracle/liboracle.so
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -I$(ROOT)/include $< -o $@ -L$(ROOT)/lizardfs_b200 -llzgpu -L$(ROOT)/oracle -loracle $(RPATH)
build/test_stripe_batcher_slices_cpu: test_stripe_batcher_slices.cc $(CPU_BACKEND) $(HDRS) $(ROOT)/oracle/liboracle.so
	@mkdir -p build
	$(CXX) -O1 -std=c++17 -Wall -DLZ_TEST_CPU_BACKEND -I$(ROOT)/include -I$(ROOT)/lizardfs_b200/csrc test_stripe_batcher_slices.cc $(CPU_BACKEND) \
	    -o $@ -L$(ROOT)/oracle -loracle -Wl,-rpath,'$$ORIGIN/../../../oracle'
$(ROOT)/oracle/liboracle.so:
	$(MAKE) -C $(ROOT)/oracle liboracle.so
