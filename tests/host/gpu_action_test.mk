# tests/host/gpu_action_test.mk — builds the in-Thrill integration test of Sum / Min / Max / AllReduce / Size (gpu_action_test.cpp) the way
# Makefile builds gpu_nodes_test: the reference's headers, the reference library from oracle/ref/Makefile and libthrill_gpu.so.
# Output in oracle/_ref/host/.  make -C tests/host -f gpu_action_test.mk
REF  ?= /root/reference
ROOT := $(abspath ../..)
OUT  := $(ROOT)/oracle/_ref/host
CXX  ?= g++
CXXFLAGS := -std=c++14 -O2 -march=x86-64-v3 -DNDEBUG -w -pthread -include cstdint -DTLX_DIE_WITH_EXCEPTION=1 -DTHRILL_HAVE_PIPE2=1
INCS := -I$(REF) -I$(REF)/extlib/tlx -I$(REF)/extlib/foxxll -I$(REF)/extlib/cereal/include -I$(ROOT)/oracle/_ref/include
all: $(OUT)/gpu_action_test
$(OUT)/gpu_action_test: gpu_action_test.cpp $(ROOT)/thrill_b200/host/thrill_gpu_nodes.hpp $(ROOT)/include/thrill_gpu.h
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INCS) gpu_action_test.cpp $(ROOT)/oracle/_ref/libthrill_ref.a \
	    -L$(ROOT)/thrill_b200/csrc -lthrill_gpu -Wl,-rpath,'$$ORIGIN/../../../thrill_b200/csrc' -ldl -lpthread -o $@
.PHONY: all
