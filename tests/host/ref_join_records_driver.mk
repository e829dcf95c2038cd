# tests/host/ref_join_records_driver.mk — builds the fixture driver of tests/golden/make_golden_join_records.py (ref_join_records_driver.cpp: the stock
# api::InnerJoin on records) against the reference's headers and the reference library from oracle/ref/Makefile.
# No GPU code.  Output in oracle/_ref/host/.  make -C tests/host -f ref_join_records_driver.mk
REF  ?= /root/reference
ROOT := $(abspath ../..)
OUT  := $(ROOT)/oracle/_ref/host
CXX  ?= g++
CXXFLAGS := -std=c++14 -O2 -march=x86-64-v3 -DNDEBUG -w -pthread -include cstdint -DTLX_DIE_WITH_EXCEPTION=1 -DTHRILL_HAVE_PIPE2=1
INCS := -I$(REF) -I$(REF)/extlib/tlx -I$(REF)/extlib/foxxll -I$(REF)/extlib/cereal/include -I$(ROOT)/oracle/_ref/include
all: $(OUT)/ref_join_records_driver
$(OUT)/ref_join_records_driver: ref_join_records_driver.cpp
	@mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) $(INCS) ref_join_records_driver.cpp $(ROOT)/oracle/_ref/libthrill_ref.a -ldl -lpthread -o $@
.PHONY: all
