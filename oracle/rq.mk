# TEST INFRASTRUCTURE ONLY -- the ResidualQuantizer encoding entry points (ref_rq_shim.cpp) as
# oracle/_ref/libfaiss_ref_rq.so, linked against oracle/_ref/libfaiss_ref.so (built by oracle/Makefile).
# Same compiler and flags as oracle/Makefile; no reference source is copied.
#
#   make -C oracle -f rq.mk

REF      ?= /root/reference
OUT      := _ref
CXX      := /usr/bin/g++
CXXFLAGS := -std=c++20 -O3 -fPIC -fopenmp -mavx2 -mfma -mf16c -mpopcnt -mbmi2 \
            -DCOMPILE_SIMD_AVX2 -DFINTEGER=int -DNDEBUG -w -I$(REF)

all: $(OUT)/libfaiss_ref_rq.so

$(OUT)/libfaiss_ref_rq.so: ref_rq_shim.cpp $(OUT)/libfaiss_ref.so
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_rq_shim.cpp -L$(OUT) -lfaiss_ref -Wl,-rpath,'$$ORIGIN'

.PHONY: all
