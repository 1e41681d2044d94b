# TEST INFRASTRUCTURE ONLY -- the IndexHNSWCagra entry points (ref_cagra_shim.cpp) as
# oracle/_ref/libfaiss_ref_cagra.so, linked against oracle/_ref/libfaiss_ref.so (built by oracle/Makefile).
# Same compiler and flags as oracle/Makefile; no reference source is copied.
#
#   make -C oracle -f cagra.mk

REF      ?= /root/reference
OUT      := _ref
CXX      := /usr/bin/g++
CXXFLAGS := -std=c++20 -O3 -fPIC -fopenmp -mavx2 -mfma -mf16c -mpopcnt -mbmi2 \
            -DCOMPILE_SIMD_AVX2 -DFINTEGER=int -DNDEBUG -w -I$(REF)

all: $(OUT)/libfaiss_ref_cagra.so

$(OUT)/libfaiss_ref_cagra.so: ref_cagra_shim.cpp $(OUT)/libfaiss_ref.so
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_cagra_shim.cpp -L$(OUT) -lfaiss_ref -Wl,-rpath,'$$ORIGIN'

.PHONY: all
