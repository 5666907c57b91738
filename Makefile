# Top-level build: the product library (nvcc, sm_90a), the CPU oracle and the CPU kernel simulator (tests only).
NVCC ?= nvcc
CXX ?= g++
CSRC = cerberus_b200/csrc
ARCH = -gencode arch=compute_90a,code=sm_90a
HDRS = $(wildcard $(CSRC)/*.cuh) $(CSRC)/*.inl $(CSRC)/compat.h include/cerberus_b200.h

.PHONY: all lib oracle sim prof clean
all: lib oracle sim

lib: cerberus_b200/libcerberus_b200.so
cerberus_b200/libcerberus_b200.so: $(CSRC)/cabi.cu $(HDRS)
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -Xptxas -v --shared -Xcompiler -fPIC -o $@ $(CSRC)/cabi.cu 2> $(CSRC)/ptxas.log || (cat $(CSRC)/ptxas.log; false)

# profiling-only build with per-phase cycle counters (tools/phase_profile.py); never loaded by the product or the tests
prof: tools/libcerberus_b200_prof.so
tools/libcerberus_b200_prof.so: $(CSRC)/cabi.cu $(HDRS)
	$(NVCC) $(ARCH) -O3 -lineinfo -std=c++17 -DCERB_PHASE_TIMING --shared -Xcompiler -fPIC -o $@ $(CSRC)/cabi.cu

oracle:
	$(MAKE) -s -C oracle

sim: tests/cusim/libcerberus_b200_sim.so
tests/cusim/libcerberus_b200_sim.so: $(CSRC)/cabi.cu $(HDRS) tests/cusim/cusim.h tests/cusim/cusim.cpp
	$(CXX) -O2 -std=c++17 -DCERB_CUSIM -Itests/cusim -fPIC -shared -Wall -Wno-unused-variable -Wno-unused-function -o $@ -x c++ $(CSRC)/cabi.cu tests/cusim/cusim.cpp -lpthread

clean:
	rm -f cerberus_b200/libcerberus_b200.so tests/cusim/libcerberus_b200_sim.so oracle/liboracle.so
