# Plain Makefile (SURVEY section 7: the autotools shape of the reference, without autotools): the sm_90a (H100) C-ABI library, the
# `daccord` command line, the host tools library and -- test infrastructure only -- the CPU oracle.
# daccord_b200/build.py runs the same commands from Python (what __graft_entry__.build() calls).
NVCC     ?= nvcc
# (make predefines CXX = g++; in this image that is a wrapper without libgomp.spec, so the system compiler is named -- override with make CXX=...)
CXX      := /usr/bin/g++
B        := daccord_b200/_build
CSRC     := daccord_b200/csrc
NVFLAGS  := -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC,-O3,-ffp-contract=off,-fopenmp -shared
CXXFLAGS := -O3 -g -std=c++17 -march=x86-64-v2 -ffp-contract=off -fopenmp -pthread
CUDEPS   := $(wildcard $(CSRC)/*.cu $(CSRC)/*.cuh $(CSRC)/*.hpp) include/daccord_b200.h
HOSTDEPS := $(wildcard $(CSRC)/host/*.hpp $(CSRC)/host/*.cpp) $(CSRC)/profile_core.cuh $(CSRC)/inqual_core.cuh $(CSRC)/exqual_core.cuh $(CSRC)/proper_core.cuh include/daccord_b200.h

all: $(B)/libdaccord_b200.so $(B)/libdaccord_host.so $(B)/daccord $(B)/computeintrinsicqv $(B)/computeextrinsicqv $(B)/lasfilteralignments oracle

$(B)/libdaccord_b200.so: $(CUDEPS)
	@mkdir -p $(B)
	PATH=/usr/bin:$$PATH $(NVCC) $(NVFLAGS) -o $@ $(CSRC)/dcu_lib.cu -lcudart -lgomp

$(B)/libdaccord_host.so: $(HOSTDEPS)
	@mkdir -p $(B)
	$(CXX) $(CXXFLAGS) -fPIC -shared -o $@ $(CSRC)/host/hostlib.cpp

$(B)/daccord: $(HOSTDEPS) $(B)/libdaccord_b200.so
	$(CXX) $(CXXFLAGS) -o $@ $(CSRC)/host/daccord_main.cpp -L$(B) -ldaccord_b200 -Wl,-rpath,'$$ORIGIN'

$(B)/computeintrinsicqv: $(HOSTDEPS) $(B)/libdaccord_b200.so
	$(CXX) $(CXXFLAGS) -o $@ $(CSRC)/host/computeintrinsicqv.cpp -L$(B) -ldaccord_b200 -Wl,-rpath,'$$ORIGIN'

$(B)/computeextrinsicqv: $(HOSTDEPS) $(B)/libdaccord_b200.so
	$(CXX) $(CXXFLAGS) -o $@ $(CSRC)/host/computeextrinsicqv.cpp -L$(B) -ldaccord_b200 -Wl,-rpath,'$$ORIGIN'

$(B)/lasfilteralignments: $(HOSTDEPS) $(B)/libdaccord_b200.so
	$(CXX) $(CXXFLAGS) -o $@ $(CSRC)/host/lasfilteralignments.cpp -L$(B) -ldaccord_b200 -Wl,-rpath,'$$ORIGIN'

oracle:
	$(MAKE) -s -C oracle

check: all
	python -m pytest tests -x -q -m "not gpu"

clean:
	rm -rf $(B) oracle/_build tests/emu/_build

.PHONY: all oracle check clean
