# Build the sm_90a CUDA library (C-ABI) and the CPU oracle.  nvcc cross-compiles without a GPU.
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function --expt-relaxed-constexpr -Iinclude -Icrazyara_b200/csrc
CSRC      := crazyara_b200/csrc
CU_SRCS   := $(wildcard $(CSRC)/*.cu)
CU_OBJS   := $(patsubst $(CSRC)/%.cu,build/%.o,$(CU_SRCS))
LIB       := crazyara_b200/libara_b200.so

all: $(LIB)

build/search.o: EXTRA := -fmad=false
build/rules_kernels.o: EXTRA := -fmad=false

build/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) $(wildcard include/*.h)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) $(EXTRA) -c $< -o $@

$(LIB): $(CU_OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $^

# profiling build: clock64 probes inside the descent (tools/prof_select.py with ARA_B200_LIB=build/libara_b200_fine.so)
build/search_fine.o: $(CSRC)/search.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) $(wildcard include/*.h)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -fmad=false -DARA_PROF_FINE -c $< -o $@
build/libara_b200_fine.so: build/search_fine.o $(filter-out build/search.o,$(CU_OBJS))
	$(NVCC) $(ARCH) -shared -o $@ $^
fine: build/libara_b200_fine.so

# profiling build of the trunk kernel: per-role cycle counters (tools/prof_trunk.py with ARA_B200_LIB=build/libara_b200_tprof.so)
build/rise_trunk_host_prof.o: $(CSRC)/rise_trunk_host.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) $(wildcard include/*.h)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -DARA_TRUNK_PROF -c $< -o $@
build/libara_b200_tprof.so: build/rise_trunk_host_prof.o $(filter-out build/rise_trunk_host.o,$(CU_OBJS))
	$(NVCC) $(ARCH) -shared -o $@ $^
tprof: build/libara_b200_tprof.so

clean:
	rm -rf build $(LIB)

.PHONY: all clean

# C++ host: UCI front-end over the C-ABI (no CUDA in this translation unit)
UCI := crazyara_b200/ara_uci
$(UCI): crazyara_b200/host/uci_main.cpp $(wildcard crazyara_b200/host/*.h) $(CSRC)/chess_dev.cuh include/ara_b200.h $(LIB)
	g++ -O2 -std=c++17 -Wall -pthread -Iinclude -Icrazyara_b200/host -I$(CSRC) $< -o $@ -Lcrazyara_b200 -lara_b200 -Wl,-rpath,'$$ORIGIN' -L/usr/local/cuda/lib64 -Wl,-rpath,/usr/local/cuda/lib64

all: $(UCI)
