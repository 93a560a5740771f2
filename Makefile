# Builds the product in-tree:
#   roc_b200/lib/libroc_b200.so  — sm_90a kernels + C ABI (include/roc_b200.h) + C++ host (include/roc_gnn.h, roc_host.h)
#   roc_b200/bin/roc_gnn         — stand-alone driver with the reference's CLI
# and the test infrastructure (oracle/Makefile): oracle/libroc_oracle.so, oracle/_ref/libroc_ref.so
CUDA   ?= /usr/local/cuda
NVCC   ?= $(CUDA)/bin/nvcc
CXX    := g++
ARCH   := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Iinclude -Iroc_b200/csrc
CXXFLAGS := -O2 -std=c++17 -fPIC -Iinclude -Iroc_b200/csrc -Iroc_b200/csrc/host -I$(CUDA)/include -Wall -Wno-unused-function

BUILD := build
CU_SRCS := sg elementwise linear_simt linear linear_tc linear_tc_dw halo batchnorm layernorm attn_scores
HOST_SRCS := runtime graph model capi
CU_OBJS := $(CU_SRCS:%=$(BUILD)/%.o)
HOST_OBJS := $(HOST_SRCS:%=$(BUILD)/host_%.o)
LIB := roc_b200/lib/libroc_b200.so
BIN := roc_b200/bin/roc_gnn

all: $(LIB) $(BIN) oracle

$(BUILD)/%.o: roc_b200/csrc/%.cu roc_b200/csrc/common.cuh roc_b200/csrc/tc_common.cuh include/roc_b200.h
	@mkdir -p $(BUILD)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(BUILD)/host_%.o: roc_b200/csrc/host/%.cc roc_b200/csrc/host/host_internal.h include/roc_gnn.h include/roc_host.h include/roc_b200.h
	@mkdir -p $(BUILD)
	$(CXX) $(CXXFLAGS) -c $< -o $@

$(LIB): $(CU_OBJS) $(HOST_OBJS)
	@mkdir -p roc_b200/lib
	$(NVCC) $(ARCH) -shared -o $@ $^ -lcudart -lcurand -ldl

$(BIN): $(BUILD)/host_main.o $(LIB)
	@mkdir -p roc_b200/bin
	$(CXX) -o $@ $< -Lroc_b200/lib -lroc_b200 -L$(CUDA)/lib64 -lcudart -Wl,-rpath,'$$ORIGIN/../lib'

oracle:
	$(MAKE) -C oracle all

# compute-sanitizer (memcheck + racecheck) over the tiny configuration; needs a GPU
sanitize: $(LIB)
	tools/sanitize.sh

# tensor-pipe rate of m64n32k8 against m64n64k8 / m64n128k8 (tf32, A from registers); needs a GPU to run
$(BUILD)/bench_wgmma_n: tools/bench_wgmma_n.cu roc_b200/csrc/tc_common.cuh
	@mkdir -p $(BUILD)
	$(NVCC) $(ARCH) -O3 -std=c++17 -Iroc_b200/csrc $< -o $@

clean:
	rm -rf $(BUILD) $(LIB) $(BIN)
	$(MAKE) -C oracle clean

.PHONY: all oracle clean sanitize
