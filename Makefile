# In-tree build of the C-ABI library (sm_90a only) and the CPU oracle.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr -Iinclude
CSRC := $(wildcard visionllm_b200/csrc/*.cu)
OBJ := $(patsubst visionllm_b200/csrc/%.cu,build/%.o,$(CSRC))
LIB := visionllm_b200/lib/libvllm_b200.so

all: $(LIB) oracle

HDRS := $(wildcard visionllm_b200/csrc/*.cuh) include/vllm_b200.h
build/%.o: visionllm_b200/csrc/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; false)

$(LIB): $(OBJ)
	@mkdir -p visionllm_b200/lib
	$(NVCC) -shared $(ARCH) -o $@ $(OBJ) -lcudart

oracle:
	$(MAKE) -C oracle

clean:
	rm -rf build visionllm_b200/lib oracle/*.so oracle/_ref

.PHONY: all oracle clean
