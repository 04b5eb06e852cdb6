# Build the sm_90a shared library (C ABI in include/loftr_b200.h) and the test helpers.
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC
LIB       := loftr_b200/lib/libloftr_b200.so
CSRC      := loftr_b200/csrc
HDRS      := $(wildcard $(CSRC)/*.cuh) include/loftr_b200.h

all: $(LIB) build/bringup

$(LIB): $(CSRC)/engine.cu $(HDRS)
	@mkdir -p loftr_b200/lib
	$(NVCC) $(NVFLAGS) -shared $(CSRC)/engine.cu -o $@ -ldl

build/bringup: tests/cuda/bringup.cu $(LIB)
	@mkdir -p build
	$(NVCC) $(ARCH) -O2 -std=c++17 tests/cuda/bringup.cu -o $@ -Lloftr_b200/lib -lloftr_b200 -Xlinker -rpath -Xlinker '$$ORIGIN/../loftr_b200/lib'

clean:
	rm -rf build loftr_b200/lib

.PHONY: all clean
