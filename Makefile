# Builds the sm_90a CUDA library (C ABI) and the stand-alone kernel test drivers.
NVCC      ?= nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall
CSRC      := segtran_b200/csrc
LIB_SRCS  := $(filter-out $(CSRC)/test_%.cu,$(wildcard $(CSRC)/*.cu))
LIB_OBJS  := $(patsubst $(CSRC)/%.cu,build/%.o,$(LIB_SRCS))
HDRS      := $(wildcard $(CSRC)/*.cuh) include/segtran_b200.h
LIB       := segtran_b200/libsegtran_b200.so
TESTS     := build/test_gemm

all: $(LIB) $(TESTS) oracle

build/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(LIB_OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $^ -lcudart_static -lpthread -ldl -lrt

build/test_%: $(CSRC)/test_%.cu $(LIB)
	$(NVCC) $(NVFLAGS) $< -o $@ -Lsegtran_b200 -lsegtran_b200 -Xlinker -rpath -Xlinker '$$ORIGIN/../segtran_b200'

oracle:
	@true

clean:
	rm -rf build $(LIB)

.PHONY: all clean oracle
