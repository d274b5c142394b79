# Builds the in-tree native library (sm_90a only) and the CPU oracle.
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
EXTRA     ?=
NVCCFLAGS := $(EXTRA) -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v
CSRC      := parsec_b200/csrc
LIB       := parsec_b200/libparsec_b200.so
CU_SRCS   := $(CSRC)/pb2_engine.cu $(CSRC)/pb2_engine_prio.cu $(CSRC)/pb2_engine_trace.cu $(CSRC)/pb2_engine_prio_trace.cu \
             $(CSRC)/pb2_stream.cu
CPP_SRCS  := $(wildcard $(CSRC)/*.cpp)
HDRS      := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) $(wildcard $(CSRC)/*.hpp) $(wildcard include/*.h)

all: $(LIB) oracle

$(LIB): $(CU_SRCS) $(CPP_SRCS) $(HDRS)
	$(NVCC) $(NVCCFLAGS) -shared -o $@ $(CU_SRCS) $(CPP_SRCS) -Iinclude 2> build_ptxas.log || (cat build_ptxas.log; exit 1)
	@grep -E "error|warning" build_ptxas.log | grep -v "ptxas info" || true

oracle:
	$(MAKE) -C oracle

clean:
	rm -f $(LIB) build_ptxas.log
	$(MAKE) -C oracle clean

.PHONY: all oracle clean
