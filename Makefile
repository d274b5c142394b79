# Builds the in-tree native library (sm_90a only) and the CPU oracle.
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
EXTRA     ?=
NVCCFLAGS := $(EXTRA) -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v
CSRC      := parsec_b200/csrc
LIB       := parsec_b200/libparsec_b200.so
CU_SRCS   := $(CSRC)/pb2_engine.cu $(CSRC)/pb2_stream.cu
CPP_SRCS  := $(wildcard $(CSRC)/*.cpp)
HDRS      := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) $(wildcard $(CSRC)/*.hpp) $(wildcard include/*.h)
# the built-in window kernels, one object (and one ptxas log) per variant v = (queue_policy 1) + 2 * (trace)
WINDOW_OBJS  := $(foreach v,0 1 2 3,build/pb2_window_kernels_$(v).o)
WINDOW_LOGS  := $(WINDOW_OBJS:.o=.log)
# the HBM window kernel with application bodies: relocatable device code, linked at run time (pb2_engine_link_bodies)
LINKED_CUBIN := build/pb2_engine_linked.cubin
# the GEMM window kernel with application bodies, linked only when asked for (PB2_LINK_GEMM_WINDOWS)
LINKED_GEMM_CUBIN := build/pb2_engine_linked_gemm.cubin
# both again with the group call of linked readers compiled in, linked instead of them with PB2_LINK_READER_GROUPS
LINKED_GROUPS_CUBIN := build/pb2_engine_linked_groups.cubin
LINKED_GEMM_GROUPS_CUBIN := build/pb2_engine_linked_gemm_groups.cubin
# the GEMM window kernel that calls GEMM-worker bodies through pb2_linked_gemm_body, with and without the group call,
# linked instead of the two above with PB2_LINK_GEMM_BODY_ENTRY
LINKED_GEMM_ENTRY_CUBIN := build/pb2_engine_linked_gemm_entry.cubin
LINKED_GEMM_ENTRY_GROUPS_CUBIN := build/pb2_engine_linked_gemm_entry_groups.cubin
LINKED_OBJ   := build/pb2_linked_image.o
# the device bodies the GPU tests link (tests/test_linked_bodies_gpu.py, tests/test_checked_linked_gpu.py,
# tests/test_linked_readers_gpu.py, tests/test_reader_groups_linked_gpu.py, tests/test_gemm_worker_bodies_gpu.py,
# tests/test_gemm_body_entry_gpu.py, tests/test_gemm_body_parts_gpu.py), as relocatable cubins and as PTX
TEST_BODIES  := tests/cuda/linked_bodies.cubin tests/cuda/linked_bodies.ptx \
                tests/cuda/checked_bodies.cubin tests/cuda/checked_bodies.ptx \
                tests/cuda/reader_bodies.cubin tests/cuda/reader_bodies.ptx \
                tests/cuda/reader_group_bodies.cubin tests/cuda/reader_group_bodies.ptx \
                tests/cuda/gemm_worker_bodies.cubin tests/cuda/gemm_worker_bodies.ptx \
                tests/cuda/gemm_entry_bodies.cubin tests/cuda/gemm_entry_bodies.ptx \
                tests/cuda/gemm_entry_group_bodies.cubin \
                tests/cuda/gemm_part_bodies.cubin tests/cuda/gemm_part_group_bodies.cubin

all: $(LIB) linked_bodies oracle

$(LIB): $(CU_SRCS) $(CPP_SRCS) $(HDRS) $(WINDOW_OBJS) $(LINKED_OBJ)
	$(NVCC) $(NVCCFLAGS) -shared -o $@ $(CU_SRCS) $(CPP_SRCS) $(WINDOW_OBJS) $(LINKED_OBJ) -Iinclude 2> build_ptxas.log || (cat build_ptxas.log; exit 1)
	@cat $(WINDOW_LOGS) >> build_ptxas.log
	@grep -E "error|warning" build_ptxas.log | grep -v "ptxas info" || true

build/pb2_window_kernels_%.o: $(CSRC)/pb2_window_kernels.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -DPB2_WINDOW_VARIANT=$* -c -o $@ $< -Iinclude 2> build/pb2_window_kernels_$*.log || (cat build/pb2_window_kernels_$*.log; exit 1)

$(LINKED_CUBIN): $(CSRC)/pb2_engine_linked.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -rdc=true -cubin -o $@ $< -Iinclude 2> build/linked_ptxas.log || (cat build/linked_ptxas.log; exit 1)

$(LINKED_GEMM_CUBIN): $(CSRC)/pb2_engine_linked_gemm.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -rdc=true -cubin -o $@ $< -Iinclude 2> build/linked_gemm_ptxas.log || (cat build/linked_gemm_ptxas.log; exit 1)

$(LINKED_GROUPS_CUBIN): $(CSRC)/pb2_engine_linked.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -DPB2_LINKED_READER_GROUPS -rdc=true -cubin -o $@ $< -Iinclude 2> build/linked_groups_ptxas.log || (cat build/linked_groups_ptxas.log; exit 1)

$(LINKED_GEMM_GROUPS_CUBIN): $(CSRC)/pb2_engine_linked_gemm.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -DPB2_LINKED_READER_GROUPS -rdc=true -cubin -o $@ $< -Iinclude 2> build/linked_gemm_groups_ptxas.log || (cat build/linked_gemm_groups_ptxas.log; exit 1)

$(LINKED_GEMM_ENTRY_CUBIN): $(CSRC)/pb2_engine_linked_gemm.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -DPB2_LINKED_GEMM_BODY_ENTRY -rdc=true -cubin -o $@ $< -Iinclude 2> build/linked_gemm_entry_ptxas.log || (cat build/linked_gemm_entry_ptxas.log; exit 1)

$(LINKED_GEMM_ENTRY_GROUPS_CUBIN): $(CSRC)/pb2_engine_linked_gemm.cu $(HDRS)
	@mkdir -p build
	$(NVCC) $(NVCCFLAGS) -DPB2_LINKED_GEMM_BODY_ENTRY -DPB2_LINKED_READER_GROUPS -rdc=true -cubin -o $@ $< -Iinclude 2> build/linked_gemm_entry_groups_ptxas.log || (cat build/linked_gemm_entry_groups_ptxas.log; exit 1)

$(LINKED_OBJ): $(CSRC)/pb2_linked_image.S $(LINKED_CUBIN) $(LINKED_GEMM_CUBIN) $(LINKED_GROUPS_CUBIN) $(LINKED_GEMM_GROUPS_CUBIN) \
               $(LINKED_GEMM_ENTRY_CUBIN) $(LINKED_GEMM_ENTRY_GROUPS_CUBIN)
	gcc -c -DPB2_LINKED_CUBIN='"$(abspath $(LINKED_CUBIN))"' -DPB2_LINKED_GEMM_CUBIN='"$(abspath $(LINKED_GEMM_CUBIN))"' \
	    -DPB2_LINKED_GROUPS_CUBIN='"$(abspath $(LINKED_GROUPS_CUBIN))"' \
	    -DPB2_LINKED_GEMM_GROUPS_CUBIN='"$(abspath $(LINKED_GEMM_GROUPS_CUBIN))"' \
	    -DPB2_LINKED_GEMM_ENTRY_CUBIN='"$(abspath $(LINKED_GEMM_ENTRY_CUBIN))"' \
	    -DPB2_LINKED_GEMM_ENTRY_GROUPS_CUBIN='"$(abspath $(LINKED_GEMM_ENTRY_GROUPS_CUBIN))"' -o $@ $<

linked_bodies: $(TEST_BODIES)

tests/cuda/linked_bodies.cubin: tests/cuda/linked_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -Iinclude -o $@ $<

tests/cuda/linked_bodies.ptx: tests/cuda/linked_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 -arch=compute_90a -rdc=true -ptx -Iinclude -o $@ $<

tests/cuda/checked_bodies.cubin: tests/cuda/checked_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -Iinclude -o $@ $<

tests/cuda/checked_bodies.ptx: tests/cuda/checked_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 -arch=compute_90a -rdc=true -ptx -Iinclude -o $@ $<

tests/cuda/reader_bodies.cubin: tests/cuda/reader_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -Iinclude -o $@ $<

tests/cuda/reader_bodies.ptx: tests/cuda/reader_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 -arch=compute_90a -rdc=true -ptx -Iinclude -o $@ $<

# -maxrregcount=80: the group form keeps a count per member in registers; capped, it fits the HBM window kernels'
# 80-register budget, which the link enforces (the only stack it takes is the call ABI's saved registers)
tests/cuda/reader_group_bodies.cubin: tests/cuda/reader_group_bodies.cu tests/cuda/reader_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -maxrregcount=80 -Iinclude -o $@ $<

tests/cuda/reader_group_bodies.ptx: tests/cuda/reader_group_bodies.cu tests/cuda/reader_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 -arch=compute_90a -rdc=true -ptx -Iinclude -o $@ $<

# -maxrregcount=80: the image is linked into the HBM window kernels as well, whose budget (80) the link enforces
tests/cuda/gemm_worker_bodies.cubin: tests/cuda/gemm_worker_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -maxrregcount=80 -Xptxas -v -Iinclude -o $@ $< 2> tests/cuda/gemm_worker_bodies.log || (cat tests/cuda/gemm_worker_bodies.log; exit 1)

tests/cuda/gemm_worker_bodies.ptx: tests/cuda/gemm_worker_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 -arch=compute_90a -rdc=true -ptx -maxrregcount=80 -Iinclude -o $@ $<

# -maxrregcount=168: pb2_linked_gemm_body is reached from the GEMM window kernels only, whose budget (168) the link
# enforces; pb2_linked_body still reaches the HBM kernels too, and ptxas fits it in their 80 (the link checks that)
tests/cuda/gemm_entry_bodies.cubin: tests/cuda/gemm_entry_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -maxrregcount=168 -Xptxas -v -Iinclude -o $@ $< 2> tests/cuda/gemm_entry_bodies.log || (cat tests/cuda/gemm_entry_bodies.log; exit 1)

tests/cuda/gemm_entry_bodies.ptx: tests/cuda/gemm_entry_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 -arch=compute_90a -rdc=true -ptx -maxrregcount=168 -Iinclude -o $@ $<

# the same image with the group form of its reader, pb2_linked_reader_group (PB2_LINK_READER_GROUPS)
tests/cuda/gemm_entry_group_bodies.cubin: tests/cuda/gemm_entry_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -maxrregcount=168 -DGEMM_ENTRY_READER_GROUP -Iinclude -o $@ $<

# GEMM-worker bodies that split their tasks by part (pb2_engine_set_gemm_body_parts), at the GEMM kernels' 168
# registers, and with the group form of their reader
tests/cuda/gemm_part_bodies.cubin: tests/cuda/gemm_part_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -maxrregcount=168 -Xptxas -v -Iinclude -o $@ $< 2> tests/cuda/gemm_part_bodies.log || (cat tests/cuda/gemm_part_bodies.log; exit 1)

tests/cuda/gemm_part_group_bodies.cubin: tests/cuda/gemm_part_bodies.cu include/pb2_device_body.h
	$(NVCC) -O3 -std=c++17 $(ARCH) -rdc=true -cubin -maxrregcount=168 -DGEMM_PART_READER_GROUP -Iinclude -o $@ $<

oracle:
	$(MAKE) -C oracle

clean:
	rm -f $(LIB) build_ptxas.log $(WINDOW_OBJS) $(WINDOW_LOGS) $(LINKED_CUBIN) $(LINKED_GEMM_CUBIN) $(LINKED_OBJ) build/linked_ptxas.log \
	      build/linked_gemm_ptxas.log $(LINKED_GROUPS_CUBIN) $(LINKED_GEMM_GROUPS_CUBIN) build/linked_groups_ptxas.log \
	      build/linked_gemm_groups_ptxas.log $(LINKED_GEMM_ENTRY_CUBIN) $(LINKED_GEMM_ENTRY_GROUPS_CUBIN) \
	      build/linked_gemm_entry_ptxas.log build/linked_gemm_entry_groups_ptxas.log $(TEST_BODIES) \
	      tests/cuda/gemm_worker_bodies.log tests/cuda/gemm_entry_bodies.log tests/cuda/gemm_part_bodies.log
	$(MAKE) -C oracle clean

.PHONY: all linked_bodies oracle clean
