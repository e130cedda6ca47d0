# Builds libpaimon_gpu.so (sm_90a only) in-tree, and the parity oracle.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Iinclude -Ipaimon_b200/csrc
SRCS := paimon_b200/csrc/merge.cu paimon_b200/csrc/emit.cu paimon_b200/csrc/api.cu \
	paimon_b200/csrc/parquet_decode.cu paimon_b200/csrc/parquet_encode.cu paimon_b200/csrc/parquet_meta.cc \
	paimon_b200/csrc/arrow_export.cu paimon_b200/csrc/upload.cu paimon_b200/csrc/readback.cu paimon_b200/csrc/orc_decode.cu paimon_b200/csrc/orc_meta.cc \
	paimon_b200/csrc/orc_encode.cu paimon_b200/csrc/encoded_file.cu paimon_b200/csrc/file_index.cu
HDRS := include/paimon_gpu.h paimon_b200/csrc/pg_internal.h paimon_b200/csrc/device_utils.cuh paimon_b200/csrc/parquet_meta.h \
	paimon_b200/csrc/zstd_device.cuh paimon_b200/csrc/zstd_encode_device.cuh paimon_b200/csrc/inflate_device.cuh paimon_b200/csrc/lz4_device.cuh paimon_b200/csrc/snappy_device.cuh paimon_b200/csrc/orc_device.cuh paimon_b200/csrc/orc_meta.h \
	paimon_b200/csrc/orc_encode_device.cuh paimon_b200/csrc/encoded_file.h paimon_b200/csrc/xxhash64_device.cuh paimon_b200/csrc/murmur3_device.cuh \
	paimon_b200/csrc/scan_kernels.cuh paimon_b200/csrc/range_reader.h paimon_b200/csrc/device_layout.h paimon_b200/csrc/sbbf_device.cuh
LIB := paimon_b200/libpaimon_gpu.so

all: $(LIB) oracle

# one object per source (build/ is scratch), linked into the shared library
OBJDIR ?= build
OBJS := $(patsubst paimon_b200/csrc/%,$(OBJDIR)/%.o,$(SRCS))

# the Makefile is a prerequisite too: a change of ARCH or flags rebuilds every object
$(OBJDIR)/%.o: paimon_b200/csrc/% $(HDRS) Makefile
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) $(EXTRA_DEFS) -x cu -c -o $@ $<

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS)

ptxas-info: $(SRCS) $(HDRS)
	$(NVCC) $(NVFLAGS) -Xptxas -v -c -o /dev/null paimon_b200/csrc/merge.cu
	$(NVCC) $(NVFLAGS) -Xptxas -v -c -o /dev/null paimon_b200/csrc/file_index.cu
	$(NVCC) $(NVFLAGS) -Xptxas -v -c -o /dev/null paimon_b200/csrc/parquet_encode.cu
	$(NVCC) $(NVFLAGS) -Xptxas -v -c -o /dev/null paimon_b200/csrc/orc_encode.cu

# the JNI shim against the JNI specification's signatures (no JDK in the image: jni/stub/jni.h)
jni-check:
	g++ -std=c++17 -fsyntax-only -Wall -Ijni/stub -Iinclude jni/paimon_gpu_jni.cc

oracle:
	$(MAKE) -C oracle -s

clean:
	rm -rf $(LIB) $(OBJDIR)
	$(MAKE) -C oracle clean

.PHONY: all oracle clean ptxas-info jni-check
