# Build the C-ABI CUDA library (sm_90a only) and the oracle's C/compiled pieces.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall --expt-relaxed-constexpr
CSRC := pixray_b200/csrc
OBJDIR := build/obj
SRCS := $(wildcard $(CSRC)/*.cu)
OBJS := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(SRCS))
LIB := pixray_b200/lib/libpixray_b200.so

all: $(LIB)

$(OBJDIR)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.inc) $(wildcard $(CSRC)/*.h) include/pixray_b200.h
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	@mkdir -p pixray_b200/lib
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -ldl

clean:
	rm -rf build $(LIB)

.PHONY: all clean
