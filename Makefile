# Builds the C-ABI shared library (sm_90a only).
NVCC      ?= /usr/local/cuda/bin/nvcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
             --expt-relaxed-constexpr
CSRC      := videopose3d_b200/csrc
LIBDIR    := videopose3d_b200/_lib
LIB       := $(LIBDIR)/libvp3d_b200.so
SRCS      := $(CSRC)/conv_gemm.cu $(CSRC)/wgrad_gemm.cu $(CSRC)/pack.cu $(CSRC)/train_ops.cu $(CSRC)/api.cu $(CSRC)/train_api.cu $(CSRC)/gather.cu $(CSRC)/step_ops.cu $(CSRC)/semi_loss.cu $(CSRC)/pose_loss.cu $(CSRC)/stream.cu $(CSRC)/clips.cu $(CSRC)/calib.cu $(CSRC)/detections.cu
OBJS      := $(SRCS:$(CSRC)/%.cu=$(LIBDIR)/%.o)
HDRS      := $(wildcard $(CSRC)/*.cuh) include/vp3d_b200.h

all: $(LIB)

$(LIBDIR)/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p $(LIBDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -Xlinker --exclude-libs=ALL

# Debug build with in-kernel time stamps (tools/timeline.py): a second library next to the product one.
DBGDIR    := $(LIBDIR)/dbg
DBGOBJS   := $(SRCS:$(CSRC)/%.cu=$(DBGDIR)/%.o)
$(DBGDIR)/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p $(DBGDIR)
	$(NVCC) $(NVFLAGS) -DVP3D_TIMELINE -c $< -o $@
dbg: $(DBGOBJS)
	$(NVCC) $(ARCH) -shared -o $(DBGDIR)/libvp3d_b200.so $(DBGOBJS) -Xlinker --exclude-libs=ALL

micro: tools/micro/pack_bench.cu $(CSRC)/pack.cu $(HDRS)
	@mkdir -p $(DBGDIR)
	$(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo tools/micro/pack_bench.cu $(CSRC)/pack.cu -o $(DBGDIR)/pack_bench

clean:
	rm -rf $(LIBDIR)

.PHONY: all clean dbg micro
