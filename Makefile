# Builds the C-ABI kernel library (sm_90a only): stable-video-infinity_b200/lib/libsvi_b200.so
NVCC ?= nvcc
PKG := stable-video-infinity_b200
CSRC := $(PKG)/csrc
LIB := $(PKG)/lib/libsvi_b200.so
NVFLAGS := -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC
SRCS := $(CSRC)/runtime.cu $(CSRC)/gemm_wgmma.cu $(CSRC)/attn_wgmma.cu $(CSRC)/sp_exchange.cu $(CSRC)/elementwise.cu $(CSRC)/conv3d_wgmma.cu $(CSRC)/vae_elementwise.cu $(CSRC)/encoder_kernels.cu $(CSRC)/audio_kernels.cu $(CSRC)/rife_kernels.cu $(CSRC)/esrgan_kernels.cu $(CSRC)/fastblend_kernels.cu $(CSRC)/window_kernels.cu $(CSRC)/replace_kernels.cu $(CSRC)/quality_kernels.cu $(CSRC)/reward_kernels.cu $(CSRC)/processor_kernels.cu
OBJS := $(patsubst $(CSRC)/%.cu,build/%.o,$(SRCS))

all: $(LIB)

build/%.o: $(CSRC)/%.cu $(CSRC)/common.cuh $(CSRC)/wgmma.cuh include/svi_b200.h include/svi_b200_lora.h include/svi_b200_rife.h include/svi_b200_esrgan.h include/svi_b200_fastblend.h include/svi_b200_fastblend_modes.h include/svi_b200_unianimate.h include/svi_b200_replace.h include/svi_b200_quality.h include/svi_b200_reward.h include/svi_b200_processors.h
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -Xptxas -v -c $< -o $@ 2> build/$*.ptxas.log || (cat build/$*.ptxas.log; exit 1)

$(LIB): $(OBJS)
	@mkdir -p $(PKG)/lib
	$(NVCC) -shared -o $@ $(OBJS) -cudart shared

clean:
	rm -rf build $(LIB)
.PHONY: all clean
