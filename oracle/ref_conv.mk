# oracle/ref_conv.mk — builds the reference's cudamat_conv.cuh library.  TEST INFRASTRUCTURE ONLY.
#   _ref/libcudamat_conv_ref.so : cudamat_conv_others.cu with the four files its extern "C" block links against (the
#                                 source list of libcudamat_conv.so in $(REF)/cudamat/Makefile), compiled UNMODIFIED
#                                 for sm_90 with the flags of $(REF)/cudamat/Makefile:12-17 (arch list replaced), like
#                                 _ref/libcudamat_conv_gemm_ref.so in Makefile.  The GPU-side oracle of ResponseNorm /
#                                 ContrastNorm / their undos / RGBToYUV (tests/test_gpu_abi_rest.py); the product never
#                                 loads it.  Only where $(REF) exists; elsewhere the prebuilt file (if any) is kept.
#   make -C oracle -f ref_conv.mk
REF ?= /root/reference
NVCC ?= /usr/local/cuda/bin/nvcc
CUDA_LIB ?= /usr/local/cuda/lib64

REF_CONV_SRC := $(addprefix $(REF)/cudamat/,cudamat_conv_filteracts.cu cudamat_conv_imgacts.cu \
                cudamat_conv_weightacts.cu cudamat_conv_others.cu cudamat_conv_util.cu)

all:
	@if [ -d $(REF)/cudamat ]; then $(MAKE) -f ref_conv.mk _ref/libcudamat_conv_ref.so; \
	 else echo "oracle: $(REF) absent - keeping prebuilt _ref/libcudamat_conv_ref.so (if any)"; fi

_ref/libcudamat_conv_ref.so: $(REF_CONV_SRC)
	mkdir -p _ref
	$(NVCC) -O3 --use_fast_math -w -gencode arch=compute_90,code=sm_90 --compiler-options '-fPIC' --shared \
	  -Xlinker -rpath -Xlinker $(CUDA_LIB) -o $@ $(REF_CONV_SRC) -lcublas -L$(CUDA_LIB)

.PHONY: all
