# TEST INFRASTRUCTURE ONLY (see DESIGN.md §6).
#
#   make -f oracle/sample_params_gpu.mk -> oracle/_ref/libmxref_sample_params_gpu.so: the reference's
#   own GPU multi-sample samplers (uniform, normal, gamma, exponential with typed parameter arrays),
#   for the H100 tests and bench_sample_params.py. It compiles src/common/random_generator.cu where it
#   lies under $(REF), with the harness ref_sample_params_gpu.cu, for sm_90a with the reference's GPU
#   flags, those of oracle/sample_gpu.mk (-O3, nvcc's default -fmad=true contraction, no fast math).
#   The .so is all that stays (oracle/_ref/ is git-ignored); it links the CUDA runtime statically.
REF ?= /root/reference
NVCC ?= /usr/local/cuda/bin/nvcc
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

REF_NVCC_FLAGS = -std=c++14 -Xcompiler -D_FORCE_INLINES -O3 -gencode arch=compute_90a,code=sm_90a \
  -Xcompiler -fPIC -shared -w -DNDEBUG -cudart static \
  -DMSHADOW_USE_CUDA=1 -DMXNET_USE_CUDA=1 -DMSHADOW_USE_CUDNN=0 -DMXNET_USE_CUDNN=0 \
  -DMSHADOW_USE_CBLAS=0 -DMSHADOW_USE_MKL=0 -DMXNET_USE_OPENCV=0 -DMXNET_USE_MKLDNN=0 \
  -DMXNET_USE_LAPACK=0 -DDMLC_USE_CXX11=1 -DMSHADOW_IN_CXX11=1 -DDMLC_LOG_STACK_TRACE=0 \
  -DMXNET_USE_NCCL=0 -DMSHADOW_USE_NVML=0 \
  -I$(REF)/include -I$(REF)/src -I$(REF)/3rdparty/mshadow -I$(REF)/3rdparty/dmlc-core/include \
  -I$(REF)/3rdparty/tvm/nnvm/include -I$(REF)/3rdparty/tvm/include -I$(REF)/3rdparty/dlpack/include

ref_sample_params_gpu: $(HERE)_ref/libmxref_sample_params_gpu.so

$(HERE)_ref/libmxref_sample_params_gpu.so: $(HERE)ref_sample_params_gpu.cu
	@if [ -f "$(REF)/src/common/random_generator.cu" ]; then \
	  mkdir -p $(HERE)_ref && \
	  env -u CC -u CXX $(NVCC) $(REF_NVCC_FLAGS) -o $@ $(REF)/src/common/random_generator.cu $< -lcublas_static -lcublasLt_static -lculibos && \
	  echo "built oracle/_ref/libmxref_sample_params_gpu.so from $(REF)"; \
	else echo "reference tree $(REF) not present: keeping any prebuilt oracle/_ref/libmxref_sample_params_gpu.so"; fi

.PHONY: ref_sample_params_gpu
