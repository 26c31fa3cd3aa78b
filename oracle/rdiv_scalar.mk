# TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -f oracle/rdiv_scalar.mk -> oracle/_ref/libmxref_rdiv.so: the reference's _rdiv_scalar
#   (ref_rdiv_scalar.cc, which includes ref_arith_ops.cc and ref_ndarray_ops.cc) over its own functor
#   and attribute parser, compiled from src/operator/ where they lie under $(REF). Same flags as
#   oracle/arith_ops.mk (the reference's CPU build); outputs only into oracle/_ref/ (git-ignored).
REF ?= /root/reference
CXX := g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

REF_FLAGS = -std=c++11 -O3 -msse3 -funroll-loops -fopenmp -fPIC -shared -w -DNDEBUG \
  -DMSHADOW_USE_CUDA=0 -DMSHADOW_USE_CBLAS=0 -DMSHADOW_USE_MKL=0 -DMXNET_USE_CUDA=0 \
  -DMXNET_USE_OPENCV=0 -DMXNET_USE_MKLDNN=0 -DMXNET_USE_LAPACK=0 -DDMLC_USE_CXX11=1 \
  -DMSHADOW_IN_CXX11=1 -DDMLC_LOG_STACK_TRACE=0 -DMSHADOW_USE_F16C=0 \
  -I$(REF)/include -I$(REF)/src -I$(REF)/3rdparty/mshadow -I$(REF)/3rdparty/dmlc-core/include \
  -I$(REF)/3rdparty/tvm/nnvm/include -I$(REF)/3rdparty/tvm/include -I$(REF)/3rdparty/dlpack/include

ref_rdiv_scalar: $(HERE)_ref/libmxref_rdiv.so

$(HERE)_ref/libmxref_rdiv.so: $(HERE)ref_rdiv_scalar.cc $(HERE)ref_arith_ops.cc $(HERE)ref_ndarray_ops.cc
	@if [ -f "$(REF)/src/operator/tensor/matrix_op-inl.h" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(CXX) $(REF_FLAGS) -I$(HERE) -Wl,--no-undefined -o $@ $< && \
	  echo "built oracle/_ref/libmxref_rdiv.so from $(REF)"; \
	else echo "reference tree $(REF) not present: keeping any prebuilt oracle/_ref/libmxref_rdiv.so"; fi

.PHONY: ref_rdiv_scalar
