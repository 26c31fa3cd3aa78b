# TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -f oracle/group_adagrad.mk -> oracle/_ref/libmxref_group_adagrad.so: the reference's own CPU
#   kernel of _contrib_group_adagrad_update (ref_group_adagrad.cc), compiled from the header where it
#   lies under $(REF). Same flags as oracle/sparse_update_ops.mk (the reference's CPU build, no FMA
#   contraction); outputs only into oracle/_ref/ (git-ignored).
REF ?= /root/reference
CXX := g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

REF_FLAGS = -std=c++11 -O3 -msse3 -funroll-loops -fopenmp -fPIC -shared -w -DNDEBUG \
  -DMSHADOW_USE_CUDA=0 -DMSHADOW_USE_CBLAS=0 -DMSHADOW_USE_MKL=0 -DMXNET_USE_CUDA=0 \
  -DMXNET_USE_OPENCV=0 -DMXNET_USE_MKLDNN=0 -DMXNET_USE_LAPACK=0 -DDMLC_USE_CXX11=1 \
  -DMSHADOW_IN_CXX11=1 -DDMLC_LOG_STACK_TRACE=0 -DMSHADOW_USE_F16C=0 \
  -I$(REF)/include -I$(REF)/src -I$(REF)/3rdparty/mshadow -I$(REF)/3rdparty/dmlc-core/include \
  -I$(REF)/3rdparty/tvm/nnvm/include -I$(REF)/3rdparty/tvm/include -I$(REF)/3rdparty/dlpack/include

ref_group_adagrad: $(HERE)_ref/libmxref_group_adagrad.so

$(HERE)_ref/libmxref_group_adagrad.so: $(HERE)ref_group_adagrad.cc
	@if [ -f "$(REF)/src/operator/contrib/optimizer_op-inl.h" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(CXX) $(REF_FLAGS) -Wl,--no-undefined -o $@ $< && \
	  echo "built oracle/_ref/libmxref_group_adagrad.so from $(REF)"; \
	else echo "reference tree $(REF) not present: keeping any prebuilt oracle/_ref/libmxref_group_adagrad.so"; fi

.PHONY: ref_group_adagrad
