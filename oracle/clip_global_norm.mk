# TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -f oracle/clip_global_norm.mk -> oracle/_ref/libmxref_clip.so: the scalar arithmetic of
#   gluon.utils.clip_global_norm and amp.unscale (ref_clip_global_norm.cc) over the reference's own
#   functors, compiled from src/operator/mshadow_op.h where it lies under $(REF). Same flags as
#   oracle/update_ops.mk (the reference's CPU build); outputs only into oracle/_ref/ (git-ignored).
REF ?= /root/reference
CXX := g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

REF_FLAGS = -std=c++11 -O3 -msse3 -funroll-loops -fopenmp -fPIC -shared -w -DNDEBUG \
  -DMSHADOW_USE_CUDA=0 -DMSHADOW_USE_CBLAS=0 -DMSHADOW_USE_MKL=0 -DMXNET_USE_CUDA=0 \
  -DMXNET_USE_OPENCV=0 -DMXNET_USE_MKLDNN=0 -DMXNET_USE_LAPACK=0 -DDMLC_USE_CXX11=1 \
  -DMSHADOW_IN_CXX11=1 -DDMLC_LOG_STACK_TRACE=0 -DMSHADOW_USE_F16C=0 \
  -I$(REF)/include -I$(REF)/src -I$(REF)/3rdparty/mshadow -I$(REF)/3rdparty/dmlc-core/include \
  -I$(REF)/3rdparty/tvm/nnvm/include -I$(REF)/3rdparty/tvm/include -I$(REF)/3rdparty/dlpack/include

ref_clip_global_norm: $(HERE)_ref/libmxref_clip.so

$(HERE)_ref/libmxref_clip.so: $(HERE)ref_clip_global_norm.cc
	@if [ -f "$(REF)/src/operator/mshadow_op.h" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(CXX) $(REF_FLAGS) -Wl,--no-undefined -o $@ $< && \
	  echo "built oracle/_ref/libmxref_clip.so from $(REF)"; \
	else echo "reference tree $(REF) not present: keeping any prebuilt oracle/_ref/libmxref_clip.so"; fi

.PHONY: ref_clip_global_norm
