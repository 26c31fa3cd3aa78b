# TEST INFRASTRUCTURE ONLY (see oracle/README.md).
#
#   make -f oracle/add_n.mk -> oracle/_ref/libmxref_add_n.so: the reference's own add_n arithmetic
#   (ref_add_n.cc), compiled where it lies under $(REF): ElementWiseSumCompute_ from the header
#   src/operator/tensor/elemwise_sum.h, and two function templates cut out at build time, as
#   oracle/Makefile cuts the row_sparse reduce: ElementwiseSumContainsDnsImpl from
#   src/ndarray/ndarray_function.cc and CastStorageRspDnsImpl (the storage fallback's densify) from
#   src/operator/tensor/cast_storage-inl.h. The excerpts live in oracle/_ref/ for the duration of the
#   compile only; the .so is all that stays (oracle/_ref/ is git-ignored). Same flags as
#   oracle/update_ops.mk (the reference's CPU build, no FMA contraction).
REF ?= /root/reference
CXX := g++
HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))

REF_FLAGS = -std=c++11 -O3 -msse3 -funroll-loops -fopenmp -fPIC -shared -w -DNDEBUG \
  -DMSHADOW_USE_CUDA=0 -DMSHADOW_USE_CBLAS=0 -DMSHADOW_USE_MKL=0 -DMXNET_USE_CUDA=0 \
  -DMXNET_USE_OPENCV=0 -DMXNET_USE_MKLDNN=0 -DMXNET_USE_LAPACK=0 -DDMLC_USE_CXX11=1 \
  -DMSHADOW_IN_CXX11=1 -DDMLC_LOG_STACK_TRACE=0 -DMSHADOW_USE_F16C=0 \
  -I$(REF)/include -I$(REF)/src -I$(REF)/3rdparty/mshadow -I$(REF)/3rdparty/dmlc-core/include \
  -I$(REF)/3rdparty/tvm/nnvm/include -I$(REF)/3rdparty/tvm/include -I$(REF)/3rdparty/dlpack/include

# $(1): file, $(2): the function's first line (a grep pattern), $(3): excerpt name. From the line
# above that one (its template<...> line, or a blank line) to the first closing brace in column 0.
define EXCERPT
	s=$$(grep -n '$(2)' $(1) | head -1 | cut -d: -f1); \
	e=$$(awk -v s=$$s 'NR>s && /^}/ {print NR; exit}' $(1)); \
	test -n "$$s" && test -n "$$e" && sed -n "$$((s-1)),$${e}p" $(1) > $(HERE)_ref/$(3)
endef

ref_add_n: $(HERE)_ref/libmxref_add_n.so

$(HERE)_ref/libmxref_add_n.so: $(HERE)ref_add_n.cc
	@if [ -f "$(REF)/src/operator/tensor/elemwise_sum.h" ]; then \
	  mkdir -p $(HERE)_ref && \
	  $(call EXCERPT,$(REF)/src/ndarray/ndarray_function.cc,^void ElementwiseSumContainsDnsImpl,excerpt_sum_contains_dns.inc) && \
	  $(call EXCERPT,$(REF)/src/operator/tensor/cast_storage-inl.h,^void CastStorageRspDnsImpl,excerpt_cast_rsp_dns.inc) && \
	  $(CXX) $(REF_FLAGS) -I$(HERE) -Wl,--no-undefined -o $@ $<; rc=$$?; \
	  rm -f $(HERE)_ref/excerpt_sum_contains_dns.inc $(HERE)_ref/excerpt_cast_rsp_dns.inc; \
	  test $$rc -eq 0 && echo "built oracle/_ref/libmxref_add_n.so from $(REF)"; \
	else echo "reference tree $(REF) not present: keeping any prebuilt oracle/_ref/libmxref_add_n.so"; fi

.PHONY: ref_add_n
