# The reference's GPU NMS kernel as a test oracle (see ref_nms.cu), next to the `ref` target of Makefile:
#   make -f ref_nms.mk      -> _ref/libref_nms.so exporting ref_gpu_nms (only where a checkout of the reference exists)
NVCC ?= /usr/local/cuda/bin/nvcc
CXX := $(shell test -x /usr/bin/g++ && echo /usr/bin/g++ || echo g++)
REF ?= /root/reference

_ref/libref_nms.so: ref_nms.cu ref_nms.mk $(REF)/lib/nms/nms_kernel.cu
	@mkdir -p _ref
	$(NVCC) -ccbin $(CXX) -gencode arch=compute_90a,code=sm_90a -std=c++17 -Xcompiler -fPIC -shared -w \
	  -DREF_ROOT=$(REF) -I $(REF)/lib/nms -o $@ ref_nms.cu
