# ORACLE build recipe for the reference's depth renderer — test infrastructure only.
#   make -f depth.mk   -> _ref/libref_depth.so: the reference's uav_simulator/local_sensing/src/depth_render.cu compiled unmodified, where
#                         it lies, with ref_depth_wrap.cu, for sm_90a at -O3 (nvcc's default contraction, as the reference's CUDA build).
# Only possible where the reference tree exists; elsewhere a prebuilt library (or none) is kept and the tests run from
# tests/golden/sense_reference.npz.
NVCC ?= nvcc
REFERENCE ?= /root/reference
SENSE_DIR := $(REFERENCE)/src/uav_simulator/local_sensing/src
DEPTH_SRC := $(SENSE_DIR)/depth_render.cu
DEPTH_HDR := $(SENSE_DIR)/depth_render.cuh $(SENSE_DIR)/device_image.cuh $(SENSE_DIR)/cuda_exception.cuh $(SENSE_DIR)/helper_math.h

ifneq ($(wildcard $(DEPTH_SRC)),)
_ref/libref_depth.so: ref_depth_wrap.cu depth.mk $(DEPTH_SRC) $(DEPTH_HDR)
	mkdir -p _ref && $(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++14 -Xcompiler -fPIC -w -I$(SENSE_DIR) \
	  -shared -o $@ ref_depth_wrap.cu $(DEPTH_SRC) && echo "built $@"
else
_ref/libref_depth.so:
	@echo "reference tree absent: keeping prebuilt $@ if any"
endif
