# ORACLE build recipe for the reference's distance field — test infrastructure only.
#   make -f esdf.mk   -> _ref/libref_esdf.so: the reference's map_manager/src/Gridmap3D.cpp compiled unmodified with ref_esdf_wrap.cpp,
#                        against the eager Eigen stand-in and the ROS stand-ins, with the reference's flags (-O3, no -march: no FMA).
# A library of its own, with the reference sources among its prerequisites, so that make rebuilds it whenever the wrapper or the reference
# changes and never mistakes an older grid library for it. Only possible where the reference tree exists; elsewhere a prebuilt library
# (or none) is kept and the tests run from tests/golden/esdf_reference.npz.
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
REFERENCE ?= /root/reference
GRID_SRC := $(REFERENCE)/src/map_manager/src/Gridmap3D.cpp
GRID_HDR := $(REFERENCE)/src/map_manager/include/map_manager/GridMap3D.h

ifneq ($(wildcard $(GRID_SRC)),)
_ref/libref_esdf.so: ref_esdf_wrap.cpp esdf.mk _shim_dyn/Eigen/Eigen _shim_dyn/ros/ros.h $(GRID_SRC) $(GRID_HDR)
	mkdir -p _ref && $(CXX) -O3 -std=c++14 -fPIC -ffp-contract=off -w -I_shim_dyn -I$(REFERENCE)/src/map_manager/include \
	  -shared -o $@ ref_esdf_wrap.cpp $(GRID_SRC) && echo "built $@"
else
_ref/libref_esdf.so:
	@echo "reference tree absent: keeping prebuilt $@ if any"
endif
