# ORACLE build recipe for the reference's world generators — test infrastructure only.
#   make -f world.mk   -> _ref/libref_world.so: the reference's map_manager/src/globalmap_gene.cpp (main renamed) and
#                         uav_simulator/mockamap/src/maps.cpp + perlinnoise.cpp, compiled unmodified where they lie, with ref_world_wrap.cpp,
#                         with the reference's flags (-O3, no -march: no FMA) and libstdc++ (std::shuffle, std::default_random_engine,
#                         std::uniform_real_distribution as the reference build links them).
# Stand-ins, found first on the include path (oracle/_shim_world; see each header): ROS (NodeHandle::param returning the wrapper's values),
# PCL (PointCloud<PointXYZ>, toROSMsg, PCDReader), sensor_msgs / geometry_msgs, and the Eigen the files use (Vector3d for geneRoad,
# MatrixXi for the maze code, which compiles but is never pinned). -Bsymbolic binds the library's own time() calls to the wrapper's time().
# Only possible where the reference tree exists; elsewhere a prebuilt library (or none) is kept and the tests run from
# tests/golden/world_reference.npz.
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
REFERENCE ?= /root/reference
GSRC := $(REFERENCE)/src/map_manager/src/globalmap_gene.cpp
MOCKA := $(REFERENCE)/src/uav_simulator/mockamap
MSRC := $(MOCKA)/src/maps.cpp $(MOCKA)/src/perlinnoise.cpp
SHIMS := $(wildcard _shim_world/*/*)

ifneq ($(wildcard $(GSRC)),)
_ref/libref_world.so: ref_world_wrap.cpp world.mk $(SHIMS) $(GSRC) $(MSRC)
	mkdir -p _ref && $(CXX) -O3 -std=c++14 -fPIC -w -Dmain=globalmap_gene_main -I_shim_world -I$(MOCKA)/include -shared \
	  -Wl,-Bsymbolic -o $@ ref_world_wrap.cpp $(GSRC) $(MSRC) && echo "built $@"
else
_ref/libref_world.so:
	@echo "reference tree absent: keeping prebuilt $@ if any"
endif
