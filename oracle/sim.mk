# ORACLE build recipe for the reference's closed-loop simulator — test infrastructure only.
#   make -f sim.mk   -> _ref/libref_sim.so: the reference's so3_quadrotor_simulator/src/dynamics/Quadrotor.cpp, so3_control/src/SO3Control.cpp
#                       and (through ref_sim_wrap.cpp, for its static getControl, main renamed) quadrotor_simulator_so3.cpp, with
#                       uav_utils/geometry_utils.h, utils/trajectory.hpp and the vendored odeint under so3_quadrotor_simulator/include/ode,
#                       all compiled unmodified where they lie, with the reference's flags (-O3, no -march: no FMA).
# Stand-ins, found first on the include path (oracle/_shim_sim; see each header):
#   Eigen: restates Eigen's algorithms for the fixed sizes these files use, so the pin is to a tolerance, not to the bit;
#   Boost: boost_standin.hpp behind one generated forwarding header per Boost header name (under _ref/sim_boost); defined where odeint's
#          integrate path runs, declared where it only parses;
#   odeint: the vendored forward header ode/boost/numeric/odeint.hpp pulls in every stepper, rosenbrock4's uBLAS matrices among them, which
#          would need far more Boost than odeint::integrate does; _shim_sim/ode/boost/numeric/odeint.hpp stands in for it and includes
#          the vendored integrate/integrate.hpp unmodified and nothing else;
#   ROS: ros/ros.h and the node's message headers, declared just enough to compile;
#   utils/root_finder.hpp: oracle/_shim_dyn's declarations-only stand-in (as for libref_minco.so).
# Only possible where the reference tree exists; elsewhere a prebuilt library (or none) is kept and the tests run from
# tests/golden/sim_reference.npz.
CXX := $(shell [ -x /usr/bin/g++ ] && echo /usr/bin/g++ || echo g++)
REFERENCE ?= /root/reference
SIM := $(REFERENCE)/src/uav_simulator
QSRC := $(SIM)/so3_quadrotor_simulator/src/dynamics/Quadrotor.cpp
CSRC := $(SIM)/so3_control/src/SO3Control.cpp
NODE := $(SIM)/so3_quadrotor_simulator/src/quadrotor_simulator_so3.cpp
BOOST_NAMES := array bind config range range/config range/algorithm/copy ref static_assert type_traits type_traits/integral_constant \
  type_traits/is_same type_traits/remove_reference utility/enable_if mpl/and mpl/bool mpl/end mpl/find_if mpl/has_xxx mpl/if \
  mpl/placeholders mpl/size_t units/get_dimension units/get_system units/quantity fusion/include/all fusion/include/for_each \
  fusion/include/front fusion/include/is_sequence fusion/include/make_fused fusion/include/vector fusion/include/zip_view
SHIMS := $(wildcard _shim_sim/*.hpp _shim_sim/*/* _shim_sim/ode/boost/numeric/*) _shim_dyn/utils/root_finder.hpp
INC := -I_shim_sim -I_ref/sim_boost -I_shim_dyn -I$(SIM)/so3_quadrotor_simulator/include -I$(SIM)/so3_quadrotor_simulator/include/ode \
  -I$(SIM)/so3_control/include -I$(SIM)/so3_quadrotor_simulator/src -I$(REFERENCE)/src/common/uav_utils/include -I$(REFERENCE)/src/utils/include

ifneq ($(wildcard $(QSRC)),)
_ref/libref_sim.so: ref_sim_wrap.cpp sim.mk ../include/isdf.h $(SHIMS) $(QSRC) $(CSRC) $(NODE)
	mkdir -p _ref/sim_boost/boost
	for h in $(BOOST_NAMES); do mkdir -p _ref/sim_boost/boost/$$(dirname $$h); echo '#include <boost_standin.hpp>' > _ref/sim_boost/boost/$$h.hpp; done
	$(CXX) -O3 -std=c++17 -fPIC -ffp-contract=off -w -Dmain=quadrotor_simulator_so3_main $(INC) -shared -o $@ ref_sim_wrap.cpp $(QSRC) $(CSRC) \
	  && echo "built $@"
else
_ref/libref_sim.so:
	@echo "reference tree absent: keeping prebuilt $@ if any"
endif
