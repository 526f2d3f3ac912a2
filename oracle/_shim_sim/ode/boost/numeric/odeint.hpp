// ORACLE — TEST INFRASTRUCTURE ONLY.
// Stand-in for the vendored ode/boost/numeric/odeint.hpp, found first on the include path when the reference's Quadrotor.cpp is compiled for
// oracle/_ref/libref_sim.so. The vendored forward header includes every odeint stepper (rosenbrock4 and its uBLAS matrices, Bulirsch-Stoer,
// Adams-Bashforth-Moulton, ...); Quadrotor::step uses only odeint::integrate. This file includes the vendored integrate.hpp, unmodified, and
// nothing else, so the integrator the library runs is the reference's own controlled_runge_kutta<runge_kutta_dopri5> and integrate_adaptive.
#pragma once
#include <boost/numeric/odeint/integrate/integrate.hpp>
