// ORACLE — TEST INFRASTRUCTURE ONLY.
// Stand-in for <ros/ros.h>, declared just far enough for the reference's Quadrotor.cpp, SO3Control.cpp and quadrotor_simulator_so3.cpp to
// compile unmodified for oracle/_ref/libref_sim.so. The node's main (renamed at compile time) and its callbacks compile against these
// declarations but are never called; getControl, the one piece of that file the wrapper uses, touches no ROS.
#pragma once
#include <string>
#include <memory>
#define ROS_ASSERT(x) ((void)0)
#define ROS_ERROR(...) ((void)0)
#define ROS_WARN(...) ((void)0)
#define ROS_INFO(...) ((void)0)
namespace ros {
struct Duration { explicit Duration(double) {} };
struct Time {
    static Time now() { return Time(); }
    bool operator>=(const Time &) const { return true; }
    Time &operator+=(const Duration &) { return *this; }
};
struct Rate { explicit Rate(double) {} void sleep() {} };
struct Header { std::string frame_id; Time stamp; };
struct TransportHints { TransportHints &tcpNoDelay() { return *this; } };
struct Publisher { template <class M> void publish(const M &) const {} };
struct Subscriber {};
struct NodeHandle {
    explicit NodeHandle(const std::string & = "") {}
    template <class M> Publisher advertise(const std::string &, int) { return Publisher(); }
    template <class F> Subscriber subscribe(const std::string &, int, F, const TransportHints &) { return Subscriber(); }
    template <class T, class U> void param(const std::string &, T &v, const U &d) { v = d; }
    bool ok() const { return false; }
};
inline void init(int &, char **, const std::string &) {}
inline void spinOnce() {}
}  // namespace ros
