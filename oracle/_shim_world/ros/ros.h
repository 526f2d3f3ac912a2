// ORACLE — TEST INFRASTRUCTURE ONLY.
// Stand-in for <ros/ros.h>, declared just far enough for the reference's globalmap_gene.cpp and mockamap's maps.cpp to compile unmodified
// for oracle/_ref/libref_world.so. NodeHandle::param reads the values oracle/ref_world_wrap.cpp sets (ref_world_params), else the default
// the call gives; the node's main (renamed at compile time) and its publishers compile but are never called.
#pragma once
#include <iostream>
#include <map>
#include <string>
#define ROS_INFO(...) ((void)0)
#define ROS_WARN(...) ((void)0)
#define ROS_ERROR(...) ((void)0)
namespace ros {
std::map<std::string, double> &ref_world_params();
struct Duration { explicit Duration(double) {} void sleep() const {} };
struct Rate { explicit Rate(double) {} void sleep() {} };
struct Publisher { template <class M> void publish(const M &) const {} };
struct NodeHandle {
    explicit NodeHandle(const std::string & = "") {}
    template <class M> Publisher advertise(const std::string &, int) { return Publisher(); }
    template <class T, class U> bool param(const std::string &name, T &v, const U &d) {
        const auto it = ref_world_params().find(name);
        v = it == ref_world_params().end() ? (T)d : (T)it->second;
        return true;
    }
    bool param(const std::string &, std::string &v, const std::string &d) { v = d; return true; }
    template <class T> bool getParam(const std::string &, T &) { return false; }
};
inline void init(int &, char **, const std::string &) {}
inline void spin() {}
inline void spinOnce() {}
inline bool ok() { return false; }
}  // namespace ros
