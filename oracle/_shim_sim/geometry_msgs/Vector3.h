// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in message for the simulator node's compile (see ros/ros.h).
#pragma once
#include <ros/ros.h>
namespace geometry_msgs {
struct Vector3 { double x = 0, y = 0, z = 0; typedef std::shared_ptr<const Vector3> ConstPtr; };
struct Quaternion { double x = 0, y = 0, z = 0, w = 1; };
struct Point { double x = 0, y = 0, z = 0; };
}  // namespace geometry_msgs
