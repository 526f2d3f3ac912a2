// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in message for the simulator node's compile (see ros/ros.h).
#pragma once
#include <geometry_msgs/Vector3.h>
namespace sensor_msgs {
struct Imu { ros::Header header; geometry_msgs::Quaternion orientation; geometry_msgs::Vector3 angular_velocity, linear_acceleration; };
}  // namespace sensor_msgs
