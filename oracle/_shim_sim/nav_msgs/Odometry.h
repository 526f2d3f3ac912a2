// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in message for the simulator node's compile (see ros/ros.h).
#pragma once
#include <geometry_msgs/Vector3.h>
namespace nav_msgs {
struct Odometry {
    ros::Header header;
    std::string child_frame_id;
    struct { struct { geometry_msgs::Point position; geometry_msgs::Quaternion orientation; } pose; } pose;
    struct { struct { geometry_msgs::Vector3 linear, angular; } twist; } twist;
};
}  // namespace nav_msgs
