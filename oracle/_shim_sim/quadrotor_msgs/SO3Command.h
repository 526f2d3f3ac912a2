// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in message for the simulator node's compile (see ros/ros.h).
#pragma once
#include <geometry_msgs/Vector3.h>
namespace quadrotor_msgs {
struct SO3Command {
    geometry_msgs::Vector3 force;
    geometry_msgs::Quaternion orientation;
    double kR[3], kOm[3];
    struct { double kf_correction, angle_corrections[2], current_yaw; bool use_external_yaw; } aux;
    typedef std::shared_ptr<const SO3Command> ConstPtr;
};
}  // namespace quadrotor_msgs
