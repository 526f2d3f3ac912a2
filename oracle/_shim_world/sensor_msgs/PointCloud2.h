// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in for <sensor_msgs/PointCloud2.h>: a header with a frame id, nothing else.
#pragma once
#include <string>
namespace sensor_msgs { struct PointCloud2 { struct { std::string frame_id; } header; }; }
