// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in for <pcl_conversions/pcl_conversions.h>: toROSMsg converts nothing, and PCDReader (which
// globalmap_gene.cpp reaches through this header) reads nothing: the PCD path is never taken.
#pragma once
#include <string>
#include <pcl/point_cloud.h>
#include <sensor_msgs/PointCloud2.h>
namespace pcl {
template <class P> void toROSMsg(const PointCloud<P> &, sensor_msgs::PointCloud2 &) {}
struct PCDReader { template <class P> int read(const std::string &, PointCloud<P> &) { return -1; } };
}  // namespace pcl
