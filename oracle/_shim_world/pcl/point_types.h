// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in for <pcl/point_types.h>: PointXYZ as PCL lays it out, x, y, z and a fourth float that the
// constructor sets to 1.0f (PCL's PointXYZ() : x, y, z = 0, data[3] = 1.0f).
#pragma once
namespace pcl {
struct PointXYZ {
    union { float data[4]; struct { float x, y, z; }; };
    PointXYZ() { x = y = z = 0.0f; data[3] = 1.0f; }
    PointXYZ(float x_, float y_, float z_) { x = x_; y = y_; z = z_; data[3] = 1.0f; }
};
}  // namespace pcl
