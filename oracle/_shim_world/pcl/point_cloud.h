// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in for <pcl/point_cloud.h>: the points vector, width / height / is_dense and push_back as PCL
// keeps them. Real PCL pulls in Eigen, which mockamap's maps.hpp relies on for Eigen::MatrixXi.
#pragma once
#include <Eigen/Core>
#include <cstdint>
#include <memory>
#include <vector>
#include "point_types.h"
namespace pcl {
template <class P> struct PointCloud {
    typedef std::shared_ptr<PointCloud> Ptr;
    std::vector<P> points;
    uint32_t width = 0, height = 0;
    bool is_dense = true;
    void push_back(const P &p) { points.push_back(p); width = (uint32_t)points.size(); height = 1; }
    size_t size() const { return points.size(); }
};
}  // namespace pcl
