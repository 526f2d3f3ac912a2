// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in for <geometry_msgs/TransformStamped.h> (included, unused by globalmap_gene.cpp).
#pragma once
namespace geometry_msgs { struct TransformStamped {}; }
