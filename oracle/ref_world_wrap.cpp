// ORACLE — TEST INFRASTRUCTURE ONLY. A C API over the reference's own world generators for oracle/_ref/libref_world.so (oracle/world.mk):
//   ref_world_globalmap  globalmap_gene.cpp's mapGene(map_id) (compiled unmodified, main renamed), on the node's cloud_resolution and
//                        init_*, after srand(rand_seed); time() is defined here, so the srand(time(NULL)) of maps 4 and 11 receives
//                        srand_seed (the library is linked -Bsymbolic, so its own calls bind to this definition)
//   ref_world_perlin / ref_world_boxes  mockamap's Maps::generate(1 / 2) (maps.cpp, perlinnoise.cpp unmodified) on a BasicInfo of the
//                        given sizes, scale and seed, the parameters read through the ros::NodeHandle stand-in
// Each writes the first cap records (x, y, z, data[3]) and returns the cloud's size; ref_world_perlin returns -1 where perlin3D throws.
#include <ros/ros.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#include <sensor_msgs/PointCloud2.h>
#include <cstdlib>
#include <ctime>
#include <stdexcept>
#include "maps.hpp"

extern double cloud_resolution, init_x, init_y, init_z;
extern pcl::PointCloud<pcl::PointXYZ> global_map_pcl_cloud;
void mapGene(int id);

static time_t g_time;
extern "C" time_t time(time_t *t) { if (t) *t = g_time; return g_time; }

namespace ros {
std::map<std::string, double> &ref_world_params() { static std::map<std::string, double> m; return m; }
}

static long long copy_out(const std::vector<pcl::PointXYZ> &pts, size_t n, float *out, long long cap) {
    for (size_t i = 0; i < n && (long long)i < cap; i++)
        for (int a = 0; a < 4; a++) out[4 * i + a] = pts[i].data[a];
    return (long long)n;
}

extern "C" {

long long ref_world_globalmap(int id, uint32_t rand_seed, uint32_t srand_seed, double res, const double *init, float *out, long long cap) {
    global_map_pcl_cloud.points.clear();
    cloud_resolution = res; init_x = init[0]; init_y = init[1]; init_z = init[2];
    g_time = (time_t)srand_seed;
    srand(rand_seed);
    mapGene(id);
    return copy_out(global_map_pcl_cloud.points, global_map_pcl_cloud.points.size(), out, cap);
}

static long long run_mocka(int type, uint32_t seed, int X, int Y, int Z, double scale, float *out, long long cap) {
    ros::NodeHandle nh("~");
    pcl::PointCloud<pcl::PointXYZ> cloud;
    sensor_msgs::PointCloud2 output;
    mocka::Maps::BasicInfo info;
    info.nh_private = &nh; info.sizeX = X; info.sizeY = Y; info.sizeZ = Z; info.seed = (int)seed; info.scale = scale;
    info.output = &output; info.cloud = &cloud;
    mocka::Maps map;
    map.setInfo(info);
    try {
        map.generate(type);
    } catch (const std::out_of_range &) {
        return -1;
    }
    return copy_out(cloud.points, (size_t)cloud.width * cloud.height, out, cap);
}

long long ref_world_perlin(uint32_t seed, int X, int Y, int Z, double scale, double complexity, double fill, double attenuation, int fractal,
                           float *out, long long cap) {
    auto &p = ros::ref_world_params();
    p.clear();
    p["complexity"] = complexity; p["fill"] = fill; p["attenuation"] = attenuation; p["fractal"] = fractal;
    return run_mocka(1, seed, X, Y, Z, scale, out, cap);
}

long long ref_world_boxes(uint32_t seed, int X, int Y, int Z, double scale, int obstacles, double wmin, double wmax, float *out, long long cap) {
    auto &p = ros::ref_world_params();
    p.clear();
    p["width_min"] = wmin; p["width_max"] = wmax; p["obstacle_number"] = obstacles;
    return run_mocka(2, seed, X, Y, Z, scale, out, cap);
}

}  // extern "C"
