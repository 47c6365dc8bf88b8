/*
 * voxel_grid.hpp — header-only C++ host layer for the reference's VoxelGrid (planning_ros_utils/include/planning_ros_utils/
 * voxel_grid.h, src/mapping_utils/voxel_grid.cpp) over the C ABI of include/mplb.h: the same public members and signatures,
 * with both grids on the GPU.  getMap / getInflatedMap return planning_ros_msgs::VoxelMap when that message header is on the
 * include path, otherwise a struct with the same field names (origin.x/y/z, dim.x/y/z, resolution, data), so cloud_to_map.cpp
 * and map_replanner_node.cpp compile against it with or without ROS.  writeMap(MapUtil<3> &) is setMap(map_util, getMap())
 * without leaving the device.  Errors print mplb_last_error(), as map_planner.hpp does.
 */
#ifndef MPL_B200_VOXEL_GRID_HPP
#define MPL_B200_VOXEL_GRID_HPP
#include <cstdint>
#include <cstdio>
#include <vector>

#include "map_planner.hpp"

#if defined(__has_include)
#if __has_include(<planning_ros_msgs/VoxelMap.h>)
#include <planning_ros_msgs/VoxelMap.h>
#define MPL_B200_HAS_VOXELMAP_MSG 1
#endif
#endif

namespace mpl_b200 {
#ifdef MPL_B200_HAS_VOXELMAP_MSG
typedef planning_ros_msgs::VoxelMap VoxelMap;
#else
struct VoxelMap { /* the fields of planning_ros_msgs/VoxelMap.msg that VoxelGrid writes */
  struct { double x, y, z; } origin, dim;
  float resolution;
  std::vector<int8_t> data;
};
#endif
}  // namespace mpl_b200

class VoxelGrid {
 public:
  VoxelGrid(Vec3f origin, Vec3f dim, float res) { /* vg:3-10 */
    const double o[3] = {origin(0), origin(1), origin(2)}, d[3] = {dim(0), dim(1), dim(2)};
    if (mplb_voxel_grid_create(o, d, res, &h_) != MPLB_OK) std::printf("[VoxelGrid] create failed: %s\n", mplb_last_error());
  }
  ~VoxelGrid() { mplb_voxel_grid_destroy(h_); }
  VoxelGrid(const VoxelGrid &) = delete;
  VoxelGrid &operator=(const VoxelGrid &) = delete;

  void clear() { report(mplb_voxel_grid_clear(h_)); } /* vg:12-16 */
  vec_Vec3f getCloud() { return cloud(mplb_voxel_grid_get_cloud(h_, nullptr, 0), nullptr); } /* vg:18-29 */
  vec_Vec3f getLocalCloud(const Vec3f &pos, const Vec3f &ori, const Vec3f &dim) { /* vg:47-69 */
    const double p[3] = {pos(0), pos(1), pos(2)}, o[3] = {ori(0), ori(1), ori(2)}, d[3] = {dim(0), dim(1), dim(2)};
    const double *box[3] = {p, o, d};
    return cloud(mplb_voxel_grid_get_local_cloud(h_, p, o, d, nullptr, 0), box);
  }
  mpl_b200::VoxelMap getMap() { return map(0); }         /* vg:71-98 */
  mpl_b200::VoxelMap getInflatedMap() { return map(1); } /* vg:100-127 */
  bool allocate(const Vec3f &new_dim_d, const Vec3f &new_ori_d) { /* vg:129-172 */
    const double d[3] = {new_dim_d(0), new_dim_d(1), new_dim_d(2)}, o[3] = {new_ori_d(0), new_ori_d(1), new_ori_d(2)};
    int32_t changed = 0;
    report(mplb_voxel_grid_allocate(h_, d, o, &changed));
    return changed != 0;
  }
  void addCloud(const vec_Vec3f &pts) { /* vg:174-180 */
    const std::vector<double> p = flat(pts);
    report(mplb_voxel_grid_add_cloud(h_, p.data(), (int64_t)pts.size()));
  }
  vec_Vec3i addCloud(const vec_Vec3f &pts, const vec_Vec3i &ns) { /* vg:182-199 */
    const std::vector<double> p = flat(pts);
    std::vector<int32_t> n3;
    for (const auto &it : ns) { n3.push_back(it(0)); n3.push_back(it(1)); n3.push_back(it(2)); }
    int32_t dim[3] = {0, 0, 0};
    mplb_voxel_grid_get_info(h_, dim, nullptr, nullptr, nullptr);
    const int64_t ncell = (int64_t)dim[0] * dim[1] * dim[2], want = (int64_t)pts.size() * (int64_t)ns.size();
    const int64_t cap = want < ncell ? want : ncell; /* one call emits a cell at most once */
    std::vector<int32_t> out((size_t)(cap > 0 ? cap : 1) * 3);
    const int64_t k = mplb_voxel_grid_add_cloud_inflated(h_, p.data(), (int64_t)pts.size(), n3.data(), (int)ns.size(), out.data(), cap);
    vec_Vec3i r;
    if (k < 0) { report((int)k); return r; }
    for (int64_t i = 0; i < k && i < cap; i++) r.push_back(Vec3i(out[3 * i], out[3 * i + 1], out[3 * i + 2]));
    return r;
  }
  void decay() { report(mplb_voxel_grid_decay(h_)); } /* vg:214-225 */
  void fill(int nx, int ny) { const int32_t c[3] = {nx, ny, 0}; report(mplb_voxel_grid_fill(h_, c, 1, 1)); }           /* vg:35-39 */
  void fill(int nx, int ny, int nz) { const int32_t c[3] = {nx, ny, nz}; report(mplb_voxel_grid_fill(h_, c, 1, 0)); }   /* vg:41-45 */
  void clear(int nx, int ny) { const int32_t c[3] = {nx, ny, 0}; report(mplb_voxel_grid_clear_columns(h_, c, 1)); }    /* vg:31-33 */

  /* setMap(map_util, getMap() / getInflatedMap()) on the device; map_util must already have the grid's geometry */
  bool writeMap(MPL::MapUtil<3> &map_util, bool inflated = false) {
    return report(mplb_voxel_grid_write_map(h_, inflated ? 1 : 0, map_util.handle()));
  }
  mplb_voxel_grid *handle() const { return h_; }

 private:
  bool report(int rc) {
    if (rc < 0) std::printf("[VoxelGrid] %s\n", mplb_last_error());
    return rc >= 0;
  }
  static std::vector<double> flat(const vec_Vec3f &pts) {
    std::vector<double> p;
    p.reserve(pts.size() * 3);
    for (const auto &it : pts) { p.push_back(it(0)); p.push_back(it(1)); p.push_back(it(2)); }
    return p;
  }
  vec_Vec3f cloud(int64_t n, const double *const *box) {
    vec_Vec3f r;
    if (n <= 0) { if (n < 0) report((int)n); return r; }
    std::vector<double> p((size_t)n * 3);
    n = box ? mplb_voxel_grid_get_local_cloud(h_, box[0], box[1], box[2], p.data(), n) : mplb_voxel_grid_get_cloud(h_, p.data(), n);
    for (int64_t i = 0; i < n; i++) r.push_back(Vec3f(p[3 * i], p[3 * i + 1], p[3 * i + 2]));
    return r;
  }
  mpl_b200::VoxelMap map(int inflated) {
    mpl_b200::VoxelMap m;
    int32_t dim[3] = {0, 0, 0};
    double ori[3] = {0, 0, 0};
    float res = 0;
    mplb_voxel_grid_get_info(h_, dim, nullptr, ori, &res);
    m.origin.x = ori[0]; m.origin.y = ori[1]; m.origin.z = ori[2];
    m.dim.x = dim[0]; m.dim.y = dim[1]; m.dim.z = dim[2];
    m.resolution = res;
    m.data.resize((size_t)dim[0] * dim[1] * dim[2], 0);
    if (!m.data.empty()) report(mplb_voxel_grid_get_map(h_, inflated, reinterpret_cast<int8_t *>(m.data.data()), m.data.size()));
    return m;
  }
  mplb_voxel_grid *h_ = nullptr;
};
#endif
