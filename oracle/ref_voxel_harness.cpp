// ref_voxel_harness.cpp — C entry points over the REFERENCE'S OWN VoxelGrid (planning_ros_utils/src/mapping_utils/voxel_grid.cpp,
// compiled unmodified from where it lies, against the stand-in Eigen / Boost / planning_ros_msgs headers of oracle/shim/).
// TEST INFRASTRUCTURE ONLY.  Every call has the shape of the oracle's orv_ call of the same name (oracle/voxel_oracle.cpp), so
// oracle/voxel.py drives both through one class.  Inputs where the reference is undefined (clear(nx, ny) outside the grid,
// a geometry beyond int32) are never passed here.
#include <mpl_collision/map_util.h>
#include <planning_ros_utils/voxel_grid.h>

#include <cstdint>
#include <cstring>

namespace {
Vec3f v3(const double *p) { return Vec3f(p[0], p[1], p[2]); }
int64_t put_cloud(const vec_Vec3f &pts, double *out, int64_t cap) {
  for (int64_t k = 0; k < (int64_t)pts.size() && k < cap; k++)
    for (int i = 0; i < 3; i++) out[3 * k + i] = pts[k](i);
  return (int64_t)pts.size();
}
}  // namespace

extern "C" {

void *rvx_create(const double *origin, const double *dim_m, float res) { return new VoxelGrid(v3(origin), v3(dim_m), res); }
void rvx_destroy(void *h) { delete (VoxelGrid *)h; }
int rvx_allocate(void *h, const double *dim_m, const double *origin) { return ((VoxelGrid *)h)->allocate(v3(dim_m), v3(origin)) ? 1 : 0; }
void rvx_info(void *h, int32_t *dim, int32_t *ori, double *origin_d, float *res) {
  // VoxelGrid keeps its geometry private; getMap reports dim_, origin_d_ and res_ (origin_ is not observable)
  planning_ros_msgs::VoxelMap m = ((VoxelGrid *)h)->getMap();
  dim[0] = (int32_t)m.dim.x; dim[1] = (int32_t)m.dim.y; dim[2] = (int32_t)m.dim.z;
  origin_d[0] = m.origin.x; origin_d[1] = m.origin.y; origin_d[2] = m.origin.z;
  ori[0] = ori[1] = ori[2] = INT32_MIN;
  *res = m.resolution;
}
void rvx_clear(void *h) { ((VoxelGrid *)h)->clear(); }
void rvx_add_cloud(void *h, const double *pts, int64_t n) {
  vec_Vec3f v;
  for (int64_t i = 0; i < n; i++) v.push_back(v3(pts + 3 * i));
  ((VoxelGrid *)h)->addCloud(v);
}
int64_t rvx_add_cloud_inflated(void *h, const double *pts, int64_t n, const int32_t *ns, int n_ns, int32_t *out, int64_t cap) {
  vec_Vec3f v;
  for (int64_t i = 0; i < n; i++) v.push_back(v3(pts + 3 * i));
  vec_Vec3i vn;
  for (int j = 0; j < n_ns; j++) vn.push_back(Vec3i(ns[3 * j], ns[3 * j + 1], ns[3 * j + 2]));
  vec_Vec3i r = ((VoxelGrid *)h)->addCloud(v, vn);
  for (int64_t k = 0; k < (int64_t)r.size() && k < cap; k++)
    for (int i = 0; i < 3; i++) out[3 * k + i] = r[k](i);
  return (int64_t)r.size();
}
void rvx_decay(void *h) { ((VoxelGrid *)h)->decay(); }
void rvx_fill(void *h, const int32_t *cells3, int n, int column) {
  for (int k = 0; k < n; k++) {
    if (column) ((VoxelGrid *)h)->fill(cells3[3 * k], cells3[3 * k + 1]);
    else ((VoxelGrid *)h)->fill(cells3[3 * k], cells3[3 * k + 1], cells3[3 * k + 2]);
  }
}
void rvx_clear_columns(void *h, const int32_t *cells3, int n) {
  for (int k = 0; k < n; k++) ((VoxelGrid *)h)->clear(cells3[3 * k], cells3[3 * k + 1]);
}
int64_t rvx_get_cloud(void *h, double *out, int64_t cap) { return put_cloud(((VoxelGrid *)h)->getCloud(), out, cap); }
int64_t rvx_get_local_cloud(void *h, const double *pos, const double *ori, const double *dim, double *out, int64_t cap) {
  return put_cloud(((VoxelGrid *)h)->getLocalCloud(v3(pos), v3(ori), v3(dim)), out, cap);
}
int64_t rvx_get_map(void *h, int inflated, int8_t *out, int64_t cap) {
  planning_ros_msgs::VoxelMap m = inflated ? ((VoxelGrid *)h)->getInflatedMap() : ((VoxelGrid *)h)->getMap();
  if (cap < (int64_t)m.data.size()) return -1;
  std::memcpy(out, m.data.data(), m.data.size());
  return (int64_t)m.data.size();
}

// ---- the reference's MapUtil<3> (mpl_collision/map_util.h) as map_replanner_node.cpp uses it beside the grid
void *rvx_mu_create(const double *origin, const int32_t *dim, double res, const int8_t *data) {
  MPL::VoxelMapUtil *m = new MPL::VoxelMapUtil();
  m->setMap(v3(origin), Vec3i(dim[0], dim[1], dim[2]), MPL::Tmap(data, data + (size_t)dim[0] * dim[1] * dim[2]), res);
  return m;
}
void rvx_mu_destroy(void *m) { delete (MPL::VoxelMapUtil *)m; }
int64_t rvx_mu_ray_trace(void *m, const double *p1, const double *p2, int32_t *out, int64_t cap) { // map_util.h:117-134
  vec_Vec3i pns = ((MPL::VoxelMapUtil *)m)->rayTrace(v3(p1), v3(p2));
  for (int64_t k = 0; k < (int64_t)pns.size() && k < cap; k++)
    for (int i = 0; i < 3; i++) out[3 * k + i] = pns[k](i);
  return (int64_t)pns.size();
}
// addCloudCallback / clearCloudCallback (map_replanner_node.cpp:175-232) on the grid and the MapUtil, without the planner
// call: the ray of the message's first and last point, the edit of the grid, then setMap(map_util, voxel_mapper_->getMap()).
// Returns the new_obs / new_clear list the node hands to updateBlockedNodes / updateClearedNodes.
int64_t rvx_node_edit(void *h, void *mu, int add, const double *p1, const double *p2, int32_t *out, int64_t cap) {
  VoxelGrid *g = (VoxelGrid *)h;
  MPL::VoxelMapUtil *map_util = (MPL::VoxelMapUtil *)mu;
  vec_Vec3i pns = map_util->rayTrace(v3(p1), v3(p2));
  vec_Vec3i cells;
  if (add) {
    vec_Vec3i ns;
    for (int nx = -2; nx <= 2; nx++)
      for (int ny = -2; ny <= 2; ny++) ns.push_back(Vec3i(nx, ny, 0));
    for (const auto &it : pns)
      for (const auto &itt : ns) {
        Vec3i pn = it + itt;
        if (map_util->isFree(pn)) {
          g->fill(pn(0), pn(1));
          cells.push_back(pn);
        }
      }
  } else {
    for (const auto &pn : pns)
      if (map_util->isOccupied(pn)) {
        g->clear(pn(0), pn(1));
        cells.push_back(pn);
      }
  }
  planning_ros_msgs::VoxelMap map = g->getMap(); // setMap(map_util, map), planning_ros_utils mapping_utils.h
  map_util->setMap(Vec3f(map.origin.x, map.origin.y, map.origin.z), Vec3i(map.dim.x, map.dim.y, map.dim.z),
                   MPL::Tmap(map.data.begin(), map.data.end()), map.resolution);
  for (int64_t k = 0; k < (int64_t)cells.size() && k < cap; k++)
    for (int i = 0; i < 3; i++) out[3 * k + i] = cells[k](i);
  return (int64_t)cells.size();
}

}  // extern "C"
