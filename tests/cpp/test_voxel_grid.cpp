/* cloud_to_map.cpp's processCloud and map_replanner_node.cpp's start-up and edit callbacks (:175-232, :326-336) re-typed
 * without ROS against include/planning_ros_utils/voxel_grid.h (the compat name of include/mpl_b200/voxel_grid.hpp):
 * VoxelGrid(origin, dim, res) + addCloud + getMap; addCloud(pts, ns); then the MapUtil built from getMap, the ray of the
 * add_cloud message, the 5 x 5 isFree columns filled, writeMap, and the ray of the clear_cloud message, its isOccupied columns
 * cleared, writeMap.  Prints counts and FNV-1a hashes in a fixed format; tests/test_gpu_voxel_grid.py compares them with the
 * fixture recorded from the reference.  argv[1]: origin[3] dim_m[3] (f64), res (f32), n (i64), n x 3 f32 points, then the two
 * points of add_cloud and of clear_cloud (4 x 3 f32). */
#include <planning_ros_utils/voxel_grid.h>

#include <cstdio>
#include <fstream>

static unsigned long long fnv(const void *p, size_t n) {
  unsigned long long h = 1469598103934665603ull;
  for (size_t i = 0; i < n; i++) { h ^= ((const unsigned char *)p)[i]; h *= 1099511628211ull; }
  return h;
}
template <class M>
static unsigned long long map_hash(const M &m) { return fnv(m.data.data(), m.data.size()); }
static unsigned long long cells_hash(const vec_Vec3i &c) {
  std::vector<int32_t> v;
  for (const auto &it : c) { v.push_back(it(0)); v.push_back(it(1)); v.push_back(it(2)); }
  return fnv(v.data(), v.size() * 4);
}

int main(int argc, char **argv) {
  if (argc < 2) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  double o[3], d[3];
  float res;
  long long n;
  f.read((char *)o, sizeof(o)); f.read((char *)d, sizeof(d)); f.read((char *)&res, sizeof(res)); f.read((char *)&n, sizeof(n));
  std::vector<float> raw((size_t)n * 3 + 12);
  f.read((char *)raw.data(), raw.size() * sizeof(float));
  vec_Vec3f cloud; /* cloud_to_vec: float32 points widened */
  for (long long i = 0; i < n; i++) cloud.push_back(Vec3f(raw[3 * i], raw[3 * i + 1], raw[3 * i + 2]));
  const float *ex = raw.data() + 3 * n;
  const Vec3f add1(ex[0], ex[1], ex[2]), add2(ex[3], ex[4], ex[5]), clr1(ex[6], ex[7], ex[8]), clr2(ex[9], ex[10], ex[11]);

  /* cloud_to_map.cpp processCloud */
  VoxelGrid voxel_grid(Vec3f(o[0], o[1], o[2]), Vec3f(d[0], d[1], d[2]), res);
  voxel_grid.addCloud(cloud);
  auto map = voxel_grid.getMap();
  size_t occ = 0;
  for (auto v : map.data) occ += v == 100;
  std::printf("cloud_to_map: dim %d %d %d occupied %zu hash %llu cloud %zu\n", (int)map.dim.x, (int)map.dim.y, (int)map.dim.z, occ,
              map_hash(map), voxel_grid.getCloud().size());

  /* addCloud(pts, ns) with the node's 5 x 5 x 1 offsets on a fresh grid */
  vec_Vec3i ns;
  for (int nx = -2; nx <= 2; nx++)
    for (int ny = -2; ny <= 2; ny++) ns.push_back(Vec3i(nx, ny, 0));
  VoxelGrid inflated(Vec3f(o[0], o[1], o[2]), Vec3f(d[0], d[1], d[2]), res);
  vec_Vec3i obs = inflated.addCloud(cloud, ns);
  std::printf("inflated: new_obs %zu hash %llu\n", obs.size(), cells_hash(obs));

  /* map_replanner_node: map_util from getMap, freeUnknown; addCloudCallback; clearCloudCallback */
  std::shared_ptr<MPL::VoxelMapUtil> map_util(new MPL::VoxelMapUtil);
  map_util->setMap(Vec3f(map.origin.x, map.origin.y, map.origin.z), Vec3i(map.dim.x, map.dim.y, map.dim.z),
                   MPL::Tmap(map.data.begin(), map.data.end()), map.resolution);
  map_util->freeUnknown();
  vec_Vec3i new_obs;
  for (const auto &it : map_util->rayTrace(add1, add2))
    for (const auto &itt : ns) {
      const Vec3i pn(it(0) + itt(0), it(1) + itt(1), it(2) + itt(2));
      if (map_util->isFree(pn)) {
        voxel_grid.fill(pn(0), pn(1));
        new_obs.push_back(pn);
      }
    }
  voxel_grid.writeMap(*map_util);
  MPL::Tmap after = map_util->getMap();
  std::printf("add_cloud: new_obs %zu hash %llu map %llu\n", new_obs.size(), cells_hash(new_obs), fnv(after.data(), after.size()));
  vec_Vec3i new_clear;
  for (const auto &pn : map_util->rayTrace(clr1, clr2))
    if (map_util->isOccupied(pn)) {
      voxel_grid.clear(pn(0), pn(1));
      new_clear.push_back(pn);
    }
  voxel_grid.writeMap(*map_util);
  after = map_util->getMap();
  std::printf("clear_cloud: new_clear %zu hash %llu map %llu\n", new_clear.size(), cells_hash(new_clear), fnv(after.data(), after.size()));
  return 0;
}
