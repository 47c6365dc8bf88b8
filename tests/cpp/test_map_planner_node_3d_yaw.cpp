/* The planning block of map_planner_node (mpl_test_node/src/map_planner_node.cpp:106-196) with use_3d and use_yaw, typed
 * against this repo's header: {-u, 0, u}^3 x {-u_yaw, 0, u_yaw}, 81 rows of (dx, dy, dz, dyaw), ACCxYAW waypoints.
 * argv[1]: a 3-D map (dims, origin, res, start, goal, cells); argv[2], argv[3]: yaw_max and wyaw.
 * Prints "plan <ok> <cost> <n_seg>" and one "wp" line per waypoint (position and yaw in hex floats);
 * tests/test_gpu_shaped_wide_cpp.py compares them with the oracle. */
#include <mpl_b200/map_planner.hpp>

#include <cstdio>
#include <cstdlib>
#include <fstream>

using namespace MPL;

int main(int argc, char **argv) {
  if (argc < 4) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  int nd[3];
  double ori[3], res, st[3], gl[3];
  f.read((char *)nd, sizeof(nd)); f.read((char *)ori, sizeof(ori)); f.read((char *)&res, sizeof(res));
  f.read((char *)st, sizeof(st)); f.read((char *)gl, sizeof(gl));
  Tmap data((size_t)nd[0] * nd[1] * nd[2]);
  f.read((char *)data.data(), data.size());
  const double yaw_max = std::atof(argv[2]), wyaw = std::atof(argv[3]);

  std::shared_ptr<VoxelMapUtil> map_util = std::make_shared<VoxelMapUtil>();
  map_util->setMap(Vec3f(ori[0], ori[1], ori[2]), Vec3i(nd[0], nd[1], nd[2]), data, res);
  map_util->freeUnknown();

  const double v_max = 2.0, a_max = 1.0, dt = 1.0, u = 1.0, u_yaw = 0.3;
  const int num = 1;
  vec_E<VecDf> U;
  const decimal_t du = u / num;
  for (decimal_t dx = -u; dx <= u; dx += du)
    for (decimal_t dy = -u; dy <= u; dy += du)
      for (decimal_t dz = -u; dz <= u; dz += du)
        for (decimal_t dyaw = -u_yaw; dyaw <= u_yaw; dyaw += u_yaw) {
          VecDf vec(4);
          vec[0] = dx; vec[1] = dy; vec[2] = dz; vec[3] = dyaw;
          U.push_back(vec);
        }

  Waypoint3D start;
  start.pos = Vec3f(st[0], st[1], st[2]);
  start.vel = Vec3f(0, 0, 0);
  start.acc = Vec3f(0, 0, 0);
  start.jrk = Vec3f(0, 0, 0);
  start.yaw = 0;
  start.use_pos = true;
  start.use_vel = true;
  start.use_acc = false;
  start.use_jrk = false;
  start.use_yaw = true;

  Waypoint3D goal(start.control);
  goal.pos = Vec3f(gl[0], gl[1], gl[2]);
  goal.vel = Vec3f(0, 0, 0);
  goal.acc = Vec3f(0, 0, 0);
  goal.jrk = Vec3f(0, 0, 0);

  std::unique_ptr<VoxelMapPlanner> planner_ptr;
  planner_ptr.reset(new VoxelMapPlanner(false));
  planner_ptr->setMapUtil(map_util);
  planner_ptr->setVmax(v_max);
  planner_ptr->setAmax(a_max);
  planner_ptr->setYawmax(yaw_max);
  planner_ptr->setWyaw(wyaw);
  planner_ptr->setDt(dt);
  planner_ptr->setU(U);
  planner_ptr->setTol(0.5);

  const bool valid = planner_ptr->plan(start, goal);
  const auto ws = planner_ptr->getTraj().getWaypoints();
  std::printf("plan %d %a %d\n", valid ? 1 : 0, planner_ptr->getTrajCost(), valid ? (int)ws.size() - 1 : 0);
  if (valid)
    for (const auto &w : ws) std::printf("wp %a %a %a %a\n", w.pos(0), w.pos(1), w.pos(2), w.yaw);
  return 0;
}
