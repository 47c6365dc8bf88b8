/* Two replanners of the replanner node (mpl_test_node/src/map_replanner_node.cpp:107-241) driven through the fleet members of
 * this repo's header (planLPABatch, getLinkedNodesBatch, updateBlockedNodesBatch, updateClearedNodesBatch, getSubStateSpaceBatch,
 * MapUtil::traceCells) and, side by side, a second pair driven by the single members.  After every step it prints one digest
 * line per mode; tests/test_gpu_cpp_fleet.py checks that the two modes print the same lines.  argv[1]: corridor.bin. */
#include <mpl_b200/map_planner.hpp>

#include <cstdio>
#include <fstream>

using namespace MPL;

static unsigned long long mix(unsigned long long h, double v) {
  unsigned long long b;
  std::memcpy(&b, &v, 8);
  return (h ^ b) * 0x100000001B3ull;
}

int main(int argc, char **argv) {
  if (argc < 2) return 2;
  std::ifstream f(argv[1], std::ios::binary);
  int nd[2];
  double ori[2], res, st[2], gl[2];
  f.read((char *)nd, sizeof(nd)); f.read((char *)ori, sizeof(ori)); f.read((char *)&res, sizeof(res));
  f.read((char *)st, sizeof(st)); f.read((char *)gl, sizeof(gl));
  Tmap data((size_t)nd[0] * nd[1]);
  f.read((char *)data.data(), data.size());

  vec_E<VecDf> U;
  for (decimal_t dx = -0.5; dx <= 0.5; dx += 0.5)
    for (decimal_t dy = -0.5; dy <= 0.5; dy += 0.5) { VecDf u(2); u[0] = dx; u[1] = dy; U.push_back(u); }

  /* mode 0: fleet members, mode 1: single members; every replanner has its own map */
  std::shared_ptr<OccMapUtil> maps[2][2];
  std::unique_ptr<OccMapPlanner> pls[2][2];
  vec_E<Waypoint2D> starts[2], gs[2];
  for (int m = 0; m < 2; m++)
    for (int i = 0; i < 2; i++) {
      maps[m][i].reset(new OccMapUtil);
      maps[m][i]->setMap(Vec2f(ori[0], ori[1]), Vec2i(nd[0], nd[1]), data, res);
      maps[m][i]->freeUnknown();
      pls[m][i].reset(new OccMapPlanner(false));
      OccMapPlanner &p = *pls[m][i];
      p.setMapUtil(maps[m][i]); p.setVmax(1.0); p.setAmax(1.0); p.setDt(1.0); p.setU(U); p.setLPAstar(true);
      Waypoint2D s, g;
      s.pos = Vec2f(st[0], st[1]); s.vel = Vec2f::Zero(); s.acc = Vec2f::Zero(); s.jrk = Vec2f::Zero();
      s.use_pos = true; s.use_vel = true; s.use_acc = false; s.use_jrk = false; s.use_yaw = false;
      g = s;
      g.pos = Vec2f(gl[0], gl[1]);
      starts[m].push_back(s);
      gs[m].push_back(g);
    }
  std::vector<OccMapPlanner *> fleet = {pls[0][0].get(), pls[0][1].get()};

  auto digest = [&](const char *tag) {
    for (int m = 0; m < 2; m++) {
      unsigned long long h = 0xCBF29CE484222325ull;
      size_t n = 0;
      for (int i = 0; i < 2; i++) {
        OccMapPlanner &p = *pls[m][i];
        h = mix(h, p.getTrajCost());
        for (const auto &w : p.getTraj().getWaypoints()) { h = mix(h, w.pos(0)); h = mix(h, w.pos(1)); n++; }
        for (const auto &q : p.getCloseSet()) { h = mix(h, q(0)); h = mix(h, q(1)); }
        h = mix(h, (double)p.getOpenSet().size());
      }
      std::printf("%s mode %d: waypoints %zu digest %016llx\n", tag, m, n, h);
    }
  };
  auto plan = [&](const char *tag) { /* true when every planner found a trajectory of at least three waypoints */
    std::vector<bool> ok;
    OccMapPlanner::planLPABatch(fleet, starts[0], gs[0], &ok);
    bool all = ok[0] && ok[1];
    for (int i = 0; i < 2; i++) all = pls[1][i]->plan(starts[1][i], gs[1][i]) && all;
    std::printf("%s: ok batched %d %d\n", tag, (int)ok[0], (int)ok[1]);
    digest(tag);
    for (int m = 0; m < 2; m++) for (int i = 0; i < 2; i++) all = all && pls[m][i]->getTraj().getWaypoints().size() >= 3;
    return all;
  };
  if (!plan("first")) return 1;

  /* getLinkedNodes, then the add-cloud edit: a ray across each trajectory, its isFree cells of a 5 x 5 stencil become occupied */
  auto linked = OccMapPlanner::getLinkedNodesBatch(fleet);
  for (int i = 0; i < 2; i++) std::printf("linked %d: %zu %zu\n", i, linked[i].size(), pls[1][i]->getLinkedNodes().size());
  vec_Veci<2> ns;
  for (int x = -2; x <= 2; x++) for (int y = -2; y <= 2; y++) ns.push_back(Vec2i(x, y));
  std::vector<vec_Veci<2>> blocked[2];
  for (int m = 0; m < 2; m++)
    for (int i = 0; i < 2; i++) {
      const auto ws = pls[m][i]->getTraj().getWaypoints();
      const size_t k = (size_t)(ws.size() * 0.45);
      const vec_Vecf<2> a = {ws[k].pos}, b = {ws[k + 1].pos}; /* one segment of the path, as the node's two script points */
      vec_Veci<2> cells = maps[m][i]->traceCells(a, b, ns, MPLB_TRACE_FREE);
      Tmap mm = maps[m][i]->getMap();
      for (const auto &pn : cells) mm[pn(0) + nd[0] * pn(1)] = 100;
      maps[m][i]->setMap(maps[m][i]->getOrigin(), maps[m][i]->getDim(), mm, maps[m][i]->getRes());
      blocked[m].push_back(cells);
    }
  std::printf("blocked %zu %zu\n", blocked[0][0].size(), blocked[0][1].size());
  OccMapPlanner::updateBlockedNodesBatch(fleet, blocked[0]);
  for (int i = 0; i < 2; i++) pls[1][i]->updateBlockedNodes(blocked[1][i]);
  plan("blocked");

  /* clear-cloud: half of the cells are free again (the second replanner clears none) */
  OccMapPlanner::getLinkedNodesBatch(fleet);
  for (int i = 0; i < 2; i++) pls[1][i]->getLinkedNodes();
  std::vector<vec_Veci<2>> cleared[2];
  for (int m = 0; m < 2; m++)
    for (int i = 0; i < 2; i++) {
      vec_Veci<2> c(blocked[m][i].begin(), blocked[m][i].begin() + (i == 0 ? blocked[m][i].size() / 2 : 0));
      Tmap mm = maps[m][i]->getMap();
      for (const auto &pn : c) mm[pn(0) + nd[0] * pn(1)] = 0;
      maps[m][i]->setMap(maps[m][i]->getOrigin(), maps[m][i]->getDim(), mm, maps[m][i]->getRes());
      cleared[m].push_back(c);
    }
  OccMapPlanner::updateClearedNodesBatch(fleet, cleared[0]);
  for (int i = 0; i < 2; i++) pls[1][i]->updateClearedNodes(cleared[1][i]);
  const bool cleared_ok = plan("cleared");

  /* subtree: the roots move one and zero steps */
  if (!cleared_ok) return 1;
  for (int m = 0; m < 2; m++)
    for (int i = 0; i < 2; i++) starts[m][i] = pls[m][i]->getTraj().getWaypoints()[1 - i];
  OccMapPlanner::getSubStateSpaceBatch(fleet, {1, 0});
  pls[1][0]->getSubStateSpace(1);
  pls[1][1]->getSubStateSpace(0);
  plan("subtree");
  return 0;
}
