/* One replan cycle of two replanners (mpl_test_node/src/map_replanner_node.cpp:107-253) through the device members of this repo's
 * header: planLPABatchDevice, serializeLPABatch, trajectoryWaypointsBatch, getSubStateSpaceBatch, planLPABatchDevice from the
 * device starts, refineLPABatch.  A second pair runs the same cycle through planLPABatch and the host members.  After every plan it
 * prints, per mode, a digest of each planner's record, retained trajectory (mplb_get_actions / mplb_get_seg_states) and message
 * bytes (the host pair's rows uploaded into the plan-batch layout and serialised by the same member); the device mode also checks
 * its own rows and records against its retained trajectory.  tests/test_gpu_cpp_fleet_device.py compares the modes.
 * argv[1]: corridor.bin. */
#include <cuda_runtime.h>
#include <mpl_b200/map_planner.hpp>

#include <cstdio>
#include <cstring>
#include <fstream>

using namespace MPL;

static const int N = 2, MAX_SEG = 128;

static unsigned long long mix(unsigned long long h, const void *p, size_t n) {
  const unsigned char *b = (const unsigned char *)p;
  for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 0x100000001B3ull;
  return h;
}

static mplb_waypoint wp(const Waypoint2D &w) {
  mplb_waypoint c;
  std::memset(&c, 0, sizeof(c));
  for (int k = 0; k < 2; k++) { c.pos[k] = w.pos(k); c.vel[k] = w.vel(k); c.acc[k] = w.acc(k); c.jrk[k] = w.jrk(k); }
  c.yaw = w.yaw; c.t = w.t; c.control = (int)w.control;
  return c;
}

struct Layout { /* the plan-batch layout on the device */
  mplb_result *res = nullptr;
  int *act = nullptr;
  double *seg = nullptr;
  unsigned char *msg = nullptr;
  unsigned *len = nullptr;
  size_t stride = 0;
  Layout() {
    stride = mplb_trajectory_msg_size(MAX_SEG, "map");
    cudaMalloc((void **)&res, N * sizeof(mplb_result));
    cudaMalloc((void **)&act, (size_t)N * MAX_SEG * sizeof(int));
    cudaMalloc((void **)&seg, (size_t)N * MAX_SEG * 13 * sizeof(double));
    cudaMalloc((void **)&msg, N * stride);
    cudaMalloc((void **)&len, N * sizeof(unsigned));
  }
  ~Layout() { cudaFree(res); cudaFree(act); cudaFree(seg); cudaFree(msg); cudaFree(len); }
};

/* record, retained trajectory and message of every planner of one mode */
static void digest(const char *tag, int mode, std::vector<OccMapPlanner *> &pls, const Layout &L) {
  std::vector<OccMapPlanner *> fleet(pls.begin(), pls.end());
  if (!OccMapPlanner::serializeLPABatch(fleet, L.res, L.act, L.seg, MAX_SEG, L.msg, L.stride, L.len, 0.0, "map", 7, 1, 2)) {
    std::printf("%s mode %d: serialize failed\n", tag, mode);
    return;
  }
  std::vector<unsigned char> msg(N * L.stride);
  std::vector<unsigned> len(N);
  cudaMemcpy(msg.data(), L.msg, msg.size(), cudaMemcpyDeviceToHost);
  cudaMemcpy(len.data(), L.len, N * sizeof(unsigned), cudaMemcpyDeviceToHost);
  for (int i = 0; i < N; i++) {
    mplb_planner *h = pls[i]->handle();
    const int n = mplb_get_actions(h, nullptr, 0);
    std::vector<int> a(n > 0 ? n : 1);
    std::vector<double> s((size_t)(n > 0 ? n : 1) * 13);
    mplb_get_actions(h, a.data(), n);
    mplb_get_seg_states(h, s.data(), n);
    unsigned long long d = mix(0xCBF29CE484222325ull, a.data(), (size_t)std::max(n, 0) * sizeof(int));
    d = mix(d, s.data(), (size_t)std::max(n, 0) * 13 * sizeof(double));
    d = mix(d, msg.data() + i * L.stride, len[i]);
    std::printf("%s mode %d planner %d: n_seg %d len %u digest %016llx\n", tag, mode, i, n, len[i], d);
  }
}

/* the host pair's records and retained rows into the plan-batch layout */
static void upload(std::vector<OccMapPlanner *> &pls, const Layout &L) {
  std::vector<mplb_result> r(N);
  std::vector<int> a((size_t)N * MAX_SEG, -1);
  std::vector<double> s((size_t)N * MAX_SEG * 13, 0.0);
  for (int i = 0; i < N; i++) {
    r[i] = pls[i]->result();
    if (r[i].status != MPLB_PLAN_OK) continue;
    mplb_get_actions(pls[i]->handle(), &a[(size_t)i * MAX_SEG], MAX_SEG);
    mplb_get_seg_states(pls[i]->handle(), &s[(size_t)i * MAX_SEG * 13], MAX_SEG);
  }
  cudaMemcpy(L.res, r.data(), N * sizeof(mplb_result), cudaMemcpyHostToDevice);
  cudaMemcpy(L.act, a.data(), a.size() * sizeof(int), cudaMemcpyHostToDevice);
  cudaMemcpy(L.seg, s.data(), s.size() * sizeof(double), cudaMemcpyHostToDevice);
}

/* the device pair's own rows and records against its retained trajectory: 1 when they agree */
static int rows_match(std::vector<OccMapPlanner *> &pls, const Layout &L) {
  std::vector<mplb_result> r(N);
  std::vector<int> a((size_t)N * MAX_SEG);
  std::vector<double> s((size_t)N * MAX_SEG * 13);
  cudaMemcpy(r.data(), L.res, N * sizeof(mplb_result), cudaMemcpyDeviceToHost);
  cudaMemcpy(a.data(), L.act, a.size() * sizeof(int), cudaMemcpyDeviceToHost);
  cudaMemcpy(s.data(), L.seg, s.size() * sizeof(double), cudaMemcpyDeviceToHost);
  for (int i = 0; i < N; i++) {
    if (r[i].status != MPLB_PLAN_OK || r[i].n_seg > MAX_SEG) return 0;
    std::vector<int> ra(r[i].n_seg);
    std::vector<double> rs((size_t)r[i].n_seg * 13);
    if (mplb_get_actions(pls[i]->handle(), ra.data(), r[i].n_seg) != r[i].n_seg) return 0;
    mplb_get_seg_states(pls[i]->handle(), rs.data(), r[i].n_seg);
    if (std::memcmp(ra.data(), &a[(size_t)i * MAX_SEG], ra.size() * sizeof(int))) return 0;
    if (std::memcmp(rs.data(), &s[(size_t)i * MAX_SEG * 13], rs.size() * sizeof(double))) return 0;
    for (int j = r[i].n_seg; j < MAX_SEG; j++) if (a[(size_t)i * MAX_SEG + j] != -1) return 0;
  }
  return 1;
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

  /* mode 0: host members, mode 1: device members; every replanner has its own map; replanner 1 uses dt = 0.5 */
  std::shared_ptr<OccMapUtil> maps[2][N];
  std::unique_ptr<OccMapPlanner> owned[2][N];
  std::vector<OccMapPlanner *> pls[2];
  vec_E<Waypoint2D> starts, goals;
  for (int i = 0; i < N; i++) {
    Waypoint2D s, g;
    s.pos = Vec2f(st[0], st[1]); s.vel = Vec2f::Zero(); s.acc = Vec2f::Zero(); s.jrk = Vec2f::Zero();
    s.use_pos = true; s.use_vel = true; s.use_acc = false; s.use_jrk = false; s.use_yaw = false;
    g = s;
    g.pos = Vec2f(gl[0], gl[1]);
    starts.push_back(s);
    goals.push_back(g);
  }
  for (int m = 0; m < 2; m++)
    for (int i = 0; i < N; i++) {
      maps[m][i].reset(new OccMapUtil);
      maps[m][i]->setMap(Vec2f(ori[0], ori[1]), Vec2i(nd[0], nd[1]), data, res);
      maps[m][i]->freeUnknown();
      owned[m][i].reset(new OccMapPlanner(false));
      OccMapPlanner &p = *owned[m][i];
      p.setMapUtil(maps[m][i]); p.setVmax(1.0); p.setAmax(1.0); p.setDt(i == 0 ? 1.0 : 0.5); p.setU(U); p.setLPAstar(true);
      pls[m].push_back(&p);
    }
  Layout host_rows, dev_rows;
  mplb_waypoint *d_s = nullptr, *d_g = nullptr;
  int *d_k = nullptr, *d_ok = nullptr;
  cudaMalloc((void **)&d_s, N * sizeof(mplb_waypoint));
  cudaMalloc((void **)&d_g, N * sizeof(mplb_waypoint));
  cudaMalloc((void **)&d_k, N * sizeof(int));
  cudaMalloc((void **)&d_ok, N * sizeof(int));
  std::vector<mplb_waypoint> hs(N), hg(N);
  for (int i = 0; i < N; i++) { hs[i] = wp(starts[i]); hg[i] = wp(goals[i]); }
  cudaMemcpy(d_s, hs.data(), N * sizeof(mplb_waypoint), cudaMemcpyHostToDevice);
  cudaMemcpy(d_g, hg.data(), N * sizeof(mplb_waypoint), cudaMemcpyHostToDevice);

  auto plan = [&](const char *tag, const vec_E<Waypoint2D> &host_starts) {
    OccMapPlanner::planLPABatch(pls[0], host_starts, goals);
    upload(pls[0], host_rows);
    const bool ok = OccMapPlanner::planLPABatchDevice(pls[1], d_s, d_g, dev_rows.res, dev_rows.act, dev_rows.seg, MAX_SEG);
    std::printf("%s: device call %d rows %d\n", tag, (int)ok, rows_match(pls[1], dev_rows));
    digest(tag, 0, pls[0], host_rows);
    digest(tag, 1, pls[1], dev_rows);
  };
  plan("first", starts);

  /* the next start: getWaypoints()[1] on the host (mode 0) and on the device (mode 1), then getSubStateSpace(1) */
  vec_E<Waypoint2D> next = starts;
  for (int i = 0; i < N; i++) next[i] = pls[0][i]->getTraj().getWaypoints()[1];
  const int one[N] = {1, 1};
  cudaMemcpy(d_k, one, sizeof(one), cudaMemcpyHostToDevice);
  const bool wok = OccMapPlanner::trajectoryWaypointsBatch(pls[1], dev_rows.res, dev_rows.act, dev_rows.seg, MAX_SEG, d_k, d_s, d_ok);
  std::vector<mplb_waypoint> dn(N);
  int okv[N];
  cudaMemcpy(dn.data(), d_s, N * sizeof(mplb_waypoint), cudaMemcpyDeviceToHost);
  cudaMemcpy(okv, d_ok, sizeof(okv), cudaMemcpyDeviceToHost);
  for (int i = 0; i < N; i++) {
    const mplb_waypoint h = wp(next[i]);
    std::printf("next %d: call %d ok %d same %d\n", i, (int)wok, okv[i],
                (int)(std::memcmp(h.pos, dn[i].pos, sizeof(h.pos)) == 0 && std::memcmp(h.vel, dn[i].vel, sizeof(h.vel)) == 0 &&
                      h.t == dn[i].t));
  }
  OccMapPlanner::getSubStateSpaceBatch(pls[0], {1, 1});
  OccMapPlanner::getSubStateSpaceBatch(pls[1], {1, 1});
  plan("subtree", next);

  /* the refinement of both modes' rows: the same coefficient rows */
  double *d_c[2];
  std::vector<int32_t> ns[2];
  const size_t nc = (size_t)N * MAX_SEG * 3 * 6;
  std::vector<double> c[2];
  for (int m = 0; m < 2; m++) {
    cudaMalloc((void **)&d_c[m], nc * sizeof(double));
    const Layout &L = m == 0 ? host_rows : dev_rows;
    const bool ok = OccMapPlanner::refineLPABatch(pls[m], L.res, L.act, L.seg, MAX_SEG, d_c[m], &ns[m]);
    c[m].resize(nc);
    cudaMemcpy(c[m].data(), d_c[m], nc * sizeof(double), cudaMemcpyDeviceToHost);
    std::printf("refine mode %d: call %d n_segs %d %d digest %016llx\n", m, (int)ok, ns[m][0], ns[m][1],
                mix(0xCBF29CE484222325ull, c[m].data(), nc * sizeof(double)));
    cudaFree(d_c[m]);
  }
  cudaFree(d_s); cudaFree(d_g); cudaFree(d_k); cudaFree(d_ok);
  return 0;
}
