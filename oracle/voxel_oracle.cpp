// voxel_oracle.cpp — literal sequential restatement of planning_ros_utils' VoxelGrid (include/planning_ros_utils/voxel_grid.h,
// src/mapping_utils/voxel_grid.cpp, cited vg:<line>).  TEST INFRASTRUCTURE ONLY: the checker the GPU grid is compared with, and
// itself pinned to the reference's own voxel_grid.cpp (oracle/ref_voxel_harness.cpp exports the same orv_-shaped calls as rvx_).
//
// Storage is the reference's [x][y][z] (z fastest); outputs are the reference's (getMap x fastest, clouds x outermost).  Where
// the reference is undefined the oracle does what include/mplb.h defines: a NaN or beyond-int32 quotient is outside, clear(nx,
// ny) outside the grid is ignored, and allocate rejects a negative / beyond-int32 geometry (returns -1, nothing changes).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

struct Grid {
  int dim[3] = {0, 0, 0};
  int ori[3] = {0, 0, 0};
  double origin_d[3] = {0, 0, 0};
  float res = 0;
  std::vector<int8_t> map, inf; // [x][y][z]

  size_t at(int x, int y, int z) const { return ((size_t)x * dim[1] + y) * dim[2] + z; }
  bool outside(const int *n) const {
    return n[0] < 0 || n[0] >= dim[0] || n[1] < 0 || n[1] >= dim[1] || n[2] < 0 || n[2] >= dim[2];
  }
  // floatToInt (vg:201-203) on axis i; INT32_MIN where cast<int> is undefined
  int to_int1(double p, int i) const {
    const double q = (p - origin_d[i]) / (double)res;
    return (q > -2147483649.0 && q < 2147483648.0) ? (int)q : INT32_MIN;
  }
  // floatToInt (vg:201-203); false = cast<int> undefined (treated as outside)
  bool to_int(const double *pt, int *n) const {
    for (int i = 0; i < 3; i++) {
      const double q = (pt[i] - origin_d[i]) / (double)res;
      if (!(q > -2147483649.0 && q < 2147483648.0)) return false;
      n[i] = (int)q;
    }
    return true;
  }
  // intToFloat (vg:205-207)
  void to_float(const int *n, double *pt) const {
    for (int i = 0; i < 3; i++) pt[i] = ((double)n[i] + 0.5) * (double)res + origin_d[i];
  }
};

int allocate(Grid &g, const double *dim_m, const double *origin) { // vg:129-172; 1 changed, 0 unchanged, -1 rejected
  int nd[3], no[3];
  for (int i = 0; i < 3; i++) {
    const double qd = dim_m[i] / (double)g.res, qo = origin[i] / (double)g.res;
    if (!(qd > -1.0 && qd < 2147483648.0) || !(qo > -2147483649.0 && qo < 2147483648.0)) return -1;
    nd[i] = (int)qd;
    no[i] = (int)qo;
  }
  if (nd[2] == 0 && no[2] == 0) nd[2] = 1;
  if (nd[0] == g.dim[0] && nd[1] == g.dim[1] && nd[2] == g.dim[2] && no[0] == g.ori[0] && no[1] == g.ori[1] && no[2] == g.ori[2])
    return 0;
  const size_t n = (size_t)nd[0] * nd[1] * nd[2];
  if (n > 0x7fffffffull) return -1;
  std::vector<int8_t> nm(n, 0);
  for (int l = 0; l < nd[0]; l++)
    for (int w = 0; w < nd[1]; w++)
      for (int h = 0; h < nd[2]; h++)
        if (l + no[0] >= g.ori[0] && w + no[1] >= g.ori[1] && h + no[2] >= g.ori[2] && l + no[0] < g.ori[0] + g.dim[0] &&
            w + no[1] < g.ori[1] + g.dim[1] && h + no[2] < g.ori[2] + g.dim[2])
          nm[((size_t)l * nd[1] + w) * nd[2] + h] = g.map[g.at(l + no[0] - g.ori[0], w + no[1] - g.ori[1], h + no[2] - g.ori[2])];
  g.map = nm;
  g.inf = nm;
  for (int i = 0; i < 3; i++) { g.dim[i] = nd[i]; g.ori[i] = no[i]; g.origin_d[i] = origin[i]; }
  return 1;
}

int64_t cloud(const Grid &g, const std::vector<int8_t> &grid, const int *lo, const int *up, double *out, int64_t cap) {
  int64_t k = 0;
  int n[3];
  for (n[0] = lo[0]; n[0] < up[0]; n[0]++)
    for (n[1] = lo[1]; n[1] < up[1]; n[1]++)
      for (n[2] = lo[2]; n[2] < up[2]; n[2]++)
        if (grid[g.at(n[0], n[1], n[2])] > 0) {
          if (k < cap) g.to_float(n, out + 3 * k);
          k++;
        }
  return k;
}

}  // namespace

extern "C" {

void *orv_create(const double *origin, const double *dim_m, float res) { // vg:3-10
  Grid *g = new Grid();
  g->res = res;
  if (allocate(*g, dim_m, origin) < 0) { delete g; return nullptr; }
  return g;
}
void orv_destroy(void *h) { delete (Grid *)h; }
int orv_allocate(void *h, const double *dim_m, const double *origin) { return allocate(*(Grid *)h, dim_m, origin); }
void orv_info(void *h, int32_t *dim, int32_t *ori, double *origin_d, float *res) {
  const Grid &g = *(Grid *)h;
  for (int i = 0; i < 3; i++) { dim[i] = g.dim[i]; ori[i] = g.ori[i]; origin_d[i] = g.origin_d[i]; }
  *res = g.res;
}
void orv_clear(void *h) { // vg:12-16
  Grid &g = *(Grid *)h;
  std::fill(g.map.begin(), g.map.end(), 0);
  std::fill(g.inf.begin(), g.inf.end(), 0);
}
void orv_add_cloud(void *h, const double *pts, int64_t n) { // vg:174-180
  Grid &g = *(Grid *)h;
  for (int64_t i = 0; i < n; i++) {
    int c[3];
    if (!g.to_int(pts + 3 * i, c) || g.outside(c)) continue;
    g.map[g.at(c[0], c[1], c[2])] = 100;
  }
}
int64_t orv_add_cloud_inflated(void *h, const double *pts, int64_t n, const int32_t *ns, int n_ns, int32_t *out, int64_t cap) {
  Grid &g = *(Grid *)h; // vg:182-199
  int64_t k = 0;
  for (int64_t i = 0; i < n; i++) {
    int c[3];
    if (!g.to_int(pts + 3 * i, c) || g.outside(c)) continue;
    if (g.map[g.at(c[0], c[1], c[2])] != 100) {
      for (int j = 0; j < n_ns; j++) {
        const int c2[3] = {c[0] + ns[3 * j], c[1] + ns[3 * j + 1], c[2] + ns[3 * j + 2]};
        if (!g.outside(c2) && g.inf[g.at(c2[0], c2[1], c2[2])] != 100) {
          g.inf[g.at(c2[0], c2[1], c2[2])] = 100;
          if (k < cap) std::memcpy(out + 3 * k, c2, sizeof(c2));
          k++;
        }
      }
    }
    g.map[g.at(c[0], c[1], c[2])] = 100;
  }
  return k;
}
void orv_decay(void *h) { // vg:214-225
  Grid &g = *(Grid *)h;
  for (size_t i = 0; i < g.map.size(); i++) {
    if (g.map[i] > 0) g.map[i]--;
    if (g.inf[i] > 0) g.inf[i]--;
  }
}
void orv_fill(void *h, const int32_t *cells3, int n, int column) { // vg:35-45
  Grid &g = *(Grid *)h;
  for (int k = 0; k < n; k++) {
    const int x = cells3[3 * k], y = cells3[3 * k + 1], z = cells3[3 * k + 2];
    if (column) {
      if (x >= 0 && x < g.dim[0] && y >= 0 && y < g.dim[1])
        for (int nz = 0; nz < g.dim[2]; nz++) g.map[g.at(x, y, nz)] = 100;
    } else if (x >= 0 && x < g.dim[0] && y >= 0 && y < g.dim[1] && z >= 0 && z < g.dim[2]) {
      g.map[g.at(x, y, z)] = 100;
    }
  }
}
void orv_clear_columns(void *h, const int32_t *cells3, int n) { // vg:31-33 (outside ignored)
  Grid &g = *(Grid *)h;
  for (int k = 0; k < n; k++) {
    const int x = cells3[3 * k], y = cells3[3 * k + 1];
    if (x < 0 || x >= g.dim[0] || y < 0 || y >= g.dim[1]) continue;
    for (int nz = 0; nz < g.dim[2]; nz++) g.map[g.at(x, y, nz)] = 0;
  }
}
int64_t orv_get_cloud(void *h, double *out, int64_t cap) { // vg:18-29
  Grid &g = *(Grid *)h;
  const int lo[3] = {0, 0, 0};
  return cloud(g, g.map, lo, g.dim, out, cap);
}
int64_t orv_get_local_cloud(void *h, const double *pos, const double *ori, const double *dim, double *out, int64_t cap) {
  Grid &g = *(Grid *)h; // vg:47-69
  double a[3], b[3];
  for (int i = 0; i < 3; i++) { a[i] = pos[i] + ori[i]; b[i] = a[i] + dim[i]; }
  int lo[3], up[3];
  for (int i = 0; i < 3; i++) { // where cast<int> is undefined, x86 gives INT_MIN: an empty / unclipped bound
    const int n1 = g.to_int1(a[i], i), n2 = g.to_int1(b[i], i);
    lo[i] = n1 < 0 ? 0 : n1;
    up[i] = n2 > g.dim[i] ? g.dim[i] : n2;
  }
  return cloud(g, g.inf, lo, up, out, cap);
}
int64_t orv_get_map(void *h, int inflated, int8_t *out, int64_t cap) { // vg:71-127, x fastest
  Grid &g = *(Grid *)h;
  const std::vector<int8_t> &grid = inflated ? g.inf : g.map;
  const int64_t n = (int64_t)g.map.size();
  if (cap < n) return -1;
  for (int x = 0; x < g.dim[0]; x++)
    for (int y = 0; y < g.dim[1]; y++)
      for (int z = 0; z < g.dim[2]; z++)
        out[x + (int64_t)g.dim[0] * y + (int64_t)g.dim[0] * g.dim[1] * z] = grid[g.at(x, y, z)] > 0 ? 100 : 0;
  return n;
}

// MapUtil::rayTrace (map_util.h:117-134) on a grid of (origin, dim, res), with MapUtil::floatToInt's std::round
// (half away from zero, map_util.h:103-108); the replanner node traces its edit rays with it.
int64_t orv_map_ray_trace(const double *origin, const int32_t *dim, double res, const double *p1, const double *p2, int32_t *out,
                          int64_t cap) {
  double diff[3], q = 0;
  for (int i = 0; i < 3; i++) {
    diff[i] = p2[i] - p1[i];
    q = std::max(q, std::fabs(diff[i] / res)); // lpNorm<Infinity>
  }
  const int max_diff = (int)(q / 0.8);
  const double s = 1.0 / max_diff;
  int prev[3] = {-1, -1, -1};
  int64_t k = 0;
  for (int n = 1; n < max_diff; n++) {
    int pn[3];
    bool out_side = false;
    for (int i = 0; i < 3; i++) {
      const double pt = p1[i] + (diff[i] * s) * n;
      pn[i] = (int)std::round((pt - origin[i]) / res - 0.5);
      out_side = out_side || pn[i] < 0 || pn[i] >= dim[i];
    }
    if (out_side) break;
    if (pn[0] != prev[0] || pn[1] != prev[1] || pn[2] != prev[2]) {
      if (k < cap) std::memcpy(out + 3 * k, pn, sizeof(pn));
      k++;
    }
    std::memcpy(prev, pn, sizeof(pn));
  }
  return k;
}

}  // extern "C"
