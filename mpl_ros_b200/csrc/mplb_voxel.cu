/*
 * mplb_voxel.cu — VoxelGrid on the GPU: the map builder of planning_ros_utils (include/planning_ros_utils/voxel_grid.h,
 * src/mapping_utils/voxel_grid.cpp, cited vg:<line>) with both int8 grids resident in HBM, x fastest.
 *
 * Kernels (all memory bound):
 *   k_vg_shift          allocate's copy of map_ into the new geometry (vg:139-160)
 *   k_vg_add            addCloud(pts): one thread per point (vg:174-180); equal writes of 100 race benignly
 *   k_vg_point_keys / k_vg_point_first / k_vg_cand_keys / k_vg_cand_first / k_vg_emit
 *                       addCloud(pts, ns) (vg:182-199), whose output depends on the point order: per pass of consecutive
 *                       points, (cell, point) and (cell, candidate id = i * |ns| + j) pairs are radix-sorted (stable, so equal
 *                       cells keep id order) and the first claim of each cell wins; the winners are compacted in id order
 *   k_vg_decay          decay (vg:214-225)
 *   k_vg_fill / k_vg_clear_cols    fill / clear(nx, ny) (vg:31-45)
 *   k_vg_row_count / k_vg_row_emit getCloud / getLocalCloud (vg:18-69): counts per (x, y) row, scan, ordered write
 *   k_vg_binarize       getMap / getInflatedMap data (vg:71-127), also straight into an mplb_map's cells
 * The sorts and scans are CUB's device-wide primitives.  Scratch scales with points x |ns| of one pass (about 32 B per
 * candidate with CUB's sort storage) and with the x-y footprint for the clouds, never with the cell count (DESIGN.md 4.13).
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/mplb.h"
#include "mplb_internal.h"
#include "mplb_ref.h"

using namespace mplb_ref;

namespace {

/* geometry as the kernels see it */
struct Geo {
  int nd[3];
  double origin_d[3];
  float res;
};

int blocks_for(size_t n) { return (int)std::min<size_t>((n + 255) / 256, (size_t)148 * 32); }

__device__ __forceinline__ double load_pt(const void *pts, int fp32, long long k) {
  return fp32 ? (double)((const float *)pts)[k] : ((const double *)pts)[k];
}
/* floatToInt + isOutSide (vg:201-212): the linear x-fastest cell index, or -1 */
__device__ __forceinline__ long long point_cell(const Geo &g, const void *pts, int fp32, long long i, int *c) {
  for (int a = 0; a < 3; a++) {
    if (!vg_float_to_cell(load_pt(pts, fp32, i * 3 + a), g.origin_d[a], g.res, &c[a])) return -1;
    if (c[a] < 0 || c[a] >= g.nd[a]) return -1;
  }
  return (long long)c[0] + (long long)g.nd[0] * c[1] + (long long)g.nd[0] * g.nd[1] * c[2];
}

/* allocate (vg:139-160): new cell (l, w, h) takes old cell (l, w, h) + new_ori - ori when that is inside the old grid */
__global__ void k_vg_shift(const int8_t *old_map, int ox, int oy, int oz, int8_t *out, int nx, int ny, int nz, int sx, int sy,
                           int sz) {
  const size_t total = (size_t)nx * ny * nz;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const long long l = (long long)(i % nx) + sx, w = (long long)((i / nx) % ny) + sy, h = (long long)(i / ((size_t)nx * ny)) + sz;
    int8_t v = 0;
    if (l >= 0 && l < ox && w >= 0 && w < oy && h >= 0 && h < oz) v = old_map[l + (long long)ox * w + (long long)ox * oy * h];
    out[i] = v;
  }
}

__global__ void k_vg_add(Geo g, const void *pts, int fp32, long long n, int8_t *map) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    int c[3];
    const long long idx = point_cell(g, pts, fp32, i, c);
    if (idx >= 0) map[idx] = 100;
  }
}

/* one pass of addCloud(pts, ns) over points [i0, i0 + np): key = cell (ncell when outside), value = point */
__global__ void k_vg_point_keys(Geo g, const void *pts, int fp32, long long i0, int np, unsigned ncell, unsigned *key, unsigned *val) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < np; i += gridDim.x * blockDim.x) {
    int c[3];
    const long long idx = point_cell(g, pts, fp32, i0 + i, c);
    key[i] = idx >= 0 ? (unsigned)idx : ncell;
    val[i] = (unsigned)i;
  }
}
/* point i dilates iff it is inside, the first of the pass on its cell, and map_ there was not 100 when the pass began
 * (earlier passes have written their cells; later points of this pass on the same cell see the 100 point i writes) */
__global__ void k_vg_point_first(const unsigned *key, const unsigned *val, int np, unsigned ncell, const int8_t *map,
                                 unsigned *pcell) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x) {
    const unsigned c = key[k];
    const bool first = c < ncell && (k == 0 || key[k - 1] != c);
    pcell[val[k]] = (first && map[c] != 100) ? c : ncell; /* ncell: no dilation */
  }
}
/* candidate id = i * n_ns + j: key = cell n_i + ns_j when point i dilates, that cell is inside and inflated_map_ there was not
 * 100 when the pass began; ncell otherwise */
__global__ void k_vg_cand_keys(const unsigned *pcell, int np, const int *ns, int n_ns, int nx, int ny, int nz, unsigned ncell,
                               const int8_t *inf, unsigned *key, unsigned *val) {
  const long long total = (long long)np * n_ns;
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total; id += (long long)gridDim.x * blockDim.x) {
    const int i = (int)(id / n_ns), j = (int)(id % n_ns);
    const unsigned c = pcell[i];
    unsigned out = ncell;
    if (c < ncell) {
      const int x = (int)(c % (unsigned)nx) + ns[j * 3], y = (int)((c / (unsigned)nx) % (unsigned)ny) + ns[j * 3 + 1],
                z = (int)(c / ((unsigned)nx * (unsigned)ny)) + ns[j * 3 + 2];
      if (x >= 0 && x < nx && y >= 0 && y < ny && z >= 0 && z < nz) {
        const unsigned c2 = (unsigned)x + (unsigned)nx * y + (unsigned)nx * ny * z;
        if (inf[c2] != 100) out = c2;
      }
    }
    key[id] = out;
    val[id] = (unsigned)id;
  }
}
/* the first candidate (lowest id) on each cell is emitted: flag[id] = 1 */
__global__ void k_vg_cand_first(const unsigned *key, const unsigned *val, long long total, unsigned ncell, int *flag) {
  for (long long k = blockIdx.x * (long long)blockDim.x + threadIdx.x; k < total; k += (long long)gridDim.x * blockDim.x) {
    const unsigned c = key[k];
    flag[val[k]] = (c < ncell && (k == 0 || key[k - 1] != c)) ? 1 : 0;
  }
}
/* emitted candidates in id order: row base + pos[id] of new_obs (when < cap); inflated_map_ there becomes 100.  Then
 * every inside point's cell of map_ becomes 100 (k_vg_add over the same points). */
__global__ void k_vg_emit(const int *flag, const int *pos, const unsigned *pcell, long long total, const int *ns, int n_ns, int nx,
                          int ny, int8_t *inf, int *out, long long base, long long cap) {
  for (long long id = blockIdx.x * (long long)blockDim.x + threadIdx.x; id < total; id += (long long)gridDim.x * blockDim.x) {
    if (!flag[id]) continue;
    const int i = (int)(id / n_ns), j = (int)(id % n_ns);
    const unsigned c = pcell[i];
    const int x = (int)(c % (unsigned)nx) + ns[j * 3], y = (int)((c / (unsigned)nx) % (unsigned)ny) + ns[j * 3 + 1],
              z = (int)(c / ((unsigned)nx * (unsigned)ny)) + ns[j * 3 + 2];
    inf[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z] = 100;
    const long long r = base + pos[id];
    if (r < cap) { out[r * 3] = x; out[r * 3 + 1] = y; out[r * 3 + 2] = z; }
  }
}

__global__ void k_vg_decay(int8_t *a, int8_t *b, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    if (a[i] > 0) a[i]--;
    if (b[i] > 0) b[i]--;
  }
}

/* fill(nx, ny) (column) / fill(nx, ny, nz) / clear(nx, ny) (value 0, column) on map_, cells outside ignored */
__global__ void k_vg_fill(int8_t *map, const int *cells3, int n, int column, int8_t value, int nx, int ny, int nz) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int x = cells3[k * 3], y = cells3[k * 3 + 1], z = cells3[k * 3 + 2];
  if (x < 0 || x >= nx || y < 0 || y >= ny) return;
  if (column) {
    for (int h = 0; h < nz; h++) map[(size_t)x + (size_t)nx * y + (size_t)nx * ny * h] = value;
  } else if (z >= 0 && z < nz) {
    map[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z] = value;
  }
}

/* clouds over the box [lo, up): one thread per (x, y) with x fastest across threads (coalesced reads down each z);
 * row r = (x - lo0) * by + (y - lo1) is the reference's x-outermost order */
__global__ void k_vg_row_count(const int8_t *grid, int nx, int ny, int lo0, int lo1, int lo2, int bx, int by, int up2, int *cnt) {
  const long long rows = (long long)bx * by;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < rows; t += (long long)gridDim.x * blockDim.x) {
    const int x = lo0 + (int)(t % bx), y = lo1 + (int)(t / bx);
    int c = 0;
    for (int z = lo2; z < up2; z++) c += grid[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z] > 0;
    cnt[(long long)(x - lo0) * by + (y - lo1)] = c;
  }
}
__global__ void k_vg_row_emit(const int8_t *grid, Geo g, int lo0, int lo1, int lo2, int bx, int by, int up2, const int *off,
                              double *out, long long cap) {
  const int nx = g.nd[0], ny = g.nd[1];
  const long long rows = (long long)bx * by;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < rows; t += (long long)gridDim.x * blockDim.x) {
    const int x = lo0 + (int)(t % bx), y = lo1 + (int)(t / bx);
    long long r = off[(long long)(x - lo0) * by + (y - lo1)];
    for (int z = lo2; z < up2 && r < cap; z++) {
      if (grid[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z] <= 0) continue;
      out[r * 3] = vg_cell_to_float(x, g.origin_d[0], g.res);
      out[r * 3 + 1] = vg_cell_to_float(y, g.origin_d[1], g.res);
      out[r * 3 + 2] = vg_cell_to_float(z, g.origin_d[2], g.res);
      r++;
    }
  }
}

__global__ void k_vg_binarize(const int8_t *src, int8_t *dst, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = src[i] > 0 ? 100 : 0;
}

__global__ void k_map_get_cells(const int8_t *grid, int dim, int nx, int ny, int nz, const int *cells3, int n, int *values) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int x = cells3[k * 3], y = cells3[k * 3 + 1], z = dim == 3 ? cells3[k * 3 + 2] : 0;
  values[k] = (x < 0 || x >= nx || y < 0 || y >= ny || z < 0 || z >= nz) ? INT_MIN
                                                                          : (int)grid[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z];
}

/* ---- MapUtil::rayTrace (mu:117-134) and the replanner node's cell selection (map_replanner_node.cpp:199-219,221-229).
 * Ray r examines its points n = 1 .. len[r] (slot r * B + n - 1; B bounds the points a ray can have inside the map), cut[r] is
 * its first point outside the map (or len[r] + 1), and a point is traced when it comes before the cut and its cell differs
 * from the previous point's. */
__device__ __forceinline__ void ray_ends(const MplbMapView &m, const double *p1s, const double *p2s, long long r, double *a, double *b) {
  for (int k = 0; k < m.dim; k++) { a[k] = p1s[r * 3 + k]; b[k] = p2s[r * 3 + k]; }
}
__device__ __forceinline__ void ray_cell(const MplbMapView &m, const double *a, const double *diff, double s, int n, int *pn) {
  double pt[3];
  for (int k = 0; k < m.dim; k++) pt[k] = ray_point(a[k], diff[k], s, n);
  float_to_int(m, pt, pn);
}
__device__ __forceinline__ bool trace_keep(const MplbMapView &m, const int *c, int select) {
  if (select == MPLB_TRACE_ALL) return true;
  if (outside(m, c)) return false; /* isFree / isOccupied are false outside (mu:44-69) */
  const int8_t v = m.d_grid[(size_t)c[0] + (size_t)m.nd[0] * c[1] + (m.dim == 3 ? (size_t)m.nd[0] * m.nd[1] * c[2] : 0)];
  return select == MPLB_TRACE_FREE ? (v >= 0 && v < 100) : v == 100;
}

/* one thread per ray: the endpoint checks, the points to examine, the initial cut */
__global__ void k_trace_rays(MplbMapView m, const double *p1s, const double *p2s, int n_rays, int B, int *len, int *cut, int *bad) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rays) return;
  double a[3], b[3], diff[3];
  ray_ends(m, p1s, p2s, r, a, b);
  bool ok = true;
  for (int k = 0; k < m.dim; k++) ok = ok && isfinite(a[k]) && isfinite(b[k]);
  ok = ok && ray_span(m.dim, m.res, a, b, diff) < 2147483648.0;
  int l = 0;
  if (ok) {
    double s;
    l = min(ray_setup(m.dim, m.res, a, b, diff, &s) - 1, B);
    if (l < 0) l = 0;
  } else {
    atomicOr(bad, 1);
  }
  len[r] = l;
  cut[r] = l + 1;
}
/* one thread per slot: the first point outside the map cuts the ray */
__global__ void k_trace_cut(MplbMapView m, const double *p1s, const double *p2s, long long slots, int B, const int *len, int *cut) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < slots; t += (long long)gridDim.x * blockDim.x) {
    const long long r = t / B;
    const int n = (int)(t % B) + 1;
    if (n > len[r]) continue;
    double a[3], b[3], diff[3], s;
    ray_ends(m, p1s, p2s, r, a, b);
    ray_setup(m.dim, m.res, a, b, diff, &s);
    int pn[3];
    ray_cell(m, a, diff, s, n, pn);
    if (outside(m, pn)) atomicMin(&cut[r], n);
  }
}
/* slot t's traced cell (false when the slot traces none) */
__device__ __forceinline__ bool slot_cell(const MplbMapView &m, const double *p1s, const double *p2s, long long t, int B, const int *cut,
                                          int *pn) {
  const long long r = t / B;
  const int n = (int)(t % B) + 1;
  if (n >= cut[r]) return false;
  double a[3], b[3], diff[3], s;
  ray_ends(m, p1s, p2s, r, a, b);
  ray_setup(m.dim, m.res, a, b, diff, &s);
  ray_cell(m, a, diff, s, n, pn);
  if (n == 1) return true; /* the reference's previous cell starts at -1, never a cell inside */
  int pp[3];
  ray_cell(m, a, diff, s, n - 1, pp);
  return pn[0] != pp[0] || pn[1] != pp[1] || pn[2] != pp[2];
}
/* one thread per slot: how many of its candidates pn + ns[k] the selection keeps */
__global__ void k_trace_count(MplbMapView m, const double *p1s, const double *p2s, long long slots, int B, const int *cut, const int *ns,
                              int n_ns, int select, int *cnt) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < slots; t += (long long)gridDim.x * blockDim.x) {
    int pn[3];
    int c = 0;
    if (slot_cell(m, p1s, p2s, t, B, cut, pn))
      for (int k = 0; k < n_ns; k++) {
        const int q[3] = {pn[0] + ns[k * 3], pn[1] + ns[k * 3 + 1], m.dim == 3 ? pn[2] + ns[k * 3 + 2] : 0};
        c += trace_keep(m, q, select);
      }
    cnt[t] = c;
  }
}
/* one thread per slot: its kept candidates at their place in (ray, point, offset) order (pos = exclusive scan of the counts),
 * the first `cap` rows only; offsets[r] and, from slot 0, offsets[n_rays] and the total (-1: an endpoint was rejected) */
__global__ void k_trace_emit(MplbMapView m, const double *p1s, const double *p2s, int n_rays, long long slots, int B, const int *cut,
                             const int *ns, int n_ns, int select, const int *cnt, const int *pos, const int *bad, int *out, long long cap,
                             long long *offsets, long long *total) {
  if (*bad) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *total = -1;
    return;
  }
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < slots; t += (long long)gridDim.x * blockDim.x) {
    long long w = pos[t];
    if (offsets && t % B == 0) offsets[t / B] = w;
    if (t == 0) {
      const long long all = (long long)pos[slots - 1] + cnt[slots - 1];
      if (offsets) offsets[n_rays] = all;
      *total = all;
    }
    int pn[3];
    if (w >= cap || !slot_cell(m, p1s, p2s, t, B, cut, pn)) continue;
    for (int k = 0; k < n_ns && w < cap; k++) {
      const int q[3] = {pn[0] + ns[k * 3], pn[1] + ns[k * 3 + 1], m.dim == 3 ? pn[2] + ns[k * 3 + 2] : 0};
      if (!trace_keep(m, q, select)) continue;
      out[w * 3] = q[0]; out[w * 3 + 1] = q[1]; out[w * 3 + 2] = q[2];
      w++;
    }
  }
}

int key_bits(unsigned ncell) { /* radix-sort bits covering keys 0 .. ncell */
  int b = 1;
  while (b < 32 && (1ull << b) <= ncell) b++;
  return b;
}

}  // namespace

struct mplb_voxel_grid {
  int dim[3] = {0, 0, 0};
  int ori[3] = {0, 0, 0};
  double origin_d[3] = {0, 0, 0};
  float res = 0;
  size_t ncell = 0;
  int device = 0;
  DevBuf<int8_t> d_map, d_inf;
  long long chunk_points = 0;
  /* scratch of the inflated insertion and of the clouds */
  DevBuf<unsigned> k0, k1, v0, v1, pcell;
  DevBuf<int> flag, pos, ns, cells, rows, obs;
  DevBuf<double> pts;
  DevBuf<char> tmp;
  DevBuf<int8_t> bytes;

  Geo geo() const {
    Geo g;
    for (int i = 0; i < 3; i++) { g.nd[i] = dim[i]; g.origin_d[i] = origin_d[i]; }
    g.res = res;
    return g;
  }
};

namespace {

int vg_allocate(mplb_voxel_grid *g, const double *dim_m, const double *origin, int32_t *changed) {
  int nd[3], no[3];
  for (int i = 0; i < 3; i++) { /* Vec3i new_dim(new_dim_d(i) / res_, ...), the float res_ widened (vg:130-131) */
    const double qd = dim_m[i] / (double)g->res, qo = origin[i] / (double)g->res;
    if (!(qd > -1.0 && qd < 2147483648.0)) return mplb_internal_fail(MPLB_ERR_ARG, "voxel grid dimension negative, NaN or beyond int32");
    if (!(qo > -2147483649.0 && qo < 2147483648.0)) return mplb_internal_fail(MPLB_ERR_ARG, "voxel grid origin NaN or beyond int32");
    nd[i] = (int)qd;
    no[i] = (int)qo;
  }
  if (nd[2] == 0 && no[2] == 0) nd[2] = 1; /* vg:132 */
  if (changed) *changed = 0;
  if (nd[0] == g->dim[0] && nd[1] == g->dim[1] && nd[2] == g->dim[2] && no[0] == g->ori[0] && no[1] == g->ori[1] &&
      no[2] == g->ori[2])
    return MPLB_OK; /* vg:134-137 */
  const size_t ncell = (size_t)nd[0] * nd[1] * nd[2];
  if (ncell > 0x7fffffffull) return mplb_internal_fail(MPLB_ERR_ARG, "voxel grid of more than 2^31 - 1 cells");
  DevBuf<int8_t> m, f;
  if (ncell) {
    MPLB_CUDA_TRY(m.reserve(ncell));
    MPLB_CUDA_TRY(f.reserve(ncell));
    k_vg_shift<<<blocks_for(ncell), 256>>>(g->d_map.p, g->dim[0], g->dim[1], g->dim[2], m.p, nd[0], nd[1], nd[2], no[0] - g->ori[0],
                                            no[1] - g->ori[1], no[2] - g->ori[2]);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
    MPLB_CUDA_TRY(cudaMemcpy(f.p, m.p, ncell, cudaMemcpyDeviceToDevice)); /* inflated_map_ = new_map (vg:163-164) */
  }
  g->d_map = std::move(m); /* frees the old grids */
  g->d_inf = std::move(f);
  g->ncell = ncell;
  for (int i = 0; i < 3; i++) { g->dim[i] = nd[i]; g->ori[i] = no[i]; g->origin_d[i] = origin[i]; }
  if (changed) *changed = 1;
  return MPLB_OK;
}

/* the CUB temporary storage of one call */
template <class F>
int with_tmp(mplb_voxel_grid *g, F f) {
  size_t bytes = 0;
  MPLB_CUDA_TRY(f((void *)nullptr, bytes));
  MPLB_CUDA_TRY(g->tmp.reserve(std::max<size_t>(bytes, 1)));
  MPLB_CUDA_TRY(f((void *)g->tmp.p, bytes));
  return MPLB_OK;
}

/* addCloud(pts, ns) over device points; new_obs rows go to `out` (device) from row 0, the first `cap` of them */
long long vg_add_inflated(mplb_voxel_grid *g, const void *d_pts, long long n, int fp32, const int *h_ns, int n_ns, int *out,
                          long long cap, cudaStream_t s) {
  if (n <= 0 || n_ns <= 0 || g->ncell == 0) {
    if (n > 0 && g->ncell) { /* no offsets: only map_ changes */
      k_vg_add<<<blocks_for((size_t)n), 256, 0, s>>>(g->geo(), d_pts, fp32, n, g->d_map.p);
      mplb_internal_count_launches(1);
      MPLB_CUDA_TRY(cudaGetLastError());
      MPLB_CUDA_TRY(cudaStreamSynchronize(s));
    }
    return 0;
  }
  long long chunk = g->chunk_points > 0 ? g->chunk_points : std::max<long long>(1, (1ll << 22) / n_ns);
  chunk = std::min<long long>(chunk, std::max<long long>(1, 0x7fffffffll / n_ns)); /* candidate ids stay below 2^31 */
  chunk = std::min(chunk, n);
  const long long cand = chunk * n_ns;
  const unsigned ncell = (unsigned)g->ncell;
  const int bits = key_bits(ncell);
  MPLB_CUDA_TRY(g->ns.reserve((size_t)n_ns * 3));
  MPLB_CUDA_TRY(cudaMemcpyAsync(g->ns.p, h_ns, (size_t)n_ns * 3 * sizeof(int), cudaMemcpyHostToDevice, s));
  MPLB_CUDA_TRY(g->k0.reserve((size_t)cand)); MPLB_CUDA_TRY(g->k1.reserve((size_t)cand));
  MPLB_CUDA_TRY(g->v0.reserve((size_t)cand)); MPLB_CUDA_TRY(g->v1.reserve((size_t)cand));
  MPLB_CUDA_TRY(g->pcell.reserve((size_t)chunk));
  MPLB_CUDA_TRY(g->flag.reserve((size_t)cand)); MPLB_CUDA_TRY(g->pos.reserve((size_t)cand));
  const Geo geo = g->geo();
  long long total = 0;
  for (long long i0 = 0; i0 < n; i0 += chunk) {
    const int np = (int)std::min(chunk, n - i0);
    const long long nc = (long long)np * n_ns;
    k_vg_point_keys<<<blocks_for(np), 256, 0, s>>>(geo, d_pts, fp32, i0, np, ncell, g->k0.p, g->v0.p);
    MPLB_CUDA_TRY(cudaGetLastError());
    int rc = with_tmp(g, [&](void *t, size_t &b) {
      return cub::DeviceRadixSort::SortPairs(t, b, g->k0.p, g->k1.p, g->v0.p, g->v1.p, np, 0, bits, s);
    });
    if (rc) return rc;
    k_vg_point_first<<<blocks_for(np), 256, 0, s>>>(g->k1.p, g->v1.p, np, ncell, g->d_map.p, g->pcell.p);
    k_vg_cand_keys<<<blocks_for(nc), 256, 0, s>>>(g->pcell.p, np, g->ns.p, n_ns, g->dim[0], g->dim[1], g->dim[2], ncell, g->d_inf.p,
                                                  g->k0.p, g->v0.p);
    MPLB_CUDA_TRY(cudaGetLastError());
    rc = with_tmp(g, [&](void *t, size_t &b) {
      return cub::DeviceRadixSort::SortPairs(t, b, g->k0.p, g->k1.p, g->v0.p, g->v1.p, (int)nc, 0, bits, s);
    });
    if (rc) return rc;
    k_vg_cand_first<<<blocks_for(nc), 256, 0, s>>>(g->k1.p, g->v1.p, nc, ncell, g->flag.p);
    MPLB_CUDA_TRY(cudaGetLastError());
    rc = with_tmp(g, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, g->flag.p, g->pos.p, (int)nc, s); });
    if (rc) return rc;
    k_vg_emit<<<blocks_for(nc), 256, 0, s>>>(g->flag.p, g->pos.p, g->pcell.p, nc, g->ns.p, n_ns, g->dim[0], g->dim[1], g->d_inf.p,
                                             out, total, cap);
    k_vg_add<<<blocks_for(np), 256, 0, s>>>(geo, (const char *)d_pts + i0 * 3 * (fp32 ? 4 : 8), fp32, np, g->d_map.p);
    mplb_internal_count_launches(9);
    MPLB_CUDA_TRY(cudaGetLastError());
    int last[2];
    MPLB_CUDA_TRY(cudaMemcpyAsync(&last[0], g->pos.p + nc - 1, sizeof(int), cudaMemcpyDeviceToHost, s));
    MPLB_CUDA_TRY(cudaMemcpyAsync(&last[1], g->flag.p + nc - 1, sizeof(int), cudaMemcpyDeviceToHost, s));
    MPLB_CUDA_TRY(cudaStreamSynchronize(s));
    total += (long long)last[0] + last[1];
  }
  return total;
}

/* getCloud / getLocalCloud over the box [lo, up) of `grid` into device rows `out` */
long long vg_cloud(mplb_voxel_grid *g, const int8_t *grid, const int *lo, const int *up, double *out, long long cap, cudaStream_t s) {
  for (int i = 0; i < 3; i++) if (up[i] <= lo[i]) return 0;
  const int bx = up[0] - lo[0], by = up[1] - lo[1];
  const long long rows = (long long)bx * by;
  MPLB_CUDA_TRY(g->rows.reserve((size_t)rows + 1));
  MPLB_CUDA_TRY(g->flag.reserve((size_t)rows + 1));
  k_vg_row_count<<<blocks_for(rows), 256, 0, s>>>(grid, g->dim[0], g->dim[1], lo[0], lo[1], lo[2], bx, by, up[2], g->flag.p);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cudaMemsetAsync(g->flag.p + rows, 0, sizeof(int), s));
  int rc = with_tmp(g, [&](void *t, size_t &b) { return cub::DeviceScan::ExclusiveSum(t, b, g->flag.p, g->rows.p, (int)rows + 1, s); });
  if (rc) return rc;
  if (out && cap > 0) {
    k_vg_row_emit<<<blocks_for(rows), 256, 0, s>>>(grid, g->geo(), lo[0], lo[1], lo[2], bx, by, up[2], g->rows.p, out, cap);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  mplb_internal_count_launches(out && cap > 0 ? 3 : 2);
  int total = 0;
  MPLB_CUDA_TRY(cudaMemcpyAsync(&total, g->rows.p + rows, sizeof(int), cudaMemcpyDeviceToHost, s));
  MPLB_CUDA_TRY(cudaStreamSynchronize(s));
  return total;
}

long long host_cloud(mplb_voxel_grid *g, const int8_t *grid, const int *lo, const int *up, double *pts, long long cap) {
  long long n = vg_cloud(g, grid, lo, up, nullptr, 0, 0);
  if (n <= 0 || !pts || cap <= 0) return n;
  const long long w = std::min(n, cap);
  MPLB_CUDA_TRY(g->pts.reserve((size_t)w * 3));
  long long rc = vg_cloud(g, grid, lo, up, g->pts.p, w, 0);
  if (rc < 0) return rc;
  MPLB_CUDA_TRY(cudaMemcpy(pts, g->pts.p, (size_t)w * 3 * sizeof(double), cudaMemcpyDeviceToHost));
  return n;
}

int check_grid(const mplb_voxel_grid *g) {
  if (!g) return mplb_internal_fail(MPLB_ERR_ARG, "null voxel grid");
  if (mplb_internal_set_device(g->device)) return mplb_internal_fail(MPLB_ERR_CUDA, "cannot select the voxel grid's device");
  return MPLB_OK;
}

int upload_cells(mplb_voxel_grid *g, const int32_t *cells3, int n) {
  MPLB_CUDA_TRY(g->cells.reserve((size_t)n * 3));
  MPLB_CUDA_TRY(cudaMemcpy(g->cells.p, cells3, (size_t)n * 3 * sizeof(int), cudaMemcpyHostToDevice));
  return MPLB_OK;
}

/* fill / clear with the cell rows on the host (device = false) or already on the grid's device, read on `stream` */
int vg_edit(mplb_voxel_grid *g, const int32_t *cells3, int n, int column, int8_t value, bool device, cudaStream_t stream) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0 || (n > 0 && !cells3)) return mplb_internal_fail(MPLB_ERR_ARG, "bad cell buffer");
  if (n == 0 || !g->ncell) return MPLB_OK;
  const int *d_cells = (const int *)cells3;
  if (!device) {
    rc = upload_cells(g, cells3, n);
    if (rc) return rc;
    d_cells = g->cells.p;
  }
  k_vg_fill<<<(n + 255) / 256, 256, 0, stream>>>(g->d_map.p, d_cells, n, column, value, g->dim[0], g->dim[1], g->dim[2]);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(device ? cudaStreamSynchronize(stream) : cudaDeviceSynchronize());
  return MPLB_OK;
}

/* scratch of the ray tracer, per host thread (re-created when the thread's current device changes) */
struct TraceScratch {
  int device = -1;
  DevBuf<int> len, cut, ns, bad, out, cnt, pos;
  DevBuf<long long> total, offs;
  DevBuf<double> pts;
  DevBuf<char> tmp;
};
thread_local TraceScratch g_trace;
TraceScratch &trace_scratch(int device) {
  if (g_trace.device != device) { g_trace = TraceScratch(); g_trace.device = device; }
  return g_trace;
}

/* rays examine up to B points each: consecutive points are at least 0.8 res apart on the ray's dominant axis, so no ray has
 * more points inside the map before its first one outside */
int trace_points_per_ray(const MplbMapView &v) {
  int max_nd = 0;
  for (int k = 0; k < v.dim; k++) max_nd = std::max(max_nd, v.nd[k]);
  return (int)((max_nd + 2.0) / 0.8) + 2;
}
/* the most rows a call can select */
int64_t trace_bound(const MplbMapView &v, int n_rays, int n_ns) {
  return (int64_t)n_rays * trace_points_per_ray(v) * std::max(n_ns, 1);
}

/* rays (d_p1s, d_p2s: device rows of 3 doubles) through map view v on stream st: the first `cap` selected cells to d_out, the
 * n_rays + 1 offsets to d_offsets (may be NULL); returns the total count or an error */
int64_t trace_cells(const MplbMapView &v, const double *d_p1s, const double *d_p2s, int n_rays, const int32_t *ns, int n_ns,
                    int select, int *d_out, int64_t cap, long long *d_offsets, cudaStream_t st) {
  TraceScratch &g = trace_scratch(v.device);
  if (n_rays == 0) {
    if (d_offsets) MPLB_CUDA_TRY(cudaMemsetAsync(d_offsets, 0, sizeof(long long), st));
    MPLB_CUDA_TRY(cudaStreamSynchronize(st));
    return 0;
  }
  const int zero3[3] = {0, 0, 0};
  if (n_ns == 0) { ns = zero3; n_ns = 1; } /* the offset 0 alone: the ray's own cells */
  const int B = trace_points_per_ray(v);
  const long long slots = (long long)n_rays * B;
  if (slots * n_ns > 0x7fffffff) return mplb_internal_fail(MPLB_ERR_ARG, "trace_cells: more than 2^31 - 1 candidate cells to examine");
  MPLB_CUDA_TRY(g.len.reserve(n_rays));
  MPLB_CUDA_TRY(g.cut.reserve(n_rays));
  MPLB_CUDA_TRY(g.bad.reserve(1));
  MPLB_CUDA_TRY(g.total.reserve(1));
  MPLB_CUDA_TRY(g.ns.reserve((size_t)n_ns * 3));
  MPLB_CUDA_TRY(g.cnt.reserve(slots));
  MPLB_CUDA_TRY(g.pos.reserve(slots));
  MPLB_CUDA_TRY(cudaMemcpyAsync(g.ns.p, ns, (size_t)n_ns * 3 * sizeof(int), cudaMemcpyHostToDevice, st));
  MPLB_CUDA_TRY(cudaMemsetAsync(g.bad.p, 0, sizeof(int), st));
  size_t tmp_bytes = 0;
  MPLB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, g.cnt.p, g.pos.p, (int)slots, st));
  MPLB_CUDA_TRY(g.tmp.reserve(std::max<size_t>(tmp_bytes, 1)));
  k_trace_rays<<<(n_rays + 127) / 128, 128, 0, st>>>(v, d_p1s, d_p2s, n_rays, B, g.len.p, g.cut.p, g.bad.p);
  k_trace_cut<<<blocks_for((size_t)slots), 256, 0, st>>>(v, d_p1s, d_p2s, slots, B, g.len.p, g.cut.p);
  k_trace_count<<<blocks_for((size_t)slots), 256, 0, st>>>(v, d_p1s, d_p2s, slots, B, g.cut.p, g.ns.p, n_ns, select, g.cnt.p);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cub::DeviceScan::ExclusiveSum(g.tmp.p, tmp_bytes, g.cnt.p, g.pos.p, (int)slots, st));
  k_trace_emit<<<blocks_for((size_t)slots), 256, 0, st>>>(v, d_p1s, d_p2s, n_rays, slots, B, g.cut.p, g.ns.p, n_ns, select, g.cnt.p,
                                                           g.pos.p, g.bad.p, d_out, cap, d_offsets, g.total.p);
  mplb_internal_count_launches(5);
  MPLB_CUDA_TRY(cudaGetLastError());
  long long total = 0;
  MPLB_CUDA_TRY(cudaMemcpyAsync(&total, g.total.p, sizeof(total), cudaMemcpyDeviceToHost, st));
  MPLB_CUDA_TRY(cudaStreamSynchronize(st));
  if (total < 0) return mplb_internal_fail(MPLB_ERR_ARG, "trace_cells: an endpoint is not finite, or a ray has 2^31 or more steps");
  return total;
}

int check_trace_args(const mplb_map *m, int n_rays, bool rays, const int32_t *ns, int n_ns, int select, bool out, int64_t cap) {
  if (!m) return mplb_internal_fail(MPLB_ERR_ARG, "null map");
  if (n_rays < 0 || (n_rays > 0 && !rays)) return mplb_internal_fail(MPLB_ERR_ARG, "bad ray buffers");
  if (n_ns < 0 || (n_ns > 0 && !ns)) return mplb_internal_fail(MPLB_ERR_ARG, "bad stencil");
  if (select != MPLB_TRACE_ALL && select != MPLB_TRACE_FREE && select != MPLB_TRACE_OCCUPIED)
    return mplb_internal_fail(MPLB_ERR_ARG, "unknown selection");
  if (cap < 0 || (cap > 0 && !out)) return mplb_internal_fail(MPLB_ERR_ARG, "bad output buffer");
  return MPLB_OK;
}

}  // namespace

extern "C" {

int mplb_voxel_grid_create(const double *origin, const double *dim_m, float res, mplb_voxel_grid **out) {
  if (!origin || !dim_m || !out) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  if (!(res > 0) || !std::isfinite(res)) return mplb_internal_fail(MPLB_ERR_ARG, "voxel grid resolution must be finite and > 0");
  mplb_voxel_grid *g = new mplb_voxel_grid();
  g->res = res;
  if (cudaGetDevice(&g->device) != cudaSuccess) { delete g; return mplb_internal_fail(MPLB_ERR_CUDA, "no CUDA device (libmplb has no CPU path)"); }
  int rc = vg_allocate(g, dim_m, origin, nullptr);
  if (rc == MPLB_OK && cudaDeviceSynchronize() != cudaSuccess) rc = mplb_internal_fail(MPLB_ERR_CUDA, "voxel grid allocation");
  if (rc != MPLB_OK) { delete g; return rc; }
  *out = g;
  return MPLB_OK;
}

void mplb_voxel_grid_destroy(mplb_voxel_grid *g) {
  if (!g) return;
  mplb_internal_set_device(g->device);
  delete g;
}

int mplb_voxel_grid_allocate(mplb_voxel_grid *g, const double *dim_m, const double *origin, int32_t *changed) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!dim_m || !origin) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  rc = vg_allocate(g, dim_m, origin, changed);
  if (rc) return rc;
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  return MPLB_OK;
}

int mplb_voxel_grid_get_info(const mplb_voxel_grid *g, int32_t *dim, int32_t *origin_i, double *origin_d, float *res) {
  if (!g) return mplb_internal_fail(MPLB_ERR_ARG, "null voxel grid");
  for (int i = 0; i < 3; i++) {
    if (dim) dim[i] = g->dim[i];
    if (origin_i) origin_i[i] = g->ori[i];
    if (origin_d) origin_d[i] = g->origin_d[i];
  }
  if (res) *res = g->res;
  return MPLB_OK;
}

int mplb_voxel_grid_clear(mplb_voxel_grid *g) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!g->ncell) return MPLB_OK;
  MPLB_CUDA_TRY(cudaMemset(g->d_map.p, 0, g->ncell));
  MPLB_CUDA_TRY(cudaMemset(g->d_inf.p, 0, g->ncell));
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  return MPLB_OK;
}

int mplb_voxel_grid_add_cloud_device(mplb_voxel_grid *g, const void *d_pts, int64_t n, int fp32, void *stream) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0 || (n > 0 && !d_pts)) return mplb_internal_fail(MPLB_ERR_ARG, "bad point buffer");
  if (n == 0 || !g->ncell) return MPLB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  k_vg_add<<<blocks_for((size_t)n), 256, 0, s>>>(g->geo(), d_pts, fp32 ? 1 : 0, n, g->d_map.p);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cudaStreamSynchronize(s));
  return MPLB_OK;
}

int mplb_voxel_grid_add_cloud(mplb_voxel_grid *g, const double *pts, int64_t n) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0 || (n > 0 && !pts)) return mplb_internal_fail(MPLB_ERR_ARG, "bad point buffer");
  if (n == 0 || !g->ncell) return MPLB_OK;
  MPLB_CUDA_TRY(g->pts.reserve((size_t)n * 3));
  MPLB_CUDA_TRY(cudaMemcpy(g->pts.p, pts, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice));
  return mplb_voxel_grid_add_cloud_device(g, g->pts.p, n, 0, nullptr);
}

int64_t mplb_voxel_grid_add_cloud_inflated_device(mplb_voxel_grid *g, const void *d_pts, int64_t n, int fp32, const int32_t *ns,
                                                  int n_ns, void *d_new_obs, int64_t cap, void *stream) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0 || (n > 0 && !d_pts) || n_ns < 0 || (n_ns > 0 && !ns) || cap < 0 || (cap > 0 && !d_new_obs))
    return mplb_internal_fail(MPLB_ERR_ARG, "bad argument");
  return vg_add_inflated(g, d_pts, n, fp32 ? 1 : 0, ns, n_ns, (int *)d_new_obs, cap, (cudaStream_t)stream);
}

int64_t mplb_voxel_grid_add_cloud_inflated(mplb_voxel_grid *g, const double *pts, int64_t n, const int32_t *ns, int n_ns,
                                           int32_t *new_obs, int64_t cap) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (n < 0 || (n > 0 && !pts) || n_ns < 0 || (n_ns > 0 && !ns) || cap < 0 || (cap > 0 && !new_obs))
    return mplb_internal_fail(MPLB_ERR_ARG, "bad argument");
  if (n == 0) return 0;
  cap = std::min<int64_t>(cap, (int64_t)g->ncell); /* one call emits a cell at most once: the rows past ncell stay unused */
  MPLB_CUDA_TRY(g->pts.reserve((size_t)n * 3));
  MPLB_CUDA_TRY(cudaMemcpy(g->pts.p, pts, (size_t)n * 3 * sizeof(double), cudaMemcpyHostToDevice));
  if (cap > 0) MPLB_CUDA_TRY(g->obs.reserve((size_t)cap * 3));
  const long long count = vg_add_inflated(g, g->pts.p, n, 0, ns, n_ns, g->obs.p, cap, 0);
  if (count > 0 && cap > 0)
    MPLB_CUDA_TRY(cudaMemcpy(new_obs, g->obs.p, (size_t)std::min<long long>(count, cap) * 3 * sizeof(int), cudaMemcpyDeviceToHost));
  return count;
}

int mplb_voxel_grid_set_chunk_points(mplb_voxel_grid *g, int64_t points) {
  if (!g || points < 0) return mplb_internal_fail(MPLB_ERR_ARG, "bad argument");
  g->chunk_points = points;
  return MPLB_OK;
}

int mplb_voxel_grid_decay(mplb_voxel_grid *g) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!g->ncell) return MPLB_OK;
  k_vg_decay<<<blocks_for(g->ncell), 256>>>(g->d_map.p, g->d_inf.p, g->ncell);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  return MPLB_OK;
}

int mplb_voxel_grid_fill(mplb_voxel_grid *g, const int32_t *cells3, int n, int column) {
  return vg_edit(g, cells3, n, column ? 1 : 0, 100, false, nullptr);
}

int mplb_voxel_grid_clear_columns(mplb_voxel_grid *g, const int32_t *cells3, int n) { return vg_edit(g, cells3, n, 1, 0, false, nullptr); }

int mplb_voxel_grid_fill_device(mplb_voxel_grid *g, const void *d_cells3, int n, int column, void *stream) {
  return vg_edit(g, (const int32_t *)d_cells3, n, column ? 1 : 0, 100, true, (cudaStream_t)stream);
}

int mplb_voxel_grid_clear_columns_device(mplb_voxel_grid *g, const void *d_cells3, int n, void *stream) {
  return vg_edit(g, (const int32_t *)d_cells3, n, 1, 0, true, (cudaStream_t)stream);
}

int64_t mplb_voxel_grid_get_cloud(mplb_voxel_grid *g, double *pts, int64_t cap) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (cap < 0) return mplb_internal_fail(MPLB_ERR_ARG, "negative capacity");
  const int lo[3] = {0, 0, 0};
  return host_cloud(g, g->d_map.p, lo, g->dim, pts, cap);
}

int64_t mplb_voxel_grid_get_local_cloud(mplb_voxel_grid *g, const double *pos, const double *ori, const double *dim, double *pts,
                                        int64_t cap) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!pos || !ori || !dim || cap < 0) return mplb_internal_fail(MPLB_ERR_ARG, "bad argument");
  int lo[3], up[3];
  for (int i = 0; i < 3; i++) { /* vg:49-55: floatToInt(pos + ori) clamped >= 0, floatToInt(pos + ori + dim) clamped <= dim_ */
    const double a = pos[i] + ori[i], b = a + dim[i];
    int na, nb;
    if (!vg_float_to_cell(a, g->origin_d[i], g->res, &na)) na = INT_MIN; /* cast<int> undefined: x86's INT_MIN */
    if (!vg_float_to_cell(b, g->origin_d[i], g->res, &nb)) nb = INT_MIN;
    lo[i] = na < 0 ? 0 : na;
    up[i] = nb > g->dim[i] ? g->dim[i] : nb;
  }
  return host_cloud(g, g->d_inf.p, lo, up, pts, cap);
}

int mplb_voxel_grid_get_map(mplb_voxel_grid *g, int inflated, int8_t *out, size_t cap) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!out && g->ncell) return mplb_internal_fail(MPLB_ERR_ARG, "null output");
  if (cap < g->ncell) return mplb_internal_fail(MPLB_ERR_ARG, "output buffer smaller than the grid");
  if (!g->ncell) return MPLB_OK;
  MPLB_CUDA_TRY(g->bytes.reserve(g->ncell));
  k_vg_binarize<<<blocks_for(g->ncell), 256>>>(inflated ? g->d_inf.p : g->d_map.p, g->bytes.p, g->ncell);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cudaMemcpy(out, g->bytes.p, g->ncell, cudaMemcpyDeviceToHost));
  return MPLB_OK;
}

int mplb_voxel_grid_write_map(mplb_voxel_grid *g, int inflated, mplb_map *m) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!m) return mplb_internal_fail(MPLB_ERR_ARG, "null map");
  MplbMapView v;
  mplb_internal_map_view(m, &v);
  if (v.dim != 3 || v.device != g->device || v.res != (double)g->res)
    return mplb_internal_fail(MPLB_ERR_ARG, "map is not 3D on the grid's device with the grid's resolution");
  for (int i = 0; i < 3; i++)
    if (v.nd[i] != g->dim[i] || v.origin[i] != g->origin_d[i]) return mplb_internal_fail(MPLB_ERR_ARG, "map geometry differs from the grid's");
  k_vg_binarize<<<blocks_for(g->ncell), 256>>>(inflated ? g->d_inf.p : g->d_map.p, v.d_grid, g->ncell);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  rc = mplb_internal_map_cells_changed(m, nullptr);
  if (rc) return rc;
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  return MPLB_OK;
}

int mplb_voxel_grid_create_map(mplb_voxel_grid *g, int inflated, mplb_map **out) {
  int rc = check_grid(g);
  if (rc) return rc;
  if (!out) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  if (!g->ncell) return mplb_internal_fail(MPLB_ERR_ARG, "the grid has no cells");
  MPLB_CUDA_TRY(g->bytes.reserve(g->ncell));
  k_vg_binarize<<<blocks_for(g->ncell), 256>>>(inflated ? g->d_inf.p : g->d_map.p, g->bytes.p, g->ncell);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  return mplb_map_create_from_device(3, g->dim, g->origin_d, (double)g->res, g->bytes.p, nullptr, out);
}

int mplb_map_get_cells(const mplb_map *m, const int32_t *cells3, int n, int32_t *values) {
  if (!m || n < 0 || (n > 0 && (!cells3 || !values))) return mplb_internal_fail(MPLB_ERR_ARG, "bad argument");
  if (n == 0) return MPLB_OK;
  MplbMapView v;
  mplb_internal_map_view(const_cast<mplb_map *>(m), &v);
  if (mplb_internal_set_device(v.device)) return mplb_internal_fail(MPLB_ERR_CUDA, "cannot select the map's device");
  DevBuf<int> d;
  MPLB_CUDA_TRY(d.reserve((size_t)n * 4));
  MPLB_CUDA_TRY(cudaMemcpy(d.p, cells3, (size_t)n * 3 * sizeof(int), cudaMemcpyHostToDevice));
  k_map_get_cells<<<(n + 255) / 256, 256>>>(v.d_grid, v.dim, v.nd[0], v.nd[1], v.nd[2], d.p, n, d.p + (size_t)n * 3);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  MPLB_CUDA_TRY(cudaMemcpy(values, d.p + (size_t)n * 3, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  return MPLB_OK;
}

int64_t mplb_map_trace_cells(const mplb_map *m, const double *p1s, const double *p2s, int n_rays, const int32_t *ns, int n_ns,
                             int select, int32_t *cells3, int64_t cap, int64_t *offsets) {
  int rc = check_trace_args(m, n_rays, p1s && p2s, ns, n_ns, select, cells3 != nullptr, cap);
  if (rc) return rc;
  MplbMapView v;
  mplb_internal_map_view(const_cast<mplb_map *>(m), &v);
  if (mplb_internal_set_device(v.device)) return mplb_internal_fail(MPLB_ERR_CUDA, "cannot select the map's device");
  TraceScratch &g = trace_scratch(v.device);
  const int64_t rows = std::min<int64_t>(cap, trace_bound(v, n_rays, n_ns));
  MPLB_CUDA_TRY(g.pts.reserve((size_t)std::max(n_rays, 1) * 6));
  MPLB_CUDA_TRY(g.out.reserve((size_t)std::max<int64_t>(rows, 1) * 3));
  MPLB_CUDA_TRY(g.offs.reserve((size_t)n_rays + 1));
  if (n_rays > 0) {
    MPLB_CUDA_TRY(cudaMemcpy(g.pts.p, p1s, (size_t)n_rays * 3 * sizeof(double), cudaMemcpyHostToDevice));
    MPLB_CUDA_TRY(cudaMemcpy(g.pts.p + (size_t)n_rays * 3, p2s, (size_t)n_rays * 3 * sizeof(double), cudaMemcpyHostToDevice));
  }
  const int64_t total = trace_cells(v, g.pts.p, g.pts.p + (size_t)n_rays * 3, n_rays, ns, n_ns, select, g.out.p, rows, g.offs.p, 0);
  if (total < 0) return total;
  if (offsets) MPLB_CUDA_TRY(cudaMemcpy(offsets, g.offs.p, ((size_t)n_rays + 1) * sizeof(int64_t), cudaMemcpyDeviceToHost));
  const int64_t got = std::min<int64_t>(total, rows);
  if (got > 0) MPLB_CUDA_TRY(cudaMemcpy(cells3, g.out.p, (size_t)got * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return total;
}

int64_t mplb_map_trace_cells_device(const mplb_map *m, const void *d_p1s, const void *d_p2s, int n_rays, const int32_t *ns, int n_ns,
                                    int select, void *d_cells3, int64_t cap, void *d_offsets, void *stream) {
  int rc = check_trace_args(m, n_rays, d_p1s && d_p2s, ns, n_ns, select, d_cells3 != nullptr, cap);
  if (rc) return rc;
  MplbMapView v;
  mplb_internal_map_view(const_cast<mplb_map *>(m), &v);
  if (mplb_internal_set_device(v.device)) return mplb_internal_fail(MPLB_ERR_CUDA, "cannot select the map's device");
  trace_scratch(v.device);
  return trace_cells(v, (const double *)d_p1s, (const double *)d_p2s, n_rays, ns, n_ns, select, (int *)d_cells3, cap,
                     (long long *)d_offsets, (cudaStream_t)stream);
}

}  // extern "C"
