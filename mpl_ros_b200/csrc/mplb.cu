/*
 * mplb.cu — host runtime + C ABI of libmplb.so (see include/mplb.h).
 *
 * Host side of the drop-in boundary: map objects (MapUtil, map_util.h), planner objects
 * (PlannerBase / MapPlanner, planner_base.h, map_planner.cpp:6-18), batch orchestration over arena tiers,
 * and result getters.  All compute runs in the sm_90a kernels of mplb_search.cuh; there is no CPU path.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mplb.h"
#include "mplb_internal.h"
#include "mplb_search.cuh"

using namespace mplb;

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};

int fail(int code, const std::string &msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e__ = (expr);                                                                   \
    if (e__ != cudaSuccess)                                                                     \
      return fail(MPLB_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__));          \
  } while (0)

template <typename T>
struct DevBuf { /* grow-only device buffer */
  T *p = nullptr;
  size_t n = 0;
  cudaError_t reserve(size_t want) {
    if (want <= n) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr; n = 0;
    cudaError_t e = cudaMalloc((void **)&p, want * sizeof(T));
    if (e == cudaSuccess) n = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};

/* ------------------------------------------------------------------ map kernels */
__global__ void k_free_unknown(int8_t *g, size_t n) { /* mu:259-276 */
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    if (g[i] == -1) g[i] = 0;
}

/* mu:221-257: out = in; every neighbour offset of an occupied cell becomes occupied (writes race benignly: same value) */
__global__ void k_dilate(const int8_t *in, int8_t *out, int dim, int nx, int ny, int nz, const int *ns, int n_ns) {
  size_t total = (size_t)nx * ny * nz;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    if (in[i] != 100) continue;
    int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((size_t)nx * ny));
    for (int k = 0; k < n_ns; k++) {
      int xx = x + ns[k * dim], yy = y + ns[k * dim + 1], zz = dim == 3 ? z + ns[k * dim + 2] : 0;
      if (xx < 0 || xx >= nx || yy < 0 || yy >= ny || zz < 0 || zz >= nz) continue;
      out[(size_t)xx + (size_t)nx * yy + (size_t)nx * ny * zz] = 100;
    }
  }
}

/* Pack occupancy (value == 100, mu:48) into 64-bit bricks: 4x4x4 voxels (3D) / 8x8 cells (2D) per word. */
__global__ void k_build_bricks(const int8_t *g, unsigned long long *bricks, int dim, int nx, int ny, int nz, int bx, int by,
                               int bz) {
  size_t nb = (size_t)bx * by * bz;
  for (size_t b = blockIdx.x * (size_t)blockDim.x + threadIdx.x; b < nb; b += (size_t)gridDim.x * blockDim.x) {
    int ix = (int)(b % bx), iy = (int)((b / bx) % by), iz = (int)(b / ((size_t)bx * by));
    unsigned long long w = 0;
    if (dim == 3) {
      for (int bit = 0; bit < 64; bit++) {
        int x = ix * 4 + (bit & 3), y = iy * 4 + ((bit >> 2) & 3), z = iz * 4 + (bit >> 4);
        if (x < nx && y < ny && z < nz && g[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z] == 100) w |= 1ull << bit;
      }
    } else {
      for (int bit = 0; bit < 64; bit++) {
        int x = ix * 8 + (bit & 7), y = iy * 8 + (bit >> 3);
        if (x < nx && y < ny && g[(size_t)x + (size_t)nx * y] == 100) w |= 1ull << bit;
      }
    }
    bricks[b] = w;
  }
}


/* ---- scheduling hints (never influence results): free-space connected components and a longest-first plan order.
 * A batch finishes when its longest plan does, and plans whose goal lies in another free-space component exhaust
 * their whole reachable set, so they should start first (longest-processing-time-first list scheduling). */
__global__ void k_label_init(const int8_t *g, int *lab, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    lab[i] = (g[i] == 100) ? -1 : (int)i;
}
__global__ void k_label_step(int *lab, int nx, int ny, int nz, int *changed) {
  size_t total = (size_t)nx * ny * nz;
  bool any = false;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int l = lab[i];
    if (l < 0) continue;
    int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((size_t)nx * ny));
    int m = l;
    /* follow the current label once (pointer jumping) and look at the six neighbours */
    int r = lab[l]; if (r >= 0 && r < m) m = r;
    if (x > 0) { int v = lab[i - 1]; if (v >= 0 && v < m) m = v; }
    if (x + 1 < nx) { int v = lab[i + 1]; if (v >= 0 && v < m) m = v; }
    if (y > 0) { int v = lab[i - nx]; if (v >= 0 && v < m) m = v; }
    if (y + 1 < ny) { int v = lab[i + nx]; if (v >= 0 && v < m) m = v; }
    if (z > 0) { int v = lab[i - (size_t)nx * ny]; if (v >= 0 && v < m) m = v; }
    if (z + 1 < nz) { int v = lab[i + (size_t)nx * ny]; if (v >= 0 && v < m) m = v; }
    if (m < l) { lab[i] = m; any = true; }
  }
  if (any) *changed = 1;
}
__global__ void k_label_count(const int *lab, int *cnt, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    int l = lab[i];
    if (l >= 0) atomicAdd(&cnt[l], 1);
  }
}
__global__ void k_plan_keys(const mplb_waypoint *starts, const mplb_waypoint *goals, int n, const int *lab, const int *comp_size,
                            int dim, int nx, int ny, int nz, double ox, double oy, double oz, double res, unsigned *keys) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double o[3] = {ox, oy, oz};
  const int nd[3] = {nx, ny, nz};
  int cs[3] = {0, 0, 0}, cg[3] = {0, 0, 0};
  bool in_s = true, in_g = true;
  unsigned dist = 0;
  for (int ax = 0; ax < dim; ax++) {
    cs[ax] = (int)floor((starts[i].pos[ax] - o[ax]) / res);
    cg[ax] = (int)floor((goals[i].pos[ax] - o[ax]) / res);
    in_s = in_s && cs[ax] >= 0 && cs[ax] < nd[ax];
    in_g = in_g && cg[ax] >= 0 && cg[ax] < nd[ax];
    unsigned d = (unsigned)abs(cs[ax] - cg[ax]);
    dist = d > dist ? d : dist;
  }
  unsigned key = dist > 0xffffffu ? 0xffffffu : dist;
  if (lab && in_s && in_g) {
    int ls = lab[(size_t)cs[0] + (size_t)nx * cs[1] + (size_t)nx * ny * cs[2]];
    int lg = lab[(size_t)cg[0] + (size_t)nx * cg[1] + (size_t)nx * ny * cg[2]];
    if (ls >= 0 && ls != lg) { /* goal not in the start's free-space component: the search exhausts that component */
      unsigned sz = comp_size ? (unsigned)comp_size[ls] >> 3 : 0u;
      key = (1u << 30) | (sz > 0xffffffu ? 0xffffffu : sz);
    }
  }
  keys[i] = key;
}
__global__ void k_plan_order(const unsigned *keys, int n, int *order) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned k = keys[i];
  int rank = 0;
  for (int j = 0; j < n; j++) { unsigned kj = keys[j]; rank += (kj > k) || (kj == k && j < i); }
  order[rank] = i;
}


/* ---- potential map (map_planner.cpp:286-391).  tmp[q] collects max over sources s of mask[q - s]; the reference's
 * sequential loop is order independent because the mask values never exceed H_MAX = 100 (see DESIGN.md). */
__global__ void k_pot_stamp(const int8_t *src, int *tmp, int dim, int nx, int ny, int nz, int x1, int y1, int z1, int x2,
                            int y2, int z2, const int *moff, const int *mval, int nmask) {
  __shared__ int list[256];
  __shared__ int cnt;
  const long long bx = x2 - x1, by = y2 - y1, bz = z2 - z1;
  const long long total = bx * by * bz;
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += (long long)gridDim.x * blockDim.x) {
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    long long i = base + threadIdx.x;
    if (i < total) {
      int x = x1 + (int)(i % bx), y = y1 + (int)((i / bx) % by), z = z1 + (int)(i / (bx * by));
      size_t idx = (size_t)x + (size_t)nx * y + (size_t)nx * ny * z;
      if (src[idx] > 0) list[atomicAdd(&cnt, 1)] = (int)i;
    }
    __syncthreads();
    const long long work = (long long)cnt * nmask;
    for (long long w = threadIdx.x; w < work; w += blockDim.x) {
      const long long si = list[(int)(w / nmask)];
      const int m = (int)(w % nmask);
      int x = x1 + (int)(si % bx) + moff[m * 3], y = y1 + (int)((si / bx) % by) + moff[m * 3 + 1],
          z = z1 + (int)(si / (bx * by)) + moff[m * 3 + 2];
      if (x < 0 || x >= nx || y < 0 || y >= ny || z < 0 || z >= nz) continue;
      atomicMax(&tmp[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z], mval[m]);
    }
    __syncthreads();
  }
}
__global__ void k_pot_merge(int8_t *grid, const int *tmp, int nx, int ny, int nz, int x1, int y1, int z1, int x2, int y2,
                            int z2) {
  size_t total = (size_t)nx * ny * nz;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int x = (int)(i % nx), y = (int)((i / nx) % ny), z = (int)(i / ((size_t)nx * ny));
    int v = (int)grid[i];
    bool src = v > 0 && x >= x1 && x < x2 && y >= y1 && y < y2 && z >= z1 && z < z2;
    int t = tmp[i];
    grid[i] = (int8_t)(src ? 100 : (t > v ? t : v));
  }
}
__global__ void k_fill_int(int *a, int v, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) a[i] = v;
}

/* ---- planning_ros_msgs/Trajectory, ROS 1 wire format.  One warp per (plan, primitive): lane l writes bytes l, l+32, ...
 * of the 216-byte Primitive record (4 x {uint32 6, float64[6]} + float64 t), so stores of a warp are contiguous. */
struct MsgArgs {
  const mplb_result *results;
  const int *actions;
  const double *segs;
  int n, max_seg, dim, ord, use_yaw;
  const double *U, *Uyaw;
  double dt, z;
  unsigned seq, sec, nsec, frame_len;
  unsigned char frame[64];
  unsigned char *out;
  size_t stride;
  unsigned *len;
};
__device__ __forceinline__ unsigned char byte_of(double v, int b) { return (unsigned char)((unsigned long long)__double_as_longlong(v) >> (8 * b)); }
__device__ __forceinline__ unsigned char byte_of(unsigned v, int b) { return (unsigned char)(v >> (8 * b)); }
__global__ void k_serialize_traj(const __grid_constant__ MsgArgs a) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const long long total = (long long)a.n * (a.max_seg + 1); /* slot 0 of every plan: header, counts, length */
  for (long long w = (long long)blockIdx.x * wpb + (threadIdx.x >> 5); w < total; w += (long long)gridDim.x * wpb) {
    const int plan = (int)(w / (a.max_seg + 1)), k = (int)(w % (a.max_seg + 1)) - 1;
    const mplb_result r = a.results[plan];
    const int n_seg = (r.status == MPLB_PLAN_OK) ? r.n_seg : 0;
    const size_t head = 16 + (size_t)a.frame_len + 4; /* seq, stamp.sec, stamp.nsec, frame_id length + bytes, primitive count */
    const size_t need = head + (size_t)n_seg * 216 + 4;
    const bool fits = n_seg <= a.max_seg && need <= a.stride;
    unsigned char *o = a.out + (size_t)plan * a.stride;
    if (k < 0) {
      if (lane == 0) a.len[plan] = fits ? (unsigned)need : 0u;
      if (!fits) continue;
      for (int b = lane; b < (int)head; b += 32) {
        unsigned char v;
        if (b < 4) v = byte_of(a.seq, b);
        else if (b < 8) v = byte_of(a.sec, b - 4);
        else if (b < 12) v = byte_of(a.nsec, b - 8);
        else if (b < 16) v = byte_of(a.frame_len, b - 12);
        else if (b < 16 + (int)a.frame_len) v = a.frame[b - 16];
        else v = byte_of((unsigned)n_seg, b - 16 - (int)a.frame_len);
        o[b] = v;
      }
      if (lane < 4) o[need - 4 + lane] = 0; /* LambdaSeg[] lambda: empty */
      continue;
    }
    if (!fits || k >= n_seg) continue;
    const double *row = a.segs + ((size_t)plan * a.max_seg + k) * 13;
    const int act = a.actions[(size_t)plan * a.max_seg + k];
    unsigned char *po = o + head + (size_t)k * 216;
    for (int b = lane; b < 216; b += 32) {
      unsigned char v;
      if (b >= 208) v = byte_of(a.dt, b - 208);
      else {
        const int arr = b / 52, off = b % 52; /* arr: 0 cx, 1 cy, 2 cz, 3 cyaw */
        if (off < 4) v = byte_of(6u, off);
        else {
          const int ci = (off - 4) >> 3, bb = (off - 4) & 7; /* coefficient index 0..5, highest order first (pr:35-52) */
          double c = 0.0;
          if (arr < a.dim) {
            const int d = 5 - ci; /* derivative held by this coefficient */
            if (d < a.ord) c = row[d * 3 + arr];
            else if (d == a.ord) c = a.U[act * 3 + arr];
          } else if (arr == 2) c = (ci == 5) ? a.z : 0.0; /* 2D: cz = (0,0,0,0,0,z) */
          else if (arr == 3 && a.use_yaw) c = (ci == 5) ? row[12] : (ci == 4 ? a.Uyaw[act] : 0.0);
          v = byte_of(c, bb);
        }
      }
      po[b] = v;
    }
  }
}

/* plans that fit no arena tier get a complete MPLB_PLAN_NOMEM record: whatever the buffers held before (an earlier
 * batch's record, the counters of an aborted smaller tier, a caller's stale data) must not show through */
__global__ void k_mark_status(mplb_result *results, int *actions, int max_seg, const int *work, int n_work, int status) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_work) return;
  const int pid = work ? work[i] : i;
  mplb_result r;
  r.status = status; r.n_seg = 0; r.cost = __longlong_as_double(0x7ff0000000000000ll);
  r.pops = 0; r.n_nodes = 0; r.n_open = 0; r.n_closed = 0;
  r.n_prims = 0; r.n_samples = 0; r.n_valid = 0;
  r.pop_hash = 0ull; r.closed_hash = 0ull; r.device_ms = 0.0;
  results[pid] = r;
  if (actions)
    for (int k = 0; k < max_seg; k++) actions[(size_t)pid * max_seg + k] = -1;
}

__global__ void k_sincos_cr(const double *x, int n, double *s, double *c) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) trig::sincos_cr(x[i], &s[i], &c[i]);
}

}  // namespace

/* ================================================================== objects */
struct mplb_map {
  int dim = 3;
  int nd[3] = {1, 1, 1};
  int bd[3] = {1, 1, 1};
  double origin[3] = {0, 0, 0};
  double res = 1;
  size_t ncell = 0, nbrick = 0;
  int device = 0;
  int8_t *d_grid = nullptr;
  unsigned long long *d_bricks = nullptr;
  int *d_labels = nullptr; /* free-space component label per cell (scheduling hint), built lazily */
  int *d_comp_size = nullptr; /* number of cells carrying each label */
  unsigned long long labels_version = ~0ull;
  unsigned long long version = 0;

  int rebuild_bricks(cudaStream_t s) {
    int blocks = (int)std::min<size_t>((nbrick + 255) / 256, 148 * 16);
    k_build_bricks<<<blocks, 256, 0, s>>>(d_grid, d_bricks, dim, nd[0], nd[1], nd[2], bd[0], bd[1], bd[2]);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    version++;
    return MPLB_OK;
  }
};

namespace { struct BatchRun; }

struct mplb_planner {
  int dim = 3;
  int verbose = 0;
  int device = 0;
  mplb_map *map = nullptr;
  /* env_base defaults eb:368-392, planner defaults pb:337-339 */
  double v_max = -1, a_max = -1, j_max = -1, yaw_max = -1, dt = 1.0, w = 10.0, eps = 1.0;
  double tol_pos = 0.5, tol_vel = -1, tol_acc = -1, t_max = INFINITY;
  int max_num = -1;
  double mem_fraction = 0.6;
  int max_slots = 0; /* 0 = as many CTAs as are resident */
  int resident_sig = -1, resident_cached = 0, hcap_big_cached = 0, sm_count = 0;
  size_t budget_bytes = 0; /* arena budget, measured at the first batch (reset by MPLB_MEM_FRACTION / MPLB_ARENA_BYTES) */
  size_t arena_bytes = 0;  /* MPLB_ARENA_BYTES: upper bound on the budget, 0 = unset */
  int lpa_init_nodes = 1 << 16, lpa_init_preds = 1 << 20; /* MPLB_LPA_INIT_NODES / _PREDS: LPA* array sizes at allocation */
  std::vector<double> U; /* nU x 3 */
  std::vector<double> Uyaw; /* nU yaw rates when the rows have Dim + 1 entries (pr:217), else empty */
  int nU = 0;
  double wyaw = 1.0; /* eb:372 */
  /* cost shaping (em:104-128): defaults em:196-197 */
  double pot_w = 0.1, grad_w = 0.0;
  DevBuf<int8_t> d_pot;
  size_t pot_cells = 0; /* 0 = no potential map */
  DevBuf<unsigned> d_region;
  std::vector<uint8_t> h_region; /* empty = no search region */
  /* prior trajectory (pb:249-252): coefficient rows cx, cy, cz, cyaw (6 each, highest order first) and duration per segment */
  int prior_nseg = 0, prior_control = 0;
  std::vector<double> prior_coeffs, prior_ts;
  double prior_start_t = 0; /* t of the start waypoints of the batch being planned (the table is indexed by depth) */
  double cfg_prior_start_t = 0;
  DevBuf<double> d_prior;
  BatchRun *run = nullptr; /* the batch in flight (run_batch_begin / run_batch_end) */
  cudaStream_t own_stream = nullptr; /* stream of the asynchronous host-buffer entry points */
  std::vector<mplb_waypoint> h_ls, h_lg; /* staged stripe of the asynchronous host-buffer entry points */
  int async_n = 0, async_per = 0, async_ms = 0;
  int exact_preds = -1; /* predecessor log: -1 = where the running best predecessor is not provably exact, 0 = never, 1 = always */
  bool log_mode = false;

  /* device-side configuration, rebuilt when dirty */
  bool dirty = true;
  int cfg_control = 0;
  unsigned long long cfg_map_version = ~0ull;
  DevCfg cfg;
  DevBuf<double> d_U, d_ttab, d_Uyaw;
  DevBuf<int> d_toff, d_tcnt;
  int kfields = 0;
  int key_bits = 0; /* bits the packed key spans, word 0's padding included */

  /* scratch */
  DevBuf<unsigned char> arena;
  DevBuf<int> d_ctrl; /* [0] work counter, [1] overflow count */
  DevBuf<int> d_work, d_over, d_slot;
  DevBuf<unsigned> d_keys;
  DevBuf<mplb_waypoint> d_starts, d_goals;
  DevBuf<mplb_result> d_results;
  DevBuf<int> d_actions;
  DevBuf<double> d_segs;
  DevBuf<long long> d_phase; /* diagnostics build only */
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;

  /* last batch */
  double last_ms = 0;
  int last_launches = 0, last_tiers = 0;
  std::vector<mplb_tier_info> last_tier_rows; /* one per tier pass (mplb_last_batch_tiers) */
  /* retained single plan */
  bool retained = false;
  bool ret_arena = false; /* the retained plan's search state is in the arena (false after MPLB_PLAN_NOMEM) */
  bool ret_lpa = false; /* the retained plan came from the LPA* unit: no A* arena behind the node getters */
  mplb_result ret_result;
  int ret_cap = 0, ret_ns = 0, ret_slot = 0;
  size_t ret_stride = 0, ret_off_state = 0, ret_off_heap = 0, ret_off_poplog = 0, ret_row_bytes = 0;
  std::vector<int> ret_actions;
  std::vector<double> ret_segs;
};

namespace {

size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

struct Layout {
  size_t off_rows, off_heap, off_table, off_poplog, off_log, stride, row_bytes;
  int tsize_max, log_cap;
};

/* Large tiers (hundreds of MB per plan) trade probe length for room: load factor <= 1/2 instead of 1/4. */
int load_inv_of(int cap) { return cap > 262144 ? 2 : MPLB_LOAD_INV; }

Layout make_layout(int cap, int ns, int nU, bool want_poplog, bool log_mode) {
  Layout L;
  long long ts = MPLB_TINIT; /* 64-bit: the last tier would overflow an int (the caller stops tiering at 2^30 table slots) */
  while (ts < (long long)load_inv_of(cap) * ((long long)cap + nU) && ts < (1ll << 30)) ts <<= 1;
  L.tsize_max = (int)ts;
  size_t o = 0;
  L.row_bytes = (sizeof(RowHdr) + (size_t)ns * sizeof(double) + 15) & ~(size_t)15;
  o += align_up((size_t)cap * sizeof(NodeHot), 256);
  L.off_rows = o;
  o += align_up((size_t)cap * L.row_bytes, 256);
  L.off_heap = o;
  o += align_up((size_t)cap * sizeof(HeapEnt), 256);
  L.off_table = o;
  o += align_up((size_t)ts * sizeof(Slot), 256);
  L.off_poplog = o;
  if (want_poplog) o += align_up((size_t)cap * sizeof(int), 256);
  L.off_log = o;
  L.log_cap = 0;
  if (log_mode) { /* predecessor records: every finite-cost edge of every expansion (gs:100-102); 6 per node of capacity */
    const long long lc = std::min<long long>(6LL * cap + nU, 0x7fffffffLL);
    L.log_cap = (int)lc;
    o += align_up((size_t)lc * sizeof(PredRec), 256);
  }
  L.stride = o;
  return L;
}

int control_order(int control) { /* control.h:10-20: the yaw variants add bit 16 to the base pattern */
  switch (control & 15) {
    case MPLB_CONTROL_VEL: return 1;
    case MPLB_CONTROL_ACC: return 2;
    case MPLB_CONTROL_JRK: return 3;
    case MPLB_CONTROL_SNP: return 4;
    default: return 0;
  }
}

double margin_cells(double vmax_eff, double dt, double res) { return std::max(2.0, 2.0 * vmax_eff * dt) / res; }

int bits_for(long long range) {
  int b = 1;
  while ((1ll << b) < range) b++;
  return b;
}

/* Build the device configuration: control table, sample-time tables (em:95-99), key packing. */
int build_cfg(mplb_planner *p, int control) {
  if (!p->map) return fail(MPLB_ERR_STATE, "planner has no map (setMapUtil not called)");
  if (p->nU <= 0) return fail(MPLB_ERR_STATE, "planner has no control set (setU not called)");
  if (p->nU > MPLB_MAXU) return fail(MPLB_ERR_ARG, "more than 128 controls are not supported");
  int ord = (control & ~31) ? 0 : control_order(control);
  if (ord == 0) return fail(MPLB_ERR_ARG, "unsupported control flag on the start waypoint");
  const bool use_yaw = (control & 16) != 0;
  if (use_yaw && p->Uyaw.empty())
    return fail(MPLB_ERR_ARG, "the start waypoint uses yaw but the control rows have no yaw column (setU rows need Dim + 1 entries)");
  if (p->map->dim != p->dim) return fail(MPLB_ERR_ARG, "map dimension does not match planner dimension");
  if (!(p->dt > 0)) return fail(MPLB_ERR_ARG, "dt must be > 0");
  if (ord >= 2 && !(p->v_max > 0))
    return fail(MPLB_ERR_ARG, "v_max must be > 0 for ACC/JRK/SNP controls (the sample divisor of env_map.h:95 is unbounded otherwise)");
  if (p->tol_vel >= 0 && ord < 2) return fail(MPLB_ERR_ARG, "tol_vel >= 0 needs a control order with velocity in the state");
  if (p->tol_acc >= 0 && ord < 3) return fail(MPLB_ERR_ARG, "tol_acc >= 0 needs a control order with acceleration in the state");
  if (!p->dirty && p->cfg_control == control && p->cfg_map_version == p->map->version &&
      (p->prior_nseg == 0 || p->cfg_prior_start_t == p->prior_start_t))
    return MPLB_OK;

  mplb_map *m = p->map;
  DevCfg &c = p->cfg;
  std::memset(&c, 0, sizeof(c));
  c.dim = p->dim; c.ord = ord; c.control = control; c.nU = p->nU;
  const bool shaped = use_yaw || p->pot_cells || !p->h_region.empty();
  c.ns = p->dim * ord + (shaped ? 1 : 0); /* the cost-shaping / yaw kernels keep a yaw slot after the polynomial state */
  c.max_num = p->max_num;
  c.dt = p->dt; c.w = p->w; c.eps = p->eps; c.v_max = p->v_max; c.a_max = p->a_max; c.j_max = p->j_max;
  c.tol_pos = p->tol_pos; c.tol_vel = p->tol_vel; c.tol_acc = p->tol_acc;
  for (int i = 0; i < 3; i++) { c.nd[i] = m->nd[i]; c.bd[i] = m->bd[i]; c.origin[i] = m->origin[i]; }
  c.res = m->res;
  c.grid = m->d_grid;
  c.bricks = m->d_bricks;

  /* controls */
  CUDA_TRY(p->d_U.reserve((size_t)p->nU * 3));
  CUDA_TRY(cudaMemcpy(p->d_U.p, p->U.data(), (size_t)p->nU * 3 * sizeof(double), cudaMemcpyHostToDevice));
  c.U = p->d_U.p;
  double umax = 0;
  for (double u : p->U) umax = std::max(umax, std::fabs(u));
  double vmax_eff = ord >= 2 ? p->v_max : umax;

  /* sample-time tables: exactly the reference loop `for (t = 0; t < T; t += T/n)` for every divisor n */
  int n_hi = std::max(5, (int)std::ceil(vmax_eff * p->dt / m->res)) + 1;
  if (n_hi > 4096) return fail(MPLB_ERR_ARG, "v_max*dt/res is too large (more than 4096 samples per primitive)");
  std::vector<double> ttab;
  std::vector<int> toff(n_hi + 1, 0), tcnt(n_hi + 1, 0);
  for (int n = 5; n <= n_hi; n++) {
    toff[n] = (int)ttab.size();
    double dts = p->dt / n;
    int cnt = 0;
    for (double t = 0; t < p->dt; t += dts) { ttab.push_back(t); cnt++; }
    tcnt[n] = cnt;
  }
  CUDA_TRY(p->d_ttab.reserve(ttab.size()));
  CUDA_TRY(p->d_toff.reserve(toff.size()));
  CUDA_TRY(p->d_tcnt.reserve(tcnt.size()));
  CUDA_TRY(cudaMemcpy(p->d_ttab.p, ttab.data(), ttab.size() * sizeof(double), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(p->d_toff.p, toff.data(), toff.size() * sizeof(int), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(p->d_tcnt.p, tcnt.data(), tcnt.size() * sizeof(int), cudaMemcpyHostToDevice));
  c.ttab = p->d_ttab.p; c.toff = p->d_toff.p; c.tcnt = p->d_tcnt.p; c.n_hi = n_hi;
  c.tt_total = (int)ttab.size();
  c.inv_res = 1.0 / m->res;
  /* Guard band of the filtered sampler (filtered_w, clear_of_tie), in cells.  u = 2^-53 is the unit roundoff.
   * M = largest cell coordinate a sampled parent can have (map extent + margin, maxc + margin_cells) + the largest
   * displacement terms over one primitive (dsum: the dynamic bounds of a validated primitive, and |u| for the top
   * coefficient, times dt^d / d! / res) + 2.  P = largest absolute coordinate a sample can take, in metres:
   * max over the axes of |origin| + extent + margin.
   * - The filter's w differs from the real value y = (p(t) - origin)/res - 0.5 by less than 8u * M: y0, the
   *   coefficients and the Horner steps each round once or twice relative to numbers bounded by M.  Documented (and
   *   tested) as < 2^-45 * M.
   * - The reference's own value y_ref = fl(fl(fl(p) - origin)/res) - 0.5 (mu:103-108) differs from y by its rounding of
   *   p (pr:128-131): the last add p = s + p0 happens at the magnitude of the absolute coordinate, <= u * P metres or
   *   u * P / res cells, plus roundings relative to the cell coordinate and displacement, < 8u * M.
   * (|p| <= P holds for every sample that can land inside the map: one farther out is outside whichever neighbouring
   * cell it rounds to.)
   * So |w - y_ref| < 2^-49 * M + 2^-53 * P / res, and the band 2^-40 * M + 2^-50 * P / res holds it with 8x headroom
   * on the term that grows with the origin (UTM-style map frames: origins of 5e5 .. 1e7 m).  That term stays small
   * enough for use_fast at such origins (about 2e-7 cells at 1e7 m and res = 0.05). */
  {
    double bnd[5] = {0, p->v_max, p->a_max, p->j_max, 0};
    bnd[ord] = umax; /* the control itself is the top coefficient */
    bool known = true;
    double dsum = 0, tp = 1, fact = 1;
    for (int d = 1; d <= ord; d++) {
      tp *= p->dt; fact *= d;
      if (!(bnd[d] > 0) && d < ord) known = false;
      dsum += std::fabs(bnd[d]) * tp / fact / m->res;
    }
    double maxc = 0, maxp = 0;
    const double margin_m = std::max(2.0, 2.0 * vmax_eff * p->dt);
    for (int i = 0; i < p->dim; i++) {
      maxc = std::max(maxc, (double)m->nd[i]);
      maxp = std::max(maxp, std::fabs(m->origin[i]) + m->nd[i] * m->res + margin_m);
    }
    double delta = std::ldexp(maxc + margin_cells(vmax_eff, p->dt, m->res) + dsum + 2.0, -40) + std::ldexp(maxp / m->res, -50);
    c.use_fast = (known && n_hi < MPLB_NCAP && c.tt_total <= MPLB_TT_CAP && delta <= 1e-6) ? 1 : 0;
    c.fast_delta = delta;
  }
  /* cost shaping (em:104-128) */
  c.pot = nullptr; c.region = nullptr; c.pot_w = p->pot_w; c.grad_w = p->grad_w;
  c.use_yaw = use_yaw ? 1 : 0; c.nkey = p->dim * ord + (use_yaw ? 1 : 0);
  c.yaw_max = p->yaw_max; c.wyaw = p->wyaw; c.cos_yaw_max = 1.0; c.Uyaw = nullptr;
  if (use_yaw) {
    CUDA_TRY(p->d_Uyaw.reserve((size_t)p->nU));
    CUDA_TRY(cudaMemcpy(p->d_Uyaw.p, p->Uyaw.data(), (size_t)p->nU * sizeof(double), cudaMemcpyHostToDevice));
    c.Uyaw = p->d_Uyaw.p;
    if (p->yaw_max > 0) {
      if (!(p->yaw_max < 1e5)) return fail(MPLB_ERR_ARG, "yaw_max is out of range");
      double sn;
      trig::sincos_cr(p->yaw_max, &sn, &c.cos_yaw_max); /* cos(my) of pr:521, correctly rounded like the device side */
    }
  }
  if (shaped) {
    if (p->pot_cells && p->pot_cells != m->ncell) return fail(MPLB_ERR_STATE, "potential map size does not match the planner's map");
    if (!p->h_region.empty() && p->h_region.size() != m->ncell) return fail(MPLB_ERR_STATE, "search region size does not match the planner's map");
    if (p->nU > 32) return fail(MPLB_ERR_ARG, "search region / potential map / yaw controls need a control set of at most 32 rows");
    if (!c.use_fast) return fail(MPLB_ERR_ARG, "search region / potential map / yaw controls need positive dynamic bounds for every derivative of the control order");
    if (p->pot_cells) c.pot = p->d_pot.p;
    if (!p->h_region.empty()) c.region = p->d_region.p;
  }
  /* prior trajectory (eb:46-53, em:187-225 without a potential map) */
  c.prior = nullptr; c.prior_n = 0; c.prior_on = 0;
  if (p->prior_nseg > 0) {
    if (p->pot_cells) return fail(MPLB_ERR_ARG, "a prior trajectory together with a potential map is not supported (em:199-214 is unpinned)");
    const int D = p->dim, n = p->prior_nseg;
    std::vector<double> taus(1, 0.0);
    for (int i = 0; i < n; i++) taus.push_back(p->prior_ts[i] + taus.back()); /* trajectory.h:52-57 */
    const double total = taus.back();
    auto evaluate = [&](double time, mplb_waypoint *out) { /* trajectory.h:66-86 */
      double tau = time;
      if (tau < 0) tau = 0;
      if (tau > total) tau = total;
      std::memset(out, 0, sizeof(*out));
      for (int id = 0; id < n; id++) {
        if ((tau >= taus[id] && tau < taus[id + 1]) || id == n - 1) {
          tau -= taus[id];
          const double *cs = &p->prior_coeffs[(size_t)id * 24];
          mplb_ref::Prim1 q[4]; /* the segment's Primitive1D per axis, then yaw */
          std::memcpy(q, cs, sizeof(q));
          for (int j = 0; j < D; j++) {
            out->pos[j] = mplb_ref::pr_p(q[j], tau);
            out->vel[j] = mplb_ref::pr_v(q[j], tau);
            out->acc[j] = mplb_ref::pr_a(q[j], tau);
            out->jrk[j] = mplb_ref::pr_j(q[j], tau);
          }
          out->yaw = mplb_ref::normalize_angle(mplb_ref::pr_p(q[3], tau));
          out->control = p->prior_control;
          return;
        }
      }
    };
    /* em:196-223: costs[k] = w t (no potential map), total_cost = traverse_trajectory (0: a collision-free prior is assumed,
     * as in MPL/test/test_planner_2d_with_prior_traj.cpp) + w total; prior_traj_[k] = (evaluate(t), total_cost - costs[int(t/dt)]) */
    std::vector<double> costs;
    for (double t = 0; t < total; t += p->dt) costs.push_back(p->w * t);
    const double total_cost = 0.0 + p->w * total;
    std::vector<mplb_waypoint> pw;
    std::vector<double> pc;
    for (double t = 0; t < total; t += p->dt) {
      const int id = (int)(t / p->dt);
      mplb_waypoint wq;
      evaluate(t, &wq);
      pw.push_back(wq);
      pc.push_back(total_cost - costs[std::min<size_t>((size_t)std::max(id, 0), costs.size() - 1)]);
    }
    evaluate(total, &c.prior_goal); /* em:224 */
    /* rows by depth: a depth-d state carries t = start.t + dt + ... + dt (em:161), eb:48-51 indexes with size_t(t / dt) */
    std::vector<double> rows;
    double t = p->prior_start_t;
    for (int d = 0; d < (1 << 20); d++) {
      const double q = t / p->dt;
      if (!(q >= 0) || q >= (double)pw.size()) break;
      const size_t id = (size_t)q;
      if (id >= pw.size()) break;
      for (int k = 0; k < 3; k++) rows.push_back(pw[id].pos[k]);
      rows.push_back(pc[id]);
      t += p->dt;
    }
    c.prior_on = 1;
    c.prior_n = (int)(rows.size() / 4);
    if (c.prior_n > 0) {
      CUDA_TRY(p->d_prior.reserve(rows.size()));
      CUDA_TRY(cudaMemcpy(p->d_prior.p, rows.data(), rows.size() * sizeof(double), cudaMemcpyHostToDevice));
      c.prior = p->d_prior.p;
    }
    p->cfg_prior_start_t = p->prior_start_t;
  }
  /* predecessor log (see PredRec): needed wherever a node's g can still drop after it was used to relax a successor */
  p->log_mode = p->exact_preds > 0 || (p->exact_preds < 0 && (p->eps > 1.0 || p->prior_nseg > 0 || (ord == 1 && !(p->v_max >= umax))));
  {
    int e = 0;
    double mant = std::frexp(p->v_max, &e);
    c.vmax_rcp_exact = (p->v_max > 0 && mant == 0.5 && e > -500 && e < 500) ? 1.0 / p->v_max : 0.0;
  }
  /* key packing: field f = axis*ord + d; pos fields cover the map plus a margin (end states are not collision
   * tested at t = T, em:99), derivative fields cover their dynamic bound (validated primitives, pr:449-496). */
  double margin = std::max(2.0, 2.0 * vmax_eff * p->dt);
  double bounds[4] = {0, p->v_max, p->a_max, p->j_max};
  int bitpos = 0;
  for (int ax = 0; ax < p->dim; ax++) {
    for (int d = 0; d < ord; d++) {
      int f = ax * ord + d;
      long long lo, hi;
      if (d == 0) {
        /* the reference's (int)std::round(pos / 0.01) (wp:97-99) is only defined while the quotient fits an int */
        const double qlo = std::floor((m->origin[ax] - margin) / 0.01) - 2, qhi = std::ceil((m->origin[ax] + m->nd[ax] * m->res + margin) / 0.01) + 2;
        if (!(qlo >= -2147483648.0 && qhi <= 2147483647.0))
          return fail(MPLB_ERR_ARG, "map too far from the origin: lattice position keys round(pos / 0.01) leave the int32 range (|pos| must stay below about 2.1e7)");
        lo = (long long)qlo;
        hi = (long long)qhi;
      } else {
        double B = bounds[d] > 0 ? bounds[d] : 100.0;
        hi = (long long)std::ceil(B / 0.1) + 2;
        lo = -hi;
      }
      int bits = bits_for(hi - lo + 1);
      if (bits > 31) return fail(MPLB_ERR_ARG, "lattice key field too wide");
      int word = bitpos / 64;
      if ((bitpos % 64) + bits > 64) { word++; bitpos = word * 64; }
      if (word > 1) return fail(MPLB_ERR_ARG, "lattice key does not fit 128 bits for this map / bounds");
      c.koff[f] = (int)lo; c.kbits[f] = (unsigned char)bits; c.kshift[f] = (unsigned char)(bitpos % 64);
      c.kword[f] = (unsigned char)word;
      bitpos += bits;
    }
  }
  if (shaped) { /* yaw field (wp:114-117): normalised yaw / 0.1 lies in [-32, 32]; a raw start yaw gets some slack */
    const int f = p->dim * ord;
    const int bits = use_yaw ? 9 : 1;
    int word = bitpos / 64;
    if ((bitpos % 64) + bits > 64) { word++; bitpos = word * 64; }
    if (word > 1) return fail(MPLB_ERR_ARG, "lattice key does not fit 128 bits for this map / bounds");
    c.koff[f] = use_yaw ? -256 : 0; c.kbits[f] = (unsigned char)bits; c.kshift[f] = (unsigned char)(bitpos % 64);
    c.kword[f] = (unsigned char)word;
    bitpos += bits;
  }
  c.key_wide = (bitpos > 96) ? 1 : 0;
  p->key_bits = bitpos;
  p->kfields = c.nkey;
  p->cfg_control = control;
  p->cfg_map_version = m->version;
  p->dirty = false;
  return MPLB_OK;
}

/* shared memory of one CTA: the plan record, plus (|U| > 32 instantiations) `hcap` heap entries of 20 bytes behind it */
template <int DIM, int ORD, int MAXU, bool POT>
size_t smem_bytes(int hcap) {
  using SM = PlanSmem<DIM, ORD, MAXU, POT>;
  return SM::DYN_HEAP ? heap_dyn_offset<SM>() + (size_t)hcap * 20 : sizeof(SM);
}

template <int DIM, int ORD, int MAXU, bool POT>
int launch_batch(const DevCfg &c, const BatchArgs &a, int grid, cudaStream_t s) {
  size_t smem = smem_bytes<DIM, ORD, MAXU, POT>(a.hcap);
  auto kern = astar_batch_kernel<DIM, ORD, MAXU, POT>;
  if (smem > 48 * 1024) CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared); /* residency is shared-memory bound */
  /* the occupancy bricks are the only data with reuse across pops and plans: keep them resident in L2 */
  cudaLaunchConfig_t cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(MPLB_NT); cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  size_t brick_bytes = (size_t)c.bd[0] * c.bd[1] * c.bd[2] * sizeof(unsigned long long);
  static thread_local int persist_max = -1, window_max = 0;
  if (persist_max < 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&persist_max, cudaDevAttrMaxPersistingL2CacheSize, dev);
    cudaDeviceGetAttribute(&window_max, cudaDevAttrMaxAccessPolicyWindowSize, dev);
    if (persist_max > 0) cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, (size_t)persist_max / 2);
    cudaGetLastError();
  }
  if (persist_max > 0 && window_max > 0) {
    attr[0].id = cudaLaunchAttributeAccessPolicyWindow;
    attr[0].val.accessPolicyWindow.base_ptr = const_cast<unsigned long long *>(c.bricks);
    attr[0].val.accessPolicyWindow.num_bytes = std::min(brick_bytes, (size_t)window_max);
    attr[0].val.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)(persist_max / 2) / (double)std::max<size_t>(brick_bytes, 1));
    attr[0].val.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr[0].val.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    nattr = 1;
  }
  cfg.attrs = attr; cfg.numAttrs = nattr;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kern, c, a);
  g_launches++;
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("cudaLaunchKernelEx: ") + cudaGetErrorString(e));
  CUDA_TRY(cudaGetLastError());
  return MPLB_OK;
}

template <int DIM, int ORD, int MAXU, bool POT>
int resident_ctas(int device, int hcap) {
  int per_sm = 0, sms = 0;
  size_t smem = smem_bytes<DIM, ORD, MAXU, POT>(hcap);
  auto kern = astar_batch_kernel<DIM, ORD, MAXU, POT>;
  if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, MPLB_NT, smem) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
  return per_sm * sms;
}

/* the cost-shaping kernels exist for |U| <= 32 only (build_cfg rejects larger control sets with shaping) */
template <int DIM, int ORD, int MAXU>
int launch_any(bool shaped, const DevCfg &c, const BatchArgs &a, int grid, cudaStream_t s) {
  if constexpr (MAXU == 1) { if (shaped) return launch_batch<DIM, ORD, MAXU, true>(c, a, grid, s); }
  return launch_batch<DIM, ORD, MAXU, false>(c, a, grid, s);
}
template <int DIM, int ORD, int MAXU>
int resident_any(bool shaped, int device, int hcap) {
  if constexpr (MAXU == 1) { if (shaped) return resident_ctas<DIM, ORD, MAXU, true>(device, hcap); }
  return resident_ctas<DIM, ORD, MAXU, false>(device, hcap);
}
/* largest shared-memory heap of a |U| > 32 launch that runs one plan per SM */
template <int DIM, int ORD, int MAXU>
int hcap_big(int device) {
  int optin = 0;
  if (cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device) != cudaSuccess) return MPLB_HCAP_SMALL;
  const long long room = (long long)optin - (long long)heap_dyn_offset<PlanSmem<DIM, ORD, MAXU, false>>() - 1024;
  long long h = room / 20 / 256 * 256;
  return (int)std::max<long long>(MPLB_HCAP_SMALL, std::min<long long>(h, 8192));
}

#define DISPATCH_U(D, O, nu, CALL) do { if ((nu) <= 32) { CALL(D, O, 1); } else { CALL(D, O, 4); } } while (0)
#ifdef MPLB_BENCH_ONLY /* tuning builds (tools/ab_bench.py): only the two bench instantiations, seconds to compile */
#define DISPATCH(dim, ord, nu, CALL)                                                          \
  do {                                                                                        \
    if (dim == 3 && ord == 2 && (nu) <= 32) { CALL(3, 2, 1); } else if (dim == 3 && ord == 3 && (nu) > 32) { CALL(3, 3, 4); } \
    else return fail(MPLB_ERR_ARG, "tuning build: only the bench configurations are compiled in");                         \
  } while (0)
#else
#define DISPATCH(dim, ord, nu, CALL)                                                          \
  do {                                                                                        \
    if (dim == 2 && ord == 1) DISPATCH_U(2, 1, nu, CALL); else if (dim == 2 && ord == 2) DISPATCH_U(2, 2, nu, CALL); \
    else if (dim == 2 && ord == 3) DISPATCH_U(2, 3, nu, CALL); else if (dim == 2 && ord == 4) DISPATCH_U(2, 4, nu, CALL); \
    else if (dim == 3 && ord == 1) DISPATCH_U(3, 1, nu, CALL); else if (dim == 3 && ord == 2) DISPATCH_U(3, 2, nu, CALL); \
    else if (dim == 3 && ord == 3) DISPATCH_U(3, 3, nu, CALL); else DISPATCH_U(3, 4, nu, CALL); \
  } while (0)
#endif

/* Core: device-resident batch over arena tiers. */
/* One batch over arena tiers, in two halves so that a caller can keep one batch in flight per planner:
 * run_batch_begin enqueues everything up to and including the first tier's search launch and returns without waiting;
 * run_batch_end waits for it, re-runs overflowed plans in larger tiers (synchronously) and closes the timing.  Two planners
 * on two streams overlap the drain of one batch (a launch ends with its longest plan) with the start of the next. */
struct BatchRun {
  bool active = false;
  const mplb_waypoint *d_starts = nullptr, *d_goals = nullptr;
  mplb_result *d_results = nullptr;
  int *d_actions = nullptr;
  double *d_segs = nullptr;
  int n = 0, max_seg = 0;
  bool retain = false, shaped = false, identity = true, finished = false;
  cudaStream_t s = nullptr;
  int n_work = 0, cap = 0, resident = 0, slots = 0, n_this_tier = 0;
  long long cap_bound = 0;
  size_t budget = 0;
  Layout L;
};

/* the body of one tier up to its launch; sets R.finished when nothing is left to launch (NOMEM marking) */
int batch_launch_tier(mplb_planner *p, BatchRun &R) {
  const DevCfg &c = p->cfg;
  cudaStream_t s = R.s;
  int rc = MPLB_OK;
  R.L = make_layout(R.cap, c.ns, c.nU, R.retain, p->log_mode);
  const Layout &L = R.L;
  int slots = std::min(R.n_work, R.resident);
  if (p->max_slots > 0) slots = std::min(slots, p->max_slots);
  if ((size_t)slots * L.stride > R.budget) slots = (int)(R.budget / L.stride);
  mplb_tier_info row;
  std::memset(&row, 0, sizeof(row));
  row.cap = R.cap; row.slots = slots; row.n_work = R.n_work; row.load_inv = load_inv_of(R.cap); row.tsize_max = L.tsize_max;
  row.log_cap = L.log_cap; row.stride_bytes = (int64_t)L.stride; row.ordered = R.identity ? 0 : 1; row.resident = R.resident;
  if (slots <= 0 || (long long)load_inv_of(R.cap) * ((long long)R.cap + c.nU) > (1ll << 30)) {
    /* nothing larger fits (or the table would pass 2^30 slots): the remaining plans report NOMEM.  In the first tier
     * the work list may be the identity (no id array was written), later tiers carry the overflow list. */
    k_mark_status<<<(R.n_work + 255) / 256, 256, 0, s>>>(R.d_results, R.d_actions, R.max_seg, R.identity ? nullptr : p->d_work.p,
                                                         R.n_work, MPLB_PLAN_NOMEM);
    g_launches++;
    CUDA_TRY(cudaGetLastError());
    row.nomem = 1;
    p->last_tier_rows.push_back(row);
    R.finished = true;
    return MPLB_OK;
  }
  if (p->arena.n < (size_t)slots * L.stride) {
    CUDA_TRY(cudaStreamSynchronize(s));
    if (p->arena.reserve((size_t)slots * L.stride) != cudaSuccess) {
      cudaGetLastError();
      return fail(MPLB_ERR_NOMEM, "cannot allocate the search arena");
    }
  }
  CUDA_TRY(cudaMemsetAsync(p->d_ctrl.p, 0, 2 * sizeof(int), s));
  BatchArgs a;
  std::memset(&a, 0, sizeof(a));
  a.starts = R.d_starts; a.goals = R.d_goals; a.results = R.d_results; a.actions = R.d_actions; a.seg_states = R.d_segs;
  a.max_seg = R.max_seg; a.work = R.identity ? nullptr : p->d_work.p; a.n_work = R.n_work;
  a.work_counter = p->d_ctrl.p; a.arena = p->arena.p; a.stride = L.stride; a.cap = R.cap; a.tsize_max = L.tsize_max; a.load_inv = load_inv_of(R.cap);
  a.off_rows = L.off_rows; a.off_heap = L.off_heap; a.off_table = L.off_table; a.off_poplog = L.off_poplog;
  a.off_log = L.off_log; a.log_cap = L.log_cap;
  /* |U| > 32: when memory leaves at most one plan per SM anyway, that plan gets a much larger shared-memory heap top */
  a.hcap = (c.nU > 32 && slots <= p->sm_count && p->hcap_big_cached > 0) ? p->hcap_big_cached : MPLB_HCAP_SMALL;
  a.want_poplog = R.retain ? 1 : 0; a.slot_of_plan = R.retain ? p->d_slot.p : nullptr;
  a.overflow_count = p->d_ctrl.p + 1; a.overflow_list = p->d_over.p;
#ifdef MPLB_PHASE_TIMING
  CUDA_TRY(p->d_phase.reserve((size_t)R.n * 16));
  a.phase_cycles = p->d_phase.p;
#endif
  const bool shaped = R.shaped;
#define LAUNCH_CALL(D, O, M) rc = launch_any<D, O, M>(shaped, c, a, slots, s)
  DISPATCH(c.dim, c.ord, c.nU, LAUNCH_CALL);
  if (rc != MPLB_OK) return rc;
  p->last_launches++; p->last_tiers++;
  row.hcap = c.nU > 32 ? a.hcap : MPLB_HCAP; /* the |U| <= 32 instantiations keep a fixed top in their static shared memory */
  p->last_tier_rows.push_back(row);
  R.slots = slots;
  R.n_this_tier = R.n_work;
  return MPLB_OK;
}

int run_batch_begin(mplb_planner *p, const mplb_waypoint *d_starts, const mplb_waypoint *d_goals, int n, mplb_result *d_results,
                    int *d_actions, double *d_segs, int max_seg, int control, bool retain, cudaStream_t s) {
  BatchRun &R = *p->run;
  if (R.active) return fail(MPLB_ERR_STATE, "a batch is already in flight on this planner (mplb_*_end not called)");
  int rc = build_cfg(p, control);
  if (rc != MPLB_OK) return rc;
  const DevCfg &c = p->cfg;
  p->retained = false;
  if (!p->ev0) { CUDA_TRY(cudaEventCreate(&p->ev0)); CUDA_TRY(cudaEventCreate(&p->ev1)); }
  CUDA_TRY(p->d_ctrl.reserve(2));
  CUDA_TRY(p->d_over.reserve((size_t)n));
  CUDA_TRY(p->d_work.reserve((size_t)n));
  if (retain) CUDA_TRY(p->d_slot.reserve((size_t)n));

  /* resident CTAs of this kernel instantiation and the memory budget are looked up once per configuration: both
   * calls cost on the order of a millisecond, comparable to a small batch */
  const bool shaped = c.pot != nullptr || c.region != nullptr || c.use_yaw != 0;
  const int cfg_sig = (shaped ? 1000 : 0) + c.dim * 100 + c.ord * 10 + (c.nU <= 32 ? 1 : 4);
  if (p->resident_sig != cfg_sig) {
    int r = 0;
#define RES_CALL(D, O, M) do { r = resident_any<D, O, M>(shaped, p->device, MPLB_HCAP_SMALL); if (M > 1) p->hcap_big_cached = hcap_big<D, O, M>(p->device); } while (0)
    DISPATCH(c.dim, c.ord, c.nU, RES_CALL);
    p->resident_cached = r;
    p->resident_sig = cfg_sig;
  }
  const int resident = p->resident_cached;
  if (p->sm_count == 0) cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, p->device);
  if (resident <= 0) return fail(MPLB_ERR_CUDA, "no resident CTA for the search kernel (is this an sm_90 device?)");

  if (p->budget_bytes == 0) {
    size_t free_b = 0, total_b = 0;
    CUDA_TRY(cudaMemGetInfo(&free_b, &total_b));
    p->budget_bytes = (size_t)((double)(free_b + p->arena.n) * p->mem_fraction);
    if (p->arena_bytes > 0) p->budget_bytes = std::min(p->budget_bytes, p->arena_bytes);
  }

  R = BatchRun();
  R.d_starts = d_starts; R.d_goals = d_goals; R.d_results = d_results; R.d_actions = d_actions; R.d_segs = d_segs;
  R.n = n; R.max_seg = max_seg; R.retain = retain; R.shaped = shaped; R.s = s; R.resident = resident; R.budget = p->budget_bytes;
  R.n_work = n;
  R.identity = true;
  int cap = 32768;
  /* MaxExpandStep bounds the node count by max_num * |U| (every pop creates at most |U| nodes): no tier needs more */
  R.cap_bound = c.max_num > 0 ? std::min<long long>((long long)c.max_num * c.nU + 2LL * c.nU + 64, 1ll << 30) : (1ll << 30);
  if (c.max_num > 0) { /* start in the tier that is likely to fit */
    while (cap < R.cap_bound && cap < 262144) cap *= 8;
  }
  R.cap = (int)std::min<long long>(cap, std::max<long long>(R.cap_bound, 1024));
  p->last_launches = 0; p->last_tiers = 0;
  p->last_tier_rows.clear();
  p->ret_arena = false;
  bool ev0_done = false;
  if (n > resident / 2 && n <= 65536) { /* longest-first order (scheduling only): see k_plan_keys */
    mplb_map *m = p->map;
    if (m->ncell <= (1ull << 26) && m->labels_version != m->version) {
      if (!m->d_labels && cudaMalloc((void **)&m->d_labels, m->ncell * sizeof(int)) != cudaSuccess) { cudaGetLastError(); m->d_labels = nullptr; }
      if (m->d_labels) {
        int blocks = (int)std::min<size_t>((m->ncell + 255) / 256, 148 * 32);
        k_label_init<<<blocks, 256, 0, s>>>(m->d_grid, m->d_labels, m->ncell);
        g_launches++;
        int *d_changed = p->d_ctrl.p; /* reuse: reset before every check */
        for (int it = 0; it < 4096; it += 8) {
          CUDA_TRY(cudaMemsetAsync(d_changed, 0, sizeof(int), s));
          for (int k = 0; k < 8; k++) { k_label_step<<<blocks, 256, 0, s>>>(m->d_labels, m->nd[0], m->nd[1], m->nd[2], d_changed); g_launches++; }
          int changed = 0;
          CUDA_TRY(cudaMemcpyAsync(&changed, d_changed, sizeof(int), cudaMemcpyDeviceToHost, s));
          CUDA_TRY(cudaStreamSynchronize(s));
          if (!changed) break;
        }
        if (!m->d_comp_size && cudaMalloc((void **)&m->d_comp_size, m->ncell * sizeof(int)) != cudaSuccess) { cudaGetLastError(); m->d_comp_size = nullptr; }
        if (m->d_comp_size) {
          CUDA_TRY(cudaMemsetAsync(m->d_comp_size, 0, m->ncell * sizeof(int), s));
          k_label_count<<<blocks, 256, 0, s>>>(m->d_labels, m->d_comp_size, m->ncell);
          g_launches++;
        }
        CUDA_TRY(cudaStreamSynchronize(s)); /* another planner's stream may read the labels next */
        m->labels_version = m->version;
      }
    }
    CUDA_TRY(p->d_keys.reserve((size_t)n));
    CUDA_TRY(cudaEventRecord(p->ev0, s)); /* the per-batch ordering kernels are inside the timed region */
    ev0_done = true;
    int nb = (n + 127) / 128;
    const bool have_labels = (m->labels_version == m->version) && m->d_labels;
    k_plan_keys<<<nb, 128, 0, s>>>(d_starts, d_goals, n, have_labels ? m->d_labels : nullptr, have_labels ? m->d_comp_size : nullptr,
                                 m->dim, m->nd[0], m->nd[1], m->nd[2], m->origin[0], m->origin[1], m->origin[2], m->res, p->d_keys.p);
    k_plan_order<<<nb, 128, 0, s>>>(p->d_keys.p, n, p->d_work.p);
    g_launches += 2;
    p->last_launches += 2;
    CUDA_TRY(cudaGetLastError());
    R.identity = false;
  }
  if (!ev0_done) CUDA_TRY(cudaEventRecord(p->ev0, s));
  rc = batch_launch_tier(p, R);
  if (rc != MPLB_OK) return rc;
  R.active = true;
  return MPLB_OK;
}

int run_batch_end(mplb_planner *p) {
  BatchRun &R = *p->run;
  if (!R.active) return fail(MPLB_ERR_STATE, "no batch in flight on this planner");
  R.active = false;
  const DevCfg &c = p->cfg;
  cudaStream_t s = R.s;
  while (!R.finished) {
    int n_over = 0;
    CUDA_TRY(cudaMemcpyAsync(&n_over, p->d_ctrl.p + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    p->last_tier_rows.back().n_overflow = n_over;
    if (R.retain && R.n == 1 && n_over == 0) {
      p->ret_cap = R.cap; p->ret_ns = c.ns; p->ret_stride = R.L.stride; p->ret_off_state = R.L.off_rows; p->ret_row_bytes = R.L.row_bytes;
      p->ret_off_heap = R.L.off_heap; p->ret_off_poplog = R.L.off_poplog;
      p->ret_arena = true;
    }
    if (n_over == 0) break;
    /* next tier: overflowed plans restart from scratch (the search is deterministic) with 8x the arena */
    std::swap(p->d_work, p->d_over);
    R.n_work = n_over;
    R.identity = false;
    if (R.cap >= R.cap_bound || R.cap > (1 << 27)) R.cap = 1 << 30; /* beyond every budget: the next pass reports NOMEM */
    /* with a MaxExpandStep bound and most plans of this tier overflowing (a search that does not terminate early, like the
     * jerk lattice of BASELINE configs[4]) the remaining tiers would only repeat work: go straight to the bound */
    else if (c.max_num > 0 && 2 * n_over > R.n_this_tier) R.cap = (int)R.cap_bound;
    else R.cap = (int)std::min<long long>((long long)R.cap * 8, R.cap_bound);
    int rc = batch_launch_tier(p, R);
    if (rc != MPLB_OK) return rc;
  }
  CUDA_TRY(cudaEventRecord(p->ev1, s));
  CUDA_TRY(cudaEventSynchronize(p->ev1));
  float ms = 0;
  CUDA_TRY(cudaEventElapsedTime(&ms, p->ev0, p->ev1));
  p->last_ms = ms;
  return MPLB_OK;
}

int run_batch(mplb_planner *p, const mplb_waypoint *d_starts, const mplb_waypoint *d_goals, int n, mplb_result *d_results,
              int *d_actions, double *d_segs, int max_seg, int control, bool retain, cudaStream_t s) {
  int rc = run_batch_begin(p, d_starts, d_goals, n, d_results, d_actions, d_segs, max_seg, control, retain, s);
  if (rc != MPLB_OK) return rc;
  return run_batch_end(p);
}

int set_device_of(int device) {
  int cur = -1;
  if (cudaGetDevice(&cur) != cudaSuccess) return -1;
  if (cur != device && cudaSetDevice(device) != cudaSuccess) return -1;
  return 0;
}

int map_alloc(int dim, const int32_t *ndim, const double *origin, double res, mplb_map **out) {
  if (!out || !ndim || !origin) return fail(MPLB_ERR_ARG, "null argument");
  if (dim != 2 && dim != 3) return fail(MPLB_ERR_ARG, "dim must be 2 or 3");
  if (!(res > 0)) return fail(MPLB_ERR_ARG, "resolution must be > 0");
  mplb_map *m = new mplb_map();
  m->dim = dim;
  m->res = res;
  size_t n = 1;
  for (int i = 0; i < dim; i++) {
    if (ndim[i] <= 0) { delete m; return fail(MPLB_ERR_ARG, "map dimensions must be positive"); }
    m->nd[i] = ndim[i];
    m->origin[i] = origin[i];
    n *= (size_t)ndim[i];
  }
  if (n > 0x7fffffffull) { delete m; return fail(MPLB_ERR_ARG, "more than 2^31-1 cells (the reference indexes cells with int, map_util.h:33-41)"); }
  m->ncell = n;
  if (dim == 3) { m->bd[0] = (m->nd[0] + 3) / 4; m->bd[1] = (m->nd[1] + 3) / 4; m->bd[2] = (m->nd[2] + 3) / 4; }
  else { m->bd[0] = (m->nd[0] + 7) / 8; m->bd[1] = (m->nd[1] + 7) / 8; m->bd[2] = 1; }
  m->nbrick = (size_t)m->bd[0] * m->bd[1] * m->bd[2];
  if (cudaGetDevice(&m->device) != cudaSuccess) { delete m; return fail(MPLB_ERR_CUDA, "no CUDA device (libmplb has no CPU path)"); }
  if (cudaMalloc((void **)&m->d_grid, n) != cudaSuccess || cudaMalloc((void **)&m->d_bricks, m->nbrick * 8) != cudaSuccess) {
    std::string e = cudaGetErrorString(cudaGetLastError());
    if (m->d_grid) cudaFree(m->d_grid);
    delete m;
    return fail(MPLB_ERR_CUDA, "cudaMalloc(map): " + e);
  }
  *out = m;
  return MPLB_OK;
}

}  // namespace

int mplb_internal_fail(int code, const char *msg) { return fail(code, msg ? msg : ""); }
void mplb_internal_count_launches(int n) { g_launches += n; }
int mplb_internal_planner_cfg(mplb_planner *p, MplbLpaHostCfg *o) {
  std::memset(o, 0, sizeof(*o));
  o->dim = p->dim; o->nU = p->nU; o->max_num = p->max_num; o->device = p->device; o->verbose = p->verbose;
  o->v_max = p->v_max; o->a_max = p->a_max; o->j_max = p->j_max; o->dt = p->dt; o->w = p->w; o->eps = p->eps;
  o->tol_pos = p->tol_pos; o->tol_vel = p->tol_vel; o->tol_acc = p->tol_acc;
  o->lpa_init_nodes = p->lpa_init_nodes; o->lpa_init_preds = p->lpa_init_preds;
  o->U = p->U.data();
  o->Uyaw = p->Uyaw.empty() ? nullptr : p->Uyaw.data();
  o->shaped = (p->pot_cells != 0 || !p->h_region.empty() || p->prior_nseg != 0 || !p->Uyaw.empty()) ? 1 : 0;
  o->has_map = p->map != nullptr;
  if (p->map) {
    for (int i = 0; i < 3; i++) { o->nd[i] = p->map->nd[i]; o->origin[i] = p->map->origin[i]; }
    o->res = p->map->res;
    o->d_grid = p->map->d_grid;
  }
  return MPLB_OK;
}
void mplb_internal_map_view(mplb_map *m, MplbMapView *o) {
  o->dim = m->dim; o->device = m->device; o->res = m->res; o->ncell = m->ncell; o->d_grid = m->d_grid;
  for (int i = 0; i < 3; i++) { o->nd[i] = m->nd[i]; o->origin[i] = m->origin[i]; }
}
int mplb_internal_map_cells_changed(mplb_map *m, void *stream) { return m->rebuild_bricks((cudaStream_t)stream); }
void mplb_internal_set_retained(mplb_planner *p, const mplb_result *res, const int *actions, const double *segs13, int n_seg) {
  p->ret_result = *res;
  p->ret_actions.assign(actions, actions + n_seg);
  p->ret_segs.assign(segs13, segs13 + (size_t)n_seg * 13);
  p->retained = true;
  p->ret_lpa = true;
}

/* one thread per edited cell (MapUtil::setMap with an edited copy of getMap(), map_replanner_node.cpp:181-196) */
__global__ void k_set_cells(int8_t *g, const int *cells3, int n, int dim, int nx, int ny, int nz, int8_t value) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = cells3[i * 3], y = cells3[i * 3 + 1], z = dim == 3 ? cells3[i * 3 + 2] : 0;
  if (x < 0 || x >= nx || y < 0 || y >= ny || z < 0 || z >= nz) return;
  g[(size_t)x + (size_t)nx * y + (size_t)nx * ny * z] = value;
}

/* ================================================================== C ABI */
extern "C" {

const char *mplb_last_error(void) { return g_err.c_str(); }

int mplb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int64_t mplb_launch_count(void) { return (int64_t)g_launches.load(); }

int mplb_map_create(int dim, const int32_t *ndim, const double *origin, double res, const int8_t *data, mplb_map **out) {
  if (!data) return fail(MPLB_ERR_ARG, "null map data");
  mplb_map *m = nullptr;
  int rc = map_alloc(dim, ndim, origin, res, &m);
  if (rc != MPLB_OK) return rc;
  if (cudaMemcpy(m->d_grid, data, m->ncell, cudaMemcpyHostToDevice) != cudaSuccess) {
    std::string e = cudaGetErrorString(cudaGetLastError());
    mplb_map_destroy(m);
    return fail(MPLB_ERR_CUDA, "cudaMemcpy(map): " + e);
  }
  rc = m->rebuild_bricks(0);
  if (rc != MPLB_OK) { mplb_map_destroy(m); return rc; }
  CUDA_TRY(cudaStreamSynchronize(0));
  *out = m;
  return MPLB_OK;
}

int mplb_map_create_from_device(int dim, const int32_t *ndim, const double *origin, double res, const void *dev_data,
                                void *stream, mplb_map **out) {
  if (!dev_data) return fail(MPLB_ERR_ARG, "null device map data");
  mplb_map *m = nullptr;
  int rc = map_alloc(dim, ndim, origin, res, &m);
  if (rc != MPLB_OK) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  if (cudaMemcpyAsync(m->d_grid, dev_data, m->ncell, cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
    std::string e = cudaGetErrorString(cudaGetLastError());
    mplb_map_destroy(m);
    return fail(MPLB_ERR_CUDA, "cudaMemcpyAsync(map d2d): " + e);
  }
  rc = m->rebuild_bricks(s);
  if (rc != MPLB_OK) { mplb_map_destroy(m); return rc; }
  CUDA_TRY(cudaStreamSynchronize(s));
  *out = m;
  return MPLB_OK;
}

int mplb_map_free_unknown(mplb_map *m) {
  if (!m) return fail(MPLB_ERR_ARG, "null map");
  if (set_device_of(m->device)) return fail(MPLB_ERR_CUDA, "cannot select the map's device");
  int blocks = (int)std::min<size_t>((m->ncell + 255) / 256, 148 * 16);
  k_free_unknown<<<blocks, 256>>>(m->d_grid, m->ncell);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  int rc = m->rebuild_bricks(0);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(0));
  return MPLB_OK;
}

int mplb_map_set_data(mplb_map *m, const int8_t *data) {
  if (!m || !data) return fail(MPLB_ERR_ARG, "null argument");
  if (set_device_of(m->device)) return fail(MPLB_ERR_CUDA, "cannot select the map's device");
  CUDA_TRY(cudaMemcpy(m->d_grid, data, m->ncell, cudaMemcpyHostToDevice));
  int rc = m->rebuild_bricks(0);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(0));
  return MPLB_OK;
}

int mplb_map_set_cells(mplb_map *m, const int32_t *cells3, int n, int value) {
  if (!m || (n > 0 && !cells3)) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if (set_device_of(m->device)) return fail(MPLB_ERR_CUDA, "cannot select the map's device");
  int *d = nullptr;
  CUDA_TRY(cudaMalloc((void **)&d, (size_t)n * 3 * sizeof(int)));
  cudaError_t e = cudaMemcpy(d, cells3, (size_t)n * 3 * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    k_set_cells<<<(n + 255) / 256, 256>>>(m->d_grid, d, n, m->dim, m->nd[0], m->nd[1], m->nd[2], (int8_t)value);
    g_launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaFree(d);
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("map_set_cells: ") + cudaGetErrorString(e));
  int rc = m->rebuild_bricks(0);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(0));
  return MPLB_OK;
}

int mplb_map_dilate(mplb_map *m, const int32_t *ns, int n) {
  if (!m || (n > 0 && !ns)) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if (set_device_of(m->device)) return fail(MPLB_ERR_CUDA, "cannot select the map's device");
  int8_t *tmp = nullptr;
  int *d_ns = nullptr;
  CUDA_TRY(cudaMalloc((void **)&tmp, m->ncell));
  CUDA_TRY(cudaMalloc((void **)&d_ns, (size_t)n * m->dim * sizeof(int)));
  CUDA_TRY(cudaMemcpy(d_ns, ns, (size_t)n * m->dim * sizeof(int), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(tmp, m->d_grid, m->ncell, cudaMemcpyDeviceToDevice));
  int blocks = (int)std::min<size_t>((m->ncell + 255) / 256, 148 * 16);
  k_dilate<<<blocks, 256>>>(tmp, m->d_grid, m->dim, m->nd[0], m->nd[1], m->nd[2], d_ns, n);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  int rc = m->rebuild_bricks(0);
  CUDA_TRY(cudaStreamSynchronize(0));
  cudaFree(tmp);
  cudaFree(d_ns);
  return rc;
}

int mplb_map_get_info(const mplb_map *m, int32_t *dim, int32_t *ndim, double *origin, double *res) {
  if (!m) return fail(MPLB_ERR_ARG, "null map");
  if (dim) *dim = m->dim;
  for (int i = 0; i < m->dim; i++) { if (ndim) ndim[i] = m->nd[i]; if (origin) origin[i] = m->origin[i]; }
  if (res) *res = m->res;
  return MPLB_OK;
}

int mplb_map_get_data(const mplb_map *m, int8_t *out, size_t cap) {
  if (!m || !out) return fail(MPLB_ERR_ARG, "null argument");
  if (cap < m->ncell) return fail(MPLB_ERR_ARG, "output buffer smaller than the map");
  if (set_device_of(m->device)) return fail(MPLB_ERR_CUDA, "cannot select the map's device");
  CUDA_TRY(cudaMemcpy(out, m->d_grid, m->ncell, cudaMemcpyDeviceToHost));
  return MPLB_OK;
}

void mplb_map_destroy(mplb_map *m) {
  if (!m) return;
  if (m->d_grid) cudaFree(m->d_grid);
  if (m->d_bricks) cudaFree(m->d_bricks);
  if (m->d_labels) cudaFree(m->d_labels);
  if (m->d_comp_size) cudaFree(m->d_comp_size);
  delete m;
}

int mplb_planner_create(int dim, int verbose, mplb_planner **out) {
  if (!out) return fail(MPLB_ERR_ARG, "null argument");
  if (dim != 2 && dim != 3) return fail(MPLB_ERR_ARG, "dim must be 2 or 3");
  mplb_planner *p = new mplb_planner();
  p->dim = dim;
  p->verbose = verbose;
  if (cudaGetDevice(&p->device) != cudaSuccess) { delete p; return fail(MPLB_ERR_CUDA, "no CUDA device (libmplb has no CPU path)"); }
  p->run = new BatchRun();
  if (verbose) std::printf("[MapPlanner] PLANNER VERBOSE ON\n");
  *out = p;
  return MPLB_OK;
}

void mplb_planner_destroy(mplb_planner *p) {
  if (!p) return;
  mplb_internal_lpa_drop(p);
  p->d_U.release(); p->d_ttab.release(); p->d_toff.release(); p->d_tcnt.release(); p->arena.release();
  p->d_ctrl.release(); p->d_work.release(); p->d_over.release(); p->d_slot.release(); p->d_starts.release();
  p->d_goals.release(); p->d_results.release(); p->d_actions.release(); p->d_segs.release();
  p->d_keys.release(); p->d_phase.release(); p->d_pot.release(); p->d_region.release(); p->d_Uyaw.release(); p->d_prior.release();
  if (p->ev0) cudaEventDestroy(p->ev0);
  if (p->ev1) cudaEventDestroy(p->ev1);
  if (p->own_stream) cudaStreamDestroy(p->own_stream);
  delete p->run;
  delete p;
}

int mplb_planner_set_map(mplb_planner *p, mplb_map *m) {
  if (!p || !m) return fail(MPLB_ERR_ARG, "null argument");
  if (m->dim != p->dim) return fail(MPLB_ERR_ARG, "map dimension does not match planner dimension");
  if (m->device != p->device) return fail(MPLB_ERR_ARG, "map and planner live on different devices");
  p->map = m;
  p->dirty = true;
  p->retained = false;
  return MPLB_OK;
}

int mplb_planner_set_param(mplb_planner *p, int key, double v) {
  if (!p) return fail(MPLB_ERR_ARG, "null planner");
  switch (key) {
    case MPLB_V_MAX: p->v_max = v; break;
    case MPLB_A_MAX: p->a_max = v; break;
    case MPLB_J_MAX: p->j_max = v; break;
    case MPLB_YAW_MAX: p->yaw_max = v; break;
    case MPLB_DT: p->dt = v; break;
    case MPLB_W: p->w = v; break;
    case MPLB_EPSILON: p->eps = v; break;
    case MPLB_MAX_NUM: p->max_num = (int)v; break;
    case MPLB_TOL_POS: p->tol_pos = v; break;
    case MPLB_TOL_VEL: p->tol_vel = v; break;
    case MPLB_TOL_ACC: p->tol_acc = v; break;
    case MPLB_T_MAX: p->t_max = v; break;
    case MPLB_POTENTIAL_WEIGHT: p->pot_w = v; break;
    case MPLB_GRADIENT_WEIGHT: p->grad_w = v; break;
    case MPLB_WYAW: p->wyaw = v; break;
    case MPLB_MEM_FRACTION:
      if (!(v > 0 && v <= 0.95)) return fail(MPLB_ERR_ARG, "mem fraction must be in (0, 0.95]");
      p->mem_fraction = v;
      p->budget_bytes = 0;
      break;
    case MPLB_ARENA_BYTES:
      if (!(v >= 0 && v < 9.0e18)) return fail(MPLB_ERR_ARG, "arena bytes must be >= 0 (0 = unset)");
      p->arena_bytes = (size_t)v;
      p->budget_bytes = 0;
      break;
    case MPLB_LPA_INIT_NODES:
    case MPLB_LPA_INIT_PREDS:
      if (!(v >= MPLB_LPA_MIN_CAP && v <= MPLB_LPA_MAX_INIT && v == std::floor(v)))
        return fail(MPLB_ERR_ARG, "LPA* initial sizes must be whole numbers in [MPLB_LPA_MIN_CAP, MPLB_LPA_MAX_INIT]");
      (key == MPLB_LPA_INIT_NODES ? p->lpa_init_nodes : p->lpa_init_preds) = (int)v;
      break;
    case MPLB_MAX_SLOTS: p->max_slots = (int)v; break;
    case MPLB_EXACT_PREDS: p->exact_preds = (int)v; break;
    default: return fail(MPLB_ERR_ARG, "unknown parameter key");
  }
  p->dirty = true;
  if (p->verbose) std::printf("[PlannerBase] set param %d: %f\n", key, v);
  return MPLB_OK;
}

int mplb_planner_set_controls(mplb_planner *p, const double *U, int n, int udim) {
  if (!p || !U) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0 || n > MPLB_MAXU) return fail(MPLB_ERR_ARG, "control set must have 1..128 rows");
  if (udim != p->dim && udim != p->dim + 1) return fail(MPLB_ERR_ARG, "control rows must have Dim entries, or Dim + 1 with a yaw rate (pr:217)");
  p->U.assign((size_t)n * 3, 0.0);
  p->Uyaw.clear();
  if (udim == p->dim + 1) p->Uyaw.assign((size_t)n, 0.0);
  for (int i = 0; i < n; i++) {
    for (int k = 0; k < p->dim; k++) p->U[(size_t)i * 3 + k] = U[(size_t)i * udim + k];
    if (udim == p->dim + 1) p->Uyaw[i] = U[(size_t)i * udim + p->dim];
  }
  p->nU = n;
  p->dirty = true;
  return MPLB_OK;
}


/* ---- cost shaping: search region (eb:301-303, map_planner.cpp:46-95) and potential map (em:182, map_planner.cpp:286-391) */
namespace {
int upload_region(mplb_planner *p) {
  const size_t n = p->h_region.size();
  std::vector<unsigned> bits((n + 31) / 32, 0u);
  for (size_t i = 0; i < n; i++)
    if (p->h_region[i]) bits[i >> 5] |= 1u << (i & 31);
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  CUDA_TRY(p->d_region.reserve(bits.size()));
  CUDA_TRY(cudaMemcpy(p->d_region.p, bits.data(), bits.size() * sizeof(unsigned), cudaMemcpyHostToDevice));
  p->dirty = true;
  return MPLB_OK;
}
}  // namespace

int mplb_planner_set_search_region(mplb_planner *p, const uint8_t *in_region, size_t n) {
  if (!p) return fail(MPLB_ERR_ARG, "null planner");
  if (!in_region || n == 0) { p->h_region.clear(); p->dirty = true; return MPLB_OK; }
  if (!p->map) return fail(MPLB_ERR_STATE, "planner has no map (setMapUtil not called)");
  if (n != p->map->ncell) return fail(MPLB_ERR_ARG, "search region must have one entry per map cell");
  p->h_region.assign(in_region, in_region + n);
  return upload_region(p);
}

int mplb_planner_set_search_region_path(mplb_planner *p, const double *path, int npts, int dense, const double *radius) {
  if (!p || !radius || (npts > 0 && !path)) return fail(MPLB_ERR_ARG, "null argument");
  if (!p->map) return fail(MPLB_ERR_STATE, "planner has no map (setMapUtil not called)");
  const mplb_map *m = p->map;
  const int D = m->dim;
  /* cells along the path: rayTrace (mu:117-134) between consecutive points plus each end point */
  std::vector<int> cells; /* 3 ints per cell */
  auto push = [&](const int *pn) { cells.push_back(pn[0]); cells.push_back(pn[1]); cells.push_back(pn[2]); };
  if (!dense) {
    for (int i = 1; i < npts; i++) {
      const double *a = path + (size_t)(i - 1) * 3, *b = path + (size_t)i * 3;
      double diff[3] = {0, 0, 0}, s;
      const int max_diff = mplb_ref::ray_setup(D, m->res, a, b, diff, &s);
      int prev[3] = {-1, -1, -1};
      for (int n = 1; n < max_diff; n++) {
        double pt[3] = {0, 0, 0};
        int pn[3];
        for (int k = 0; k < D; k++) pt[k] = mplb_ref::ray_point(a[k], diff[k], s, n);
        mplb_ref::float_to_int(*m, pt, pn);
        if (mplb_ref::outside(*m, pn)) break;
        bool same = true;
        for (int k = 0; k < D; k++) same = same && pn[k] == prev[k];
        if (!same) push(pn);
        for (int k = 0; k < D; k++) prev[k] = pn[k];
      }
      int pe[3];
      mplb_ref::float_to_int(*m, b, pe);
      push(pe);
    }
  } else {
    for (int i = 0; i < npts; i++) { int pn[3]; mplb_ref::float_to_int(*m, path + (size_t)i * 3, pn); push(pn); }
  }
  int rn[3] = {0, 0, 0};
  for (int k = 0; k < D; k++) rn[k] = (int)std::ceil(radius[k] / m->res);
  p->h_region.assign(m->ncell, 0);
  for (size_t ci = 0; ci + 2 < cells.size(); ci += 3) {
    const int lo[3] = {std::max(cells[ci] - rn[0], 0), std::max(cells[ci + 1] - rn[1], 0), D == 3 ? std::max(cells[ci + 2] - rn[2], 0) : 0};
    const int hi[3] = {std::min(cells[ci] + rn[0], m->nd[0] - 1), std::min(cells[ci + 1] + rn[1], m->nd[1] - 1),
                       D == 3 ? std::min(cells[ci + 2] + rn[2], m->nd[2] - 1) : 0};
    for (int z = lo[2]; z <= hi[2]; z++)
      for (int y = lo[1]; y <= hi[1]; y++) {
        if (lo[0] > hi[0]) continue;
        uint8_t *row = p->h_region.data() + (size_t)m->nd[0] * y + (size_t)m->nd[0] * m->nd[1] * z;
        std::memset(row + lo[0], 1, (size_t)(hi[0] - lo[0] + 1));
      }
  }
  int rc = upload_region(p);
  if (rc == MPLB_OK && p->verbose) std::printf("[MapPlanner] set search region\n");
  return rc;
}

int64_t mplb_planner_get_search_region(mplb_planner *p, uint8_t *out, size_t cap) {
  if (!p) { fail(MPLB_ERR_ARG, "null planner"); return 0; }
  const size_t n = p->h_region.size();
  if (out && n) std::memcpy(out, p->h_region.data(), std::min(cap, n));
  return (int64_t)n;
}

int mplb_planner_set_potential_map(mplb_planner *p, const int8_t *pot, size_t n) {
  if (!p) return fail(MPLB_ERR_ARG, "null planner");
  if (!pot || n == 0) { p->pot_cells = 0; p->dirty = true; return MPLB_OK; }
  if (!p->map) return fail(MPLB_ERR_STATE, "planner has no map (setMapUtil not called)");
  if (n != p->map->ncell) return fail(MPLB_ERR_ARG, "potential map must have one entry per map cell");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  CUDA_TRY(p->d_pot.reserve(n));
  CUDA_TRY(cudaMemcpy(p->d_pot.p, pot, n, cudaMemcpyHostToDevice));
  p->pot_cells = n;
  p->dirty = true;
  return MPLB_OK;
}

int mplb_planner_update_potential_map(mplb_planner *p, const double *pos, const double *radius, const double *range,
                                      double pow_) {
  if (!p || !pos || !radius || !range) return fail(MPLB_ERR_ARG, "null argument");
  if (!p->map) return fail(MPLB_ERR_STATE, "planner has no map (setMapUtil not called)");
  mplb_map *m = p->map;
  if (m->device != p->device) return fail(MPLB_ERR_STATE, "map and planner live on different devices");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  const int D = m->dim;
  /* createMask (map_planner.cpp:286-325), evaluated on the host with the reference's libm calls */
  std::vector<int> moff, mval;
  const double h_max = 100.0;
  const int rn = (int)std::ceil(radius[0] / m->res);
  const int hn = D == 3 ? (int)std::ceil(radius[2] / m->res) : 0;
  for (int nx = -rn; nx <= rn; nx++)
    for (int ny = -rn; ny <= rn; ny++)
      for (int nz = -hn; nz <= hn; nz++) {
        const double r = std::hypot((double)nx, (double)ny);
        if (r > rn) continue;
        const double base = D == 2 ? (1 - r / rn) : (1 - r / rn) * (1 - (double)std::abs(nz) / hn);
        const double h = h_max * std::pow(base, pow_);
        if (h > 1e-3) { moff.push_back(nx); moff.push_back(ny); moff.push_back(nz); mval.push_back((int)(int8_t)h); }
      }
  /* the stamped box (map_planner.cpp:330-347): whole map, or the clamped cells of pos -+ range with an open upper end */
  int c1[3] = {0, 0, 0}, c2[3] = {m->nd[0], m->nd[1], D == 3 ? m->nd[2] : 1};
  double rnorm = 0;
  for (int k = 0; k < D; k++) rnorm += range[k] * range[k];
  if (std::sqrt(rnorm) > 0) {
    double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
    for (int k = 0; k < D; k++) { lo[k] = pos[k] - range[k]; hi[k] = pos[k] + range[k]; }
    mplb_ref::float_to_int(*m, lo, c1);
    mplb_ref::float_to_int(*m, hi, c2);
    for (int k = 0; k < D; k++) {
      c1[k] = std::min(std::max(c1[k], 0), m->nd[k] - 1);
      c2[k] = std::min(std::max(c2[k], 0), m->nd[k] - 1);
    }
    if (D == 2) { c1[2] = 0; c2[2] = 1; }
  }
  int *d_tmp = nullptr, *d_moff = nullptr, *d_mval = nullptr;
  const int nmask = (int)mval.size();
  CUDA_TRY(cudaMalloc((void **)&d_tmp, m->ncell * sizeof(int)));
  const int fill_blocks = (int)std::min<size_t>((m->ncell + 255) / 256, 148 * 16);
  k_fill_int<<<fill_blocks, 256>>>(d_tmp, -1000, m->ncell);
  g_launches++;
  cudaError_t e = cudaGetLastError();
  const long long box = (long long)std::max(c2[0] - c1[0], 0) * std::max(c2[1] - c1[1], 0) * std::max(c2[2] - c1[2], 0);
  if (e == cudaSuccess && nmask > 0 && box > 0) {
    e = cudaMalloc((void **)&d_moff, moff.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_mval, mval.size() * sizeof(int));
    if (e == cudaSuccess) e = cudaMemcpy(d_moff, moff.data(), moff.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_mval, mval.data(), mval.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      const int blocks = (int)std::min<long long>((box + 255) / 256, 148 * 16);
      k_pot_stamp<<<blocks, 256>>>(m->d_grid, d_tmp, D, m->nd[0], m->nd[1], m->nd[2], c1[0], c1[1], c1[2], c2[0], c2[1], c2[2],
                                   d_moff, d_mval, nmask);
      g_launches++;
      e = cudaGetLastError();
    }
  }
  if (e == cudaSuccess) {
    k_pot_merge<<<fill_blocks, 256>>>(m->d_grid, d_tmp, m->nd[0], m->nd[1], m->nd[2], c1[0], c1[1], c1[2], c2[0], c2[1], c2[2]);
    g_launches++;
    e = cudaGetLastError();
  }
  int rc = MPLB_OK;
  if (e == cudaSuccess) rc = m->rebuild_bricks(0); /* the map itself now holds dmap (map_planner.cpp:387) */
  if (e == cudaSuccess && rc == MPLB_OK) e = p->d_pot.reserve(m->ncell);
  if (e == cudaSuccess && rc == MPLB_OK) e = cudaMemcpy(p->d_pot.p, m->d_grid, m->ncell, cudaMemcpyDeviceToDevice); /* map_planner.cpp:388 */
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaFree(d_tmp);
  if (d_moff) cudaFree(d_moff);
  if (d_mval) cudaFree(d_mval);
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("update_potential_map: ") + cudaGetErrorString(e));
  if (rc != MPLB_OK) return rc;
  p->pot_cells = m->ncell;
  p->dirty = true;
  return MPLB_OK;
}

int mplb_planner_set_prior_trajectory(mplb_planner *p, int n_seg, const double *coeffs, const double *seg_t, int control) {
  if (!p) return fail(MPLB_ERR_ARG, "null planner");
  if (n_seg <= 0) { p->prior_nseg = 0; p->prior_coeffs.clear(); p->prior_ts.clear(); p->dirty = true; return MPLB_OK; }
  if (!coeffs || !seg_t) return fail(MPLB_ERR_ARG, "null argument");
  p->prior_nseg = n_seg;
  p->prior_control = control;
  p->prior_coeffs.assign(coeffs, coeffs + (size_t)n_seg * 24);
  p->prior_ts.assign(seg_t, seg_t + n_seg);
  p->dirty = true;
  if (p->verbose) std::printf("[PlannerBase] set prior trajectory\n");
  return MPLB_OK;
}

int mplb_plan_batch_device(mplb_planner *p, const void *d_starts, const void *d_goals, int n, void *d_results,
                           void *d_actions, void *d_seg_states, int max_seg, void *stream) {
  if (!p || !d_starts || !d_goals || !d_results) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if ((d_actions || d_seg_states) && max_seg <= 0) return fail(MPLB_ERR_ARG, "max_seg must be > 0 when trajectories are requested");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  cudaStream_t s = (cudaStream_t)stream;
  mplb_waypoint w0; /* the control mode is a property of the start waypoint (waypoint.h:46-55); its t seeds the prior-trajectory table */
  CUDA_TRY(cudaMemcpyAsync(&w0, d_starts, sizeof(w0), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  const int control = w0.control;
  p->prior_start_t = w0.t;
  return run_batch(p, (const mplb_waypoint *)d_starts, (const mplb_waypoint *)d_goals, n, (mplb_result *)d_results,
                   (int *)d_actions, (double *)d_seg_states, max_seg, control, false, s);
}

static int plan_batch_host(mplb_planner *p, const mplb_waypoint *starts, const mplb_waypoint *goals, int n,
                           mplb_result *results, int32_t *actions, double *seg_states, int max_seg, bool retain) {
  if (!p || !starts || !goals || !results) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if ((actions || seg_states) && max_seg <= 0) return fail(MPLB_ERR_ARG, "max_seg must be > 0 when trajectories are requested");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  for (int i = 0; i < n; i++) {
    if (starts[i].control != starts[0].control) return fail(MPLB_ERR_ARG, "all starts of a batch must share one control mode");
    if (starts[i].enable_t) return fail(MPLB_ERR_ARG, "enable_t waypoints are not supported");
    if (p->prior_nseg > 0 && starts[i].t != starts[0].t) return fail(MPLB_ERR_ARG, "with a prior trajectory all starts of a batch must share one t");
  }
  p->prior_start_t = starts[0].t;
  cudaStream_t s = 0;
  CUDA_TRY(p->d_starts.reserve(n));
  CUDA_TRY(p->d_goals.reserve(n));
  CUDA_TRY(p->d_results.reserve(n));
  if (actions) CUDA_TRY(p->d_actions.reserve((size_t)n * max_seg));
  if (seg_states) CUDA_TRY(p->d_segs.reserve((size_t)n * max_seg * 13));
  CUDA_TRY(cudaMemcpyAsync(p->d_starts.p, starts, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(p->d_goals.p, goals, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyHostToDevice, s));
  int rc = run_batch(p, p->d_starts.p, p->d_goals.p, n, p->d_results.p, actions ? p->d_actions.p : nullptr,
                     seg_states ? p->d_segs.p : nullptr, max_seg, starts[0].control, retain, s);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaMemcpyAsync(results, p->d_results.p, (size_t)n * sizeof(mplb_result), cudaMemcpyDeviceToHost, s));
  if (actions) CUDA_TRY(cudaMemcpyAsync(actions, p->d_actions.p, (size_t)n * max_seg * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (seg_states)
    CUDA_TRY(cudaMemcpyAsync(seg_states, p->d_segs.p, (size_t)n * max_seg * 13 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (int i = 0; i < n; i++)
    if (results[i].status == MPLB_INTERNAL_BADCTRL) return fail(MPLB_ERR_ARG, "a start waypoint has a different control mode");
  return MPLB_OK;
}

int mplb_plan_batch(mplb_planner *p, const mplb_waypoint *starts, const mplb_waypoint *goals, int n, mplb_result *results,
                    int32_t *actions, double *seg_states, int max_seg) {
  return plan_batch_host(p, starts, goals, n, results, actions, seg_states, max_seg, false);
}

int mplb_plan(mplb_planner *p, const mplb_waypoint *start, const mplb_waypoint *goal, mplb_result *out) {
  if (!p || !start || !goal || !out) return fail(MPLB_ERR_ARG, "null argument");
  if (mplb_internal_lpa_enabled(p)) return mplb_internal_lpa_plan(p, start, goal, out); /* PlannerBase::plan with use_lpastar_, pb:308-311 */
  int max_seg = 4096;
  p->ret_actions.assign(max_seg, -1);
  p->ret_segs.assign((size_t)max_seg * 13, 0.0);
  int rc = plan_batch_host(p, start, goal, 1, out, p->ret_actions.data(), p->ret_segs.data(), max_seg, true);
  if (rc != MPLB_OK) return rc;
  if (out->status == MPLB_PLAN_OK && out->n_seg > max_seg) { /* longer than the retained rows: plan again with room (deterministic) */
    max_seg = out->n_seg;
    p->ret_actions.assign(max_seg, -1);
    p->ret_segs.assign((size_t)max_seg * 13, 0.0);
    rc = plan_batch_host(p, start, goal, 1, out, p->ret_actions.data(), p->ret_segs.data(), max_seg, true);
    if (rc != MPLB_OK) return rc;
  }
  p->ret_result = *out;
  p->ret_slot = 0;
  CUDA_TRY(cudaMemcpy(&p->ret_slot, p->d_slot.p, sizeof(int), cudaMemcpyDeviceToHost));
  p->retained = true;
  p->ret_lpa = false;
  if (p->verbose) {
    if (out->status == MPLB_PLAN_START_NOT_FREE) std::printf("[PlannerBase] start is not free!\n");
    else if (out->status == MPLB_PLAN_MAX_EXPAND) std::printf("MaxExpandStep [%d] Reached!!!!!!\n\n", p->max_num);
    else if (out->status == MPLB_PLAN_QUEUE_EMPTY) std::printf("Priority queue is empty!!!!!!\n\n");
    else if (out->status == MPLB_PLAN_OK) std::printf("Reached Goal !!!!!!\n\nExpand [%d] nodes!\n", out->pops);
    if (out->status != MPLB_PLAN_OK && out->status != MPLB_PLAN_START_IS_GOAL) std::printf("[PlannerBase] Cannot find a traj!\n");
  }
  return MPLB_OK;
}

int mplb_get_actions(mplb_planner *p, int32_t *actions, int cap) {
  if (!p || !p->retained) return fail(MPLB_ERR_STATE, "no retained plan");
  int n = p->ret_result.n_seg;
  for (int i = 0; i < n && i < cap && i < (int)p->ret_actions.size() && actions; i++) actions[i] = p->ret_actions[i];
  return n;
}

int mplb_get_seg_states(mplb_planner *p, double *states13, int cap) {
  if (!p || !p->retained) return fail(MPLB_ERR_STATE, "no retained plan");
  int n = p->ret_result.n_seg;
  for (int i = 0; i < n && i < cap && (size_t)(i + 1) * 13 <= p->ret_segs.size() && states13; i++) std::memcpy(states13 + (size_t)i * 13, &p->ret_segs[(size_t)i * 13], 13 * sizeof(double));
  return n;
}

/* the node getters read the retained plan's arena slot: there is none after MPLB_PLAN_NOMEM (no tier ran it to the end) */
static int check_retained_arena(mplb_planner *p) {
  if (!p || !p->retained) return fail(MPLB_ERR_STATE, "no retained plan");
  if (p->ret_lpa) return fail(MPLB_ERR_STATE, "the retained plan is an LPA* plan: use mplb_lpa_get_nodes / mplb_lpa_get_heap");
  if (!p->ret_arena) return fail(MPLB_ERR_STATE, "the retained plan has no search state (MPLB_PLAN_NOMEM: no arena tier fit it)");
  return MPLB_OK;
}

int mplb_get_nodes(mplb_planner *p, mplb_node *nodes, int cap) {
  if (int rc = check_retained_arena(p)) return rc;
  int n = p->ret_result.n_nodes;
  if (!nodes || cap <= 0) return n;
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int m = std::min(n, cap);
  std::vector<NodeHot> hot(m);
  std::vector<unsigned char> rw((size_t)m * p->ret_row_bytes);
  unsigned char *base = p->arena.p + (size_t)p->ret_slot * p->ret_stride;
  CUDA_TRY(cudaMemcpy(hot.data(), base, (size_t)m * sizeof(NodeHot), cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(rw.data(), base + p->ret_off_state, (size_t)m * p->ret_row_bytes, cudaMemcpyDeviceToHost));
  const DevCfg &c = p->cfg;
  for (int i = 0; i < m; i++) {
    mplb_node &o = nodes[i];
    std::memset(&o, 0, sizeof(o));
    const RowHdr *rh = reinterpret_cast<const RowHdr *>(rw.data() + (size_t)i * p->ret_row_bytes);
    const double *st = reinterpret_cast<const double *>(rw.data() + (size_t)i * p->ret_row_bytes + sizeof(RowHdr));
    for (int d = 0; d < c.ord; d++)
      for (int ax = 0; ax < c.dim; ax++) o.state[d * 3 + ax] = st[d * c.dim + ax];
    if (c.use_yaw) o.state[12] = st[c.dim * c.ord];
    o.g = hot[i].g; o.h = hot[i].h;
    if (rh->k0 == MPLB_KEY_OUT_OF_RANGE && rh->k1 == MPLB_KEY_OUT_OF_RANGE) { /* the start, outside the packable range */
      for (int f = 0; f < c.nkey; f++) {
        const int d = f < c.dim * c.ord ? f % c.ord : 1, ax = f / c.ord; /* field axis * ord + d; the yaw field last */
        o.key[f] = mplb_ref::round_int(mplb_ref::ddiv(f < c.dim * c.ord ? st[d * c.dim + ax] : st[f], d == 0 ? 0.01 : 0.1));
      }
    } else {
      for (int f = 0; f < c.nkey; f++) {
        unsigned long long wv = c.kword[f] ? rh->k1 : rh->k0;
        unsigned long long v = (wv >> c.kshift[f]) & ((1ull << c.kbits[f]) - 1ull);
        o.key[f] = (int)((long long)v + c.koff[f]);
      }
    }
    o.key[15] = c.nkey;
    o.opened = (hot[i].flags & 1) ? 1 : 0;
    o.closed = (hot[i].flags & 2) ? 1 : 0;
    o.parent = rh->parent;
    o.action = hot[i].action;
  }
  return n;
}

int mplb_get_pop_log(mplb_planner *p, int32_t *node_ids, int cap) {
  if (int rc = check_retained_arena(p)) return rc;
  int n = std::min(p->ret_result.pops, p->ret_cap);
  if (!node_ids || cap <= 0) return n;
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  unsigned char *base = p->arena.p + (size_t)p->ret_slot * p->ret_stride;
  CUDA_TRY(cudaMemcpy(node_ids, base + p->ret_off_poplog, (size_t)std::min(n, cap) * sizeof(int), cudaMemcpyDeviceToHost));
  return n;
}

int mplb_get_open(mplb_planner *p, int32_t *node_ids, int cap) {
  if (int rc = check_retained_arena(p)) return rc;
  int n = p->ret_result.n_open;
  if (!node_ids || cap <= 0) return n;
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int m = std::min(n, cap);
  std::vector<HeapEnt> h(m);
  unsigned char *base = p->arena.p + (size_t)p->ret_slot * p->ret_stride;
  CUDA_TRY(cudaMemcpy(h.data(), base + p->ret_off_heap, (size_t)m * sizeof(HeapEnt), cudaMemcpyDeviceToHost));
  for (int i = 0; i < m; i++) node_ids[i] = h[i].node & 0x7fffffff;
  return n;
}

int mplb_expand(mplb_planner *p, const mplb_waypoint *states, int n, mplb_prim_trace *rows) {
  if (!p || !states || !rows) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int rc = build_cfg(p, states[0].control);
  if (rc != MPLB_OK) return rc;
  const DevCfg &c = p->cfg;
  if (c.pot || c.region || c.use_yaw) return fail(MPLB_ERR_STATE, "mplb_expand traces the plain-map get_succ only (no search region / potential map / yaw controls)");
  mplb_waypoint *d_s = nullptr;
  mplb_prim_trace *d_r = nullptr;
  CUDA_TRY(cudaMalloc((void **)&d_s, (size_t)n * sizeof(mplb_waypoint)));
  CUDA_TRY(cudaMalloc((void **)&d_r, (size_t)n * c.nU * sizeof(mplb_prim_trace)));
  CUDA_TRY(cudaMemcpy(d_s, states, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyHostToDevice));
  int grid = std::min(n, 148 * 8);
#define EXPAND_CALL(D, O, M)                                                                                \
  do {                                                                                                      \
    size_t smem = sizeof(PlanSmem<D, O, M>);                                                                \
    auto kern = expand_trace_kernel<D, O, M>;                                                                \
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
    kern<<<grid, MPLB_NT, smem>>>(c, d_s, n, d_r);                                                          \
  } while (0)
  DISPATCH(c.dim, c.ord, c.nU, EXPAND_CALL);
  g_launches++;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(rows, d_r, (size_t)n * c.nU * sizeof(mplb_prim_trace), cudaMemcpyDeviceToHost);
  cudaFree(d_s);
  cudaFree(d_r);
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("expand: ") + cudaGetErrorString(e));
  return MPLB_OK;
}

int mplb_probe_samples(mplb_planner *p, const mplb_waypoint *states, int n, mplb_sample_probe *rows, int cap,
                       int32_t *use_fast, double *fast_delta) {
  if (!p || (n > 0 && !states) || (cap > 0 && !rows)) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return 0;
  if (cap < 0) cap = 0;
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int rc = build_cfg(p, states[0].control);
  if (rc != MPLB_OK) return rc;
  const DevCfg &c = p->cfg;
  if (c.pot || c.region || c.use_yaw) return fail(MPLB_ERR_STATE, "mplb_probe_samples probes the plain-map sampler only (no search region / potential map / yaw controls)");
  if (use_fast) *use_fast = c.use_fast;
  if (fast_delta) *fast_delta = c.fast_delta;
  mplb_waypoint *d_s = nullptr;
  mplb_sample_probe *d_r = nullptr;
  int *d_count = nullptr;
  CUDA_TRY(cudaMalloc((void **)&d_s, (size_t)n * sizeof(mplb_waypoint)));
  CUDA_TRY(cudaMalloc((void **)&d_count, sizeof(int)));
  if (cap > 0) CUDA_TRY(cudaMalloc((void **)&d_r, (size_t)cap * sizeof(mplb_sample_probe)));
  CUDA_TRY(cudaMemcpy(d_s, states, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemset(d_count, 0, sizeof(int)));
  int grid = std::min(n, 148 * 8);
#define PROBE_CALL(D, O, M)                                                                                 \
  do {                                                                                                      \
    size_t smem = sizeof(PlanSmem<D, O, M>);                                                                \
    auto kern = probe_samples_kernel<D, O, M>;                                                              \
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); \
    kern<<<grid, MPLB_NT, smem>>>(c, d_s, n, d_r, cap, d_count);                                            \
  } while (0)
  DISPATCH(c.dim, c.ord, c.nU, PROBE_CALL);
#undef PROBE_CALL
  g_launches++;
  int count = 0;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpy(&count, d_count, sizeof(int), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && cap > 0) e = cudaMemcpy(rows, d_r, (size_t)std::min(count, cap) * sizeof(mplb_sample_probe), cudaMemcpyDeviceToHost);
  cudaFree(d_s);
  cudaFree(d_r);
  cudaFree(d_count);
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("probe_samples: ") + cudaGetErrorString(e));
  return count;
}

int mplb_planner_key_layout(mplb_planner *p, int32_t control, int32_t *key_bits, int32_t *key_wide, int32_t *use_fast) {
  if (!p) return fail(MPLB_ERR_ARG, "null argument");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int rc = build_cfg(p, control);
  if (rc != MPLB_OK) return rc;
  if (key_bits) *key_bits = p->key_bits;
  if (key_wide) *key_wide = p->cfg.key_wide;
  if (use_fast) *use_fast = p->cfg.use_fast;
  return MPLB_OK;
}

#ifdef MPLB_PHASE_TIMING
/* diagnostics build only (not part of the ABI): per-plan phase cycle accumulators of the last batch */
int mplb_debug_phase_cycles(mplb_planner *p, long long *out, int n) {
  if (!p || !out) return fail(MPLB_ERR_ARG, "null argument");
  CUDA_TRY(cudaMemcpy(out, p->d_phase.p, (size_t)n * 16 * sizeof(long long), cudaMemcpyDeviceToHost));
  return MPLB_OK;
}
#endif

size_t mplb_trajectory_msg_size(int n_seg, const char *frame_id) {
  return 16 + (frame_id ? std::strlen(frame_id) : 0) + 4 + (size_t)(n_seg > 0 ? n_seg : 0) * 216 + 4;
}

int mplb_serialize_trajectories_device(mplb_planner *p, const void *d_results, const void *d_actions, const void *d_seg_states,
                                       int n, int max_seg, double z, uint32_t seq, uint32_t stamp_sec, uint32_t stamp_nsec,
                                       const char *frame_id, void *d_out, size_t stride, void *d_len, void *stream) {
  if (!p || !d_results || !d_actions || !d_seg_states || !d_out || !d_len) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if (max_seg <= 0) return fail(MPLB_ERR_ARG, "max_seg must be > 0");
  if (p->dirty || !p->map) return fail(MPLB_ERR_STATE, "no batch has been planned with the current configuration");
  const size_t fl = frame_id ? std::strlen(frame_id) : 0;
  if (fl > 64) return fail(MPLB_ERR_ARG, "frame_id longer than 64 bytes");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  const DevCfg &c = p->cfg;
  MsgArgs a;
  std::memset(&a, 0, sizeof(a));
  a.results = (const mplb_result *)d_results; a.actions = (const int *)d_actions; a.segs = (const double *)d_seg_states;
  a.n = n; a.max_seg = max_seg; a.dim = c.dim; a.ord = c.ord; a.use_yaw = c.use_yaw; a.U = c.U; a.Uyaw = c.Uyaw;
  a.dt = c.dt; a.z = z; a.seq = seq; a.sec = stamp_sec; a.nsec = stamp_nsec; a.frame_len = (unsigned)fl;
  if (fl) std::memcpy(a.frame, frame_id, fl);
  a.out = (unsigned char *)d_out; a.stride = stride; a.len = (unsigned *)d_len;
  const long long warps = (long long)n * (max_seg + 1);
  const int blocks = (int)std::min<long long>((warps + 7) / 8, 148 * 8);
  k_serialize_traj<<<blocks, 256, 0, (cudaStream_t)stream>>>(a);
  g_launches++;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return MPLB_OK;
}

int mplb_serialize_trajectories(mplb_planner *p, const mplb_result *results, const int32_t *actions, const double *seg_states,
                                int n, int max_seg, double z, uint32_t seq, uint32_t stamp_sec, uint32_t stamp_nsec,
                                const char *frame_id, uint8_t *out, size_t stride, uint32_t *len) {
  if (!p || !results || !actions || !seg_states || !out || !len) return fail(MPLB_ERR_ARG, "null argument");
  if (n <= 0) return MPLB_OK;
  if (max_seg <= 0) return fail(MPLB_ERR_ARG, "max_seg must be > 0");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  unsigned char *d = nullptr;
  const size_t b_res = align_up((size_t)n * sizeof(mplb_result), 256), b_act = align_up((size_t)n * max_seg * sizeof(int), 256),
               b_seg = align_up((size_t)n * max_seg * 13 * sizeof(double), 256), b_len = align_up((size_t)n * sizeof(unsigned), 256),
               b_out = (size_t)n * stride;
  CUDA_TRY(cudaMalloc((void **)&d, b_res + b_act + b_seg + b_len + b_out));
  cudaError_t e = cudaMemcpy(d, results, (size_t)n * sizeof(mplb_result), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d + b_res, actions, (size_t)n * max_seg * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d + b_res + b_act, seg_states, (size_t)n * max_seg * 13 * sizeof(double), cudaMemcpyHostToDevice);
  int rc = MPLB_OK;
  if (e == cudaSuccess)
    rc = mplb_serialize_trajectories_device(p, d, d + b_res, d + b_res + b_act, n, max_seg, z, seq, stamp_sec, stamp_nsec, frame_id,
                                            d + b_res + b_act + b_seg + b_len, stride, d + b_res + b_act + b_seg, nullptr);
  if (e == cudaSuccess && rc == MPLB_OK) e = cudaMemcpy(len, d + b_res + b_act + b_seg, (size_t)n * sizeof(unsigned), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess && rc == MPLB_OK) e = cudaMemcpy(out, d + b_res + b_act + b_seg + b_len, b_out, cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("mplb_serialize_trajectories: ") + cudaGetErrorString(e));
  return rc;
}

int mplb_sincos_cr(const double *x, int n, double *s, double *c) {
  if (n <= 0) return MPLB_OK;
  if (!x || !s || !c) return fail(MPLB_ERR_ARG, "null argument");
  double *d = nullptr;
  CUDA_TRY(cudaMalloc((void **)&d, (size_t)n * 3 * sizeof(double)));
  cudaError_t e = cudaMemcpy(d, x, (size_t)n * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) {
    k_sincos_cr<<<(n + 127) / 128, 128>>>(d, n, d + n, d + 2 * (size_t)n);
    g_launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(s, d + n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost);
  if (e == cudaSuccess) e = cudaMemcpy(c, d + 2 * (size_t)n, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost);
  cudaFree(d);
  if (e != cudaSuccess) return fail(MPLB_ERR_CUDA, std::string("mplb_sincos_cr: ") + cudaGetErrorString(e));
  return MPLB_OK;
}

int mplb_last_batch_stats(mplb_planner *p, double *kernel_ms, int32_t *launches, int32_t *tiers) {
  if (!p) return fail(MPLB_ERR_ARG, "null planner");
  if (kernel_ms) *kernel_ms = p->last_ms;
  if (launches) *launches = p->last_launches;
  if (tiers) *tiers = p->last_tiers;
  return MPLB_OK;
}

int mplb_last_batch_tiers(mplb_planner *p, mplb_tier_info *rows, int cap) {
  if (!p) return fail(MPLB_ERR_ARG, "null planner");
  const int n = (int)p->last_tier_rows.size();
  for (int i = 0; i < n && i < cap && rows; i++) rows[i] = p->last_tier_rows[i];
  return n;
}


/* ================================================================== multi-GPU: query sharding over NCCL (SURVEY section 8e)
 * One process per GPU.  The path shards by query and only by query, so there are exactly two collectives: one
 * ncclBroadcast of the voxel grid per map and one grouped ncclSend/ncclRecv gather of fixed-stride result records (and
 * action rows) per batch.  NCCL is bound at run time (dlopen of libnccl.so.2: the copy a host application such as PyTorch
 * already loaded, else the system one), so libmplb.so itself has no link-time dependency on it. */
namespace {
struct NcclApi {
  void *h = nullptr;
  decltype(&ncclGetUniqueId) GetUniqueId = nullptr;
  decltype(&ncclCommInitRank) CommInitRank = nullptr;
  decltype(&ncclCommDestroy) CommDestroy = nullptr;
  decltype(&ncclBroadcast) Broadcast = nullptr;
  decltype(&ncclSend) Send = nullptr;
  decltype(&ncclRecv) Recv = nullptr;
  decltype(&ncclGroupStart) GroupStart = nullptr;
  decltype(&ncclGroupEnd) GroupEnd = nullptr;
  decltype(&ncclGetErrorString) GetErrorString = nullptr;
  bool ok = false;
};
NcclApi &nccl_api() {
  static NcclApi a;
  static bool tried = false;
  if (!tried) {
    tried = true;
    a.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
    if (!a.h) a.h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
    if (a.h) {
#define MPLB_NCCL_SYM(name) a.name = (decltype(a.name))dlsym(a.h, "nccl" #name)
      MPLB_NCCL_SYM(GetUniqueId); MPLB_NCCL_SYM(CommInitRank); MPLB_NCCL_SYM(CommDestroy); MPLB_NCCL_SYM(Broadcast);
      MPLB_NCCL_SYM(Send); MPLB_NCCL_SYM(Recv); MPLB_NCCL_SYM(GroupStart); MPLB_NCCL_SYM(GroupEnd); MPLB_NCCL_SYM(GetErrorString);
#undef MPLB_NCCL_SYM
      a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.Broadcast && a.Send && a.Recv && a.GroupStart && a.GroupEnd;
    }
  }
  return a;
}
#define NCCL_TRY(expr)                                                                                   \
  do {                                                                                                   \
    ncclResult_t r__ = (expr);                                                                           \
    if (r__ != ncclSuccess)                                                                              \
      return fail(MPLB_ERR_CUDA, std::string(#expr) + ": " + (N.GetErrorString ? N.GetErrorString(r__) : "nccl error")); \
  } while (0)
}  // namespace

struct mplb_comm {
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1, device = 0;
  cudaStream_t stream = nullptr;
  DevBuf<unsigned char> gres, gact, hdr; /* gather buffers on the root, header scratch */
};

int mplb_comm_unique_id(uint8_t *id128) {
  if (!id128) return fail(MPLB_ERR_ARG, "null argument");
  NcclApi &N = nccl_api();
  if (!N.ok) return fail(MPLB_ERR_STATE, "libnccl.so.2 could not be loaded");
  ncclUniqueId id;
  NCCL_TRY(N.GetUniqueId(&id));
  static_assert(sizeof(id) == MPLB_COMM_ID_BYTES, "ncclUniqueId size");
  std::memcpy(id128, &id, sizeof(id));
  return MPLB_OK;
}

int mplb_comm_create(const uint8_t *id128, int rank, int nranks, mplb_comm **out) {
  if (!id128 || !out || nranks < 1 || rank < 0 || rank >= nranks) return fail(MPLB_ERR_ARG, "bad communicator arguments");
  NcclApi &N = nccl_api();
  if (!N.ok) return fail(MPLB_ERR_STATE, "libnccl.so.2 could not be loaded");
  mplb_comm *c = new mplb_comm();
  c->rank = rank; c->nranks = nranks;
  if (cudaGetDevice(&c->device) != cudaSuccess) { delete c; return fail(MPLB_ERR_CUDA, "no CUDA device (libmplb has no CPU path)"); }
  ncclUniqueId id;
  std::memcpy(&id, id128, sizeof(id));
  ncclResult_t r = N.CommInitRank(&c->comm, nranks, id, rank);
  if (r != ncclSuccess) { delete c; return fail(MPLB_ERR_CUDA, std::string("ncclCommInitRank: ") + (N.GetErrorString ? N.GetErrorString(r) : "")); }
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) { N.CommDestroy(c->comm); delete c; return fail(MPLB_ERR_CUDA, "cudaStreamCreate"); }
  *out = c;
  return MPLB_OK;
}

void mplb_comm_destroy(mplb_comm *c) {
  if (!c) return;
  NcclApi &N = nccl_api();
  if (c->comm && N.ok) N.CommDestroy(c->comm);
  if (c->stream) cudaStreamDestroy(c->stream);
  c->gres.release(); c->gact.release(); c->hdr.release();
  delete c;
}

int mplb_comm_rank(const mplb_comm *c) { return c ? c->rank : -1; }
int mplb_comm_size(const mplb_comm *c) { return c ? c->nranks : 0; }

int mplb_comm_broadcast_map(mplb_comm *c, int root, int dim, const int32_t *ndim, const double *origin, double res,
                            const int8_t *data, mplb_map **out) {
  if (!c || !out || root < 0 || root >= c->nranks) return fail(MPLB_ERR_ARG, "bad argument");
  NcclApi &N = nccl_api();
  if (set_device_of(c->device)) return fail(MPLB_ERR_CUDA, "cannot select the communicator's device");
  double h[8] = {0, 0, 0, 0, 0, 0, 0, 0}; /* dim, origin[3], ndim[3], res */
  if (c->rank == root) {
    if (!ndim || !origin || !data || (dim != 2 && dim != 3)) return fail(MPLB_ERR_ARG, "the root must supply the map");
    h[0] = dim;
    for (int i = 0; i < dim; i++) { h[1 + i] = origin[i]; h[4 + i] = ndim[i]; }
    h[7] = res;
  }
  CUDA_TRY(c->hdr.reserve(sizeof(h)));
  CUDA_TRY(cudaMemcpyAsync(c->hdr.p, h, sizeof(h), cudaMemcpyHostToDevice, c->stream));
  NCCL_TRY(N.Broadcast(c->hdr.p, c->hdr.p, sizeof(h), ncclUint8, root, c->comm, c->stream));
  CUDA_TRY(cudaMemcpyAsync(h, c->hdr.p, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  const int d = (int)h[0];
  int32_t nd[3] = {1, 1, 1};
  double org[3] = {0, 0, 0};
  for (int i = 0; i < d && i < 3; i++) { org[i] = h[1 + i]; nd[i] = (int32_t)h[4 + i]; }
  mplb_map *m = nullptr;
  int rc = map_alloc(d, nd, org, h[7], &m);
  if (rc != MPLB_OK) return rc;
  if (c->rank == root && cudaMemcpyAsync(m->d_grid, data, m->ncell, cudaMemcpyHostToDevice, c->stream) != cudaSuccess) {
    mplb_map_destroy(m);
    return fail(MPLB_ERR_CUDA, "cudaMemcpy(map)");
  }
  ncclResult_t r = N.Broadcast(m->d_grid, m->d_grid, m->ncell, ncclInt8, root, c->comm, c->stream); /* the one map collective */
  if (r != ncclSuccess) { mplb_map_destroy(m); return fail(MPLB_ERR_CUDA, std::string("ncclBroadcast(map): ") + N.GetErrorString(r)); }
  rc = m->rebuild_bricks(c->stream);
  if (rc != MPLB_OK) { mplb_map_destroy(m); return rc; }
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  *out = m;
  return MPLB_OK;
}

/* gather of this rank's `per` result records and action rows (device buffers) into the root's gather buffers:
 * one ncclGroup of sends/receives */
static int comm_gather(mplb_comm *c, const void *d_res, const void *d_act, int per, int max_seg, int root, cudaStream_t s) {
  NcclApi &N = nccl_api();
  const size_t rb = (size_t)per * sizeof(mplb_result), ab = (size_t)per * max_seg * sizeof(int);
  if (c->rank == root) {
    CUDA_TRY(c->gres.reserve(rb * c->nranks));
    if (ab) CUDA_TRY(c->gact.reserve(ab * c->nranks));
  }
  if (c->nranks == 1) {
    CUDA_TRY(cudaMemcpyAsync(c->gres.p, d_res, rb, cudaMemcpyDeviceToDevice, s));
    if (ab) CUDA_TRY(cudaMemcpyAsync(c->gact.p, d_act, ab, cudaMemcpyDeviceToDevice, s));
    return MPLB_OK;
  }
  NCCL_TRY(N.GroupStart());
  if (c->rank == root) {
    for (int r = 0; r < c->nranks; r++) {
      if (r == root) continue;
      NCCL_TRY(N.Recv(c->gres.p + rb * r, rb, ncclUint8, r, c->comm, s));
      if (ab) NCCL_TRY(N.Recv(c->gact.p + ab * r, ab, ncclUint8, r, c->comm, s));
    }
  } else {
    NCCL_TRY(N.Send(d_res, rb, ncclUint8, root, c->comm, s));
    if (ab) NCCL_TRY(N.Send(d_act, ab, ncclUint8, root, c->comm, s));
  }
  NCCL_TRY(N.GroupEnd());
  if (c->rank == root) {
    CUDA_TRY(cudaMemcpyAsync(c->gres.p + rb * root, d_res, rb, cudaMemcpyDeviceToDevice, s));
    if (ab) CUDA_TRY(cudaMemcpyAsync(c->gact.p + ab * root, d_act, ab, cudaMemcpyDeviceToDevice, s));
  }
  return MPLB_OK;
}

int mplb_plan_stripe_gather_device(mplb_planner *p, mplb_comm *c, const void *d_starts, const void *d_goals, int n_local, int per,
                                   void *d_results, void *d_actions, int max_seg, int root, void *stream) {
  if (!p || !c || !d_results || per < n_local) return fail(MPLB_ERR_ARG, "bad argument");
  int rc = MPLB_OK;
  if (n_local > 0) rc = mplb_plan_batch_device(p, d_starts, d_goals, n_local, d_results, d_actions, nullptr, max_seg, stream);
  if (rc != MPLB_OK) return rc;
  rc = comm_gather(c, d_results, max_seg > 0 ? d_actions : nullptr, per, max_seg > 0 ? max_seg : 0, root, (cudaStream_t)stream);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return MPLB_OK;
}

/* ---- one batch in flight per planner: begin enqueues the search (no wait), end completes it and gathers.  Two planners on
 * one map overlap the drain of one batch with the start of the next (a launch ends with its longest plan). */
int mplb_plan_stripe_begin(mplb_planner *p, const void *d_starts, const void *d_goals, int n_local, void *d_results, void *d_actions,
                           int max_seg, void *stream) {
  if (!p || !d_results || (n_local > 0 && (!d_starts || !d_goals))) return fail(MPLB_ERR_ARG, "null argument");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  p->async_n = n_local;
  p->run->d_results = (mplb_result *)d_results; p->run->d_actions = (int *)d_actions; p->run->max_seg = max_seg; /* the gather needs them even for an empty stripe */
  if (n_local <= 0) return MPLB_OK;
  cudaStream_t s = (cudaStream_t)stream;
  mplb_waypoint w0;
  CUDA_TRY(cudaMemcpyAsync(&w0, d_starts, sizeof(w0), cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s)); /* this stream only: the other planner's batch keeps running */
  p->prior_start_t = w0.t;
  return run_batch_begin(p, (const mplb_waypoint *)d_starts, (const mplb_waypoint *)d_goals, n_local, (mplb_result *)d_results,
                         (int *)d_actions, nullptr, max_seg, w0.control, false, s);
}

int mplb_plan_stripe_end(mplb_planner *p, mplb_comm *c, int per, int root) {
  if (!p || !c) return fail(MPLB_ERR_ARG, "null argument");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int rc = MPLB_OK;
  if (p->async_n > 0) rc = run_batch_end(p);
  if (rc != MPLB_OK) return rc;
  /* every gather of a communicator runs on the communicator's stream, in call order (the search is complete: run_batch_end
   * synchronised the planner's stream) */
  rc = comm_gather(c, p->run->d_results, p->run->max_seg > 0 ? p->run->d_actions : nullptr, per, p->run->max_seg > 0 ? p->run->max_seg : 0, root,
                   c->stream);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  return MPLB_OK;
}

int mplb_plan_batch_sharded_begin(mplb_planner *p, mplb_comm *c, const mplb_waypoint *starts, const mplb_waypoint *goals, int n,
                                  int max_seg) {
  if (!p || !c || !starts || !goals || n <= 0) return fail(MPLB_ERR_ARG, "bad argument");
  if (p->device != c->device) return fail(MPLB_ERR_ARG, "planner and communicator live on different devices");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  if (!p->own_stream) CUDA_TRY(cudaStreamCreateWithFlags(&p->own_stream, cudaStreamNonBlocking));
  const int N = c->nranks, per = (n + N - 1) / N;
  p->h_ls.clear(); p->h_lg.clear();
  for (int i = c->rank; i < n; i += N) { p->h_ls.push_back(starts[i]); p->h_lg.push_back(goals[i]); }
  const int n_loc = (int)p->h_ls.size();
  p->async_n = n_loc; p->async_per = per; p->async_ms = max_seg;
  CUDA_TRY(p->d_starts.reserve(std::max(per, 1)));
  CUDA_TRY(p->d_goals.reserve(std::max(per, 1)));
  CUDA_TRY(p->d_results.reserve(std::max(per, 1)));
  if (max_seg > 0) CUDA_TRY(p->d_actions.reserve((size_t)per * max_seg));
  cudaStream_t s = p->own_stream;
  CUDA_TRY(cudaMemsetAsync(p->d_results.p, 0, (size_t)per * sizeof(mplb_result), s));
  if (n_loc <= 0) return MPLB_OK;
  CUDA_TRY(cudaMemcpyAsync(p->d_starts.p, p->h_ls.data(), (size_t)n_loc * sizeof(mplb_waypoint), cudaMemcpyHostToDevice, s));
  CUDA_TRY(cudaMemcpyAsync(p->d_goals.p, p->h_lg.data(), (size_t)n_loc * sizeof(mplb_waypoint), cudaMemcpyHostToDevice, s));
  p->prior_start_t = p->h_ls[0].t;
  return run_batch_begin(p, p->d_starts.p, p->d_goals.p, n_loc, p->d_results.p, max_seg > 0 ? p->d_actions.p : nullptr, nullptr, max_seg,
                         p->h_ls[0].control, false, s);
}

int mplb_plan_batch_sharded_end(mplb_planner *p, mplb_comm *c, int n, mplb_result *results, int32_t *actions, int root) {
  if (!p || !c) return fail(MPLB_ERR_ARG, "null argument");
  if (c->rank == root && !results) return fail(MPLB_ERR_ARG, "the root needs a result buffer");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  int rc = MPLB_OK;
  if (p->async_n > 0) rc = run_batch_end(p);
  if (rc != MPLB_OK) return rc;
  const int ms = p->async_ms;
  rc = comm_gather(c, p->d_results.p, ms > 0 ? p->d_actions.p : nullptr, p->async_per, ms > 0 ? ms : 0, root, c->stream);
  if (rc != MPLB_OK) return rc;
  CUDA_TRY(cudaStreamSynchronize(c->stream));
  if (c->rank == root) return mplb_comm_unstripe(c, n, p->async_per, actions ? ms : 0, results, actions);
  return MPLB_OK;
}

int mplb_comm_unstripe(mplb_comm *c, int n, int per, int max_seg, mplb_result *results, int32_t *actions) {
  if (!c || !results) return fail(MPLB_ERR_ARG, "bad argument");
  if (set_device_of(c->device)) return fail(MPLB_ERR_CUDA, "cannot select the communicator's device");
  const size_t rb = (size_t)per * sizeof(mplb_result), ab = (size_t)per * max_seg * sizeof(int);
  if (c->gres.n < rb * c->nranks) return fail(MPLB_ERR_STATE, "no gathered batch on this rank");
  std::vector<mplb_result> hr((size_t)per * c->nranks);
  std::vector<int32_t> ha(actions && max_seg > 0 ? (size_t)per * c->nranks * max_seg : 0);
  CUDA_TRY(cudaMemcpy(hr.data(), c->gres.p, rb * c->nranks, cudaMemcpyDeviceToHost));
  if (!ha.empty()) CUDA_TRY(cudaMemcpy(ha.data(), c->gact.p, ab * c->nranks, cudaMemcpyDeviceToHost));
  for (int i = 0; i < n; i++) { /* query i was planned by rank i mod N as its (i / N)-th plan */
    const int r = i % c->nranks, k = i / c->nranks;
    results[i] = hr[(size_t)r * per + k];
    if (!ha.empty()) std::memcpy(actions + (size_t)i * max_seg, &ha[((size_t)r * per + k) * max_seg], (size_t)max_seg * sizeof(int32_t));
  }
  return MPLB_OK;
}

int mplb_plan_batch_sharded(mplb_planner *p, mplb_comm *c, const mplb_waypoint *starts, const mplb_waypoint *goals, int n,
                            mplb_result *results, int32_t *actions, int max_seg, int root) {
  if (!p || !c || !starts || !goals || n <= 0) return fail(MPLB_ERR_ARG, "bad argument");
  if (c->rank == root && !results) return fail(MPLB_ERR_ARG, "the root needs a result buffer");
  if (actions && max_seg <= 0) return fail(MPLB_ERR_ARG, "max_seg must be > 0 when trajectories are requested");
  if (p->device != c->device) return fail(MPLB_ERR_ARG, "planner and communicator live on different devices");
  if (set_device_of(p->device)) return fail(MPLB_ERR_CUDA, "cannot select the planner's device");
  const int N = c->nranks, per = (n + N - 1) / N;
  std::vector<mplb_waypoint> ls, lg;
  for (int i = c->rank; i < n; i += N) { ls.push_back(starts[i]); lg.push_back(goals[i]); }
  const int n_loc = (int)ls.size();
  const int ms = actions || c->rank != root ? max_seg : 0;
  CUDA_TRY(p->d_starts.reserve(std::max(per, 1)));
  CUDA_TRY(p->d_goals.reserve(std::max(per, 1)));
  CUDA_TRY(p->d_results.reserve(std::max(per, 1)));
  if (ms > 0) CUDA_TRY(p->d_actions.reserve((size_t)per * ms));
  CUDA_TRY(cudaMemsetAsync(p->d_results.p, 0, (size_t)per * sizeof(mplb_result), c->stream));
  if (n_loc > 0) {
    CUDA_TRY(cudaMemcpyAsync(p->d_starts.p, ls.data(), (size_t)n_loc * sizeof(mplb_waypoint), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(p->d_goals.p, lg.data(), (size_t)n_loc * sizeof(mplb_waypoint), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
  }
  int rc = mplb_plan_stripe_gather_device(p, c, p->d_starts.p, p->d_goals.p, n_loc, per, p->d_results.p, ms > 0 ? p->d_actions.p : nullptr,
                                          ms, root, c->stream);
  if (rc != MPLB_OK) return rc;
  if (c->rank == root) return mplb_comm_unstripe(c, n, per, actions ? max_seg : 0, results, actions);
  return MPLB_OK;
}

}  // extern "C"
