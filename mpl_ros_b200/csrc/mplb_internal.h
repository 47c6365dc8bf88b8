/* mplb_internal.h — host helpers the translation units of libmplb.so share (not part of the ABI). */
#ifndef MPLB_INTERNAL_H
#define MPLB_INTERNAL_H
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <string>

#include "../../include/mplb.h"
#if defined(__GNUC__)
#define MPLB_HIDDEN __attribute__((visibility("hidden")))
#else
#define MPLB_HIDDEN
#endif
/* records `msg` for mplb_last_error() and returns `code` */
MPLB_HIDDEN int mplb_internal_fail(int code, const char *msg);
/* adds to the counter behind mplb_launch_count() */
MPLB_HIDDEN void mplb_internal_count_launches(int n);
/* makes `device` the calling thread's current device; 0 on success, -1 when it cannot be selected */
MPLB_HIDDEN int mplb_internal_set_device(int device);

/* returns MPLB_ERR_CUDA from the enclosing function when `expr` (a cudaError_t) is not cudaSuccess */
#define MPLB_CUDA_TRY(expr)                                                                                              \
  do {                                                                                                                   \
    cudaError_t e__ = (expr);                                                                                            \
    if (e__ != cudaSuccess)                                                                                              \
      return mplb_internal_fail(MPLB_ERR_CUDA, (std::string(#expr) + ": " + cudaGetErrorString(e__)).c_str());         \
  } while (0)

/* An owned device array of n elements of T, freed when the buffer is destroyed (the result of that cudaFree is ignored: at
 * process exit it may be cudaErrorCudartUnloading).  Movable, not copyable. */
template <class T>
struct MPLB_HIDDEN DevBuf {
  T *p = nullptr;
  size_t n = 0;

  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevBuf &operator=(DevBuf &&o) noexcept {
    if (this != &o) { release(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; }
    return *this;
  }
  ~DevBuf() { release(); }

  void release() {
    if (p) cudaFree(p);
    p = nullptr;
    n = 0;
  }
  /* at least `want` elements, contents discarded: the old array is freed before the new one is allocated */
  cudaError_t reserve(size_t want) {
    if (want <= n) return cudaSuccess;
    release();
    T *q = nullptr;
    cudaError_t e = cudaMalloc((void **)&q, want * sizeof(T));
    if (e == cudaSuccess) { p = q; n = want; }
    return e;
  }
  /* at least `want` elements keeping the first `keep`: the new array is allocated and filled before the old one is freed */
  cudaError_t grow(size_t want, size_t keep) {
    if (want <= n) return cudaSuccess;
    T *q = nullptr;
    cudaError_t e = cudaMalloc((void **)&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p && keep) e = cudaMemcpy(q, p, std::min(keep, n) * sizeof(T), cudaMemcpyDeviceToDevice);
    release();
    p = q;
    n = want;
    return e;
  }
};

/* ---- what the LPA* unit (mplb_lpa.cu) needs from the planner / map objects of mplb.cu */
struct mplb_planner;
struct mplb_result;
struct mplb_waypoint;
struct MplbLpaHostCfg {
  int dim, nU, max_num, device, verbose, has_map;
  int astar_only; /* search region / prior trajectory installed: not available under LPA* */
  int lpa_init_nodes, lpa_init_preds; /* MPLB_LPA_INIT_NODES / MPLB_LPA_INIT_PREDS */
  double v_max, a_max, j_max, dt, w, eps, tol_pos, tol_vel, tol_acc;
  int nd[3];
  double origin[3];
  double res;
  const int8_t *d_grid; /* the map's int8 cells on the planner's device */
  const double *U;      /* host, nU rows of 3 */
  const double *Uyaw;   /* host, nU yaw rates, or NULL when the control rows carry none */
  const int8_t *d_pot;  /* the planner's potential map on its device, or NULL */
  size_t pot_cells;     /* its entries (one per map cell when it matches the map) */
  double pot_w, grad_w, wyaw, yaw_max;
};
MPLB_HIDDEN int mplb_internal_planner_cfg(mplb_planner *p, MplbLpaHostCfg *out);
/* the retained single plan the getters mplb_get_actions / mplb_get_seg_states serve */
MPLB_HIDDEN void mplb_internal_set_retained(mplb_planner *p, const mplb_result *res, const int *actions, const double *segs13, int n_seg);
/* implemented by mplb_lpa.cu, called by mplb.cu */
MPLB_HIDDEN int mplb_internal_lpa_enabled(mplb_planner *p);
MPLB_HIDDEN int mplb_internal_lpa_plan(mplb_planner *p, const mplb_waypoint *start, const mplb_waypoint *goal, mplb_result *out);
MPLB_HIDDEN void mplb_internal_lpa_drop(mplb_planner *p);

/* ---- trajectory output of planned batches (the wire serialiser of mplb.cu, the waypoint gather of mplb_trajsolve.cu): what a
 * plan's rows are read with.  Entry i of a batch uses table[cfg_id[i]] (cfg_id NULL: entry 0 for all).  An A* batch passes a table
 * of one entry and no ids; an LPA* fleet passes one entry per planner (each session keeps its controls in its own device array)
 * and ids 0 .. n-1. */
struct MplbTrajCfg {
  int dim, ord;      /* ord: 1 VEL .. 4 SNP, the control order the plan was made with */
  int control;       /* the plan's Control flags (yaw bit included) */
  int use_yaw;       /* the serialiser writes cyaw rows */
  const double *U;   /* device, nU rows of 3 */
  const double *Uyaw; /* device, nU yaw rates, or NULL */
  double dt;
};
/* k_serialize_traj over n plans of the fixed-row layout (max_seg rows per plan) on `stream`; returns after it completed */
MPLB_HIDDEN int mplb_internal_serialize(const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const void *d_results, const void *d_actions,
                                        const void *d_seg_states, int n, int max_seg, double z, uint32_t seq, uint32_t stamp_sec,
                                        uint32_t stamp_nsec, const char *frame_id, void *d_out, size_t stride, void *d_len, void *stream);
/* Trajectory::getWaypoints()[pick[i]] of every plan (t the running sum of segment times), ok[i] = 0 where there is none; enqueued */
MPLB_HIDDEN int mplb_internal_pick_waypoints(const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const void *d_results, const void *d_actions,
                                             const void *d_seg_states, int n, int max_seg, const void *d_pick, void *d_wps, void *d_ok,
                                             void *stream);
/* the refinement of mplb_refine_trajectories_device for one dim, each plan with its own table entry; returns after the solve */
MPLB_HIDDEN int mplb_internal_refine(int dim, const MplbTrajCfg *d_cfgs, const int *d_cfg_id, const void *d_results, const void *d_actions,
                                     const void *d_seg_states, int n, int max_seg, int control, int yaw_control, void *d_coefs,
                                     int32_t *n_segs, void *stream);

/* ---- what the VoxelGrid unit (mplb_voxel.cu) needs from the map object of mplb.cu */
struct mplb_map;
struct MplbMapView {
  int dim, device;
  int nd[3];
  double origin[3];
  double res;
  size_t ncell;
  int8_t *d_grid; /* the map's int8 cells (x fastest) on `device` */
};
MPLB_HIDDEN void mplb_internal_map_view(mplb_map *m, MplbMapView *out);
/* after d_grid was rewritten on `stream` (a cudaStream_t): rebuild the occupancy bit-bricks, as mplb_map_set_data does */
MPLB_HIDDEN int mplb_internal_map_cells_changed(mplb_map *m, void *stream);

/* ---- what the fleet unit (mplb_fleet.cu) needs from the communicator of mplb.cu (defined in its extern "C" block) */
struct MplbCommView {
  int rank, nranks, device;
  void *stream; /* the communicator's cudaStream_t: every collective of a communicator runs on it, in call order */
};
extern "C" {
MPLB_HIDDEN void mplb_internal_comm_view(mplb_comm *c, MplbCommView *out);
/* at least `bytes` bytes of the communicator's grow-only scratch slot `slot` (< MPLB_COMM_FLEET_SLOTS) on its device, kept until
 * the communicator is destroyed; contents are not kept when it grows.  NULL (mplb_last_error set) when it cannot be allocated. */
#define MPLB_COMM_FLEET_SLOTS 8
MPLB_HIDDEN void *mplb_internal_comm_scratch(mplb_comm *c, int slot, size_t bytes);
/* rank r's bytes[r] bytes (device memory; `send` is this rank's) land at recv + bytes[0] + ... + bytes[r - 1] on every
 * rank: one group of ncclSend / ncclRecv on `stream`, enqueued only.  Every rank passes the same sizes. */
MPLB_HIDDEN int mplb_internal_comm_allgather(mplb_comm *c, const void *send, const size_t *bytes, void *recv, void *stream);
/* this rank's `per` result records and action rows (device buffers) into the root's gather buffers, which
 * mplb_comm_unstripe reads: one group of ncclSend / ncclRecv on `stream`, enqueued only */
MPLB_HIDDEN int mplb_internal_comm_gather(mplb_comm *c, const void *d_res, const void *d_act, int per, int max_seg, int root,
                                          void *stream);
}
#endif
