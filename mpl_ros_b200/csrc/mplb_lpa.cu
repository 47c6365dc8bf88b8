/*
 * mplb_lpa.cu — LPA* replanning on the GPU: kernels and host runtime around mplb_lpa_core.h (SURVEY section 8f.3).
 *
 * Reference surface (motion_primitive_library/include/mpl_planner/common/planner_base.h, planner/map_planner.h):
 *   setLPAstar :170-176, plan with use_lpastar_ :275-325, getSubStateSpace :155, reset :164-167,
 *   MapPlanner::getLinkedNodes / updateBlockedNodes / updateClearedNodes (src/mpl_planner/map_planner.cpp:125-185),
 * exercised by mpl_test_node/src/map_replanner_node.cpp:107-241.  One replanner is one CTA of one warp with its search state
 * resident in HBM between calls; mplb_lpa_plan_batch runs many replanners (robots) in one launch.  See the core header for
 * the split between the lane-parallel successor generation and the order-defining serial part.
 *
 * Kernels (all HBM/L2 latency bound pointer work except the successor rows, which are FP64):
 *   k_lpa_plan        the LPA* loop; 32 lanes generate the |U| successor rows of a popped node and then share its graph update
 *                     (key-table probes, new States, predecessor appends, rhs recomputation); lane 0 keeps what defines order:
 *                     ids, iteration-order slots and the priority-queue operations
 *   k_lpa_subtree     getSubStateSpace (a Dijkstra-like sweep over stored successor lists, serial by nature)
 *   k_lpa_link_count / k_lpa_link_scan / k_lpa_link_fill    the voxel -> edge table in insertion order (count, scan, fill)
 *   k_lpa_match       one thread per link against the changed voxels;  k_lpa_apply  sort + increaseCost / decreaseCost
 *   k_lpa_rehash      node table rebuild after the host grew the arrays
 *   k_lpa_traj        the whole trajectory of a plan longer than the batch's per-plan rows (action ids, parent coords)
 * Capacity: arrays start at MPLB_LPA_INIT_NODES nodes / MPLB_LPA_INIT_PREDS predecessor records (65 536 / 2^20 by default) and
 * double when a pop could overflow them (the kernel stops BEFORE the pop and the host grows and resumes), or before a plan whose
 * start node would not fit (plan_begin may create one node and has no stop of its own), so a search is never truncated.
 */
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/mplb.h"
#include "mplb_internal.h"
#include "mplb_lpa_core.h"

using namespace mplb_lpa;

namespace {

#define LPA_CUDA(expr)                                                                                          \
  do {                                                                                                          \
    cudaError_t e__ = (expr);                                                                                   \
    if (e__ != cudaSuccess) return mplb_internal_fail(MPLB_ERR_CUDA, (std::string(#expr) + ": " + cudaGetErrorString(e__)).c_str()); \
  } while (0)

__device__ void wp_to_state(const mplb_waypoint &w, double *st) {
  for (int k = 0; k < 3; k++) { st[k] = w.pos[k]; st[3 + k] = w.vel[k]; st[6 + k] = w.acc[k]; st[9 + k] = w.jrk[k]; }
  st[12] = w.yaw;
}

__global__ void __launch_bounds__(32)
k_lpa_plan(Ctx *ctxs, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results, int *acts, double *segs, int max_seg) {
  __shared__ Ctx x;
  __shared__ int s_code;
  __shared__ PopScratch s_pop;
  const int lane = threadIdx.x, b = blockIdx.x;
  if (lane == 0) {
    x = ctxs[b];
    int st = -1;
    if (x.h->resume == 2) st = -3; /* this session finished in an earlier launch of the same batch (another one had to grow) */
    else if (!x.h->resume) {
      double sst[13], gst[13];
      wp_to_state(starts[b], sst);
      wp_to_state(goals[b], gst);
      st = plan_begin(x, sst, starts[b].t, gst);
    }
    s_code = st;
  }
  __syncwarp();
  int code = s_code;
  if (code == -3) return;
  const int nU = x.cfg.nU;
  while (code == -1) {
    if (lane == 0) s_code = pop_begin(x);
    __syncwarp();
    const int r = s_code;
    __syncwarp();
    if (r == -1) { /* one lane per control: end state, validation, lattice key, collision samples */
      const Node &n = x.nodes[x.h->curr];
      for (int u = lane; u < nU; u += 32) succ_row(x.cfg, n.st, n.t, n.key, u, &x.rows[u]);
      __syncwarp();
    }
    if (r == -1 || r == -2) {
#ifdef MPLB_LPA_SERIAL_FINISH /* the one-lane tail, kept for A/B runs */
      if (lane == 0) s_code = pop_finish(x);
      __syncwarp();
      code = s_code;
      __syncwarp();
#else /* probes, new States, predecessor appends and rhs over the lanes; ids, slots and queue operations on lane 0 */
      pop_finish_warp(x, &s_pop);
      code = s_pop.ret;
      __syncwarp();
#endif
    } else code = r;
  }
  Hdr &h = *x.h;
  if (code == LPA_NEED_GROW) {
    if (lane == 0) { h.status = LPA_NEED_GROW; h.resume = 1; }
    return;
  }
  __shared__ int s_nseg;
  __shared__ double s_cost;
  if (lane == 0) {
    h.resume = 2; /* done: a relaunch of the batch for a growing neighbour must not plan this one again */
    int n_seg = 0;
    double cost = LPA_INF;
    if (code == LPA_OK) code = recover(x, &n_seg, &cost);
    else if (code == LPA_START_IS_GOAL) cost = 0;
    h.status = code;
    s_code = code; s_nseg = n_seg; s_cost = cost;
  }
  __syncwarp();
  code = s_code;
  /* closed set of hm_ (getCloseSet, pb:84-91): count and order-independent hash, lanes strided over the iteration order */
  int nc = 0;
  unsigned long long ch = 0;
  const bool have_state = h.initialized && code != LPA_START_NOT_FREE && code != LPA_START_IS_GOAL;
  if (have_state)
    for (int i = lane; i < h.n_order; i += 32) {
      const Node &n = x.nodes[x.order[i]];
      if (n.closed) { nc++; ch += key_hash(n.key, x.cfg.nkey); }
    }
  for (int o = 16; o > 0; o >>= 1) { nc += __shfl_down_sync(0xffffffffu, nc, o); ch += __shfl_down_sync(0xffffffffu, ch, o); }
  const int n_seg = s_nseg;
  for (int i = lane; i < n_seg && i < max_seg; i += 32) { /* trajectory: action ids and the stored coord of each segment's parent */
    acts[(size_t)b * max_seg + i] = x.traj_act[i];
    const Node &pn = x.nodes[x.best[i]];
    for (int k = 0; k < 13; k++) segs[((size_t)b * max_seg + i) * 13 + k] = pn.st[k];
  }
  if (lane == 0) {
    mplb_result r;
    memset(&r, 0, sizeof(r));
    r.status = code;
    r.n_seg = n_seg;
    r.cost = s_cost;
    r.pops = h.expand_iteration;
    if (have_state) { r.n_nodes = h.n_order; r.n_open = h.n_heap; r.n_closed = nc; r.closed_hash = ch; }
    r.n_prims = h.n_prims; r.n_samples = h.n_samples; r.n_valid = h.n_valid;
    r.pop_hash = have_state ? h.pop_hash : 0;
    results[b] = r;
  }
}

__global__ void __launch_bounds__(32) k_lpa_subtree(Ctx *ctxs, int time_step) {
  if (threadIdx.x == 0) { Ctx x = ctxs[blockIdx.x]; x.h->status = sub_state_space(x, time_step); }
}

__global__ void k_lpa_link_count(Ctx *ctxs) {
  const Ctx &x = ctxs[0];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < x.h->n_order) x.link_count[i] = link_node(x, i, nullptr);
}
__global__ void k_lpa_link_scan(Ctx *ctxs) { /* exclusive scan of the per-node counts; total -> n_links */
  const Ctx &x = ctxs[0];
  int run = 0;
  for (int i = 0; i < x.h->n_order; i++) { const int c = x.link_count[i]; x.link_count[i] = run; run += c; }
  x.h->n_links = run;
}
__global__ void k_lpa_link_fill(Ctx *ctxs) {
  const Ctx &x = ctxs[0];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < x.h->n_order) link_node(x, i, x.links + x.link_count[i]);
}
__global__ void k_lpa_match(Ctx *ctxs, const int *cells3, int n_cells) {
  const Ctx &x = ctxs[0];
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= x.h->n_links) return;
  const int vox = x.links[l].vox;
  for (int b = 0; b < n_cells; b++) {
    const int pn[3] = {cells3[b * 3], cells3[b * 3 + 1], cells3[b * 3 + 2]};
    if (cell_index(x.cfg, pn) == vox) {
      const int at = atomicAdd(&x.h->n_match, 1);
      if (at < x.h->cap_match) x.match[at] = (unsigned long long)b * (unsigned long long)x.h->n_links + (unsigned long long)l;
    }
  }
}
__global__ void k_lpa_apply(Ctx *ctxs, int blocked) { /* affected pairs in (changed voxel, link) order, then ss:207-240 */
  if (threadIdx.x != 0) return;
  Ctx x = ctxs[0];
  unsigned long long *a = x.match;
  const int n = x.h->n_match;
  for (int start = n / 2 - 1; start >= 0; start--) { /* heapsort */
    int root = start;
    while (2 * root + 1 < n) {
      int c = 2 * root + 1;
      if (c + 1 < n && a[c] < a[c + 1]) c++;
      if (a[root] < a[c]) { const unsigned long long t = a[root]; a[root] = a[c]; a[c] = t; root = c; } else break;
    }
  }
  for (int end = n - 1; end > 0; end--) {
    const unsigned long long t = a[0]; a[0] = a[end]; a[end] = t;
    int root = 0;
    while (2 * root + 1 < end) {
      int c = 2 * root + 1;
      if (c + 1 < end && a[c] < a[c + 1]) c++;
      if (a[root] < a[c]) { const unsigned long long u = a[root]; a[root] = a[c]; a[c] = u; root = c; } else break;
    }
  }
  for (int i = 0; i < n; i++) {
    const Link &l = x.links[(int)(a[i] % (unsigned long long)x.h->n_links)];
    apply_change(x, l.node, l.pred_idx, blocked != 0);
  }
}
__global__ void k_lpa_rehash(Ctx *ctxs) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  Ctx x = ctxs[0];
  for (int i = 0; i < x.h->n_nodes; i++) table_insert(x, i);
}
/* the trajectory recover() left in traj_act / best, for plans longer than k_lpa_plan's rows: one thread per segment */
__global__ void k_lpa_traj(const Ctx *ctx, int n_seg, int *acts, double *segs) {
  const Ctx &x = *ctx;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_seg) return;
  acts[i] = x.traj_act[i];
  const Node &pn = x.nodes[x.best[i]];
  for (int k = 0; k < 13; k++) segs[(size_t)i * 13 + k] = pn.st[k];
}

/* ------------------------------------------------------------------ host side */
template <typename T>
struct Buf {
  T *p = nullptr;
  size_t n = 0;
  cudaError_t grow(size_t want, size_t keep) { /* reallocate to `want` elements, keeping the first `keep` */
    if (want <= n) return cudaSuccess;
    T *q = nullptr;
    cudaError_t e = cudaMalloc((void **)&q, want * sizeof(T));
    if (e != cudaSuccess) return e;
    if (p && keep) e = cudaMemcpy(q, p, std::min(keep, n) * sizeof(T), cudaMemcpyDeviceToDevice);
    if (p) cudaFree(p);
    p = q; n = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};
template <typename T>
struct TmpBuf : Buf<T> { ~TmpBuf() { this->release(); } }; /* freed on every return path */

struct Session {
  bool on = false;
  int device = 0;
  int control = 0; /* Control flags of the first start waypoint: fixes the lattice key layout */
  Ctx h{};         /* host copy (device pointers inside) */
  Buf<Ctx> d_ctx;
  Buf<Hdr> d_hdr;
  Buf<Node> nodes;
  Buf<Succ> succ;
  Buf<Pred> preds;
  Buf<int> table, order, order2, heap_node, best, traj_act, epq_node, link_count, cells;
  Buf<double> heap_f, epq_f, U, segs;
  Buf<Row> rows;
  Buf<unsigned char> mark;
  Buf<Link> links;
  Buf<unsigned long long> match;
  Buf<mplb_waypoint> wps;
  Buf<mplb_result> res;
  Buf<int> acts;
  int cap_nodes = 0, cap_pred = 0, tsize = 0, nU = 0, n_links_host = 0;
  int init_nodes = 1 << 16, init_pred = 1 << 20; /* MPLB_LPA_INIT_NODES / _PREDS, read at every plan, used when allocating */
  int grows = 0;                                 /* doublings since the arrays were allocated */
  bool have_links = false;
  void release() {
    d_ctx.release(); d_hdr.release(); nodes.release(); succ.release(); preds.release(); table.release(); order.release();
    order2.release(); heap_node.release(); best.release(); traj_act.release(); epq_node.release(); link_count.release();
    cells.release(); heap_f.release(); epq_f.release(); U.release(); segs.release(); rows.release(); mark.release();
    links.release(); match.release(); wps.release(); res.release(); acts.release();
  }
};

std::unordered_map<mplb_planner *, Session *> g_sessions; /* planner -> its replanning session; the registry is locked, a
                                                              session itself is as non-re-entrant as its planner (env_base.h:402-404) */
std::mutex g_sessions_mu;

Session *session_of(mplb_planner *p, bool create) {
  std::lock_guard<std::mutex> lock(g_sessions_mu);
  auto it = g_sessions.find(p);
  if (it != g_sessions.end()) return it->second;
  if (!create) return nullptr;
  Session *s = new Session();
  g_sessions[p] = s;
  return s;
}

int upload_ctx(Session *s) {
  LPA_CUDA(s->d_ctx.grow(1, 0));
  LPA_CUDA(cudaMemcpy(s->d_ctx.p, &s->h, sizeof(Ctx), cudaMemcpyHostToDevice));
  return MPLB_OK;
}
int read_hdr(Session *s, Hdr *out) { LPA_CUDA(cudaMemcpy(out, s->d_hdr.p, sizeof(Hdr), cudaMemcpyDeviceToHost)); return MPLB_OK; }
int write_hdr(Session *s, const Hdr &in) { LPA_CUDA(cudaMemcpy(s->d_hdr.p, &in, sizeof(Hdr), cudaMemcpyHostToDevice)); return MPLB_OK; }

/* (re)size the node-indexed arrays to `cap` nodes and the predecessor pool to `cap_pred`; contents survive */
int ensure_capacity(Session *s, int cap, int cap_pred, bool keep) {
  Hdr hd;
  std::memset(&hd, 0, sizeof(hd));
  if (keep && s->d_hdr.p) { int rc = read_hdr(s, &hd); if (rc) return rc; }
  const size_t used = keep ? (size_t)hd.n_nodes : 0;
  const bool grow_nodes = cap > s->cap_nodes;
  if (grow_nodes) {
    LPA_CUDA(s->nodes.grow(cap, used));
    LPA_CUDA(s->succ.grow((size_t)cap * s->nU, used * s->nU));
    LPA_CUDA(s->order.grow(cap, keep ? (size_t)hd.n_order : 0));
    LPA_CUDA(s->order2.grow(cap, 0));
    LPA_CUDA(s->heap_f.grow(cap, keep ? (size_t)hd.n_heap : 0));
    LPA_CUDA(s->heap_node.grow(cap, keep ? (size_t)hd.n_heap : 0));
    LPA_CUDA(s->best.grow(cap, keep ? (size_t)hd.n_best : 0));
    LPA_CUDA(s->traj_act.grow(cap, 0));
    LPA_CUDA(s->mark.grow(cap, 0));
    LPA_CUDA(s->link_count.grow(cap, 0));
    s->cap_nodes = cap;
    int ts = 1024;
    while (ts < 2 * cap) ts <<= 1;
    if (ts > s->tsize) {
      s->table.release();
      LPA_CUDA(s->table.grow(ts, 0));
      s->tsize = ts;
    }
    LPA_CUDA(cudaMemset(s->table.p, 0xff, (size_t)s->tsize * sizeof(int)));
  }
  if (cap_pred > s->cap_pred) {
    LPA_CUDA(s->preds.grow(cap_pred, keep ? (size_t)hd.n_pred : 0));
    s->cap_pred = cap_pred;
  }
  LPA_CUDA(s->d_hdr.grow(1, 1));
  LPA_CUDA(s->rows.grow(std::max(s->nU, 32), 0)); /* >= one staging row per lane (re-created successors of a stored list) */
  s->h.h = s->d_hdr.p; s->h.nodes = s->nodes.p; s->h.succ = s->succ.p; s->h.preds = s->preds.p; s->h.table = s->table.p;
  s->h.order = s->order.p; s->h.order2 = s->order2.p; s->h.heap_f = s->heap_f.p; s->h.heap_node = s->heap_node.p;
  s->h.best = s->best.p; s->h.traj_act = s->traj_act.p; s->h.rows = s->rows.p; s->h.mark = s->mark.p;
  s->h.link_count = s->link_count.p; s->h.epq_f = s->epq_f.p; s->h.epq_node = s->epq_node.p; s->h.links = s->links.p; s->h.match = s->match.p;
  hd.cap_nodes = s->cap_nodes; hd.cap_pred = s->cap_pred; hd.tsize = s->tsize;
  int rc = write_hdr(s, hd);
  if (rc) return rc;
  rc = upload_ctx(s);
  if (rc) return rc;
  if (grow_nodes && keep && hd.n_nodes > 0) {
    k_lpa_rehash<<<1, 32>>>(s->d_ctx.p);
    mplb_internal_count_launches(1);
    LPA_CUDA(cudaGetLastError());
    LPA_CUDA(cudaDeviceSynchronize());
  }
  return MPLB_OK;
}

/* the planner's current configuration -> Cfg (device pointers), uploaded with the context */
int refresh_cfg(mplb_planner *p, Session *s, int control) {
  MplbLpaHostCfg hc;
  mplb_internal_planner_cfg(p, &hc);
  if (!hc.has_map) return mplb_internal_fail(MPLB_ERR_STATE, "LPA*: no map set");
  if (hc.nU <= 0) return mplb_internal_fail(MPLB_ERR_STATE, "LPA*: no controls set");
  if (hc.nU > LPA_MAXU) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: more than 128 controls");
  if (hc.shaped) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: potential map / search region / prior trajectory / yaw controls are A*-only on this path");
  if (control & 16) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: yaw controls are A*-only on this path");
  const int cc = control & 15;
  const int ord = cc == 1 ? 1 : cc == 3 ? 2 : cc == 7 ? 3 : cc == 15 ? 4 : 0;
  if (!ord) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the start waypoint carries no control flag");
  if (s->control && s->control != control) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the control flag changed since the first plan; call mplb_planner_reset first");
  if (s->nU && s->nU != hc.nU) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the control set changed since the first plan; call mplb_planner_reset first");
  LPA_CUDA(cudaSetDevice(hc.device));
  s->device = hc.device;
  s->nU = hc.nU;
  s->init_nodes = hc.lpa_init_nodes; s->init_pred = hc.lpa_init_preds;
  LPA_CUDA(s->U.grow((size_t)hc.nU * 3, 0));
  LPA_CUDA(cudaMemcpy(s->U.p, hc.U, (size_t)hc.nU * 3 * sizeof(double), cudaMemcpyHostToDevice));
  Cfg &c = s->h.cfg;
  c.dim = hc.dim; c.ord = ord; c.control = control; c.nU = hc.nU; c.nkey = hc.dim * ord; c.max_num = hc.max_num;
  c.dt = hc.dt; c.w = hc.w; c.eps = hc.eps; c.v_max = hc.v_max; c.a_max = hc.a_max; c.j_max = hc.j_max;
  c.tol_pos = hc.tol_pos; c.tol_vel = hc.tol_vel; c.tol_acc = hc.tol_acc;
  for (int i = 0; i < 3; i++) { c.nd[i] = hc.nd[i]; c.origin[i] = hc.origin[i]; }
  c.res = hc.res; c.grid = hc.d_grid; c.U = s->U.p;
  return MPLB_OK;
}

int reset_state(Session *s) { /* PlannerBase::reset: the next plan starts a new StateSpace (and may use other controls) */
  s->release();
  s->cap_nodes = 0; s->cap_pred = 0; s->tsize = 0; s->nU = 0; s->n_links_host = 0; s->grows = 0;
  s->have_links = false;
  s->control = 0;
  std::memset(&s->h, 0, sizeof(s->h));
  return MPLB_OK;
}

/* double every array of the session, keeping its contents */
int grow_session(Session *s) {
  s->grows++;
  return ensure_capacity(s, s->cap_nodes * 2, s->cap_pred * 2, true);
}

int plan_sessions(std::vector<mplb_planner *> &ps, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results) {
  const int n = (int)ps.size();
  if (n == 0) return MPLB_OK;
  std::vector<Session *> ss(n);
  for (int i = 0; i < n; i++) {
    Session *s = session_of(ps[i], true);
    ss[i] = s;
    int rc = refresh_cfg(ps[i], s, starts[i].control);
    if (rc) return rc;
    if (i > 0 && s->device != ss[0]->device) return mplb_internal_fail(MPLB_ERR_ARG, "LPA* batch: all planners must live on one device");
    s->control = starts[i].control;
    if (s->cap_nodes == 0) { rc = ensure_capacity(s, s->init_nodes, s->init_pred, false); if (rc) return rc; }
    else { rc = upload_ctx(s); if (rc) return rc; }
    /* room for the start node: plan_begin creates it when its key is new, and a pop may have filled the arrays exactly
       (the pop-time check keeps only n_nodes <= cap_nodes; n_order and n_heap never exceed n_nodes) */
    Hdr hd;
    rc = read_hdr(s, &hd);
    if (rc) return rc;
    if (hd.n_nodes + 1 > s->cap_nodes) { rc = grow_session(s); if (rc) return rc; }
  }
  /* the batch's contexts, contiguous */
  Session *lead = ss[0];
  const int max_seg = 4096; /* per-plan trajectory rows of the launch; longer trajectories are gathered after it */
  TmpBuf<Ctx> ctxs;
  LPA_CUDA(ctxs.grow(n, 0));
  for (int i = 0; i < n; i++) LPA_CUDA(cudaMemcpy(ctxs.p + i, &ss[i]->h, sizeof(Ctx), cudaMemcpyHostToDevice));
  LPA_CUDA(lead->wps.grow((size_t)2 * n, 0));
  LPA_CUDA(lead->res.grow(n, 0));
  LPA_CUDA(lead->acts.grow((size_t)n * max_seg, 0));
  LPA_CUDA(lead->segs.grow((size_t)n * max_seg * 13, 0));
  LPA_CUDA(cudaMemcpy(lead->wps.p, starts, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyHostToDevice));
  LPA_CUDA(cudaMemcpy(lead->wps.p + n, goals, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyHostToDevice));
  for (int i = 0; i < n; i++) { Hdr hd; int rc = read_hdr(ss[i], &hd); if (rc) return rc; hd.resume = 0; hd.status = 0; rc = write_hdr(ss[i], hd); if (rc) return rc; }
  /* every round doubles the arrays of the sessions that stopped, so 64 rounds cannot run out before int capacities do */
  for (int round = 0; round < 64; round++) {
    k_lpa_plan<<<n, 32>>>(ctxs.p, lead->wps.p, lead->wps.p + n, lead->res.p, lead->acts.p, lead->segs.p, max_seg);
    mplb_internal_count_launches(1);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) return mplb_internal_fail(MPLB_ERR_CUDA, (std::string("k_lpa_plan: ") + cudaGetErrorString(e)).c_str());
    bool again = false;
    for (int i = 0; i < n; i++) {
      Hdr hd;
      int rc = read_hdr(ss[i], &hd);
      if (rc) return rc;
      if (hd.status == LPA_NEED_GROW) { /* stopped before a pop that could overflow: double and resume */
        rc = grow_session(ss[i]);
        if (rc) return rc;
        LPA_CUDA(cudaMemcpy(ctxs.p + i, &ss[i]->h, sizeof(Ctx), cudaMemcpyHostToDevice));
        again = true;
      }
    }
    if (!again) break;
  }
  LPA_CUDA(cudaMemcpy(results, lead->res.p, (size_t)n * sizeof(mplb_result), cudaMemcpyDeviceToHost));
  std::vector<int> acts;
  std::vector<double> segs;
  for (int i = 0; i < n; i++) { /* retained trajectory for mplb_get_actions / mplb_get_seg_states (traj_ stays as it was on failure) */
    /* lhm_ is NOT refreshed by plan(): the link table stays whatever getLinkedNodes built last (map_planner.cpp:127) */
    if (results[i].status != MPLB_PLAN_OK) continue;
    const int ns = results[i].n_seg;
    acts.resize(std::max(ns, 1));
    segs.resize((size_t)std::max(ns, 1) * 13);
    const int *d_acts = lead->acts.p + (size_t)i * max_seg;
    const double *d_segs = lead->segs.p + (size_t)i * max_seg * 13;
    TmpBuf<int> long_acts;
    TmpBuf<double> long_segs;
    if (ns > max_seg) { /* the launch kept max_seg rows; traj_act / best on the device still hold the whole trajectory */
      LPA_CUDA(long_acts.grow(ns, 0));
      LPA_CUDA(long_segs.grow((size_t)ns * 13, 0));
      k_lpa_traj<<<(ns + 127) / 128, 128>>>(ctxs.p + i, ns, long_acts.p, long_segs.p);
      mplb_internal_count_launches(1);
      LPA_CUDA(cudaGetLastError());
      d_acts = long_acts.p;
      d_segs = long_segs.p;
    }
    LPA_CUDA(cudaMemcpy(acts.data(), d_acts, (size_t)ns * sizeof(int), cudaMemcpyDeviceToHost));
    LPA_CUDA(cudaMemcpy(segs.data(), d_segs, (size_t)ns * 13 * sizeof(double), cudaMemcpyDeviceToHost));
    mplb_internal_set_retained(ps[i], &results[i], acts.data(), segs.data(), ns);
  }
  return MPLB_OK;
}

Session *need(mplb_planner *p, const char *what) {
  Session *s = p ? session_of(p, false) : nullptr;
  if (!s || !s->on || !s->d_hdr.p) { mplb_internal_fail(MPLB_ERR_STATE, (std::string(what) + ": LPA* is not enabled or has not planned yet").c_str()); return nullptr; }
  cudaSetDevice(s->device);
  return s;
}

int build_links(Session *s) {
  Hdr hd;
  int rc = read_hdr(s, &hd);
  if (rc) return rc;
  s->have_links = true;
  if (hd.n_order == 0) { hd.n_links = 0; s->n_links_host = 0; return write_hdr(s, hd); }
  const int blocks = (hd.n_order + 127) / 128;
  k_lpa_link_count<<<blocks, 128>>>(s->d_ctx.p);
  k_lpa_link_scan<<<1, 1>>>(s->d_ctx.p);
  mplb_internal_count_launches(2);
  LPA_CUDA(cudaGetLastError());
  LPA_CUDA(cudaDeviceSynchronize());
  rc = read_hdr(s, &hd);
  if (rc) return rc;
  if ((size_t)hd.n_links > s->links.n) {
    LPA_CUDA(s->links.grow((size_t)hd.n_links + 1024, 0));
    s->h.links = s->links.p;
    hd.cap_links = (int)s->links.n;
    rc = write_hdr(s, hd);
    if (rc) return rc;
    rc = upload_ctx(s);
    if (rc) return rc;
  }
  if (hd.n_links > 0) {
    k_lpa_link_fill<<<blocks, 128>>>(s->d_ctx.p);
    mplb_internal_count_launches(1);
    LPA_CUDA(cudaGetLastError());
    LPA_CUDA(cudaDeviceSynchronize());
  }
  s->n_links_host = hd.n_links;
  return MPLB_OK;
}

int update_nodes(mplb_planner *p, const int32_t *cells3, int n, bool blocked) {
  Session *s = need(p, blocked ? "updateBlockedNodes" : "updateClearedNodes");
  if (!s) return MPLB_ERR_STATE;
  if (n < 0 || (n > 0 && !cells3)) return mplb_internal_fail(MPLB_ERR_ARG, "null cell list");
  if (!s->have_links || n == 0 || s->n_links_host == 0) return 0; /* lhm_ empty: nothing is linked (map_planner.cpp:164-168) */
  int rc = refresh_cfg(p, s, s->control); /* the map pointer may have been rebuilt */
  if (rc) return rc;
  LPA_CUDA(s->cells.grow((size_t)n * 3, 0));
  LPA_CUDA(cudaMemcpy(s->cells.p, cells3, (size_t)n * 3 * sizeof(int), cudaMemcpyHostToDevice));
  Hdr hd;
  for (int attempt = 0; attempt < 2; attempt++) {
    rc = read_hdr(s, &hd);
    if (rc) return rc;
    hd.n_match = 0;
    hd.cap_match = (int)s->match.n;
    rc = write_hdr(s, hd);
    if (rc) return rc;
    rc = upload_ctx(s);
    if (rc) return rc;
    k_lpa_match<<<(s->n_links_host + 127) / 128, 128>>>(s->d_ctx.p, s->cells.p, n);
    mplb_internal_count_launches(1);
    LPA_CUDA(cudaGetLastError());
    LPA_CUDA(cudaDeviceSynchronize());
    rc = read_hdr(s, &hd);
    if (rc) return rc;
    if ((size_t)hd.n_match <= s->match.n) break;
    LPA_CUDA(s->match.grow((size_t)hd.n_match + 1024, 0)); /* the pair list did not fit: size it and match again */
    s->h.match = s->match.p;
  }
  if (hd.n_match > 0) {
    k_lpa_apply<<<1, 32>>>(s->d_ctx.p, blocked ? 1 : 0);
    mplb_internal_count_launches(1);
    LPA_CUDA(cudaGetLastError());
    LPA_CUDA(cudaDeviceSynchronize());
  }
  return hd.n_match;
}

}  // namespace

int mplb_internal_lpa_enabled(mplb_planner *p) {
  Session *s = session_of(p, false);
  return s && s->on;
}
int mplb_internal_lpa_plan(mplb_planner *p, const mplb_waypoint *start, const mplb_waypoint *goal, mplb_result *out) {
  std::vector<mplb_planner *> ps(1, p);
  return plan_sessions(ps, start, goal, out);
}
void mplb_internal_lpa_drop(mplb_planner *p) {
  std::lock_guard<std::mutex> lock(g_sessions_mu);
  auto it = g_sessions.find(p);
  if (it == g_sessions.end()) return;
  it->second->release();
  delete it->second;
  g_sessions.erase(it);
}

extern "C" {

int mplb_planner_set_lpastar(mplb_planner *p, int on) {
  if (!p) return mplb_internal_fail(MPLB_ERR_ARG, "null planner");
  Session *s = session_of(p, true);
  s->on = on != 0;
  return MPLB_OK;
}

int mplb_planner_reset(mplb_planner *p) {
  if (!p) return mplb_internal_fail(MPLB_ERR_ARG, "null planner");
  Session *s = session_of(p, false);
  if (!s) return MPLB_OK;
  cudaSetDevice(s->device);
  return reset_state(s);
}

int mplb_lpa_plan_batch(mplb_planner **planners, int n, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results) {
  if (n < 0 || (n > 0 && (!planners || !starts || !goals || !results))) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  std::vector<mplb_planner *> ps(planners, planners + n);
  for (int i = 0; i < n; i++) {
    if (!ps[i] || !mplb_internal_lpa_enabled(ps[i])) return mplb_internal_fail(MPLB_ERR_STATE, "LPA* batch: every planner must have LPA* enabled");
    for (int j = 0; j < i; j++) if (ps[j] == ps[i]) return mplb_internal_fail(MPLB_ERR_ARG, "LPA* batch: a planner appears twice");
  }
  return plan_sessions(ps, starts, goals, results);
}

int mplb_get_sub_state_space(mplb_planner *p, int time_step) {
  Session *s = need(p, "getSubStateSpace");
  if (!s) return MPLB_ERR_STATE;
  Hdr hd;
  int rc = read_hdr(s, &hd);
  if (rc) return rc;
  if (hd.n_best == 0) return 0; /* ss:117 */
  if (time_step < 0 || time_step >= hd.n_best) return mplb_internal_fail(MPLB_ERR_ARG, "getSubStateSpace: time_step beyond the last trajectory");
  /* scratch of the sweep: one queue entry per stored edge at most, one predecessor record per stored edge at most */
  const size_t edges = (size_t)hd.n_nodes * s->nU + 16;
  LPA_CUDA(s->epq_f.grow(edges, 0));
  LPA_CUDA(s->epq_node.grow(edges, 0));
  s->h.epq_f = s->epq_f.p; s->h.epq_node = s->epq_node.p;
  if (edges + (size_t)s->nU > (size_t)s->cap_pred) { rc = ensure_capacity(s, s->cap_nodes, (int)std::min<size_t>(edges + s->nU, 0x7fffffff), true); if (rc) return rc; }
  rc = upload_ctx(s);
  if (rc) return rc;
  k_lpa_subtree<<<1, 32>>>(s->d_ctx.p, time_step);
  mplb_internal_count_launches(1);
  LPA_CUDA(cudaGetLastError());
  LPA_CUDA(cudaDeviceSynchronize());
  rc = read_hdr(s, &hd);
  if (rc) return rc;
  if (hd.status == LPA_FAULT) return mplb_internal_fail(MPLB_ERR_STATE, "getSubStateSpace: a stored successor is no longer in the state space (the reference dereferences a null State here, state_space.h:160-163)");
  return hd.n_order;
}

int mplb_get_linked_nodes(mplb_planner *p, double *pts3, int cap) {
  Session *s = need(p, "getLinkedNodes");
  if (!s) return MPLB_ERR_STATE;
  int rc = refresh_cfg(p, s, s->control);
  if (rc) return rc;
  rc = upload_ctx(s);
  if (rc) return rc;
  rc = build_links(s);
  if (rc) return rc;
  const int n = s->n_links_host;
  if (pts3 && cap > 0 && n > 0) {
    std::vector<Link> l(n);
    LPA_CUDA(cudaMemcpy(l.data(), s->links.p, (size_t)n * sizeof(Link), cudaMemcpyDeviceToHost));
    const Cfg &c = s->h.cfg;
    for (int i = 0; i < n && i < cap; i++) /* intToFloat (map_util.h:110-114): (pn + 0.5) * res + origin */
      for (int k = 0; k < 3; k++) pts3[(size_t)i * 3 + k] = k < c.dim ? ((double)l[i].cell[k] + 0.5) * c.res + c.origin[k] : 0.0;
  }
  return n;
}

int mplb_update_blocked_nodes(mplb_planner *p, const int32_t *cells3, int n) { return update_nodes(p, cells3, n, true); }
int mplb_update_cleared_nodes(mplb_planner *p, const int32_t *cells3, int n) { return update_nodes(p, cells3, n, false); }

static unsigned long long host_mix(unsigned long long h, unsigned long long v) { return (h ^ v) * 0x100000001B3ull; }

int mplb_lpa_get_nodes(mplb_planner *p, mplb_lpa_node *out, int cap) {
  Session *s = need(p, "lpa_get_nodes");
  if (!s) return MPLB_ERR_STATE;
  Hdr hd;
  int rc = read_hdr(s, &hd);
  if (rc) return rc;
  if (!out || cap <= 0 || hd.n_order == 0) return hd.n_order;
  std::vector<Node> nodes(hd.n_nodes);
  std::vector<Succ> succ((size_t)hd.n_nodes * s->nU);
  std::vector<Pred> preds(std::max(hd.n_pred, 1));
  std::vector<int> order(hd.n_order);
  LPA_CUDA(cudaMemcpy(nodes.data(), s->nodes.p, nodes.size() * sizeof(Node), cudaMemcpyDeviceToHost));
  LPA_CUDA(cudaMemcpy(succ.data(), s->succ.p, succ.size() * sizeof(Succ), cudaMemcpyDeviceToHost));
  if (hd.n_pred > 0) LPA_CUDA(cudaMemcpy(preds.data(), s->preds.p, (size_t)hd.n_pred * sizeof(Pred), cudaMemcpyDeviceToHost));
  LPA_CUDA(cudaMemcpy(order.data(), s->order.p, order.size() * sizeof(int), cudaMemcpyDeviceToHost));
  const int nk = s->h.cfg.nkey;
  for (int i = 0; i < hd.n_order && i < cap; i++) {
    const Node &n = nodes[order[i]];
    mplb_lpa_node &o = out[i];
    std::memset(&o, 0, sizeof(o));
    for (int k = 0; k < nk; k++) o.key[k] = n.key[k];
    o.key[15] = nk;
    for (int k = 0; k < 13; k++) o.state[k] = n.st[k];
    o.g = n.g; o.rhs = n.rhs; o.h = n.h; o.opened = n.opened; o.closed = n.closed; o.n_succ = n.n_succ; o.n_pred = n.n_pred;
    unsigned long long hs = 0xCBF29CE484222325ull, hp = hs;
    for (int k = 0; k < n.n_succ; k++) {
      const Succ &e = succ[(size_t)order[i] * s->nU + k];
      unsigned long long cb; std::memcpy(&cb, &e.cost, 8);
      hs = host_mix(host_mix(host_mix(hs, key_hash(nodes[e.node].key, nk)), (unsigned long long)e.act), cb);
    }
    for (int q = n.pred_head; q >= 0; q = preds[q].next) {
      unsigned long long cb; std::memcpy(&cb, &preds[q].cost, 8);
      hp = host_mix(host_mix(host_mix(hp, key_hash(nodes[preds[q].node].key, nk)), (unsigned long long)preds[q].act), cb);
    }
    o.succ_hash = hs; o.pred_hash = hp;
  }
  return hd.n_order;
}

int mplb_lpa_get_heap(mplb_planner *p, mplb_lpa_heap_entry *out, int cap) {
  Session *s = need(p, "lpa_get_heap");
  if (!s) return MPLB_ERR_STATE;
  Hdr hd;
  int rc = read_hdr(s, &hd);
  if (rc) return rc;
  if (!out || cap <= 0 || hd.n_heap == 0) return hd.n_heap;
  std::vector<double> f(hd.n_heap);
  std::vector<int> hn(hd.n_heap);
  std::vector<Node> nodes(hd.n_nodes);
  LPA_CUDA(cudaMemcpy(f.data(), s->heap_f.p, f.size() * sizeof(double), cudaMemcpyDeviceToHost));
  LPA_CUDA(cudaMemcpy(hn.data(), s->heap_node.p, hn.size() * sizeof(int), cudaMemcpyDeviceToHost));
  LPA_CUDA(cudaMemcpy(nodes.data(), s->nodes.p, nodes.size() * sizeof(Node), cudaMemcpyDeviceToHost));
  for (int i = 0; i < hd.n_heap && i < cap; i++) { out[i].fval = f[i]; out[i].key_hash = key_hash(nodes[hn[i]].key, s->h.cfg.nkey); }
  return hd.n_heap;
}

int mplb_lpa_get_capacity(mplb_planner *p, int32_t *cap_nodes, int32_t *cap_pred, int32_t *tsize, int32_t *n_nodes_physical,
                          int32_t *grows) {
  Session *s = need(p, "lpa_get_capacity");
  if (!s) return MPLB_ERR_STATE;
  Hdr hd;
  int rc = read_hdr(s, &hd);
  if (rc) return rc;
  if (cap_nodes) *cap_nodes = s->cap_nodes;
  if (cap_pred) *cap_pred = s->cap_pred;
  if (tsize) *tsize = s->tsize;
  if (n_nodes_physical) *n_nodes_physical = hd.n_nodes;
  if (grows) *grows = s->grows;
  return MPLB_OK;
}

int mplb_lpa_get_best_child(mplb_planner *p, mplb_lpa_node *out, int cap) {
  Session *s = need(p, "lpa_get_best_child");
  if (!s) return MPLB_ERR_STATE;
  Hdr hd;
  int rc = read_hdr(s, &hd);
  if (rc) return rc;
  if (!out || cap <= 0 || hd.n_best == 0) return hd.n_best;
  std::vector<int> best(hd.n_best);
  LPA_CUDA(cudaMemcpy(best.data(), s->best.p, best.size() * sizeof(int), cudaMemcpyDeviceToHost));
  const int nk = s->h.cfg.nkey;
  for (int i = 0; i < hd.n_best && i < cap; i++) {
    Node n;
    LPA_CUDA(cudaMemcpy(&n, s->nodes.p + best[i], sizeof(Node), cudaMemcpyDeviceToHost));
    mplb_lpa_node &o = out[i];
    std::memset(&o, 0, sizeof(o));
    for (int k = 0; k < nk; k++) o.key[k] = n.key[k];
    o.key[15] = nk;
    for (int k = 0; k < 13; k++) o.state[k] = n.st[k];
    o.g = n.g; o.rhs = n.rhs; o.h = n.h; o.opened = n.opened; o.closed = n.closed; o.n_succ = n.n_succ; o.n_pred = n.n_pred;
  }
  return hd.n_best;
}
}
