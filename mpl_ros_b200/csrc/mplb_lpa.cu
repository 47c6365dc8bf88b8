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
 *   k_lpa_plan_shaped the same loop for sessions with a potential map or yaw controls (the SH statements of the core); a batch
 *                     that mixes kinds is one launch per kind on the same stream
 *   k_lpa_subtree     getSubStateSpace (a Dijkstra-like sweep over stored successor lists, serial by nature)
 *   k_lpa_link_count / k_lpa_link_scan / k_lpa_link_fill    the voxel -> edge table in insertion order (count, scan, fill)
 *   k_lpa_match       one thread per link against the changed voxels;  k_lpa_apply  sort + increaseCost / decreaseCost
 *   k_lpa_rehash      node table rebuild after the host grew the arrays
 *   k_lpa_traj        the whole trajectory of a plan longer than the batch's per-plan rows (action ids, parent coords)
 *   k_lpa_gather_hdr  every header of a batch into one array, for one copy to the host
 * The maintenance kernels (link, match, apply, subtree) serve a batch of sessions per launch, one session per block index, and the
 * single-planner entry points are batches of one (DESIGN.md section 4.12.2).
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

/* one entry of a batched updateBlockedNodes / updateClearedNodes: its cells start at row cell0 of the batch's list */
struct EditArg {
  long long cell0;
  int n_cells;
  int cap; /* pairs the session's match array holds */
  int run; /* 0: the match launch skips this entry */
  int pad;
};

__device__ void wp_to_state(const mplb_waypoint &w, double *st) {
  for (int k = 0; k < 3; k++) { st[k] = w.pos[k]; st[3 + k] = w.vel[k]; st[6 + k] = w.acc[k]; st[9 + k] = w.jrk[k]; }
  st[12] = w.yaw;
}

template <bool SH>
__device__ __forceinline__ void lpa_plan_body(Ctx *ctxs, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results,
                                              int *acts, double *segs, int max_seg) {
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
      st = plan_begin<SH>(x, sst, starts[b].t, gst);
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
      for (int u = lane; u < nU; u += 32) succ_row<SH>(x.cfg, x.h->sh, n.st, n.t, n.key, u, &x.rows[u]);
      __syncwarp();
    }
    if (r == -1 || r == -2) {
#ifdef MPLB_LPA_SERIAL_FINISH /* the one-lane tail, kept for A/B runs */
      if (lane == 0) s_code = pop_finish<SH>(x);
      __syncwarp();
      code = s_code;
      __syncwarp();
#else /* probes, new States, predecessor appends and rhs over the lanes; ids, slots and queue operations on lane 0 */
      pop_finish_warp<SH>(x, &s_pop);
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

/* plain occupancy map: the statements without the potential / yaw branches */
__global__ void __launch_bounds__(32)
k_lpa_plan(Ctx *ctxs, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results, int *acts, double *segs, int max_seg) {
  lpa_plan_body<false>(ctxs, starts, goals, results, acts, segs, max_seg);
}
/* potential map and / or yaw controls (Hdr::sh) */
__global__ void __launch_bounds__(32)
k_lpa_plan_shaped(Ctx *ctxs, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results, int *acts, double *segs,
                  int max_seg) {
  lpa_plan_body<true>(ctxs, starts, goals, results, acts, segs, max_seg);
}

/* The map-maintenance kernels below serve a batch of sessions: session b's context is ctxs[b], taken from blockIdx.y where a
 * session spans several blocks (one thread per node or link) and from blockIdx.x where one block serves it. */

/* every session's header in one array, so the host reads a batch's scalars with one copy */
__global__ void k_lpa_gather_hdr(const Ctx *ctxs, Hdr *out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = *ctxs[i].h;
}

/* getSubStateSpace(time_steps[b]); a negative time step leaves session b alone */
__global__ void __launch_bounds__(32) k_lpa_subtree(Ctx *ctxs, const int *time_steps) {
  const int ts = time_steps[blockIdx.x];
  if (threadIdx.x == 0 && ts >= 0) { Ctx x = ctxs[blockIdx.x]; x.h->status = sub_state_space(x, ts); }
}

__global__ void k_lpa_link_count(Ctx *ctxs) {
  const Ctx &x = ctxs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < x.h->n_order) x.link_count[i] = link_node(x, i, nullptr);
}
__global__ void k_lpa_link_scan(Ctx *ctxs) { /* exclusive scan of the per-node counts; total -> n_links */
  if (threadIdx.x != 0) return;
  const Ctx &x = ctxs[blockIdx.x];
  int run = 0;
  for (int i = 0; i < x.h->n_order; i++) { const int c = x.link_count[i]; x.link_count[i] = run; run += c; }
  x.h->n_links = run;
}
__global__ void k_lpa_link_fill(Ctx *ctxs) {
  const Ctx &x = ctxs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < x.h->n_order) link_node(x, i, x.links + x.link_count[i]);
}
/* intToFloat (map_util.h:110-114) of every link cell, session b's rows from row0[b] on; rows at or past `cap` are not written */
__global__ void k_lpa_link_points(const Ctx *ctxs, const long long *row0, double *pts, long long cap) {
  const Ctx &x = ctxs[blockIdx.y];
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= x.h->n_links) return;
  const long long r = row0[blockIdx.y] + l;
  if (r >= cap) return;
  const Cfg &c = x.cfg;
  for (int k = 0; k < 3; k++)
    pts[r * 3 + k] = k < c.dim ? mplb_ref::dadd(mplb_ref::dmul(mplb_ref::dadd((double)x.links[l].cell[k], 0.5), c.res), c.origin[k]) : 0.0;
}
/* the pairs (changed cell b, link l) of session blockIdx.y whose voxels are equal; cnt[s] counts them, the first a.cap are kept */
__global__ void k_lpa_match(Ctx *ctxs, const int *cells3, const EditArg *args, int *cnt) {
  const EditArg a = args[blockIdx.y];
  if (!a.run) return;
  const Ctx &x = ctxs[blockIdx.y];
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= x.h->n_links) return;
  const int vox = x.links[l].vox;
  const int *cs = cells3 + a.cell0 * 3;
  for (int b = 0; b < a.n_cells; b++) {
    const int pn[3] = {cs[b * 3], cs[b * 3 + 1], cs[b * 3 + 2]};
    if (cell_index(x.cfg, pn) == vox) {
      const int at = atomicAdd(&cnt[blockIdx.y], 1);
      if (at < a.cap) x.match[at] = (unsigned long long)b * (unsigned long long)x.h->n_links + (unsigned long long)l;
    }
  }
}
/* affected pairs in (changed voxel, link) order, then ss:207-240; one block per session, cnt[b] pairs */
__global__ void k_lpa_apply(Ctx *ctxs, const int *cnt, int blocked) {
  if (threadIdx.x != 0) return;
  Ctx x = ctxs[blockIdx.x];
  unsigned long long *a = x.match;
  const int n = cnt[blockIdx.x];
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

/* plan_sessions' staging: entry i's start and goal into its slot, its session's header reset for a new plan with its shaping */
__global__ void k_lpa_plan_prep(const Ctx *ctxs, const int *slot, const Shape *shapes, const mplb_waypoint *starts,
                                const mplb_waypoint *goals, mplb_waypoint *wps, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int k = slot[i];
  wps[k] = starts[i];
  wps[n + k] = goals[i];
  Hdr *h = ctxs[k].h;
  h->resume = 0; h->status = 0; h->sh = shapes[k];
}
/* the trajectory of every successful plan that the launch wrote whole (n_seg <= max_rows), packed from row row0[slot] on (-1: the
   slot keeps nothing); one block per slot */
__global__ void k_lpa_pack(const mplb_result *res, const int *acts, const double *segs, int max_rows, const long long *row0, int *pacts,
                           double *psegs) {
  const int k = blockIdx.x;
  const int ns = res[k].n_seg;
  if (row0[k] < 0 || ns > max_rows) return;
  for (int i = threadIdx.x; i < ns; i += blockDim.x) {
    pacts[row0[k] + i] = acts[(size_t)k * max_rows + i];
    for (int c = 0; c < 13; c++) psegs[(row0[k] + i) * 13 + c] = segs[((size_t)k * max_rows + i) * 13 + c];
  }
}
/* the caller's layout of entry blockIdx.x (slot slot[i]): its record, and rows [i max_seg, (i + 1) max_seg) of the packed
   trajectory, -1 actions past it (seg-state rows past it are not written); one block per entry */
__global__ void k_lpa_scatter(const int *slot, const mplb_result *res, const long long *row0, const int *pacts, const double *psegs,
                              int max_seg, mplb_result *out, int *acts, double *segs) {
  const int i = blockIdx.x, k = slot[i];
  if (threadIdx.x == 0) out[i] = res[k];
  const int ns = row0[k] < 0 ? 0 : res[k].n_seg;
  for (int j = threadIdx.x; j < max_seg; j += blockDim.x) {
    const size_t o = (size_t)i * max_seg + j;
    if (acts) acts[o] = j < ns ? pacts[row0[k] + j] : -1;
    if (segs && j < ns)
      for (int c = 0; c < 13; c++) segs[o * 13 + c] = psegs[(row0[k] + j) * 13 + c];
  }
}

/* ------------------------------------------------------------------ host side */
struct Session {
  bool on = false;
  int device = 0;
  int control = 0; /* Control flags of the first start waypoint: fixes the lattice key layout */
  Ctx h{};         /* host copy (device pointers inside) */
  DevBuf<Ctx> d_ctx;
  DevBuf<Hdr> d_hdr;
  DevBuf<Node> nodes;
  DevBuf<Succ> succ;
  DevBuf<Pred> preds;
  DevBuf<int> table, order, order2, heap_node, best, traj_act, epq_node, link_count, cells;
  DevBuf<double> heap_f, epq_f, U, Uyaw, segs;
  DevBuf<Row> rows;
  DevBuf<unsigned char> mark;
  DevBuf<Link> links;
  DevBuf<unsigned long long> match;
  DevBuf<mplb_waypoint> wps;
  DevBuf<mplb_result> res;
  DevBuf<int> acts;
  int cap_nodes = 0, cap_pred = 0, tsize = 0, nU = 0, n_links_host = 0;
  int init_nodes = 1 << 16, init_pred = 1 << 20; /* MPLB_LPA_INIT_NODES / _PREDS, read at every plan, used when allocating */
  int grows = 0;                                 /* doublings since the arrays were allocated */
  bool have_links = false;
  bool shaped = false; /* potential map or yaw controls: planned by k_lpa_plan_shaped with `sh` in its header */
  Shape sh{};
  std::vector<double> U_host, Uyaw_host; /* what U / Uyaw hold, so that a refresh uploads the controls only when they changed */
  /* scratch of the batched maintenance calls whose first entry this session is (as plan_sessions keeps wps / res in its lead) */
  DevBuf<Ctx> b_ctx;
  DevBuf<Hdr> b_hdr;
  DevBuf<unsigned char> p_stage, p_pack; /* plan_sessions: contexts, shapes, slots (and host waypoints) up; packed trajectories down */
  DevBuf<long long> p_row0;
  DevBuf<unsigned char> t_stage; /* the trajectory-output calls' configuration table and ids */
  DevBuf<EditArg> b_args;
  DevBuf<int> b_cnt, b_cells, b_ts;
  DevBuf<long long> b_row0;
  DevBuf<double> b_pts;
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
  MPLB_CUDA_TRY(s->d_ctx.grow(1, 0));
  MPLB_CUDA_TRY(cudaMemcpy(s->d_ctx.p, &s->h, sizeof(Ctx), cudaMemcpyHostToDevice));
  return MPLB_OK;
}
int read_hdr(Session *s, Hdr *out) { MPLB_CUDA_TRY(cudaMemcpy(out, s->d_hdr.p, sizeof(Hdr), cudaMemcpyDeviceToHost)); return MPLB_OK; }
int write_hdr(Session *s, const Hdr &in) { MPLB_CUDA_TRY(cudaMemcpy(s->d_hdr.p, &in, sizeof(Hdr), cudaMemcpyHostToDevice)); return MPLB_OK; }

/* (re)size the node-indexed arrays to `cap` nodes and the predecessor pool to `cap_pred`; contents survive */
int ensure_capacity(Session *s, int cap, int cap_pred, bool keep) {
  Hdr hd;
  std::memset(&hd, 0, sizeof(hd));
  if (keep && s->d_hdr.p) { int rc = read_hdr(s, &hd); if (rc) return rc; }
  const size_t used = keep ? (size_t)hd.n_nodes : 0;
  const bool grow_nodes = cap > s->cap_nodes;
  if (grow_nodes) {
    MPLB_CUDA_TRY(s->nodes.grow(cap, used));
    MPLB_CUDA_TRY(s->succ.grow((size_t)cap * s->nU, used * s->nU));
    MPLB_CUDA_TRY(s->order.grow(cap, keep ? (size_t)hd.n_order : 0));
    MPLB_CUDA_TRY(s->order2.grow(cap, 0));
    MPLB_CUDA_TRY(s->heap_f.grow(cap, keep ? (size_t)hd.n_heap : 0));
    MPLB_CUDA_TRY(s->heap_node.grow(cap, keep ? (size_t)hd.n_heap : 0));
    MPLB_CUDA_TRY(s->best.grow(cap, keep ? (size_t)hd.n_best : 0));
    MPLB_CUDA_TRY(s->traj_act.grow(cap, 0));
    MPLB_CUDA_TRY(s->mark.grow(cap, 0));
    MPLB_CUDA_TRY(s->link_count.grow(cap, 0));
    s->cap_nodes = cap;
    int ts = 1024;
    while (ts < 2 * cap) ts <<= 1;
    if (ts > s->tsize) {
      s->table.release();
      MPLB_CUDA_TRY(s->table.grow(ts, 0));
      s->tsize = ts;
    }
    MPLB_CUDA_TRY(cudaMemset(s->table.p, 0xff, (size_t)s->tsize * sizeof(int)));
  }
  if (cap_pred > s->cap_pred) {
    MPLB_CUDA_TRY(s->preds.grow(cap_pred, keep ? (size_t)hd.n_pred : 0));
    s->cap_pred = cap_pred;
  }
  MPLB_CUDA_TRY(s->d_hdr.grow(1, 1));
  MPLB_CUDA_TRY(s->rows.grow(std::max(s->nU, 32), 0)); /* >= one staging row per lane (re-created successors of a stored list) */
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
    MPLB_CUDA_TRY(cudaGetLastError());
    MPLB_CUDA_TRY(cudaDeviceSynchronize());
  }
  return MPLB_OK;
}

/* buf = src[0 .. n), copied only when it differs bit for bit from the host record `have` of what buf holds */
int upload_if_changed(DevBuf<double> &buf, std::vector<double> &have, const double *src, size_t n) {
  if (buf.p && have.size() == n && std::memcmp(have.data(), src, n * sizeof(double)) == 0) return MPLB_OK;
  have.clear();
  MPLB_CUDA_TRY(buf.grow(n, 0));
  MPLB_CUDA_TRY(cudaMemcpy(buf.p, src, n * sizeof(double), cudaMemcpyHostToDevice));
  /* a pageable copy may return before it has landed; the plan may run on a caller's non-blocking stream */
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  have.assign(src, src + n);
  return MPLB_OK;
}

/* what refresh_cfg would refuse for planner configuration `hc` and start control flags `control`; nothing is changed */
int cfg_error(const MplbLpaHostCfg &hc, const Session *s, int control) {
  if (!hc.has_map) return mplb_internal_fail(MPLB_ERR_STATE, "LPA*: no map set");
  if (hc.nU <= 0) return mplb_internal_fail(MPLB_ERR_STATE, "LPA*: no controls set");
  if (hc.nU > LPA_MAXU) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: more than 128 controls");
  if (hc.astar_only) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: search region / prior trajectory are A*-only on this path");
  if (control & ~31) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: unsupported control flag on the start waypoint");
  const bool yaw = (control & 16) != 0;
  if (yaw && !hc.Uyaw)
    return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the start waypoint uses yaw but the control rows have no yaw column (setU rows need Dim + 1 entries)");
  if (yaw && hc.dim < 2) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: yaw controls need a planar velocity (Dim >= 2)");
  if (yaw && hc.yaw_max > 0 && !(hc.yaw_max < 1e5)) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: yaw_max is out of range");
  if (hc.d_pot && hc.pot_cells != (size_t)hc.nd[0] * hc.nd[1] * (hc.dim == 3 ? hc.nd[2] : 1))
    return mplb_internal_fail(MPLB_ERR_STATE, "LPA*: potential map size does not match the planner's map");
  const int cc = control & 15;
  const int ord = cc == 1 ? 1 : cc == 3 ? 2 : cc == 7 ? 3 : cc == 15 ? 4 : 0;
  if (!ord) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the start waypoint carries no control flag");
  if (s->control && s->control != control) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the control flag changed since the first plan; call mplb_planner_reset first");
  if (s->nU && s->nU != hc.nU) return mplb_internal_fail(MPLB_ERR_ARG, "LPA*: the control set changed since the first plan; call mplb_planner_reset first");
  return MPLB_OK;
}

/* the planner's current configuration -> Cfg (device pointers), uploaded with the context */
int refresh_cfg(mplb_planner *p, Session *s, int control) {
  MplbLpaHostCfg hc;
  mplb_internal_planner_cfg(p, &hc);
  if (int rc = cfg_error(hc, s, control)) return rc;
  MPLB_CUDA_TRY(cudaSetDevice(hc.device));
  const bool yaw = (control & 16) != 0;
  const int cc = control & 15;
  const int ord = cc == 1 ? 1 : cc == 3 ? 2 : cc == 7 ? 3 : 4;
  s->device = hc.device;
  s->nU = hc.nU;
  s->init_nodes = hc.lpa_init_nodes; s->init_pred = hc.lpa_init_preds;
  if (int rc = upload_if_changed(s->U, s->U_host, hc.U, (size_t)hc.nU * 3)) return rc;
  /* cost shaping and yaw (em:104-128, pr:503-525): the planner's device copy of its potential map, the yaw column of U */
  Shape &sh = s->sh;
  sh = Shape{};
  sh.pot = hc.d_pot; sh.pot_w = hc.pot_w; sh.grad_w = hc.grad_w;
  sh.use_yaw = yaw ? 1 : 0; sh.wyaw = hc.wyaw; sh.yaw_max = hc.yaw_max; sh.cos_yaw_max = 1.0;
  if (yaw) {
    if (int rc = upload_if_changed(s->Uyaw, s->Uyaw_host, hc.Uyaw, (size_t)hc.nU)) return rc;
    sh.Uyaw = s->Uyaw.p;
    if (hc.yaw_max > 0) { double sn; mplb::trig::sincos_cr(hc.yaw_max, &sn, &sh.cos_yaw_max); } /* cos(my) of pr:521 */
  }
  s->shaped = sh.pot != nullptr || yaw;
  Cfg &c = s->h.cfg;
  c.dim = hc.dim; c.ord = ord; c.control = control; c.nU = hc.nU; c.nkey = hc.dim * ord + (yaw ? 1 : 0); c.max_num = hc.max_num;
  c.dt = hc.dt; c.w = hc.w; c.eps = hc.eps; c.v_max = hc.v_max; c.a_max = hc.a_max; c.j_max = hc.j_max;
  c.tol_pos = hc.tol_pos; c.tol_vel = hc.tol_vel; c.tol_acc = hc.tol_acc;
  for (int i = 0; i < 3; i++) { c.nd[i] = hc.nd[i]; c.origin[i] = hc.origin[i]; }
  c.res = hc.res; c.grid = hc.d_grid; c.U = s->U.p;
  return MPLB_OK;
}

int reset_state(Session *s) { /* PlannerBase::reset: the next plan starts a new StateSpace (and may use other controls) */
  Session fresh; /* frees every array when it replaces *s; only the switch, the device and the initial sizes stay */
  fresh.on = s->on; fresh.device = s->device; fresh.init_nodes = s->init_nodes; fresh.init_pred = s->init_pred;
  *s = std::move(fresh);
  return MPLB_OK;
}

/* double every array of the session, keeping its contents */
int grow_session(Session *s) {
  s->grows++;
  return ensure_capacity(s, s->cap_nodes * 2, s->cap_pred * 2, true);
}

/* one LPA* plan per planner.  Starts and goals are either host arrays (h_starts / h_goals, uploaded with the staging) or device
 * arrays (d_starts / d_goals, in caller order on `stream`); results go to h_results and / or, with the fixed-row trajectory layout of
 * mplb_plan_batch_device, to d_results / d_acts / d_segs.  The host work of a call does not grow with n: one staging upload, one
 * header gather per growth round, one record copy and one packed copy of every retained trajectory (DESIGN.md section 4.12.2). */
struct PlanIO {
  const mplb_waypoint *h_starts = nullptr, *h_goals = nullptr, *d_starts = nullptr, *d_goals = nullptr;
  mplb_result *h_results = nullptr, *d_results = nullptr;
  int *d_acts = nullptr;
  double *d_segs = nullptr;
  int max_seg = 0;
  cudaStream_t stream = 0;
};

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

/* every header of `n` contexts in device memory, in one launch and one copy */
int gather_hdrs_of(Session *lead, const Ctx *d_ctxs, int n, std::vector<Hdr> &out, cudaStream_t stream) {
  MPLB_CUDA_TRY(lead->b_hdr.grow(n, 0));
  k_lpa_gather_hdr<<<(n + 127) / 128, 128, 0, stream>>>(d_ctxs, lead->b_hdr.p, n);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  out.resize(n);
  MPLB_CUDA_TRY(cudaMemcpyAsync(out.data(), lead->b_hdr.p, (size_t)n * sizeof(Hdr), cudaMemcpyDeviceToHost, stream));
  MPLB_CUDA_TRY(cudaStreamSynchronize(stream));
  return MPLB_OK;
}

int plan_sessions(std::vector<mplb_planner *> &ps, const PlanIO &io) {
  const int n = (int)ps.size();
  if (n == 0) return MPLB_OK;
  cudaStream_t stream = io.stream;
  std::vector<mplb_waypoint> dev_starts;
  const mplb_waypoint *starts = io.h_starts;
  if (!starts) { /* the control flags of device starts decide each session's key layout: one read of the starts */
    MplbLpaHostCfg hc0;
    mplb_internal_planner_cfg(ps[0], &hc0);
    MPLB_CUDA_TRY(cudaSetDevice(hc0.device));
    dev_starts.resize(n);
    MPLB_CUDA_TRY(cudaMemcpyAsync(dev_starts.data(), io.d_starts, (size_t)n * sizeof(mplb_waypoint), cudaMemcpyDeviceToHost, stream));
    MPLB_CUDA_TRY(cudaStreamSynchronize(stream));
    starts = dev_starts.data();
  }
  std::vector<Session *> ss(n);
  int device = -1;
  for (int i = 0; i < n; i++) { /* every configuration is checked before any session changes */
    ss[i] = session_of(ps[i], true);
    MplbLpaHostCfg hc;
    mplb_internal_planner_cfg(ps[i], &hc);
    if (int rc = cfg_error(hc, ss[i], starts[i].control)) return rc;
    if (i > 0 && hc.device != device) return mplb_internal_fail(MPLB_ERR_ARG, "LPA* batch: all planners must live on one device");
    device = hc.device;
  }
  bool allocated = false;
  for (int i = 0; i < n; i++) {
    Session *s = ss[i];
    int rc = refresh_cfg(ps[i], s, starts[i].control);
    if (rc) return rc;
    s->control = starts[i].control;
    if (s->cap_nodes == 0) { rc = ensure_capacity(s, s->init_nodes, s->init_pred, false); if (rc) return rc; allocated = true; }
  }
  /* the batch's contexts, contiguous: the plain sessions first, then the shaped ones, so that each kind is one launch over a
     contiguous range of slots; slot[i] is planner i's position, at[k] the planner in slot k */
  Session *lead = ss[0];
  const int max_rows = 4096; /* per-plan trajectory rows of the launch; longer trajectories are gathered after it */
  std::vector<int> slot(n), at(n);
  int n_plain = 0;
  for (int i = 0; i < n; i++) if (!ss[i]->shaped) slot[i] = n_plain++;
  for (int i = 0, k = n_plain; i < n; i++) if (ss[i]->shaped) slot[i] = k++;
  for (int i = 0; i < n; i++) at[slot[i]] = i;
  /* staging, one upload: Ctx[n] and Shape[n] in slot order, slot[n], then (host starts) starts[n] and goals[n] */
  const size_t o_sh = align256((size_t)n * sizeof(Ctx)), o_slot = o_sh + align256((size_t)n * sizeof(Shape)),
               o_wp = o_slot + align256((size_t)n * sizeof(int)), stage_bytes = o_wp + (io.h_starts ? 2 * (size_t)n * sizeof(mplb_waypoint) : 0);
  std::vector<unsigned char> stage(stage_bytes);
  Ctx *h_ctx = (Ctx *)stage.data();
  for (int k = 0; k < n; k++) {
    h_ctx[k] = ss[at[k]]->h;
    ((Shape *)(stage.data() + o_sh))[k] = ss[at[k]]->sh;
  }
  std::memcpy(stage.data() + o_slot, slot.data(), (size_t)n * sizeof(int));
  if (io.h_starts) {
    std::memcpy(stage.data() + o_wp, io.h_starts, (size_t)n * sizeof(mplb_waypoint));
    std::memcpy(stage.data() + o_wp + (size_t)n * sizeof(mplb_waypoint), io.h_goals, (size_t)n * sizeof(mplb_waypoint));
  }
  MPLB_CUDA_TRY(lead->p_stage.grow(stage_bytes, 0));
  MPLB_CUDA_TRY(lead->wps.grow((size_t)2 * n, 0));
  MPLB_CUDA_TRY(lead->res.grow(n, 0));
  MPLB_CUDA_TRY(lead->acts.grow((size_t)n * max_rows, 0));
  MPLB_CUDA_TRY(lead->segs.grow((size_t)n * max_rows * 13, 0));
  if (allocated) MPLB_CUDA_TRY(cudaDeviceSynchronize()); /* the new sessions' arrays were set up on the default stream */
  Ctx *d_ctx = (Ctx *)lead->p_stage.p;
  MPLB_CUDA_TRY(cudaMemcpyAsync(lead->p_stage.p, stage.data(), stage_bytes, cudaMemcpyHostToDevice, stream));
  /* room for the start node: plan_begin creates it when its key is new, and a pop may have filled the arrays exactly
     (the pop-time check keeps only n_nodes <= cap_nodes; n_order and n_heap never exceed n_nodes) */
  std::vector<Hdr> hd;
  int rc = gather_hdrs_of(lead, d_ctx, n, hd, stream);
  if (rc) return rc;
  auto regrow = [&](int k) -> int { /* double slot k's session and refresh its context in the staging */
    int r = grow_session(ss[at[k]]);
    if (r) return r;
    h_ctx[k] = ss[at[k]]->h;
    return MPLB_OK;
  };
  bool grown = false;
  for (int k = 0; k < n; k++)
    if (hd[k].n_nodes + 1 > ss[at[k]]->cap_nodes) { rc = regrow(k); if (rc) return rc; grown = true; }
  if (grown) {
    MPLB_CUDA_TRY(cudaDeviceSynchronize());
    MPLB_CUDA_TRY(cudaMemcpyAsync(d_ctx, h_ctx, (size_t)n * sizeof(Ctx), cudaMemcpyHostToDevice, stream));
  }
  const mplb_waypoint *d_starts = io.h_starts ? (const mplb_waypoint *)(lead->p_stage.p + o_wp) : io.d_starts;
  const mplb_waypoint *d_goals = io.h_starts ? d_starts + n : io.d_goals;
  k_lpa_plan_prep<<<(n + 127) / 128, 128, 0, stream>>>(d_ctx, (const int *)(lead->p_stage.p + o_slot), (const Shape *)(lead->p_stage.p + o_sh),
                                                       d_starts, d_goals, lead->wps.p, n);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  /* every round doubles the arrays of the sessions that stopped, so 64 rounds cannot run out before int capacities do */
  const int n_shaped = n - n_plain;
  for (int round = 0; round < 64; round++) {
    const mplb_waypoint *d_s = lead->wps.p, *d_g = lead->wps.p + n;
    if (n_plain > 0) {
      k_lpa_plan<<<n_plain, 32, 0, stream>>>(d_ctx, d_s, d_g, lead->res.p, lead->acts.p, lead->segs.p, max_rows);
      mplb_internal_count_launches(1);
      MPLB_CUDA_TRY(cudaGetLastError());
    }
    if (n_shaped > 0) {
      k_lpa_plan_shaped<<<n_shaped, 32, 0, stream>>>(d_ctx + n_plain, d_s + n_plain, d_g + n_plain, lead->res.p + n_plain,
                                                     lead->acts.p + (size_t)n_plain * max_rows,
                                                     lead->segs.p + (size_t)n_plain * max_rows * 13, max_rows);
      mplb_internal_count_launches(1);
      MPLB_CUDA_TRY(cudaGetLastError());
    }
    rc = gather_hdrs_of(lead, d_ctx, n, hd, stream);
    if (rc) return rc;
    bool again = false;
    for (int k = 0; k < n; k++)
      if (hd[k].status == LPA_NEED_GROW) { /* stopped before a pop that could overflow: double and resume */
        rc = regrow(k);
        if (rc) return rc;
        again = true;
      }
    if (!again) break;
    MPLB_CUDA_TRY(cudaDeviceSynchronize());
    MPLB_CUDA_TRY(cudaMemcpyAsync(d_ctx, h_ctx, (size_t)n * sizeof(Ctx), cudaMemcpyHostToDevice, stream));
  }
  std::vector<mplb_result> res(n); /* slot order */
  MPLB_CUDA_TRY(cudaMemcpyAsync(res.data(), lead->res.p, (size_t)n * sizeof(mplb_result), cudaMemcpyDeviceToHost, stream));
  MPLB_CUDA_TRY(cudaStreamSynchronize(stream));
  /* retained trajectory for mplb_get_actions / mplb_get_seg_states (traj_ stays as it was on failure): every successful plan's
     rows packed, then one copy.  lhm_ is NOT refreshed by plan(): the link table stays whatever getLinkedNodes built last
     (map_planner.cpp:127) */
  std::vector<long long> row0(n, -1);
  long long total = 0;
  int max_short = 0;
  for (int k = 0; k < n; k++) {
    if (res[k].status != MPLB_PLAN_OK) continue;
    row0[k] = total;
    total += res[k].n_seg;
    if (res[k].n_seg <= max_rows) max_short = std::max(max_short, res[k].n_seg);
  }
  const size_t o_segs = align256((size_t)total * sizeof(int)), pack_bytes = o_segs + (size_t)total * 13 * sizeof(double);
  MPLB_CUDA_TRY(lead->p_pack.grow(std::max<size_t>(pack_bytes, 1), 0));
  MPLB_CUDA_TRY(lead->p_row0.grow(n, 0));
  int *d_pacts = (int *)lead->p_pack.p;
  double *d_psegs = (double *)(lead->p_pack.p + o_segs);
  MPLB_CUDA_TRY(cudaMemcpyAsync(lead->p_row0.p, row0.data(), (size_t)n * sizeof(long long), cudaMemcpyHostToDevice, stream));
  if (max_short > 0) {
    k_lpa_pack<<<n, 128, 0, stream>>>(lead->res.p, lead->acts.p, lead->segs.p, max_rows, lead->p_row0.p,
                                                                     d_pacts, d_psegs);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  for (int k = 0; k < n; k++) { /* the launch kept max_rows rows; traj_act / best on the device still hold the whole trajectory */
    const int ns = res[k].n_seg;
    if (row0[k] < 0 || ns <= max_rows) continue;
    k_lpa_traj<<<(ns + 127) / 128, 128, 0, stream>>>(d_ctx + k, ns, d_pacts + row0[k], d_psegs + row0[k] * 13);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  if (io.d_results) {
    const int ms = std::max(io.max_seg, 0);
    k_lpa_scatter<<<n, 128, 0, stream>>>(
        (const int *)(lead->p_stage.p + o_slot), lead->res.p, lead->p_row0.p, d_pacts, d_psegs, ms, io.d_results, io.d_acts, io.d_segs);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  std::vector<unsigned char> pack(pack_bytes);
  if (total > 0) MPLB_CUDA_TRY(cudaMemcpyAsync(pack.data(), lead->p_pack.p, pack_bytes, cudaMemcpyDeviceToHost, stream));
  MPLB_CUDA_TRY(cudaStreamSynchronize(stream));
  for (int k = 0; k < n; k++) {
    const int i = at[k];
    if (io.h_results) io.h_results[i] = res[k];
    if (row0[k] < 0) continue;
    mplb_internal_set_retained(ps[i], &res[k], (const int *)pack.data() + row0[k], (const double *)(pack.data() + o_segs) + row0[k] * 13,
                               res[k].n_seg);
  }
  return MPLB_OK;
}

Session *need(mplb_planner *p, const char *what) {
  Session *s = p ? session_of(p, false) : nullptr;
  if (!s || !s->on || !s->d_hdr.p) { mplb_internal_fail(MPLB_ERR_STATE, (std::string(what) + ": LPA* is not enabled or has not planned yet").c_str()); return nullptr; }
  cudaSetDevice(s->device);
  return s;
}

/* ---- batched maintenance (getLinkedNodes, updateBlockedNodes / updateClearedNodes, getSubStateSpace).  A batch is a
 * contiguous Ctx array in its first session's scratch; the kernels take session b from the block index, so the launches and
 * synchronisations of a call do not depend on how many planners it serves.  The single-planner entry points are batches of
 * one. */

/* the sessions of planners[0 .. n): every one enabled, planned, distinct and on one device; nothing is changed */
int batch_sessions(mplb_planner *const *planners, int n, const char *what, std::vector<Session *> &ss) {
  if (n < 0 || (n > 0 && !planners)) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  ss.assign(n, nullptr);
  std::unordered_map<mplb_planner *, int> seen;
  for (int i = 0; i < n; i++) {
    if (!seen.emplace(planners[i], i).second && planners[i])
      return mplb_internal_fail(MPLB_ERR_ARG, (std::string(what) + " batch: a planner appears twice").c_str());
    ss[i] = need(planners[i], what);
    if (!ss[i]) return MPLB_ERR_STATE;
    if (ss[i]->device != ss[0]->device)
      return mplb_internal_fail(MPLB_ERR_ARG, (std::string(what) + " batch: all planners must live on one device").c_str());
  }
  if (n > 0) MPLB_CUDA_TRY(cudaSetDevice(ss[0]->device));
  return MPLB_OK;
}

/* the contexts of `ss` into the lead's contiguous array (one copy) */
int upload_batch(const std::vector<Session *> &ss) {
  Session *lead = ss[0];
  std::vector<Ctx> h(ss.size());
  for (size_t i = 0; i < ss.size(); i++) h[i] = ss[i]->h;
  MPLB_CUDA_TRY(lead->b_ctx.grow(ss.size(), 0));
  MPLB_CUDA_TRY(cudaMemcpy(lead->b_ctx.p, h.data(), h.size() * sizeof(Ctx), cudaMemcpyHostToDevice));
  return MPLB_OK;
}

/* every header of the uploaded batch, in one launch and one copy */
int gather_hdrs(const std::vector<Session *> &ss, std::vector<Hdr> &out) {
  Session *lead = ss[0];
  const int n = (int)ss.size();
  MPLB_CUDA_TRY(lead->b_hdr.grow(n, 0));
  k_lpa_gather_hdr<<<(n + 127) / 128, 128>>>(lead->b_ctx.p, lead->b_hdr.p, n);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  out.resize(n);
  MPLB_CUDA_TRY(cudaMemcpy(out.data(), lead->b_hdr.p, (size_t)n * sizeof(Hdr), cudaMemcpyDeviceToHost));
  return MPLB_OK;
}

/* getLinkedNodes for every session of `ss`; counts[i] = links of entry i, pts3 (may be NULL) the first `cap` rows of the
 * concatenated points */
int linked_nodes(std::vector<mplb_planner *> &ps, std::vector<Session *> &ss, int32_t *counts, double *pts3, int64_t cap) {
  const int n = (int)ss.size();
  if (n == 0) return MPLB_OK;
  for (int i = 0; i < n; i++) { int rc = refresh_cfg(ps[i], ss[i], ss[i]->control); if (rc) return rc; } /* the map may be new */
  Session *lead = ss[0];
  int rc = upload_batch(ss);
  if (rc) return rc;
  std::vector<Hdr> hd;
  rc = gather_hdrs(ss, hd);
  if (rc) return rc;
  int max_order = 0;
  for (int i = 0; i < n; i++) max_order = std::max(max_order, hd[i].n_order);
  const dim3 node_grid((max_order + 127) / 128, n);
  if (max_order > 0) {
    k_lpa_link_count<<<node_grid, 128>>>(lead->b_ctx.p);
    mplb_internal_count_launches(1);
  }
  k_lpa_link_scan<<<n, 1>>>(lead->b_ctx.p); /* sets n_links, 0 for an empty hm_ */
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  rc = gather_hdrs(ss, hd);
  if (rc) return rc;
  bool grown = false;
  int max_links = 0;
  std::vector<long long> row0(n);
  long long total = 0;
  for (int i = 0; i < n; i++) {
    Session *s = ss[i];
    s->have_links = true;
    s->n_links_host = hd[i].n_links;
    counts[i] = hd[i].n_links;
    row0[i] = total;
    total += hd[i].n_links;
    max_links = std::max(max_links, hd[i].n_links);
    if ((size_t)hd[i].n_links > s->links.n) { /* only the sessions whose table outgrew its array */
      MPLB_CUDA_TRY(s->links.grow((size_t)hd[i].n_links + 1024, 0));
      s->h.links = s->links.p;
      grown = true;
    }
  }
  if (grown) { rc = upload_batch(ss); if (rc) return rc; }
  const dim3 link_grid((max_links + 127) / 128, n);
  if (max_links > 0) {
    k_lpa_link_fill<<<node_grid, 128>>>(lead->b_ctx.p);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  const long long rows = pts3 ? std::min<long long>(total, cap) : 0;
  if (rows > 0) {
    MPLB_CUDA_TRY(lead->b_row0.grow(n, 0));
    MPLB_CUDA_TRY(cudaMemcpy(lead->b_row0.p, row0.data(), (size_t)n * sizeof(long long), cudaMemcpyHostToDevice));
    MPLB_CUDA_TRY(lead->b_pts.grow((size_t)rows * 3, 0));
    k_lpa_link_points<<<link_grid, 128>>>(lead->b_ctx.p, lead->b_row0.p, lead->b_pts.p, rows);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
    MPLB_CUDA_TRY(cudaMemcpy(pts3, lead->b_pts.p, (size_t)rows * 3 * sizeof(double), cudaMemcpyDeviceToHost));
  }
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  return MPLB_OK;
}

/* updateBlockedNodes / updateClearedNodes for every session of `ss`: entry i's cells are rows offsets[i] .. offsets[i+1]-1 of
 * d_cells (device); visited[i] = the pairs it visited */
int update_nodes(std::vector<mplb_planner *> &ps, std::vector<Session *> &ss, bool blocked, const int *d_cells,
                 const int64_t *offsets, int32_t *visited) {
  const int n = (int)ss.size();
  std::vector<EditArg> args(n);
  int max_links = 0;
  for (int i = 0; i < n; i++) {
    Session *s = ss[i];
    const long long nc = offsets[i + 1] - offsets[i];
    visited[i] = 0;
    args[i] = EditArg{offsets[i], (int)nc, (int)std::min<size_t>(s->match.n, 0x7fffffff), 0, 0};
    if (!s->have_links || nc == 0 || s->n_links_host == 0) continue; /* lhm_ empty: nothing is linked (map_planner.cpp:164-168) */
    int rc = refresh_cfg(ps[i], s, s->control); /* the map pointer may have been rebuilt */
    if (rc) return rc;
    args[i].run = 1;
    max_links = std::max(max_links, s->n_links_host);
  }
  if (max_links == 0) return MPLB_OK;
  Session *lead = ss[0];
  int rc = upload_batch(ss);
  if (rc) return rc;
  MPLB_CUDA_TRY(lead->b_args.grow(n, 0));
  MPLB_CUDA_TRY(lead->b_cnt.grow(n, 0));
  MPLB_CUDA_TRY(cudaMemset(lead->b_cnt.p, 0, (size_t)n * sizeof(int)));
  std::vector<int> cnt(n);
  const dim3 grid((max_links + 127) / 128, n);
  for (int round = 0; round < 2; round++) { /* the second round re-matches the entries whose pair list did not fit */
    MPLB_CUDA_TRY(cudaMemcpy(lead->b_args.p, args.data(), (size_t)n * sizeof(EditArg), cudaMemcpyHostToDevice));
    k_lpa_match<<<grid, 128>>>(lead->b_ctx.p, d_cells, lead->b_args.p, lead->b_cnt.p);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
    MPLB_CUDA_TRY(cudaMemcpy(cnt.data(), lead->b_cnt.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
    bool again = false;
    for (int i = 0; i < n; i++) {
      Session *s = ss[i];
      args[i].run = 0;
      if ((size_t)cnt[i] <= s->match.n) continue;
      MPLB_CUDA_TRY(s->match.grow((size_t)cnt[i] + 1024, 0)); /* size it and match this entry again */
      s->h.match = s->match.p;
      args[i].cap = (int)std::min<size_t>(s->match.n, 0x7fffffff);
      args[i].run = 1;
      cnt[i] = 0;
      again = true;
    }
    if (!again) break;
    rc = upload_batch(ss);
    if (rc) return rc;
    MPLB_CUDA_TRY(cudaMemcpy(lead->b_cnt.p, cnt.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice));
  }
  bool any = false;
  for (int i = 0; i < n; i++) { visited[i] = cnt[i]; any = any || cnt[i] > 0; }
  if (any) {
    k_lpa_apply<<<n, 32>>>(lead->b_ctx.p, lead->b_cnt.p, blocked ? 1 : 0);
    mplb_internal_count_launches(1);
    MPLB_CUDA_TRY(cudaGetLastError());
  }
  MPLB_CUDA_TRY(cudaDeviceSynchronize());
  return MPLB_OK;
}

/* the shared half of the update entry points: validation, then the host or device cell list */
int update_batch(mplb_planner **planners, int n, int blocked, const int32_t *cells3, bool device, const int64_t *offsets,
                 int32_t *visited) {
  const char *what = blocked ? "updateBlockedNodes" : "updateClearedNodes";
  if (n < 0 || (n > 0 && (!planners || !offsets || !visited))) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  std::vector<Session *> ss;
  int rc = batch_sessions(planners, n, what, ss);
  if (rc) return rc;
  if (n == 0) return MPLB_OK;
  for (int i = 0; i < n; i++)
    if (offsets[i] < 0 || offsets[i + 1] < offsets[i] || offsets[i + 1] - offsets[i] > 0x7fffffff)
      return mplb_internal_fail(MPLB_ERR_ARG, "bad cell offsets");
  const int64_t total = offsets[n];
  if (total > 0 && !cells3) return mplb_internal_fail(MPLB_ERR_ARG, "null cell list");
  std::vector<mplb_planner *> ps(planners, planners + n);
  const int *d_cells = (const int *)cells3;
  if (!device && total > 0) {
    Session *lead = ss[0];
    MPLB_CUDA_TRY(lead->b_cells.grow((size_t)total * 3, 0));
    MPLB_CUDA_TRY(cudaMemcpy(lead->b_cells.p, cells3, (size_t)total * 3 * sizeof(int), cudaMemcpyHostToDevice));
    d_cells = lead->b_cells.p;
  }
  return update_nodes(ps, ss, blocked != 0, d_cells, offsets, visited);
}

/* getSubStateSpace(time_steps[i]) for every session of `ss`; sizes[i] = hm_.size() afterwards, 0 without a trajectory, or
 * MPLB_ERR_STATE where the sweep met a successor that is no longer in the state space */
int sub_state_spaces(std::vector<Session *> &ss, const int32_t *time_steps, int32_t *sizes) {
  const int n = (int)ss.size();
  if (n == 0) return MPLB_OK;
  Session *lead = ss[0];
  int rc = upload_batch(ss);
  if (rc) return rc;
  std::vector<Hdr> hd;
  rc = gather_hdrs(ss, hd);
  if (rc) return rc;
  std::vector<int> ts(n, -1);
  for (int i = 0; i < n; i++) {
    if (hd[i].n_best == 0) continue; /* ss:117 */
    if (time_steps[i] < 0 || time_steps[i] >= hd[i].n_best)
      return mplb_internal_fail(MPLB_ERR_ARG, "getSubStateSpace: time_step beyond the last trajectory");
    ts[i] = time_steps[i];
  }
  bool any = false;
  for (int i = 0; i < n; i++) {
    sizes[i] = 0;
    if (ts[i] < 0) continue;
    any = true;
    Session *s = ss[i];
    /* scratch of the sweep: one queue entry per stored edge at most, one predecessor record per stored edge at most */
    const size_t edges = (size_t)hd[i].n_nodes * s->nU + 16;
    MPLB_CUDA_TRY(s->epq_f.grow(edges, 0));
    MPLB_CUDA_TRY(s->epq_node.grow(edges, 0));
    s->h.epq_f = s->epq_f.p; s->h.epq_node = s->epq_node.p;
    if (edges + (size_t)s->nU > (size_t)s->cap_pred) {
      rc = ensure_capacity(s, s->cap_nodes, (int)std::min<size_t>(edges + s->nU, 0x7fffffff), true);
      if (rc) return rc;
    }
  }
  if (!any) return MPLB_OK;
  rc = upload_batch(ss);
  if (rc) return rc;
  MPLB_CUDA_TRY(lead->b_ts.grow(n, 0));
  MPLB_CUDA_TRY(cudaMemcpy(lead->b_ts.p, ts.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice));
  k_lpa_subtree<<<n, 32>>>(lead->b_ctx.p, lead->b_ts.p);
  mplb_internal_count_launches(1);
  MPLB_CUDA_TRY(cudaGetLastError());
  rc = gather_hdrs(ss, hd);
  if (rc) return rc;
  int first = MPLB_OK;
  for (int i = 0; i < n; i++) {
    if (ts[i] < 0) continue;
    if (hd[i].status == LPA_FAULT) {
      sizes[i] = MPLB_ERR_STATE;
      if (first == MPLB_OK)
        first = mplb_internal_fail(MPLB_ERR_STATE, "getSubStateSpace: a stored successor is no longer in the state space (the reference dereferences a null State here, state_space.h:160-163)");
    } else {
      sizes[i] = hd[i].n_order;
    }
  }
  return first;
}

}  // namespace

int mplb_internal_lpa_enabled(mplb_planner *p) {
  Session *s = session_of(p, false);
  return s && s->on;
}
int mplb_internal_lpa_plan(mplb_planner *p, const mplb_waypoint *start, const mplb_waypoint *goal, mplb_result *out) {
  std::vector<mplb_planner *> ps(1, p);
  PlanIO io;
  io.h_starts = start; io.h_goals = goal; io.h_results = out;
  return plan_sessions(ps, io);
}
void mplb_internal_lpa_drop(mplb_planner *p) {
  std::lock_guard<std::mutex> lock(g_sessions_mu);
  auto it = g_sessions.find(p);
  if (it == g_sessions.end()) return;
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
  PlanIO io;
  io.h_starts = starts; io.h_goals = goals; io.h_results = results;
  return plan_sessions(ps, io);
}

int mplb_lpa_plan_batch_device(mplb_planner **planners, int n, const void *d_starts, const void *d_goals, void *d_results,
                               void *d_actions, void *d_seg_states, int max_seg, void *stream) {
  if (n < 0 || (n > 0 && (!planners || !d_starts || !d_goals || !d_results))) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  if (max_seg < 0) return mplb_internal_fail(MPLB_ERR_ARG, "LPA* batch: max_seg must be >= 0");
  std::vector<mplb_planner *> ps(planners, planners + n);
  std::unordered_map<mplb_planner *, int> seen;
  int device = -1;
  for (int i = 0; i < n; i++) {
    if (!ps[i]) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
    if (!seen.emplace(ps[i], i).second) return mplb_internal_fail(MPLB_ERR_ARG, "LPA* batch: a planner appears twice");
    if (!mplb_internal_lpa_enabled(ps[i])) return mplb_internal_fail(MPLB_ERR_STATE, "LPA* batch: every planner must have LPA* enabled");
    MplbLpaHostCfg hc;
    mplb_internal_planner_cfg(ps[i], &hc);
    if (i > 0 && hc.device != device) return mplb_internal_fail(MPLB_ERR_ARG, "LPA* batch: all planners must live on one device");
    device = hc.device;
  }
  PlanIO io;
  io.d_starts = (const mplb_waypoint *)d_starts; io.d_goals = (const mplb_waypoint *)d_goals;
  io.d_results = (mplb_result *)d_results; io.d_acts = (int *)d_actions; io.d_segs = (double *)d_seg_states;
  io.max_seg = max_seg; io.stream = (cudaStream_t)stream;
  return plan_sessions(ps, io);
}

/* the trajectory-output calls: every planner has planned (batch_sessions), and the table of their plan configurations goes up in
   one copy.  Every session holds its controls in its own device array, so no two entries share a configuration: entry i is
   planner i (dim, control order, control flags, yaw flag, controls and dt of its last plan) and ids[i] = i. */
static int traj_cfgs(mplb_planner **planners, int n, const char *what, std::vector<Session *> &ss, const void *d_results,
                     const void *d_actions, const void *d_seg_states, int max_seg, const MplbTrajCfg **d_cfgs, const int **d_ids,
                     cudaStream_t stream) {
  if (n < 0 || (n > 0 && (!planners || !d_results || !d_actions || !d_seg_states)))
    return mplb_internal_fail(MPLB_ERR_ARG, (std::string(what) + ": null argument").c_str());
  if (max_seg < 1) return mplb_internal_fail(MPLB_ERR_ARG, (std::string(what) + ": max_seg must be > 0").c_str());
  int rc = batch_sessions(planners, n, what, ss);
  if (rc || n == 0) return rc;
  for (int i = 0; i < n; i++)
    if (!ss[i]->control) return mplb_internal_fail(MPLB_ERR_STATE, (std::string(what) + ": a planner has not planned with LPA*").c_str());
  Session *lead = ss[0];
  const size_t o_ids = align256((size_t)n * sizeof(MplbTrajCfg)), bytes = o_ids + (size_t)n * sizeof(int);
  std::vector<unsigned char> h(bytes);
  for (int i = 0; i < n; i++) {
    const Session *s = ss[i];
    MplbTrajCfg &t = ((MplbTrajCfg *)h.data())[i];
    std::memset(&t, 0, sizeof(t));
    t.dim = s->h.cfg.dim; t.ord = s->h.cfg.ord; t.control = s->control; t.use_yaw = s->sh.use_yaw;
    t.U = s->U.p; t.Uyaw = s->sh.use_yaw ? s->sh.Uyaw : nullptr; t.dt = s->h.cfg.dt;
    ((int *)(h.data() + o_ids))[i] = i;
  }
  MPLB_CUDA_TRY(lead->t_stage.grow(bytes, 0));
  MPLB_CUDA_TRY(cudaMemcpyAsync(lead->t_stage.p, h.data(), bytes, cudaMemcpyHostToDevice, stream));
  *d_cfgs = (const MplbTrajCfg *)lead->t_stage.p;
  *d_ids = (const int *)(lead->t_stage.p + o_ids);
  return MPLB_OK;
}

int mplb_lpa_trajectory_waypoints_device(mplb_planner **planners, int n, const void *d_results, const void *d_actions,
                                         const void *d_seg_states, int max_seg, const void *d_index, void *d_waypoints, void *d_ok,
                                         void *stream) {
  if (n > 0 && (!d_index || !d_waypoints || !d_ok)) return mplb_internal_fail(MPLB_ERR_ARG, "trajectory waypoints: null argument");
  std::vector<Session *> ss;
  const MplbTrajCfg *d_cfgs = nullptr;
  const int *d_ids = nullptr;
  int rc = traj_cfgs(planners, n, "trajectory waypoints", ss, d_results, d_actions, d_seg_states, max_seg, &d_cfgs, &d_ids, (cudaStream_t)stream);
  if (rc || n == 0) return rc;
  rc = mplb_internal_pick_waypoints(d_cfgs, d_ids, d_results, d_actions, d_seg_states, n, max_seg, d_index, d_waypoints, d_ok, stream);
  if (rc) return rc;
  MPLB_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return MPLB_OK;
}

int mplb_lpa_serialize_trajectories_device(mplb_planner **planners, int n, const void *d_results, const void *d_actions,
                                           const void *d_seg_states, int max_seg, double z, uint32_t seq, uint32_t stamp_sec,
                                           uint32_t stamp_nsec, const char *frame_id, void *d_out, size_t stride, void *d_len,
                                           void *stream) {
  if (n > 0 && (!d_out || !d_len)) return mplb_internal_fail(MPLB_ERR_ARG, "serialize: null argument");
  if ((frame_id ? std::strlen(frame_id) : 0) > 64) return mplb_internal_fail(MPLB_ERR_ARG, "frame_id longer than 64 bytes");
  std::vector<Session *> ss;
  const MplbTrajCfg *d_cfgs = nullptr;
  const int *d_ids = nullptr;
  int rc = traj_cfgs(planners, n, "serialize", ss, d_results, d_actions, d_seg_states, max_seg, &d_cfgs, &d_ids, (cudaStream_t)stream);
  if (rc || n == 0) return rc;
  return mplb_internal_serialize(d_cfgs, d_ids, d_results, d_actions, d_seg_states, n, max_seg, z, seq, stamp_sec, stamp_nsec, frame_id,
                                 d_out, stride, d_len, stream);
}

int mplb_lpa_refine_trajectories_device(mplb_planner **planners, int n, const void *d_results, const void *d_actions,
                                        const void *d_seg_states, int max_seg, int control, int yaw_control, void *d_coefs,
                                        int32_t *n_segs, void *stream) {
  if (n > 0 && !d_coefs) return mplb_internal_fail(MPLB_ERR_ARG, "refine: null argument");
  std::vector<Session *> ss;
  const MplbTrajCfg *d_cfgs = nullptr;
  const int *d_ids = nullptr;
  int rc = traj_cfgs(planners, n, "refine", ss, d_results, d_actions, d_seg_states, max_seg, &d_cfgs, &d_ids, (cudaStream_t)stream);
  if (rc || n == 0) return rc;
  for (int i = 1; i < n; i++) /* one coefficient layout per call: (dim + 1) rows per segment */
    if (ss[i]->h.cfg.dim != ss[0]->h.cfg.dim) return mplb_internal_fail(MPLB_ERR_ARG, "refine: every planner of a call must plan in the same dim");
  return mplb_internal_refine(ss[0]->h.cfg.dim, d_cfgs, d_ids, d_results, d_actions, d_seg_states, n, max_seg, control, yaw_control,
                              d_coefs, n_segs, stream);
}

int mplb_get_sub_state_space(mplb_planner *p, int time_step) {
  int32_t size = 0;
  const int rc = mplb_lpa_sub_state_space_batch(&p, 1, &time_step, &size);
  return rc ? rc : size;
}

int mplb_get_linked_nodes(mplb_planner *p, double *pts3, int cap) {
  int32_t count = 0;
  const int rc = mplb_lpa_get_linked_nodes_batch(&p, 1, &count, pts3, cap > 0 ? cap : 0);
  return rc ? rc : count;
}

static int update_single(mplb_planner *p, const int32_t *cells3, int n, int blocked) {
  if (n < 0) return mplb_internal_fail(MPLB_ERR_ARG, "null cell list");
  const int64_t offsets[2] = {0, n};
  int32_t visited = 0;
  const int rc = update_batch(&p, 1, blocked, cells3, false, offsets, &visited);
  return rc ? rc : visited;
}
int mplb_update_blocked_nodes(mplb_planner *p, const int32_t *cells3, int n) { return update_single(p, cells3, n, 1); }
int mplb_update_cleared_nodes(mplb_planner *p, const int32_t *cells3, int n) { return update_single(p, cells3, n, 0); }

int mplb_lpa_get_linked_nodes_batch(mplb_planner **planners, int n, int32_t *counts, double *pts3, int64_t cap) {
  if (n < 0 || (n > 0 && !counts) || cap < 0) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  std::vector<Session *> ss;
  int rc = batch_sessions(planners, n, "getLinkedNodes", ss);
  if (rc) return rc;
  std::vector<mplb_planner *> ps(planners, planners + n);
  return linked_nodes(ps, ss, counts, pts3, cap);
}

int mplb_lpa_update_nodes_batch(mplb_planner **planners, int n, int blocked, const int32_t *cells3, const int64_t *offsets,
                                int32_t *visited) {
  return update_batch(planners, n, blocked, cells3, false, offsets, visited);
}

int mplb_lpa_update_nodes_batch_device(mplb_planner **planners, int n, int blocked, const void *d_cells3, const int64_t *offsets,
                                       int32_t *visited) {
  return update_batch(planners, n, blocked, (const int32_t *)d_cells3, true, offsets, visited);
}

int mplb_lpa_sub_state_space_batch(mplb_planner **planners, int n, const int32_t *time_steps, int32_t *sizes) {
  if (n < 0 || (n > 0 && (!time_steps || !sizes))) return mplb_internal_fail(MPLB_ERR_ARG, "null argument");
  std::vector<Session *> ss;
  int rc = batch_sessions(planners, n, "getSubStateSpace", ss);
  if (rc) return rc;
  return sub_state_spaces(ss, time_steps, sizes);
}

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
  MPLB_CUDA_TRY(cudaMemcpy(nodes.data(), s->nodes.p, nodes.size() * sizeof(Node), cudaMemcpyDeviceToHost));
  MPLB_CUDA_TRY(cudaMemcpy(succ.data(), s->succ.p, succ.size() * sizeof(Succ), cudaMemcpyDeviceToHost));
  if (hd.n_pred > 0) MPLB_CUDA_TRY(cudaMemcpy(preds.data(), s->preds.p, (size_t)hd.n_pred * sizeof(Pred), cudaMemcpyDeviceToHost));
  MPLB_CUDA_TRY(cudaMemcpy(order.data(), s->order.p, order.size() * sizeof(int), cudaMemcpyDeviceToHost));
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
  MPLB_CUDA_TRY(cudaMemcpy(f.data(), s->heap_f.p, f.size() * sizeof(double), cudaMemcpyDeviceToHost));
  MPLB_CUDA_TRY(cudaMemcpy(hn.data(), s->heap_node.p, hn.size() * sizeof(int), cudaMemcpyDeviceToHost));
  MPLB_CUDA_TRY(cudaMemcpy(nodes.data(), s->nodes.p, nodes.size() * sizeof(Node), cudaMemcpyDeviceToHost));
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
  MPLB_CUDA_TRY(cudaMemcpy(best.data(), s->best.p, best.size() * sizeof(int), cudaMemcpyDeviceToHost));
  const int nk = s->h.cfg.nkey;
  for (int i = 0; i < hd.n_best && i < cap; i++) {
    Node n;
    MPLB_CUDA_TRY(cudaMemcpy(&n, s->nodes.p + best[i], sizeof(Node), cudaMemcpyDeviceToHost));
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
