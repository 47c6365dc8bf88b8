/*
 * mplb_lpa_core.h — LPA* (Lifelong Planning A*) replanning core of libmplb.so (SURVEY section 8f.3).
 *
 * What it implements (paths under motion_primitive_library/include/mpl_planner, src/mpl_planner):
 *   GraphSearch::LPAstar                               common/graph_search.h:194-365      (gs)
 *   GraphSearch::recoverTraj                           common/graph_search.h:369-455
 *   StateSpace::getSubStateSpace / increaseCost / decreaseCost / updateNode / calculateKey
 *                                                      common/state_space.h:116-282       (ss)
 *   MapPlanner::getLinkedNodes / updateBlockedNodes / updateClearedNodes   map_planner.cpp:125-185
 *   env_map::get_succ / traverse_primitive / is_free(Primitive) / is_goal  env/env_map.h:25-172 (em)
 *   env_map::traverse_primitive with a potential map (em:104-118) and the yaw cost (em:121-128), Primitive's yaw channel and
 *   validate_yaw (pr:236-253,503-525), the yaw key field (waypoint.h:114-117)
 * for the occupancy map, with or without a potential map, and for the *xYAW controls.  Search region and prior trajectory
 * stay A*-only.  The potential / yaw statements are compiled only into the SH = true instantiations (k_lpa_plan_shaped), so
 * that the plain session kernel keeps its code.
 *
 * Shape on the GPU.  One replanner ("session") is one CTA of one warp; a batch of sessions (multi-robot replanning) is a
 * grid.  LPA* is a serial algorithm over a pointer graph; what is parallel inside one session is the successor
 * generation of a popped node (one lane per control: polynomial end state, dynamic validation, lattice key, the
 * collision samples of its primitive), the voxel -> edge link table (one thread per node, count / scan / fill) and the
 * matching of changed voxels against that table (one thread per link).  Everything that decides ORDER (heap, hm_
 * insertion order, updateNode sequence) runs on lane 0 in the reference's statement order, so that the priority queue
 * array, the key ties and therefore the expanded set are the reference's, state by state.
 *
 * Layout.  A node is identified with its lattice key for the whole life of the session: a record that the reference
 * would drop in getSubStateSpace and later re-create through `hm_[coord]` is reset in place (same id).  Successor lists
 * store the successor's node id instead of its coordinate (the coordinate is a function of (parent coord, action) and is
 * recomputed when a dropped successor has to be re-created), predecessor lists are singly linked records in insertion
 * order (recoverTraj's tie rule depends on that order).  hm_ iteration order — which Boost leaves unspecified and which
 * getSubStateSpace / getLinkedNodes observe — is defined as insertion order (`order[]`), like the stand-in container the
 * reference's own sources are compiled against for the parity tests.
 *
 * This header is plain C++ with MPLB_HD functions and no CUDA-only construct outside `#ifdef __CUDA_ARCH__`, so that the
 * test suite can compile the very same statements for the host and compare them with the CPU checker where there is no
 * GPU (tests/cpp/lpa_emul.cpp for plain sessions, tests/cpp/lpa_emul_shaped.cpp for every kind; test infrastructure, never
 * loaded by the product).  The product path is the kernels of mplb_lpa.cu; there is no CPU fallback.
 *
 * Arithmetic: the reference's Primitive and MapUtil arithmetic and the exact IEEE operations come from mplb_ref.h.
 */
#ifndef MPLB_LPA_CORE_H
#define MPLB_LPA_CORE_H
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "mplb_ref.h"
#include "mplb_trig.cuh"

namespace mplb_lpa {

using namespace mplb_ref;
using mplb_ref::dadd; /* these four also hide CUDA's global dadd / dsub / dmul / ddiv(double, double, cudaRoundMode) */
using mplb_ref::dsub;
using mplb_ref::dmul;
using mplb_ref::ddiv;

#define LPA_INF (__builtin_huge_val())
#define LPA_MAXU 128
#define LPA_NKEY 13 /* lattice key fields: pos vel acc jrk per axis + yaw (3-D SNPxYAW) */

/* statuses of a plan (same numbers as mplb_result.status) + internal ones */
enum { LPA_OK = 0, LPA_START_NOT_FREE = 1, LPA_MAX_EXPAND = 2, LPA_QUEUE_EMPTY = 3, LPA_TRACEBACK_FAILED = 4, LPA_START_IS_GOAL = 5,
       LPA_NEED_GROW = 100, LPA_FAULT = 101 };

MPLB_HD bool fIsInf(double x) { return x == LPA_INF || x == -LPA_INF; }

/* ------------------------------------------------------------------ configuration and storage */
struct Cfg {
  int dim, ord, control, nU, nkey, max_num;
  double dt, w, eps, v_max, a_max, j_max, tol_pos, tol_vel, tol_acc;
  int nd[3];
  double origin[3];
  double res;
  const int8_t *grid; /* int8 cells, x fastest (map_util.h:33-41) */
  const double *U;    /* nU rows of 3 */
};

struct Node {
  double st[13]; /* pos3 vel3 acc3 jrk3 yaw: the State's coord (first creator's values) */
  double t;
  double g, rhs, h;
  int key[LPA_NKEY];
  int heap_pos; /* -1 = not in pq_ */
  int n_succ;   /* stored successor entries; 0 = never expanded (gs:265) */
  int pred_head, pred_tail, n_pred;
  unsigned char opened, closed, in_hm, pad;
};
struct Succ { double cost; int node; int act; };
struct Pred { double cost; int node; int act; int next; int pad; };
struct Link { int vox; int node; int pred_idx; int cell[3]; };

struct Row { /* one control's result of get_succ for the popped node (staging, written by the lane that owns the control) */
  double st[13];
  double t;
  double cost;
  int key[LPA_NKEY];
  int verdict; /* 0 = no successor emitted (same state / dynamically infeasible), 1 = emitted */
  int n_samples;
  unsigned long long hash;
};

/* Cost shaping of env_map and the yaw controls of one session (em:104-128, pr:236-253,503-525, eb:372,388); all zero for a
 * plain session.  It lives in the session header (device memory) rather than in Cfg, so that the shared-memory context of
 * the plain kernel keeps its size; only the SH = true statements read it. */
struct Shape {
  const int8_t *pot;    /* potential map, one int8 per map cell (x fastest), or null */
  const double *Uyaw;   /* nU yaw rates (the Dim + 1-th entry of every control row) when use_yaw */
  double pot_w, grad_w; /* potential_weight_, gradient_weight_ (em:114-115) */
  double wyaw;          /* wyaw_ (eb:372) */
  double yaw_max;       /* yaw_max_ (eb:388); <= 0 disables the FOV check */
  double cos_yaw_max;   /* correctly rounded cos(yaw_max), prepared on the host (pr:521) */
  int use_yaw, pad;
};

struct Hdr { /* scalar state of one session */
  int n_nodes, cap_nodes, n_pred, cap_pred, n_order, n_heap, tsize;
  int start_node, goal_node; /* goal_node < 0: the detached State(Coord()) of gs:224-241 (g = rhs = inf, h = 0) */
  int expand_iteration, status, resume, initialized;
  int n_best, n_links, cap_links, n_match, cap_match, n_epq, cap_epq;
  int curr, has_rows; /* the pop in flight between the serial and the parallel half */
  int n_explored, fault;
  double start_g, start_rhs, start_t, eps;
  double goal[13]; /* requested goal (pos vel acc) */
  long long n_prims, n_valid, n_samples;
  unsigned long long pop_hash;
  int start_key[LPA_NKEY];
  double start_st[13];
  double start_tt;
  Shape sh;
};

struct Ctx { /* device view of one session: header + arrays */
  Cfg cfg;
  Hdr *h;
  Node *nodes;
  Succ *succ;   /* cap_nodes * nU */
  Pred *preds;  /* cap_pred */
  int *table;   /* tsize slots: node id or -1 */
  int *order;   /* hm_ iteration order */
  int *order2;  /* scratch of getSubStateSpace */
  double *heap_f;
  int *heap_node;
  int *best;    /* best_child_ (start .. goal) */
  int *traj_act;
  Row *rows;    /* nU */
  double *epq_f; int *epq_node;             /* scratch heap of getSubStateSpace (duplicates allowed) */
  unsigned char *mark;                      /* per node: member of new_hm */
  Link *links; int *link_count;             /* lhm_ as a flat table in insertion order; per order position counts/offsets */
  unsigned long long *match;                /* (changed voxel position, link index) pairs */
};

/* ------------------------------------------------------------------ lattice key (waypoint.h:92-125); the yaw field
 * round(yaw / 0.1) (wp:114-117) only in the SH instantiations, for a yaw session */
template <bool SH = false>
MPLB_HD void make_key(const Cfg &c, const double *st, int *key, bool yaw = false) {
  int n = 0;
  for (int i = 0; i < c.dim; i++) {
    key[n++] = round_int(ddiv(st[i], 0.01));
    if (c.ord >= 2) key[n++] = round_int(ddiv(st[3 + i], 0.1));
    if (c.ord >= 3) key[n++] = round_int(ddiv(st[6 + i], 0.1));
    if (c.ord >= 4) key[n++] = round_int(ddiv(st[9 + i], 0.1));
  }
  if (SH && yaw) key[n++] = round_int(ddiv(st[12], 0.1));
  for (; n < LPA_NKEY; n++) key[n] = 0;
}
MPLB_HD bool key_eq(const int *a, const int *b, int n) {
  for (int i = 0; i < n; i++) if (a[i] != b[i]) return false;
  return true;
}

/* ------------------------------------------------------------------ MapUtil queries on the occupancy grid (map_util.h) */
MPLB_HD bool occupied(const Cfg &c, const int *pn) { return outside(c, pn) ? false : c.grid[cell_index(c, pn)] == 100; }
MPLB_HD bool cell_free(const Cfg &c, const int *pn) {
  if (outside(c, pn)) return false;
  const int8_t v = c.grid[cell_index(c, pn)];
  return v < 100 && v >= 0;
}
MPLB_HD bool ray_hits_occupied(const Cfg &c, const double *p1, const double *p2) { /* mu:117-134 as em:38-42 uses it */
  double diff[3] = {0, 0, 0}, s;
  const int max_diff = ray_setup(c.dim, c.res, p1, p2, diff, &s);
  for (int n = 1; n < max_diff; n++) {
    double pt[3] = {0, 0, 0};
    int pn[3];
    for (int i = 0; i < c.dim; i++) pt[i] = ray_point(p1[i], diff[i], s, n);
    float_to_int(c, pt, pn);
    if (outside(c, pn)) break;
    if (c.grid[cell_index(c, pn)] == 100) return true;
  }
  return false;
}

/* ------------------------------------------------------------------ env_map */
MPLB_HD bool is_goal(const Cfg &c, const double *goal, const double *st) { /* em:25-45 */
  double m = 0;
  for (int i = 0; i < c.dim; i++) m = dmax(m, fabs(dsub(st[i], goal[i])));
  bool goaled = m <= c.tol_pos;
  if (goaled && c.tol_vel >= 0) {
    m = 0;
    for (int i = 0; i < c.dim; i++) m = dmax(m, fabs(dsub(st[3 + i], goal[3 + i])));
    goaled = m <= c.tol_vel;
  }
  if (goaled && c.tol_acc >= 0) {
    m = 0;
    for (int i = 0; i < c.dim; i++) m = dmax(m, fabs(dsub(st[6 + i], goal[6 + i])));
    goaled = m <= c.tol_acc;
  }
  if (goaled && ray_hits_occupied(c, st, goal)) return false;
  return goaled;
}
MPLB_HD double heur(const Cfg &c, const double *goal, const int *goal_key, const double *st, const int *key) { /* eb:46-64 */
  if (key_eq(goal_key, key, c.nkey)) return 0;
  double m = 0;
  for (int i = 0; i < c.dim; i++) m = dmax(m, fabs(dsub(st[i], goal[i])));
  if (c.v_max > 0) return ddiv(dmul(c.w, m), c.v_max);
  return dmul(c.w, m);
}
/* em:90-132 on the plain map: +inf when a sample is outside or occupied, else 0; samples at the accumulated times */
MPLB_HD double traverse(const Cfg &c, const Prim &pr, int *n_samples) {
  const double max_v = prim_max_v(c.dim, pr, c.dt);
  int n = (int)ceil(ddiv(dmul(max_v, c.dt), c.res));
  if (n < 5) n = 5;
  const double dts = ddiv(c.dt, (double)n);
  int tested = 0;
  for (double t = 0; t < c.dt; t = dadd(t, dts)) {
    double st[13];
    int pn[3];
    prim_eval(c.dim, pr, t, st);
    float_to_int(c, st, pn);
    tested++;
    if (outside(c, pn) || c.grid[cell_index(c, pn)] == 100) { *n_samples += tested; return LPA_INF; }
  }
  *n_samples += tested;
  return 0;
}
/* em:60-76: Primitive::sample(n) = n + 1 points at i * (T / n), occupied or outside -> false */
MPLB_HD bool prim_is_free(const Cfg &c, const Prim &pr) {
  const double max_v = prim_max_v(c.dim, pr, c.dt);
  const int n = (int)ceil(ddiv(dmul(max_v, c.dt), c.res));
  const double dts = ddiv(c.dt, (double)n);
  for (int i = 0; i <= n; i++) {
    double st[13];
    int pn[3];
    prim_eval(c.dim, pr, dmul((double)i, dts), st);
    float_to_int(c, st, pn);
    if (occupied(c, pn) || outside(c, pn)) return false;
  }
  return true;
}
/* ------------------------------------------------------------------ potential map and yaw (SH instantiations only) */
/* the yaw channel pr_yaw_ = Primitive1D(yaw0, u_yaw) (pr:36,242-253) at time t, normalised as evaluate() does (pr:328) */
MPLB_HD double yaw_at(double u_yaw, double yaw0, double t) {
  const Prim1 q = {{0, 0, 0, 0, u_yaw, yaw0}};
  return normalize_angle(pr_p(q, t));
}
/* validate_yaw (pr:503-525): the heading at both ends lies inside the semi-FOV yaw_max; the velocity is the primitive's own
 * (for VELxYAW the control), a zero velocity passes */
MPLB_HD bool validate_yaw(const Cfg &c, const Shape &sh, const Prim &pr, double yaw0, double u_yaw) {
  if (sh.yaw_max <= 0) return true;
  for (int e = 0; e < 2; e++) {
    const double t = e ? c.dt : 0.0;
    const double vx = pr_v(pr.ax[0], t), vy = pr_v(pr.ax[1], t);
    if (vx != 0 || vy != 0) {
      double sn, cs;
      mplb::trig::sincos_cr(yaw_at(u_yaw, yaw0, t), &sn, &cs);
      if (heading_dot(vx, vy, cs, sn) < sh.cos_yaw_max) return false;
    }
  }
  return true;
}
/* em:90-132 with the shaping branches: outside -> +inf; with a potential map, pot >= 100 -> +inf and 0 < pot < 100 adds
 * dt_s (w_pot pot + w_grad |vel|), without one an occupied cell -> +inf; then, for a yaw session with wyaw > 0, the heading
 * term wyaw (1 - v_hat . (cos yaw, sin yaw)) dt_s of every sample with |v_xy| > 1e-5.  Terms are summed in sample order. */
MPLB_HD double traverse_shaped(const Cfg &c, const Shape &sh, const Prim &pr, double yaw0, double u_yaw, int *n_samples) {
  const double max_v = prim_max_v(c.dim, pr, c.dt);
  int n = (int)ceil(ddiv(dmul(max_v, c.dt), c.res));
  if (n < 5) n = 5;
  const double dts = ddiv(c.dt, (double)n);
  int tested = 0;
  double cost = 0;
  for (double t = 0; t < c.dt; t = dadd(t, dts)) {
    double st[13];
    int pn[3];
    prim_eval(c.dim, pr, t, st);
    float_to_int(c, st, pn);
    tested++;
    if (outside(c, pn)) { *n_samples += tested; return LPA_INF; }
    const int idx = cell_index(c, pn);
    if (sh.pot) { /* em:113-118 */
      const int p = (int)sh.pot[idx];
      if (p >= 100) { *n_samples += tested; return LPA_INF; }
      if (p > 0) {
        double vn = 0;
        if (sh.grad_w != 0) { /* vel.norm(): sqrt of the left-to-right sum of squares */
          double ss = dmul(st[3], st[3]);
          for (int k = 1; k < c.dim; k++) ss = dadd(ss, dmul(st[3 + k], st[3 + k]));
          vn = dsqrt(ss);
        }
        cost = dadd(cost, dmul(dts, dadd(dmul(sh.pot_w, (double)p), dmul(sh.grad_w, vn))));
      }
    } else if (c.grid[idx] == 100) { *n_samples += tested; return LPA_INF; } /* em:119-120 */
    if (sh.use_yaw && sh.wyaw > 0) { /* em:121-128 */
      const double vx = st[3], vy = st[4];
      if (dsqrt(dadd(dmul(vx, vx), dmul(vy, vy))) > 1e-5) {
        double sn, cs;
        mplb::trig::sincos_cr(yaw_at(u_yaw, yaw0, t), &sn, &cs);
        cost = dadd(cost, dmul(dmul(sh.wyaw, dsub(1.0, heading_dot(vx, vy, cs, sn))), dts));
      }
    }
  }
  *n_samples += tested;
  return cost;
}

/* One control of get_succ (em:147-172) for the node with coord (st, t, key): any lane.  SH: the potential map / yaw branches
 * of `sh`; the plain instantiation never reads it. */
template <bool SH = false>
MPLB_HDN void succ_row(const Cfg &c, const Shape &sh, const double *st, double t, const int *key, int u, Row *row) {
  Prim pr;
  prim_build(c.dim, c.ord, st, c.U + 3 * u, pr);
  prim_eval(c.dim, pr, c.dt, row->st);
  const bool yaw = SH && sh.use_yaw;
  const double u_yaw = yaw ? sh.Uyaw[u] : 0.0;
  if (yaw) row->st[12] = yaw_at(u_yaw, st[12], c.dt);
  make_key<SH>(c, row->st, row->key, yaw);
  row->verdict = 0;
  row->n_samples = 0;
  row->cost = 0;
  if (key_eq(row->key, key, c.nkey)) return;          /* em:158 tn == curr */
  if (yaw && !validate_yaw(c, sh, pr, st[12], u_yaw)) return; /* pr:462-465, then the base control's bounds */
  if (!validate_primitive(c.dim, c.ord, pr, c.dt, c.v_max, c.a_max, c.j_max)) return; /* em:159 */
  row->t = dadd(t, c.dt);                              /* em:161 */
  row->verdict = 1;
  bool same = true;
  for (int k = 0; k < c.dim; k++) same = same && (st[k] == row->st[k]);
  double cost;
  if (SH) cost = same ? 0 : traverse_shaped(c, sh, pr, st[12], u_yaw, &row->n_samples);
  else cost = same ? 0 : traverse(c, pr, &row->n_samples); /* em:163 */
  if (!fIsInf(cost)) cost = dadd(cost, dadd(prim_J(c.dim, pr, c.dt, c.control), dmul(c.w, c.dt))); /* em:164-165, eb:343-345 */
  row->cost = cost;
  row->hash = key_hash(row->key, c.nkey);
}
/* the plain-map row (no potential map, no yaw) */
MPLB_HDN void succ_row(const Cfg &c, const double *st, double t, const int *key, int u, Row *row) {
  succ_row<false>(c, Shape{}, st, t, key, u, row);
}

/* ------------------------------------------------------------------ node table (hm_ lookup by lattice key) */
MPLB_HD int table_find(const Ctx &x, const int *key, unsigned long long hash) {
  const int mask = x.h->tsize - 1;
  int s = (int)(hash & (unsigned long long)mask);
  while (true) {
    const int id = x.table[s];
    if (id < 0) return -1;
    if (key_eq(x.nodes[id].key, key, x.cfg.nkey)) return id;
    s = (s + 1) & mask;
  }
}
MPLB_HD void table_insert(const Ctx &x, int id) {
  const int mask = x.h->tsize - 1;
  int s = (int)(key_hash(x.nodes[id].key, x.cfg.nkey) & (unsigned long long)mask);
  while (x.table[s] >= 0) s = (s + 1) & mask;
  x.table[s] = id;
}
/* make_shared<State>(coord): a record (new or recycled in place) with the fresh State's defaults */
MPLB_HD void node_init(Node &n, const double *st, double t, const int *key) {
  for (int k = 0; k < 13; k++) n.st[k] = st[k];
  n.t = t;
  for (int k = 0; k < LPA_NKEY; k++) n.key[k] = key[k];
  n.g = LPA_INF; n.rhs = LPA_INF; n.h = LPA_INF;
  n.heap_pos = -1; n.n_succ = 0; n.pred_head = n.pred_tail = -1; n.n_pred = 0;
  n.opened = 0; n.closed = 0; n.in_hm = 0; n.pad = 0;
}
/* hm_[coord] for a successor / start coordinate: existing member, or a fresh State inserted at the end of the iteration order */
MPLB_HD int hm_get_or_create(const Ctx &x, const double *st, double t, const int *key, unsigned long long hash, const int *goal_key, bool *created) {
  Hdr &h = *x.h;
  int id = table_find(x, key, hash);
  *created = false;
  if (id >= 0 && x.nodes[id].in_hm) return id;
  if (id < 0) {
    id = h.n_nodes++;
    node_init(x.nodes[id], st, t, key);
    table_insert(x, id);
  } else node_init(x.nodes[id], st, t, key); /* dropped by an earlier getSubStateSpace: the reference builds a new State */
  x.nodes[id].in_hm = 1;
  x.order[h.n_order++] = id;
  (void)goal_key;
  *created = true;
  return id;
}

/* ------------------------------------------------------------------ pq_: d_ary_heap<arity 2, mutable> with compare_pair (ss:15-34) */
MPLB_HD bool heap_worse(const Ctx &x, const double *hf, const int *hn, int a, int b) { /* cmp(a, b): a has lower priority */
  if (hf[a] == hf[b]) {
    const Node &na = x.nodes[hn[a]], &nb = x.nodes[hn[b]];
    return dmin(na.g, na.rhs) > dmin(nb.g, nb.rhs);
  }
  return hf[a] > hf[b];
}
MPLB_HD void heap_swap(const Ctx &x, double *hf, int *hn, int a, int b, bool track) {
  const double f = hf[a]; hf[a] = hf[b]; hf[b] = f;
  const int n = hn[a]; hn[a] = hn[b]; hn[b] = n;
  if (track) { x.nodes[hn[a]].heap_pos = a; x.nodes[hn[b]].heap_pos = b; }
}
MPLB_HD void heap_sift_up(const Ctx &x, double *hf, int *hn, int pos, bool force, bool track) {
  while (pos != 0) {
    const int parent = (pos - 1) / 2;
    if (force || heap_worse(x, hf, hn, parent, pos)) { heap_swap(x, hf, hn, parent, pos, track); pos = parent; }
    else return;
  }
}
MPLB_HD void heap_sift_down(const Ctx &x, double *hf, int *hn, int n, int pos, bool track) {
  while (2 * pos + 1 < n) {
    int c = 2 * pos + 1;
    if (c + 1 < n && heap_worse(x, hf, hn, c, c + 1)) c = c + 1; /* std::max_element: the first of equally good children */
    if (!heap_worse(x, hf, hn, c, pos)) { heap_swap(x, hf, hn, pos, c, track); pos = c; }
    else return;
  }
}
MPLB_HD void pq_push(const Ctx &x, double f, int node) {
  Hdr &h = *x.h;
  const int pos = h.n_heap++;
  x.heap_f[pos] = f; x.heap_node[pos] = node;
  x.nodes[node].heap_pos = pos;
  heap_sift_up(x, x.heap_f, x.heap_node, pos, false, true);
}
MPLB_HD void pq_pop(const Ctx &x) {
  Hdr &h = *x.h;
  const int last = --h.n_heap;
  x.nodes[x.heap_node[0]].heap_pos = -1;
  if (last > 0) {
    x.heap_f[0] = x.heap_f[last]; x.heap_node[0] = x.heap_node[last];
    x.nodes[x.heap_node[0]].heap_pos = 0;
    heap_sift_down(x, x.heap_f, x.heap_node, last, 0, true);
  }
}
MPLB_HD void pq_erase(const Ctx &x, int node) { /* Boost: sift up unconditionally to the root, then pop */
  heap_sift_up(x, x.heap_f, x.heap_node, x.nodes[node].heap_pos, true, true);
  pq_pop(x);
}
MPLB_HD double calc_key(const Ctx &x, int id) { /* ss:270-272 */
  const Node &n = x.nodes[id];
  return dadd(dmin(n.g, n.rhs), dmul(x.h->eps, n.h));
}
MPLB_HD void update_node(const Ctx &x, int id) { /* ss:242-267 */
  Node &n = x.nodes[id];
  if (n.rhs != x.h->start_rhs) {
    n.rhs = LPA_INF;
    for (int p = n.pred_head; p >= 0; p = x.preds[p].next) {
      const double v = dadd(x.nodes[x.preds[p].node].g, x.preds[p].cost);
      if (n.rhs > v) n.rhs = v;
    }
  }
  if (n.opened && !n.closed) { pq_erase(x, id); n.closed = 1; }
  if (n.g != n.rhs) {
    pq_push(x, calc_key(x, id), id);
    n.opened = 1;
    n.closed = 0;
  }
}
MPLB_HD int pred_find(const Ctx &x, int node, int pred_node) { /* index of pred_node in node's list, or -1 */
  int i = 0;
  for (int p = x.nodes[node].pred_head; p >= 0; p = x.preds[p].next, i++)
    if (x.preds[p].node == pred_node) return i;
  return -1;
}
MPLB_HD void pred_append(const Ctx &x, int node, int pred_node, double cost, int act) {
  Hdr &h = *x.h;
  const int r = h.n_pred++;
  x.preds[r].cost = cost; x.preds[r].node = pred_node; x.preds[r].act = act; x.preds[r].next = -1; x.preds[r].pad = 0;
  Node &n = x.nodes[node];
  if (n.pred_tail >= 0) x.preds[n.pred_tail].next = r; else n.pred_head = r;
  n.pred_tail = r;
  n.n_pred++;
}
MPLB_HD int pred_at(const Ctx &x, int node, int idx) {
  int p = x.nodes[node].pred_head;
  for (int i = 0; i < idx && p >= 0; i++) p = x.preds[p].next;
  return p;
}

/* ------------------------------------------------------------------ LPAstar (gs:194-365), split around the parallel get_succ */
MPLB_HD void goal_values(const Ctx &x, double *g, double *rhs, double *key) {
  const Hdr &h = *x.h;
  if (h.goal_node < 0) { *g = LPA_INF; *rhs = LPA_INF; *key = dadd(LPA_INF, dmul(h.eps, 0.0)); }
  else { *g = x.nodes[h.goal_node].g; *rhs = x.nodes[h.goal_node].rhs; *key = calc_key(x, h.goal_node); }
}
/* Entry of a plan (lane 0): pre-checks, start node, goal node.  Returns a final status, or -1 to enter the loop. */
template <bool SH = false>
MPLB_HDN int plan_begin(const Ctx &x, const double *start_st, double start_t, const double *goal_st) {
  Hdr &h = *x.h;
  const Cfg &c = x.cfg;
  h.n_prims = 0; h.n_valid = 0; h.n_samples = 0; h.n_explored = 0; h.pop_hash = 0xCBF29CE484222325ull; h.expand_iteration = 0;
  h.has_rows = 0; h.curr = -1;
  int pn[3];
  float_to_int(c, start_st, pn);
  if (!cell_free(c, pn)) return LPA_START_NOT_FREE; /* pb:283-287 */
  if (!h.initialized) { /* pb:296-304: a new StateSpace(epsilon_) only at the first plan */
    h.initialized = 1; h.eps = c.eps; h.start_g = 0; h.start_rhs = 0; h.start_t = 0; h.n_best = 0;
  }
  for (int k = 0; k < 13; k++) h.goal[k] = goal_st[k]; /* pb:306 */
  if (is_goal(c, h.goal, start_st)) return LPA_START_IS_GOAL; /* gs:200-205 */
  int key[LPA_NKEY], gkey[LPA_NKEY];
  const bool yaw = SH && h.sh.use_yaw;
  make_key<SH>(c, start_st, key, yaw);
  make_key<SH>(c, h.goal, gkey, yaw);
  for (int k = 0; k < LPA_NKEY; k++) h.start_key[k] = key[k];
  bool created;
  const int s = hm_get_or_create(x, start_st, start_t, key, key_hash(key, c.nkey), gkey, &created); /* gs:208 */
  if (created) { /* gs:209-221 */
    Node &n = x.nodes[s];
    n.g = LPA_INF; n.rhs = 0;
    n.h = h.eps == 0 ? 0 : heur(c, h.goal, gkey, start_st, key);
    pq_push(x, calc_key(x, s), s);
    n.opened = 1; n.closed = 0;
  }
  h.start_node = s;
  if (h.n_best > 0 && is_goal(c, h.goal, x.nodes[x.best[h.n_best - 1]].st)) h.goal_node = x.best[h.n_best - 1]; /* gs:224-232 */
  else h.goal_node = -1;
  return -1;
}
/* Head of one iteration (lane 0).  Returns -1 when the popped node needs its successors generated (the lanes then fill
 * rows[] and pop_finish follows), -2 when the node's stored successor list is used (pop_finish follows directly), or a
 * final / internal status when the loop ends here. */
MPLB_HDN int pop_begin(const Ctx &x) {
  Hdr &h = *x.h;
  const Cfg &c = x.cfg;
  if (h.n_heap == 0) return LPA_QUEUE_EMPTY; /* the reference reads pq_.top() of an empty heap here (undefined) */
  double gg, grhs, gkey;
  goal_values(x, &gg, &grhs, &gkey);
  if (!(x.heap_f[0] < gkey || grhs != gg)) return LPA_OK; /* gs:244-245 */
  if (h.n_nodes + c.nU > h.cap_nodes || h.n_pred + c.nU > h.cap_pred || h.n_order + c.nU > h.cap_nodes) return LPA_NEED_GROW;
  h.expand_iteration++;
  const int curr = x.heap_node[0];
  pq_pop(x);
  Node &n = x.nodes[curr];
  n.closed = 1;
  if (n.g > n.rhs) n.g = n.rhs; /* gs:252-257 */
  else { n.g = LPA_INF; update_node(x, curr); }
  h.curr = curr;
  if (n.n_succ == 0) { /* gs:265-271: get_succ */
    h.has_rows = 1;
    h.n_explored++;
    h.pop_hash = (h.pop_hash ^ key_hash(n.key, c.nkey)) * 0x100000001B3ull;
    h.n_prims += c.nU;
    return -1;
  }
  h.has_rows = 0;
  return -2;
}
/* Tail of one iteration (lane 0): gs:287-336.  Returns -1 to continue, else the final status. */
template <bool SH = false>
MPLB_HDN int pop_finish(const Ctx &x) {
  Hdr &h = *x.h;
  const Cfg &c = x.cfg;
  const int curr = h.curr;
  const bool yaw = SH && h.sh.use_yaw;
  int gkey[LPA_NKEY];
  make_key<SH>(c, h.goal, gkey, yaw);
  Succ *sl = x.succ + (size_t)curr * c.nU;
  if (h.has_rows) { /* first expansion: the emitted rows, in control order, become the stored list */
    int ns = 0;
    for (int u = 0; u < c.nU; u++) {
      const Row &r = x.rows[u];
      h.n_samples += r.n_samples;
      if (!r.verdict) continue;
      if (!fIsInf(r.cost)) h.n_valid++;
      bool created;
      const int sid = hm_get_or_create(x, r.st, r.t, r.key, r.hash, gkey, &created);
      if (created) x.nodes[sid].h = h.eps == 0 ? 0 : heur(c, h.goal, gkey, r.st, r.key); /* gs:279-281 */
      sl[ns].node = sid; sl[ns].act = u; sl[ns].cost = r.cost;
      ns++;
      if (pred_find(x, sid, curr) < 0) pred_append(x, sid, curr, r.cost, u); /* gs:296-309 */
      update_node(x, sid);
    }
    x.nodes[curr].n_succ = ns;
  } else {
    const int ns = x.nodes[curr].n_succ;
    for (int s = 0; s < ns; s++) {
      int sid = sl[s].node;
      if (!x.nodes[sid].in_hm) { /* dropped since: hm_[succ_coord[s]] builds a new State from the stored coordinate */
        Prim pr;
        double st[13];
        int key[LPA_NKEY];
        prim_build(c.dim, c.ord, x.nodes[curr].st, c.U + 3 * sl[s].act, pr);
        prim_eval(c.dim, pr, c.dt, st);
        if (yaw) st[12] = yaw_at(h.sh.Uyaw[sl[s].act], x.nodes[curr].st[12], c.dt);
        make_key<SH>(c, st, key, yaw);
        bool created;
        sid = hm_get_or_create(x, st, dadd(x.nodes[curr].t, c.dt), key, key_hash(key, c.nkey), gkey, &created);
        x.nodes[sid].h = h.eps == 0 ? 0 : heur(c, h.goal, gkey, st, key);
        sl[s].node = sid;
      }
      if (pred_find(x, sid, curr) < 0) pred_append(x, sid, curr, sl[s].cost, sl[s].act);
      update_node(x, sid);
    }
  }
  if (is_goal(c, h.goal, x.nodes[curr].st)) h.goal_node = curr;                 /* gs:319 */
  if (c.max_num > 0 && h.expand_iteration >= c.max_num) return LPA_MAX_EXPAND;  /* gs:322-328 */
  if (h.n_heap == 0) return LPA_QUEUE_EMPTY;                                     /* gs:331-336 */
  return -1;
}
/* ------------------------------------------------------------------ the same tail, spread over the warp
 * pop_finish walks the successors one by one on lane 0.  Most of what it does per successor is independent of the other
 * successors of the same pop: the key-table probe, building a new State, the scan of the successor's predecessor list for the
 * popped node, the append, and the recomputation of rhs over that list (it reads g of predecessors, and g changes only at the head
 * of a pop).  Only three things are order-defining: the ids / iteration-order slots / pool records handed out to new objects,
 * and the priority-queue operations.  pop_finish_warp therefore runs chunks of 32 successors: the lanes probe and detect
 * siblings with equal keys (the later one must see the earlier one's node, exactly as `hm_[coord]` would), lane 0 hands out ids
 * and slots in control order, the lanes build nodes / append predecessor records / recompute rhs for the first occurrence of
 * each node, and lane 0 then applies rhs and the heap operations in control order (a repeated sibling takes the plain serial
 * updateNode).  Statement for statement this leaves every array as pop_finish leaves it; the host build (tests/cpp/lpa_emul.cpp)
 * runs the same source with the lane loops serialised and is compared with the checker.
 * Written once for both builds: LPA_LANES(l) is the lane loop (one iteration per thread on the device), LPA_SYNC a warp barrier. */
#ifdef __CUDA_ARCH__
#define LPA_LANES(l) for (int l = (int)threadIdx.x, l##_go = 1; l##_go; l##_go = 0)
#define LPA_SYNC() __syncwarp()
#define LPA_LANE0 (threadIdx.x == 0)
#else
#ifdef LPA_REVERSE_LANES /* test builds: the result must not depend on the order in which lanes run inside a phase */
#define LPA_LANES(l) for (int l = 31; l >= 0; l--)
#else
#define LPA_LANES(l) for (int l = 0; l < 32; l++)
#endif
#define LPA_SYNC() ((void)0)
#define LPA_LANE0 true
#endif

struct PopScratch { /* per-warp staging (shared memory on the device) */
  int sid[32], state[32], leader[32], item[32], opos[32], prec[32];
  unsigned char active[32], need_append[32], has_rhs[32];
  double new_rhs[32];
  int ret;
};

MPLB_HD void table_insert_shared(const Ctx &x, int id) { /* several lanes insert different ids at once */
#ifdef __CUDA_ARCH__
  const int mask = x.h->tsize - 1;
  int s = (int)(key_hash(x.nodes[id].key, x.cfg.nkey) & (unsigned long long)mask);
  while (atomicCAS(&x.table[s], -1, id) != -1) s = (s + 1) & mask;
#else
  table_insert(x, id);
#endif
}
MPLB_HD void update_node_heap(const Ctx &x, int id) { /* the queue half of updateNode (ss:256-266) */
  Node &n = x.nodes[id];
  if (n.opened && !n.closed) { pq_erase(x, id); n.closed = 1; }
  if (n.g != n.rhs) {
    pq_push(x, calc_key(x, id), id);
    n.opened = 1;
    n.closed = 0;
  }
}
/* Called by all lanes of the warp (device) / once (host).  Result in S->ret: -1 to continue, else the final status. */
template <bool SH = false>
MPLB_HDN void pop_finish_warp(const Ctx &x, PopScratch *S) {
  Hdr &h = *x.h;
  const Cfg &c = x.cfg;
  const int curr = h.curr;
  const bool fresh = h.has_rows != 0;
  Succ *sl = x.succ + (size_t)curr * c.nU;
  const int n_in = fresh ? c.nU : x.nodes[curr].n_succ; /* controls (fresh) or stored entries */
  const bool yaw = SH && h.sh.use_yaw;
  int gkey[LPA_NKEY];
  make_key<SH>(c, h.goal, gkey, yaw);
  int ns = 0; /* lane 0's running count of stored entries (fresh case) */
  for (int base = 0; base < n_in; base += 32) {
    /* ---- 1: probe.  state 0 = member of hm_, 1 = known key whose State was dropped, 2 = never seen */
    LPA_LANES(l) {
      const int i = base + l;
      S->active[l] = 0; S->need_append[l] = 0; S->has_rhs[l] = 0; S->leader[l] = l; S->sid[l] = -1; S->state[l] = 0;
      if (i < n_in) {
        if (fresh) {
          const Row &r = x.rows[i];
          if (r.verdict) {
            S->active[l] = 1;
            const int id = table_find(x, r.key, r.hash);
            S->sid[l] = id;
            S->state[l] = id < 0 ? 2 : (x.nodes[id].in_hm ? 0 : 1);
          }
        } else {
          S->active[l] = 1;
          const int id = sl[i].node;
          S->sid[l] = id;
          S->state[l] = x.nodes[id].in_hm ? 0 : 1;
          if (S->state[l] == 1) { /* hm_[succ_coord[s]] will build a new State from the stored coordinate: recompute it */
            Row &r = x.rows[l];
            Prim pr;
            prim_build(c.dim, c.ord, x.nodes[curr].st, c.U + 3 * sl[i].act, pr);
            prim_eval(c.dim, pr, c.dt, r.st);
            if (yaw) r.st[12] = yaw_at(h.sh.Uyaw[sl[i].act], x.nodes[curr].st[12], c.dt);
            make_key<SH>(c, r.st, r.key, yaw);
            r.t = dadd(x.nodes[curr].t, c.dt);
            r.hash = key_hash(r.key, c.nkey);
          }
        }
      }
    }
    LPA_SYNC();
    /* ---- 2: the first sibling of this chunk with the same key (ids for stored entries) */
    LPA_LANES(l) {
      if (S->active[l]) {
        for (int k = 0; k < l; k++) {
          if (!S->active[k]) continue;
          bool same;
          if (fresh) same = x.rows[base + k].hash == x.rows[base + l].hash && key_eq(x.rows[base + k].key, x.rows[base + l].key, c.nkey);
          else same = S->sid[k] == S->sid[l];
          if (same) { S->leader[l] = k; break; }
        }
      }
    }
    LPA_SYNC();
    /* ---- 3: lane 0 hands out node ids, iteration-order slots and list positions in control order */
    if (LPA_LANE0) {
      for (int l = 0; l < 32; l++) {
        const int i = base + l;
        if (fresh && i < n_in) h.n_samples += x.rows[i].n_samples;
        if (!S->active[l]) continue;
        if (fresh) { if (!fIsInf(x.rows[i].cost)) h.n_valid++; S->item[l] = ns++; }
        if (S->leader[l] != l) continue;
        if (S->state[l] == 2) S->sid[l] = h.n_nodes++;
        if (S->state[l] != 0) S->opos[l] = h.n_order++;
      }
    }
    LPA_SYNC();
    /* ---- 4: the lanes build the new States */
    LPA_LANES(l) {
      if (S->active[l] && S->leader[l] == l && S->state[l] != 0) {
        const Row &r = fresh ? x.rows[base + l] : x.rows[l];
        Node &n = x.nodes[S->sid[l]];
        node_init(n, r.st, r.t, r.key);
        n.in_hm = 1;
        n.h = h.eps == 0 ? 0 : heur(c, h.goal, gkey, r.st, r.key); /* gs:279-281 */
        x.order[S->opos[l]] = S->sid[l];
        if (S->state[l] == 2) table_insert_shared(x, S->sid[l]);
      }
    }
    LPA_SYNC();
    /* ---- 5: stored list entry, and does the successor already list the popped node as a predecessor? (gs:296-303) */
    LPA_LANES(l) {
      if (S->active[l]) {
        if (S->leader[l] != l) S->sid[l] = S->sid[S->leader[l]];
        const int i = base + l;
        if (fresh) { Succ &e = sl[S->item[l]]; e.node = S->sid[l]; e.act = i; e.cost = x.rows[i].cost; }
        if (S->leader[l] == l) S->need_append[l] = pred_find(x, S->sid[l], curr) < 0;
      }
    }
    LPA_SYNC();
    if (LPA_LANE0)
      for (int l = 0; l < 32; l++)
        if (S->active[l] && S->need_append[l]) S->prec[l] = h.n_pred++;
    LPA_SYNC();
    /* ---- 6: append (one lane per node, so the lists never collide), then rhs over the node's own list (ss:245-253) */
    LPA_LANES(l) {
      if (S->active[l] && S->leader[l] == l) {
        const int sid = S->sid[l];
        Node &n = x.nodes[sid];
        if (S->need_append[l]) {
          const int i = base + l;
          const int r = S->prec[l];
          x.preds[r].cost = fresh ? x.rows[i].cost : sl[i].cost;
          x.preds[r].node = curr;
          x.preds[r].act = fresh ? i : sl[i].act;
          x.preds[r].next = -1; x.preds[r].pad = 0;
          if (n.pred_tail >= 0) x.preds[n.pred_tail].next = r; else n.pred_head = r;
          n.pred_tail = r;
          n.n_pred++;
        }
        if (n.rhs != h.start_rhs) {
          double v = LPA_INF;
          for (int p = n.pred_head; p >= 0; p = x.preds[p].next) {
            const double w = dadd(x.nodes[x.preds[p].node].g, x.preds[p].cost);
            if (v > w) v = w;
          }
          S->new_rhs[l] = v;
          S->has_rhs[l] = 1;
        }
      }
    }
    LPA_SYNC();
    /* ---- 7: lane 0 commits rhs and runs the queue operations in control order */
    if (LPA_LANE0) {
      for (int l = 0; l < 32; l++) {
        if (!S->active[l]) continue;
        const int sid = S->sid[l];
        if (S->leader[l] == l) {
          if (S->has_rhs[l]) x.nodes[sid].rhs = S->new_rhs[l];
          update_node_heap(x, sid);
        } else {
          update_node(x, sid); /* a repeated sibling: the plain serial statement */
        }
      }
    }
    LPA_SYNC();
  }
  if (LPA_LANE0) {
    if (fresh) x.nodes[curr].n_succ = ns;
    int ret = -1;
    if (is_goal(c, h.goal, x.nodes[curr].st)) h.goal_node = curr;            /* gs:319 */
    if (c.max_num > 0 && h.expand_iteration >= c.max_num) ret = LPA_MAX_EXPAND; /* gs:322-328 */
    else if (h.n_heap == 0) ret = LPA_QUEUE_EMPTY;                              /* gs:331-336 */
    S->ret = ret;
  }
  LPA_SYNC();
}

/* recoverTraj (gs:369-455); returns LPA_OK or LPA_TRACEBACK_FAILED; cost = goal g - start_g_ (gs:362) */
MPLB_HDN int recover(const Ctx &x, int *n_seg, double *cost) {
  Hdr &h = *x.h;
  const Cfg &c = x.cfg;
  h.n_best = 0;
  *n_seg = 0;
  *cost = LPA_INF;
  if (h.goal_node < 0) return LPA_TRACEBACK_FAILED; /* the detached goal State has no predecessors */
  int cur = h.goal_node, na = 0;
  bool found = false, cycle = false;
  while (x.nodes[cur].pred_head >= 0) {
    if (h.n_best > h.n_order) { cycle = true; break; } /* more steps than hm_ has members: a cycle of best predecessors.  The
                                                          reference's loop (gs:377-438) would never return; the trace-back fails
                                                          and best_child_ is left empty */
    x.best[h.n_best++] = cur;
    int min_p = -1;
    double min_rhs = LPA_INF, min_g = LPA_INF;
    for (int p = x.nodes[cur].pred_head; p >= 0; p = x.preds[p].next) {
      const double pg = x.nodes[x.preds[p].node].g;
      const double v = dadd(pg, x.preds[p].cost);
      if (min_rhs > v) { min_rhs = v; min_g = pg; min_p = p; }
      else if (!fIsInf(x.preds[p].cost) && min_rhs == v) {
        if (min_g < pg) { min_g = pg; min_p = p; }
      }
    }
    if (min_p < 0) break;
    x.traj_act[na++] = x.preds[min_p].act;
    cur = x.preds[min_p].node;
    if (key_eq(x.nodes[cur].key, h.start_key, c.nkey)) { x.best[h.n_best++] = cur; found = true; break; }
  }
  if (cycle) { h.n_best = 0; h.fault |= 2; return LPA_TRACEBACK_FAILED; }
  for (int i = 0; i < h.n_best / 2; i++) { const int t = x.best[i]; x.best[i] = x.best[h.n_best - 1 - i]; x.best[h.n_best - 1 - i] = t; }
  if (!found) return LPA_TRACEBACK_FAILED;
  for (int i = 0; i < na / 2; i++) { const int t = x.traj_act[i]; x.traj_act[i] = x.traj_act[na - 1 - i]; x.traj_act[na - 1 - i] = t; }
  *n_seg = na;
  *cost = dsub(x.nodes[h.goal_node].g, h.start_g);
  return LPA_OK;
}

/* ------------------------------------------------------------------ getSubStateSpace (ss:116-204), lane 0 */
MPLB_HD void epq_push(const Ctx &x, double f, int node) {
  Hdr &h = *x.h;
  const int pos = h.n_epq++;
  x.epq_f[pos] = f; x.epq_node[pos] = node;
  heap_sift_up(x, x.epq_f, x.epq_node, pos, false, false);
}
MPLB_HD int epq_pop(const Ctx &x) {
  Hdr &h = *x.h;
  const int top = x.epq_node[0];
  const int last = --h.n_epq;
  if (last > 0) {
    x.epq_f[0] = x.epq_f[last]; x.epq_node[0] = x.epq_node[last];
    heap_sift_down(x, x.epq_f, x.epq_node, last, 0, false);
  }
  return top;
}
MPLB_HDN int sub_state_space(const Ctx &x, int time_step) {
  Hdr &h = *x.h;
  const Cfg &c = x.cfg;
  if (h.n_best == 0 || time_step < 0 || time_step >= h.n_best) return LPA_OK;
  int curr = x.best[time_step];
  h.start_g = x.nodes[curr].g; h.start_rhs = x.nodes[curr].rhs; h.start_t = x.nodes[curr].t;
  for (int i = 0; i < h.n_order; i++) { /* ss:126-136: every member of hm_ (the root included) */
    Node &n = x.nodes[x.order[i]];
    n.g = LPA_INF; n.rhs = LPA_INF;
    n.pred_head = n.pred_tail = -1; n.n_pred = 0;
    x.mark[x.order[i]] = 0;
  }
  h.n_pred = 0; /* every live list is empty now: the record pool restarts */
  x.nodes[curr].g = h.start_g; x.nodes[curr].rhs = h.start_rhs;
  int n_new = 0;
  h.n_epq = 0;
  epq_push(x, x.nodes[curr].rhs, curr);
  x.mark[curr] = 1; x.order2[n_new++] = curr;
  int fault = 0;
  while (h.n_epq > 0) {
    curr = epq_pop(x);
    const Succ *sl = x.succ + (size_t)curr * c.nU;
    const int ns = x.nodes[curr].n_succ;
    for (int i = 0; i < ns; i++) {
      const int sid = sl[i].node;
      if (!x.nodes[sid].in_hm) { fault = 1; continue; } /* "critical bug!!!!" (ss:160-163): the reference dereferences a null State */
      if (!x.mark[sid]) { x.mark[sid] = 1; x.order2[n_new++] = sid; }
      if (pred_find(x, sid, curr) < 0) pred_append(x, sid, curr, sl[i].cost, sl[i].act);
      const double tentative = dadd(x.nodes[curr].rhs, sl[i].cost);
      if (tentative < x.nodes[sid].rhs) {
        x.nodes[sid].rhs = tentative;
        if (x.nodes[sid].closed) {
          x.nodes[sid].g = x.nodes[sid].rhs;
          epq_push(x, x.nodes[sid].rhs, sid);
        }
      }
    }
  }
  for (int i = 0; i < h.n_order; i++) { /* hm_ = new_hm */
    const int id = x.order[i];
    if (!x.mark[id]) { x.nodes[id].in_hm = 0; x.nodes[id].heap_pos = -1; }
  }
  for (int i = 0; i < n_new; i++) x.order[i] = x.order2[i];
  h.n_order = n_new;
  h.n_heap = 0; /* pq_.clear(), then the open members in iteration order (ss:190-199) */
  for (int i = 0; i < n_new; i++) x.nodes[x.order[i]].heap_pos = -1;
  for (int i = 0; i < n_new; i++) {
    const int id = x.order[i];
    if (x.nodes[id].opened && !x.nodes[id].closed) pq_push(x, calc_key(x, id), id);
  }
  if (fault) h.fault = 1;
  return fault ? LPA_FAULT : LPA_OK;
}

/* ------------------------------------------------------------------ getLinkedNodes (map_planner.cpp:125-158)
 * One call per position of the iteration order (any thread): the links of that node's predecessor edges, in (pred index,
 * sample) order.  out == nullptr counts, otherwise fills starting at out[0]; returns the count. */
MPLB_HDN int link_node(const Ctx &x, int order_pos, Link *out) {
  const Cfg &c = x.cfg;
  const int nid = x.order[order_pos];
  int cnt = 0, i = 0;
  for (int p = x.nodes[nid].pred_head; p >= 0; p = x.preds[p].next, i++) {
    Prim pr;
    prim_build(c.dim, c.ord, x.nodes[x.preds[p].node].st, c.U + 3 * x.preds[p].act, pr);
    const double max_v = prim_max_v(c.dim, pr, c.dt); /* std::max over the axes */
    const int n = (int)(1.0 * ceil(ddiv(dmul(max_v, c.dt), c.res)));
    const double dts = ddiv(c.dt, (double)n);
    int prev_id = -1;
    for (int s = 0; s <= n; s++) {
      double st[13];
      int pn[3];
      prim_eval(c.dim, pr, dmul((double)s, dts), st);
      float_to_int(c, st, pn);
      const int id = cell_index(c, pn);
      if (id != prev_id) {
        if (out) { Link &l = out[cnt]; l.vox = id; l.node = nid; l.pred_idx = i; l.cell[0] = pn[0]; l.cell[1] = pn[1]; l.cell[2] = pn[2]; }
        cnt++;
        prev_id = id;
      }
    }
  }
  return cnt;
}

/* ------------------------------------------------------------------ increaseCost / decreaseCost (ss:207-240) for one affected
 * (node, pred index) pair, lane 0, in the order updateBlockedNodes / updateClearedNodes produce (map_planner.cpp:160-185) */
MPLB_HDN void apply_change(const Ctx &x, int node, int pred_idx, bool blocked) {
  const Cfg &c = x.cfg;
  const int p = pred_at(x, node, pred_idx);
  if (p < 0) return;
  Pred &pr_ = x.preds[p];
  double new_cost;
  if (blocked) {
    if (fIsInf(pr_.cost)) return;
    new_cost = LPA_INF;
  } else {
    if (!fIsInf(pr_.cost)) return;
    Prim pr;
    prim_build(c.dim, c.ord, x.nodes[pr_.node].st, c.U + 3 * pr_.act, pr);
    if (!prim_is_free(c, pr)) return;
    new_cost = dadd(prim_J(c.dim, pr, c.dt, c.control), dmul(c.w, c.dt)); /* eb:343-345 */
  }
  pr_.cost = new_cost;
  update_node(x, node);
  Succ *sl = x.succ + (size_t)pr_.node * c.nU;
  const int ns = x.nodes[pr_.node].n_succ;
  for (int j = 0; j < ns; j++)
    if (sl[j].act == pr_.act) { sl[j].cost = new_cost; break; }
}

}  // namespace mplb_lpa
#endif
