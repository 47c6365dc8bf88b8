/*
 * lpa_emul.cpp — HOST BUILD OF THE DEVICE LPA* CORE, for tests only (never loaded by the product).
 *
 * mpl_ros_b200/csrc/mplb_lpa_core.h is written so that every statement the GPU executes for LPA* also compiles for the host.
 * This driver replays the orchestration of mpl_ros_b200/csrc/mplb_lpa.cu with host arrays and the kernels' lane / thread loops
 * unrolled serially (32 "lanes" generate the successor rows, "lane 0" does the graph update, one "thread" per node or per link
 * for the link table and the voxel matching, growth of the arrays between a stopped and a resumed plan), so that the CPU test
 * suite can compare the core with the checker (oracle) where no GPU exists.  g++ -O2 -ffp-contract=off.  The product has no
 * CPU path: libmplb.so does not contain this file.
 * Overruns: every array is allocated with GUARD spare elements beyond its capacity, and after every call into the core the
 * counters are checked against the capacities the core was given (n_nodes, n_order, n_heap <= cap_nodes, n_pred <= cap_pred,
 * n_links <= cap_links).  A write past a capacity therefore lands in owned memory and is reported (emu_overrun) instead of
 * being hidden by a vector's spare room or corrupting the heap.
 */
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../mpl_ros_b200/csrc/mplb_lpa_core.h"
#include "../../oracle/mpl_oracle.h"

using namespace mplb_lpa;

namespace {
constexpr int GUARD = LPA_MAXU + 1; /* spare elements behind every capacity: more than one pop or one plan entry can overrun */
struct EmuMap {
  int dim;
  int nd[3];
  double origin[3], res;
  std::vector<int8_t> data;
};
struct Emu {
  int dim = 3;
  EmuMap *map = nullptr;
  double v_max = -1, a_max = -1, j_max = -1, dt = 1, w = 10, eps = 1, tol_pos = 0.5, tol_vel = -1, tol_acc = -1;
  int max_num = -1;
  std::vector<double> U;
  int nU = 0;
  int control = 0;
  int init_cap = 1 << 16, init_pred = 1 << 20;
  int grows = 0;
  int serial_finish = 0;
  int no_start_room = 0; /* test switch: skip the host's room-for-the-start-node growth (shows what the invariant check catches) */
  std::string overrun;   /* first capacity violation seen, empty if none */
  /* "device" arrays */
  Hdr hdr{};
  std::vector<Node> nodes; std::vector<Succ> succ; std::vector<Pred> preds; std::vector<int> table, order, order2, heap_node, best, traj_act, epq_node, link_count;
  std::vector<double> heap_f, epq_f; std::vector<Row> rows; std::vector<unsigned char> mark; std::vector<Link> links; std::vector<unsigned long long> match;
  int cap_nodes = 0, cap_pred = 0, tsize = 0;
  bool have_links = false;
  orc_result last{};
  std::vector<int> last_actions;
  Ctx ctx() {
    Ctx x{};
    Cfg &c = x.cfg;
    const int cc = control & 15;
    c.dim = dim; c.ord = cc == 1 ? 1 : cc == 3 ? 2 : cc == 7 ? 3 : 4; c.control = control; c.nU = nU; c.nkey = dim * c.ord; c.max_num = max_num;
    c.dt = dt; c.w = w; c.eps = eps; c.v_max = v_max; c.a_max = a_max; c.j_max = j_max; c.tol_pos = tol_pos; c.tol_vel = tol_vel; c.tol_acc = tol_acc;
    for (int i = 0; i < 3; i++) { c.nd[i] = map->nd[i]; c.origin[i] = map->origin[i]; }
    c.res = map->res; c.grid = map->data.data(); c.U = U.data();
    x.h = &hdr; x.nodes = nodes.data(); x.succ = succ.data(); x.preds = preds.data(); x.table = table.data(); x.order = order.data();
    x.order2 = order2.data(); x.heap_f = heap_f.data(); x.heap_node = heap_node.data(); x.best = best.data(); x.traj_act = traj_act.data();
    x.rows = rows.data(); x.epq_f = epq_f.data(); x.epq_node = epq_node.data(); x.mark = mark.data(); x.links = links.data();
    x.link_count = link_count.data(); x.match = match.data();
    return x;
  }
  void check(const char *where) { /* the capacities the core was given hold after every call into it */
    const Hdr &h = hdr;
    if (!overrun.empty()) return;
    if (h.n_nodes > cap_nodes || h.n_order > cap_nodes || h.n_heap > cap_nodes || h.n_pred > cap_pred || h.n_links > h.cap_links) {
      char b[256];
      std::snprintf(b, sizeof(b), "%s: n_nodes %d n_order %d n_heap %d (cap_nodes %d), n_pred %d (cap_pred %d), n_links %d (cap_links %d)",
                    where, h.n_nodes, h.n_order, h.n_heap, cap_nodes, h.n_pred, cap_pred, h.n_links, h.cap_links);
      overrun = b;
    }
  }
  void ensure(int cap, int cpred) { /* ensure_capacity of mplb_lpa.cu */
    if (cap > cap_nodes) {
      const size_t c = (size_t)cap + GUARD;
      nodes.resize(c); succ.resize(c * nU); order.resize(c); order2.resize(c); heap_f.resize(c); heap_node.resize(c);
      best.resize(c); traj_act.resize(c); mark.resize(c); link_count.resize(c);
      cap_nodes = cap;
      int ts = 1024;
      while (ts < 2 * cap) ts <<= 1;
      tsize = std::max(tsize, ts);
      table.assign(tsize, -1);
      hdr.cap_nodes = cap_nodes; hdr.tsize = tsize;
      Ctx x = ctx();
      for (int i = 0; i < hdr.n_nodes; i++) table_insert(x, i); /* k_lpa_rehash */
    }
    if (cpred > cap_pred) { preds.resize((size_t)cpred + GUARD); cap_pred = cpred; }
    rows.resize(std::max(nU, 32));
    hdr.cap_nodes = cap_nodes; hdr.cap_pred = cap_pred; hdr.tsize = tsize;
  }
  void reset() {
    nodes.clear(); succ.clear(); preds.clear(); table.clear(); order.clear(); order2.clear(); heap_node.clear(); best.clear(); traj_act.clear();
    heap_f.clear(); mark.clear(); link_count.clear(); links.clear(); match.clear();
    cap_nodes = cap_pred = tsize = 0; have_links = false; control = 0; grows = 0;
    std::memset(&hdr, 0, sizeof(hdr));
  }
};
void wp_state(const orc_waypoint &w, double *st) {
  for (int k = 0; k < 3; k++) { st[k] = w.pos[k]; st[3 + k] = w.vel[k]; st[6 + k] = w.acc[k]; st[9 + k] = w.jrk[k]; }
  st[12] = w.yaw;
}
}  // namespace

extern "C" {
void *emu_map_create(int dim, const int32_t *nd, const double *origin, double res, const int8_t *data) {
  EmuMap *m = new EmuMap();
  m->dim = dim; m->res = res;
  size_t n = 1;
  for (int i = 0; i < 3; i++) { m->nd[i] = i < dim ? nd[i] : 1; m->origin[i] = i < dim ? origin[i] : 0; n *= (size_t)m->nd[i]; }
  m->data.assign(data, data + n);
  return m;
}
void emu_map_destroy(void *m) { delete (EmuMap *)m; }
void emu_map_free_unknown(void *m) { for (auto &v : ((EmuMap *)m)->data) if (v == -1) v = 0; }
void emu_map_set_cells(void *mm, const int32_t *c3, int n, int8_t value) { /* k_set_cells */
  EmuMap *m = (EmuMap *)mm;
  for (int i = 0; i < n; i++) {
    const int x = c3[i * 3], y = c3[i * 3 + 1], z = m->dim == 3 ? c3[i * 3 + 2] : 0;
    if (x < 0 || x >= m->nd[0] || y < 0 || y >= m->nd[1] || z < 0 || z >= m->nd[2]) continue;
    m->data[(size_t)x + (size_t)m->nd[0] * y + (size_t)m->nd[0] * m->nd[1] * z] = value;
  }
}
void *emu_planner_create(int dim) { Emu *e = new Emu(); e->dim = dim; return e; }
void emu_planner_destroy(void *p) { delete (Emu *)p; }
void emu_planner_set_map(void *p, void *m) { ((Emu *)p)->map = (EmuMap *)m; }
int emu_planner_set_param(void *pp, const char *key, double v) {
  Emu *p = (Emu *)pp;
  const std::string k(key);
  if (k == "v_max") p->v_max = v; else if (k == "a_max") p->a_max = v; else if (k == "j_max") p->j_max = v; else if (k == "dt") p->dt = v;
  else if (k == "w") p->w = v; else if (k == "epsilon") p->eps = v; else if (k == "max_num") p->max_num = (int)v; else if (k == "tol_pos") p->tol_pos = v;
  else if (k == "tol_vel") p->tol_vel = v; else if (k == "tol_acc") p->tol_acc = v; else if (k == "init_cap" || k == "lpa_init_nodes") p->init_cap = (int)v;
  else if (k == "init_pred" || k == "lpa_init_preds") p->init_pred = (int)v; else if (k == "serial_finish") p->serial_finish = (int)v;
  else if (k == "no_start_room") p->no_start_room = (int)v; else return -1;
  return 0;
}
void emu_planner_set_controls(void *pp, const double *U, int n, int udim) {
  Emu *p = (Emu *)pp;
  p->U.assign((size_t)n * 3, 0.0);
  for (int i = 0; i < n; i++) for (int k = 0; k < udim && k < 3; k++) p->U[(size_t)i * 3 + k] = U[(size_t)i * udim + k];
  p->nU = n;
}
int emu_grows(void *pp) { return ((Emu *)pp)->grows; }
const char *emu_overrun(void *pp) { return ((Emu *)pp)->overrun.c_str(); }
void emu_capacity(void *pp, int32_t *out5) { /* mplb_lpa_get_capacity */
  Emu *p = (Emu *)pp;
  out5[0] = p->cap_nodes; out5[1] = p->cap_pred; out5[2] = p->tsize; out5[3] = p->hdr.n_nodes; out5[4] = p->grows;
}
void emu_lpa_reset(void *pp) { ((Emu *)pp)->reset(); }

int emu_lpa_plan(void *pp, const orc_waypoint *start, const orc_waypoint *goal, orc_result *out) {
  Emu *p = (Emu *)pp;
  p->control = start->control;
  if (p->cap_nodes == 0) p->ensure(p->init_cap, p->init_pred);
  if (!p->no_start_room && p->hdr.n_nodes + 1 > p->cap_nodes) { p->grows++; p->ensure(p->cap_nodes * 2, p->cap_pred * 2); } /* room for the start node */
  p->hdr.resume = 0; p->hdr.status = 0;
  int code;
  while (true) { /* one iteration = one launch of k_lpa_plan */
    Ctx x = p->ctx();
    code = -1;
    if (!x.h->resume) {
      double sst[13], gst[13];
      wp_state(*start, sst); wp_state(*goal, gst);
      code = plan_begin(x, sst, start->t, gst);
      p->check("plan_begin");
    }
    while (code == -1) {
      const int r = pop_begin(x);
      p->check("pop_begin");
      if (r == -1) {
        const Node &n = x.nodes[x.h->curr];
        for (int lane = 0; lane < 32; lane++) for (int u = lane; u < x.cfg.nU; u += 32) succ_row(x.cfg, n.st, n.t, n.key, u, &x.rows[u]);
      }
      if (r == -1 || r == -2) {
        if (p->serial_finish) code = pop_finish(x);                      /* the one-lane tail */
        else { PopScratch S; pop_finish_warp(x, &S); code = S.ret; }     /* the warp-wide tail, lane loops serialised */
        p->check("pop_finish");
      } else code = r;
    }
    if (code == LPA_NEED_GROW) { p->hdr.resume = 1; p->grows++; p->ensure(p->cap_nodes * 2, p->cap_pred * 2); continue; }
    break;
  }
  Ctx x = p->ctx();
  Hdr &h = p->hdr;
  h.resume = 0;
  int n_seg = 0;
  double cost = LPA_INF;
  if (code == LPA_OK) code = recover(x, &n_seg, &cost); else if (code == LPA_START_IS_GOAL) cost = 0;
  p->check("recover");
  h.status = code;
  orc_result r;
  std::memset(&r, 0, sizeof(r));
  const bool have_state = h.initialized && code != LPA_START_NOT_FREE && code != LPA_START_IS_GOAL;
  r.status = code; r.n_seg = n_seg; r.cost = cost; r.pops = h.expand_iteration;
  if (have_state) {
    r.n_nodes = h.n_order; r.n_open = h.n_heap;
    for (int i = 0; i < h.n_order; i++) { const Node &n = x.nodes[x.order[i]]; if (n.closed) { r.n_closed++; r.closed_hash += key_hash(n.key, x.cfg.nkey); } }
    r.pop_hash = h.pop_hash;
  }
  r.n_prims = h.n_prims; r.n_samples = h.n_samples; r.n_valid = h.n_valid;
  p->last = r;
  p->last_actions.assign(x.traj_act, x.traj_act + n_seg);
  if (out) *out = r;
  return code;
}
int emu_lpa_get_sub_state_space(void *pp, int k) {
  Emu *p = (Emu *)pp;
  if (p->hdr.n_best == 0) return 0;
  const size_t edges = (size_t)p->hdr.n_nodes * p->nU + 16;
  p->epq_f.resize(edges); p->epq_node.resize(edges);
  if (edges + p->nU > (size_t)p->cap_pred) p->ensure(p->cap_nodes, (int)(edges + p->nU));
  Ctx x = p->ctx();
  const int st = sub_state_space(x, k);
  p->check("sub_state_space");
  return st == LPA_FAULT ? -1 : p->hdr.n_order;
}
int emu_lpa_get_linked_nodes(void *pp, double *pts3, int cap) {
  Emu *p = (Emu *)pp;
  Ctx x = p->ctx();
  p->have_links = true;
  for (int i = 0; i < p->hdr.n_order; i++) x.link_count[i] = link_node(x, i, nullptr); /* k_lpa_link_count */
  int run = 0;
  for (int i = 0; i < p->hdr.n_order; i++) { const int c = x.link_count[i]; x.link_count[i] = run; run += c; } /* k_lpa_link_scan */
  p->hdr.n_links = run;
  p->links.resize((size_t)run + GUARD);
  p->hdr.cap_links = run;
  x = p->ctx();
  for (int i = p->hdr.n_order - 1; i >= 0; i--) link_node(x, i, x.links + x.link_count[i]); /* k_lpa_link_fill, any thread order */
  p->check("link_node");
  for (int i = 0; i < run && i < cap; i++)
    for (int k = 0; k < 3; k++) pts3[(size_t)i * 3 + k] = k < p->dim ? ((double)p->links[i].cell[k] + 0.5) * x.cfg.res + x.cfg.origin[k] : 0.0;
  return run;
}
static int emu_update(Emu *p, const int32_t *c3, int n, bool blocked) {
  if (!p->have_links || n == 0 || p->hdr.n_links == 0) return 0;
  Ctx x = p->ctx();
  std::vector<unsigned long long> m;
  for (int l = p->hdr.n_links - 1; l >= 0; l--) /* k_lpa_match, any thread order */
    for (int b = 0; b < n; b++) {
      const int pn[3] = {c3[b * 3], c3[b * 3 + 1], c3[b * 3 + 2]};
      if (cell_index(x.cfg, pn) == p->links[l].vox) m.push_back((unsigned long long)b * (unsigned long long)p->hdr.n_links + (unsigned long long)l);
    }
  std::sort(m.begin(), m.end()); /* k_lpa_apply */
  for (unsigned long long key : m) { const Link &l = p->links[(int)(key % (unsigned long long)p->hdr.n_links)]; apply_change(x, l.node, l.pred_idx, blocked); }
  p->check(blocked ? "apply_change (blocked)" : "apply_change (cleared)");
  return (int)m.size();
}
int emu_lpa_update_blocked_nodes(void *pp, const int32_t *c3, int n) { return emu_update((Emu *)pp, c3, n, true); }
int emu_lpa_update_cleared_nodes(void *pp, const int32_t *c3, int n) { return emu_update((Emu *)pp, c3, n, false); }
static uint64_t mix(uint64_t h, uint64_t v) { return (h ^ v) * 0x100000001B3ull; }
int emu_lpa_dump_nodes(void *pp, orc_lpa_node *out, int cap) {
  Emu *p = (Emu *)pp;
  Ctx x = p->ctx();
  const int nk = x.cfg.nkey;
  for (int i = 0; i < p->hdr.n_order && i < cap; i++) {
    const int id = x.order[i];
    const Node &n = x.nodes[id];
    orc_lpa_node &o = out[i];
    std::memset(&o, 0, sizeof(o));
    for (int k = 0; k < nk; k++) o.key[k] = n.key[k];
    o.key[15] = nk;
    o.g = n.g; o.rhs = n.rhs; o.h = n.h; o.opened = n.opened; o.closed = n.closed; o.n_succ = n.n_succ; o.n_pred = n.n_pred;
    uint64_t hs = 0xCBF29CE484222325ull, hp = hs;
    for (int k = 0; k < n.n_succ; k++) { const Succ &e = x.succ[(size_t)id * p->nU + k]; uint64_t cb; std::memcpy(&cb, &e.cost, 8); hs = mix(mix(mix(hs, key_hash(x.nodes[e.node].key, nk)), (uint64_t)e.act), cb); }
    for (int q = n.pred_head; q >= 0; q = x.preds[q].next) { uint64_t cb; std::memcpy(&cb, &x.preds[q].cost, 8); hp = mix(mix(mix(hp, key_hash(x.nodes[x.preds[q].node].key, nk)), (uint64_t)x.preds[q].act), cb); }
    o.succ_hash = hs; o.pred_hash = hp;
  }
  return p->hdr.n_order;
}
int emu_lpa_dump_heap(void *pp, orc_lpa_heap_entry *out, int cap) {
  Emu *p = (Emu *)pp;
  Ctx x = p->ctx();
  for (int i = 0; i < p->hdr.n_heap && i < cap; i++) { out[i].fval = x.heap_f[i]; out[i].key_hash = key_hash(x.nodes[x.heap_node[i]].key, x.cfg.nkey); }
  return p->hdr.n_heap;
}
int emu_lpa_best_child(void *pp, int32_t *keys16, int cap) {
  Emu *p = (Emu *)pp;
  Ctx x = p->ctx();
  for (int i = 0; i < p->hdr.n_best && i < cap; i++) { int32_t *k = keys16 + (size_t)i * 16; std::memset(k, 0, 64); for (int j = 0; j < x.cfg.nkey; j++) k[j] = x.nodes[x.best[i]].key[j]; k[15] = x.cfg.nkey; }
  return p->hdr.n_best;
}
int emu_lpa_best_child_states(void *pp, double *s13, int cap) {
  Emu *p = (Emu *)pp;
  Ctx x = p->ctx();
  for (int i = 0; i < p->hdr.n_best && i < cap; i++) std::memcpy(s13 + (size_t)i * 13, x.nodes[x.best[i]].st, 13 * sizeof(double));
  return p->hdr.n_best;
}
int emu_lpa_get_actions(void *pp, int32_t *a, int cap) {
  Emu *p = (Emu *)pp;
  for (int i = 0; i < (int)p->last_actions.size() && i < cap; i++) a[i] = p->last_actions[i];
  return (int)p->last_actions.size();
}
}
