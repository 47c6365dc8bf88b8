/*
 * mpl_oracle.h — C interface of the CPU ORACLE (test infrastructure, NOT product code).
 *
 * The oracle is a plain-array, Eigen/Boost-free restatement of the reference's A* hot path
 * (sikang/mpl_ros @155014c, motion_primitive_library @547ddcd).  It exists only so that
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs can
 * check and time the reference algorithm.  Nothing under mpl_ros_b200/ may include, link or
 * call it.
 *
 * Parity pins: (1) MPL/README.md:200-202 (closed set 615, T = 35, J(VEL) = 36.75, J(ACC) = 1.5 on
 * MPL/data/corridor.yaml with MPL/test/test_planner_2d.cpp:29-62 parameters), tests/test_oracle_kat.py — the only numbers
 * the reference publishes.  (2) The reference's OWN planner sources compiled here against stand-in Eigen/Boost headers
 * (oracle/shim/, oracle/ref_harness.cpp -> oracle/_ref/libmplref.so): tests/test_oracle_vs_reference.py compares this
 * restatement with them exactly on 3D, |U| = 27, JRK, yaw controls, the search-region / potential-map branch and
 * iterativePlan.  Where that library cannot be built (no /root/reference) those configurations are "parity unpinned by
 * the reference's own tests" (test_distance_map_planner_2d*.cpp and test_planner_2d_with_yaw.cpp draw pictures and
 * publish no numbers).  For the yaw branch the reference's cos/sin come from an unpinned libm: trig_mode 0 calls this
 * machine's libm (what pin 2 exercises), trig_mode 1 evaluates them correctly rounded (the definition the CUDA path
 * uses); tests/test_oracle_yaw.py relates the two.
 *
 * The LPA* branch (lpa_* below; graph_search.h:194-365, state_space.h:116-282, map_planner.cpp:125-185) is pinned the same way:
 * tests/test_oracle_lpa.py and tests/test_oracle_lpa_fuzz.py compare it step by step with the reference's own sources (whole state
 * space in hm_ order, priority-queue array, best_child_, linked points); hm_ iteration order is insertion order on both sides
 * (oracle/shim/boost/unordered_map.hpp).  The TrajSolver restatement lives in oracle/poly_oracle.cpp (pins stated in its header).
 *
 * Third-party pieces that are NOT under /root/reference and are restated from their published
 * behaviour: Boost.Heap d_ary_heap<arity 2, mutable> (sift rules, see heap section of the .cpp),
 * Boost.Unordered (keyed here by the integer lattice tuple instead of boost::hash_combine),
 * Eigen fixed-size vector arithmetic (element-wise IEEE ops, lpNorm<Infinity> = max |x_i|).
 * Versions are unpinned upstream (apt libeigen3-dev / libboost-dev, MPL/wercker.yml:10).
 */
#ifndef MPL_ORACLE_H
#define MPL_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Same field order as the product's mplb_waypoint (include/mplb.h) so tests can share buffers. */
typedef struct orc_waypoint {
  double pos[3], vel[3], acc[3], jrk[3];
  double yaw, t;
  int32_t control;  /* Control::Control bit pattern, control.h:10-20 */
  int32_t enable_t; /* waypoint.h:57 */
} orc_waypoint;

typedef struct orc_result {
  int32_t status; /* 0 ok, 1 start not free, 2 max expand, 3 queue empty, 4 traceback failed, 5 start is goal */
  int32_t n_seg;
  double cost;      /* PlannerBase::traj_cost_ (goal g) or +inf */
  int32_t pops;     /* expand_iteration, graph_search.h:64,177 */
  int32_t n_nodes;  /* hm_.size() */
  int32_t n_open;   /* pq_.size() at return */
  int32_t n_closed; /* nodes with iterationclosed */
  int64_t n_prims;  /* (popped state, u) pairs entering env_map.h:155 */
  int64_t n_samples;/* voxel samples tested by env_map.h:99 loops (early exit respected) */
  int64_t n_valid;  /* finite-cost successors (graph_search.h:81 passes) */
  uint64_t pop_hash;/* order-dependent hash over popped lattice keys */
  uint64_t closed_hash; /* order-independent hash over closed lattice keys */
  double device_ms;  /* same slot as mplb_result.device_ms: here the wall-clock ms this plan took on its CPU thread
                        (filled by the batch entry points; 0 from orc_plan) */
} orc_result;

/* One row of the per-primitive trace of env_map::get_succ (env_map.h:147-172). */
typedef struct orc_prim_trace {
  int32_t verdict;   /* 0 self-loop, 1 dyn-reject, 2 collide/outside, 3 valid, 4 valid (pos unchanged, no collision test) */
  int32_t n;         /* sample divisor n of env_map.h:95 (0 if not sampled) */
  int32_t n_tested;  /* samples tested before return */
  int32_t block_idx; /* linear voxel index of the blocking sample, -1 if outside / none */
  double cost;       /* succ_cost entry (inf for verdict 2; 0 for verdicts 0/1 which emit no entry) */
  double succ[13];   /* pos3 vel3 acc3 jrk3 yaw of tn */
  int32_t key[16];   /* lattice key ints of tn, key[15] = count */
} orc_prim_trace;

typedef struct orc_node {
  double state[13]; /* pos3 vel3 acc3 jrk3 yaw — stored coord (first discoverer) */
  double t;
  double g, h;
  int32_t key[16];  /* key[15] = count */
  int32_t opened, closed;
} orc_node;

/* One node of the LPA* state space (State<Coord>, state_space.h:36-70) in hm_ iteration order (insertion order, see
 * oracle/shim/boost/unordered_map.hpp), for exact comparisons between the oracle, the reference's sources and the CUDA path. */
typedef struct orc_lpa_node {
  int32_t key[16];  /* lattice key ints, key[15] = count */
  double g, rhs, h;
  int32_t opened, closed, n_succ, n_pred;
  uint64_t succ_hash, pred_hash; /* order-dependent, over (key hash of the other end, action id, cost bits) of the stored lists */
} orc_lpa_node;
typedef struct orc_lpa_heap_entry { /* pq_ in its internal array order */
  double fval;
  uint64_t key_hash;
} orc_lpa_heap_entry;

void *orc_map_create(int dim, const int32_t *ndim, const double *origin, double res, const int8_t *data);
void orc_map_destroy(void *map);
void orc_map_free_unknown(void *map);
int orc_map_float_to_int(void *map, const double *pt, int32_t *pn); /* returns linear index or -1 if outside */

void *orc_planner_create(int dim);
void orc_planner_destroy(void *p);
void orc_planner_set_map(void *p, void *map);
/* keys: "v_max" "a_max" "j_max" "yaw_max" "dt" "w" "epsilon" "max_num" "tol_pos" "tol_vel" "tol_acc"
 *       "potential_weight" "gradient_weight" "pow" "wyaw" "tol_yaw" "trig_mode" (0 = libm cos/sin, 1 = correctly rounded) */
int orc_planner_set_param(void *p, const char *key, double v);
void orc_planner_set_controls(void *p, const double *U, int n, int udim);

/* cost shaping of env_map / MapPlanner (SURVEY section 8f.1): keys "search_radius" "potential_radius" "potential_map_range" */
void orc_planner_set_vec(void *p, const char *key, const double *v);
void orc_planner_set_search_region(void *p, const double *path, int n, int dense); /* map_planner.cpp:46-95; n rows of 3 doubles */
void orc_planner_set_potential_map(void *p, const int8_t *pot, int64_t n);          /* env_map.h:182; n = 0 clears */
void orc_planner_set_search_region_mask(void *p, const uint8_t *mask, int64_t n);   /* env_base.h:301-303; n = 0 clears */
/* PlannerBase::setPriorTrajectory (planner_base.h:249-252, env_base.h:46-53,249-256): the trajectory of `src`'s last plan
 * becomes the prior of `p` (NULL clears).  Oracle-only so far: the CUDA path does not implement prior trajectories. */
void orc_planner_set_prior_trajectory(void *p, void *src);
void orc_planner_clear_shaping(void *p);
int64_t orc_planner_get_search_region(void *p, uint8_t *out, int64_t cap);
void orc_planner_update_potential_map(void *p, const double *pos);                 /* map_planner.cpp:286-391 (rewrites the map) */
int64_t orc_map_get_data(void *map, int8_t *out, int64_t cap);
/* correctly rounded sin/cos (the yaw branch's reproducible definition of pr:520 / em:125), |x| < 2^20 */
void orc_sincos_cr(const double *x, int n, double *s, double *c);
int orc_plan(void *p, const orc_waypoint *start, const orc_waypoint *goal, orc_result *out);
/* getters for the last orc_plan on this planner */
int orc_get_actions(void *p, int32_t *actions, int cap);                 /* returns n_seg */
int orc_get_seg_states(void *p, double *states13, int cap);              /* n_seg rows of 13 doubles (parent coord per segment) */
int orc_get_nodes(void *p, orc_node *nodes, int cap);                    /* returns n_nodes (hash-map iteration, unordered) */
int orc_get_pop_keys(void *p, int32_t *keys16, int cap);                 /* rows of 16 ints in pop order; returns pops */
/* pq_ (Heap::q) in its array order; the same layout as the reference's d_ary_heap array as far as the stand-in
 * oracle/shim/boost/heap/d_ary_heap.hpp mirrors Boost's (tests/test_oracle_vs_reference.py compares the two) */
typedef struct orc_heap_entry {
  int32_t key[16];   /* lattice ints of the entry's node, key[15] = count */
  double f;          /* the stored priority g + eps * h at push / increase time */
  uint64_t key_hash; /* of the key, as in pop_hash / closed_hash and orc_lpa_heap_entry */
} orc_heap_entry;
int orc_get_heap(void *p, orc_heap_entry *entries, int cap);             /* returns pq_.size() */
/* Largest hm_.size(), pq_.size() and predecessor-record count (finite-cost edges so far) seen at the start of any
 * expansion of the last orc_plan, i.e. after its pop and before get_succ — where the CUDA kernel checks its arena.  A plan
 * overflows a tier of capacity C (|U| controls) exactly when nodes + |U| > C, heap + |U| + 1 > C, or, in predecessor-log
 * mode, records + |U| > log_cap. */
void orc_get_peaks(void *p, int64_t *peaks3);
int orc_get_succ_trace(void *p, const orc_waypoint *curr, orc_prim_trace *rows, int cap); /* returns |U| */

/* Batch: plans i = 0..n-1 striped over nthreads std::threads (one plan per thread at a time;
 * the reference itself is single-threaded per plan). actions may be NULL. */
int orc_plan_batch(void *p, const orc_waypoint *starts, const orc_waypoint *goals, int n, int nthreads,
                   orc_result *results, int32_t *actions, int max_seg);

/* Same, with a dynamic work queue (atomic index, optional processing `order`, optional pinning of thread i to core
 * i mod ncores) instead of a static stripe; busy_s[nthreads] (may be NULL) receives each thread's seconds inside plan(). */
int orc_plan_batch_dyn(void *p, const orc_waypoint *starts, const orc_waypoint *goals, int n, int nthreads,
                       orc_result *results, int32_t *actions, int max_seg, const int32_t *order, int pin, double *busy_s);

/* ---- LPA* (SURVEY section 8f.3): PlannerBase::setLPAstar + plan (planner_base.h:170-176,275-325 -> GraphSearch::LPAstar,
 * graph_search.h:194-365), getSubStateSpace (state_space.h:116-204), MapPlanner::getLinkedNodes / updateBlockedNodes /
 * updateClearedNodes (map_planner.cpp:125-185 -> StateSpace::increaseCost / decreaseCost / updateNode, state_space.h:207-282).
 * The search state persists across orc_lpa_plan calls until orc_lpa_reset. */
void orc_map_set_cells(void *map, const int32_t *cells3, int n, int8_t value); /* getMap / edit / setMap of the caller (map_replanner_node.cpp:181-196) */
void orc_lpa_reset(void *p);                                                   /* PlannerBase::reset, planner_base.h:164-167 */
int orc_lpa_plan(void *p, const orc_waypoint *start, const orc_waypoint *goal, orc_result *out);
int orc_lpa_get_sub_state_space(void *p, int time_step);                       /* returns hm_.size() afterwards */
int orc_lpa_get_linked_nodes(void *p, double *pts3, int cap);                  /* returns the number of linked points */
int orc_lpa_update_blocked_nodes(void *p, const int32_t *pns3, int n);         /* returns the number of (node, pred) pairs handed to increaseCost */
int orc_lpa_update_cleared_nodes(void *p, const int32_t *pns3, int n);
int orc_lpa_dump_nodes(void *p, orc_lpa_node *nodes, int cap);                 /* hm_ order; returns hm_.size() */
int orc_lpa_dump_heap(void *p, orc_lpa_heap_entry *entries, int cap);          /* pq_ array order; returns pq_.size() */
int orc_lpa_best_child(void *p, int32_t *keys16, int cap);                     /* best_child_ (start .. goal); returns its length */
int orc_lpa_best_child_states(void *p, double *states13, int cap);             /* stored coords of best_child_ (pos3 vel3 acc3 jrk3 yaw) */
int orc_lpa_last_fault(void *p); /* bit 0: getSubStateSpace met a successor that is no longer in hm_ (state_space.h:160-163 dereferences null);
                                    bit 1: the last trace-back met a predecessor cycle (graph_search.h:377-438 would not terminate) */
int orc_lpa_get_actions(void *p, int32_t *actions, int cap);                   /* action ids of the last LPA* trajectory; returns n_seg */

#ifdef __cplusplus
}
#endif
#endif
