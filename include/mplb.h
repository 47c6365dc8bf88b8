/*
 * mplb.h — C ABI of the H100-native motion-primitive lattice planner (libmplb.so).
 *
 * This is the drop-in boundary for ONE path of sikang/mpl_ros: the A* wavefront
 *   PlannerBase::plan -> GraphSearch::Astar -> env_map::get_succ -> Primitive -> traverse_primitive -> MapUtil
 * The reference has no FFI layer; the seam is the C++ class surface that mpl_test_node compiles against
 * (PlannerBase / MapPlanner / MapUtil).  Each entry point below cites the reference interface it replaces
 * (paths relative to /root/reference/motion_primitive_library/).  The header-compatible C++ shim that puts
 * the reference's class names back on top of this ABI is include/mpl_b200/map_planner.hpp; the binding a
 * maintainer adds at a ROS site is shown in INTEGRATION.md.
 *
 * Conventions: plain C types, caller-owned buffers, no exceptions, every function returns an int status
 * (MPLB_OK = 0) unless noted; nothing is printed unless the planner was created verbose.  A planner handle
 * is not re-entrant (like the reference's PlannerBase, env_base.h:402-404); distinct planners may share one
 * map as long as nobody mutates it.  There is NO CPU fallback: every call that needs the device fails with
 * MPLB_ERR_CUDA when no CUDA device / sm_90 kernel image is usable.
 */
#ifndef MPLB_H
#define MPLB_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library-level status codes (return values) */
#define MPLB_OK 0
#define MPLB_ERR_ARG -1      /* bad argument / unsupported configuration (message in mplb_last_error) */
#define MPLB_ERR_CUDA -2     /* CUDA runtime error or no device */
#define MPLB_ERR_STATE -3    /* call order problem (no map, no controls, no retained plan ...) */
#define MPLB_ERR_NOMEM -4    /* search arena does not fit in device memory */

/* ---- per-plan status (mplb_result.status); 0-4 are the reference's outcomes */
#define MPLB_PLAN_OK 0               /* trajectory found                       planner_base.h:324 */
#define MPLB_PLAN_START_NOT_FREE 1   /* "[PlannerBase] start is not free!"     planner_base.h:283-287 */
#define MPLB_PLAN_MAX_EXPAND 2       /* "MaxExpandStep [%d] Reached"           graph_search.h:149-154 */
#define MPLB_PLAN_QUEUE_EMPTY 3      /* "Priority queue is empty"              graph_search.h:157-161 */
#define MPLB_PLAN_TRACEBACK_FAILED 4 /* recoverTraj returned false             graph_search.h:414-431,180-181 */
#define MPLB_PLAN_START_IS_GOAL 5    /* Astar returned 0 before searching; plan() is true, traj untouched graph_search.h:44 */
#define MPLB_PLAN_KEY_RANGE 7        /* a lattice int the reference cannot represent: round(x / 0.01 or 0.1) beyond int32 in the
                                        start, or a successor outside the packable range (a derivative with an unset bound
                                        beyond 100); a start merely outside the packable range is planned from */
#define MPLB_PLAN_NOMEM 8            /* node arena exhausted at the largest tier that fits the arena budget.  The record is fully
                                        defined: n_seg 0, cost +inf, every counter, hash and device_ms 0, and the plan's action
                                        row (when requested) all -1; segment states are not written.  A retained NOMEM plan
                                        has no search state: mplb_get_nodes / _pop_log / _open fail with MPLB_ERR_STATE */

/* Control::Control bit patterns, include/mpl_basis/control.h:10-20 */
#define MPLB_CONTROL_VEL 1
#define MPLB_CONTROL_ACC 3
#define MPLB_CONTROL_JRK 7
#define MPLB_CONTROL_SNP 15
#define MPLB_CONTROL_VELxYAW 17 /* yaw variants: the state carries yaw, control rows have Dim + 1 entries (primitive.h:217,236-253) */
#define MPLB_CONTROL_ACCxYAW 19
#define MPLB_CONTROL_JRKxYAW 23
#define MPLB_CONTROL_SNPxYAW 31

/* Waypoint<Dim>, include/mpl_basis/waypoint.h:22-58 (Dim = 2 uses the first two components). */
typedef struct mplb_waypoint {
  double pos[3], vel[3], acc[3], jrk[3];
  double yaw, t;
  int32_t control;  /* the 5-bit use_pos..use_yaw union */
  int32_t enable_t; /* must be 0 (time-indexed keys are not on this path) */
  /* yaw is used when control has bit 16 (MPLB_CONTROL_*xYAW); cos/sin on that branch are the correctly rounded
   * functions (see mplb_sincos_cr), where the reference calls an unpinned libm */
} mplb_waypoint;

/* Outcome of one plan.  cost = PlannerBase::traj_cost_ (goal g, graph_search.h:179) or +inf. */
typedef struct mplb_result {
  int32_t status;
  int32_t n_seg;       /* number of primitives in the trajectory (Trajectory::segs.size()) */
  double cost;
  int32_t pops;        /* StateSpace::expand_iteration_ = getExpandedNum(), planner_base.h:148 */
  int32_t n_nodes;     /* hm_.size() */
  int32_t n_open;      /* pq_.size() at return = getOpenSet().size() */
  int32_t n_closed;    /* getCloseSet().size() */
  int64_t n_prims;     /* primitive expansions: (popped state, u) pairs entering env_map.h:155 */
  int64_t n_samples;   /* voxel samples the reference loop env_map.h:99 tests (early exit respected) */
  int64_t n_valid;     /* finite-cost successors (graph_search.h:81 passes) */
  uint64_t pop_hash;   /* order-dependent hash of popped lattice keys (parity artefact) */
  uint64_t closed_hash;/* order-independent hash of closed lattice keys (parity artefact) */
  double device_ms;    /* device time of this plan: from the moment a CTA picked it up to its result record (%globaltimer);
                          the per-plan latency behind the p50/p95 figures of bench.py.  Not a reference quantity. */
} mplb_result;

/* One (state, u) row of env_map::get_succ, env_map.h:147-172 (parity artefact + micro-benchmark output). */
typedef struct mplb_prim_trace {
  int32_t verdict;   /* 0 self-loop, 1 dyn-reject, 2 collide/outside, 3 valid, 4 valid with pos unchanged */
  int32_t n;         /* sample divisor of env_map.h:95 (0 when not sampled) */
  int32_t n_tested;  /* samples the reference loop tests before returning */
  int32_t block_idx; /* linear voxel index of the blocking sample, -1 if outside or none */
  double cost;       /* succ_cost entry (+inf for verdict 2, 0 for verdicts 0/1 which emit no entry) */
  double succ[13];   /* pos3 vel3 acc3 jrk3 yaw of the end state tn */
  int32_t key[16];   /* lattice ints of tn (waypoint.h:92-125 order), key[15] = count */
} mplb_prim_trace;

/* One collision sample of env_map.h:99-104 as the search kernel's filtered sampler sees it (parity artefact). */
typedef struct mplb_sample_probe {
  int32_t state, control, k;   /* k-th sample time of the control's divisor */
  int32_t sure;                /* filter decided without falling back */
  int32_t cell_fast[3], cell_exact[3];
  double t;
  double w[3];                 /* filtered cell coordinate minus 0.5, as the filter computed it */
} mplb_sample_probe;

/* One search node (State<Coord>, state_space.h:36-70) of a retained single plan. */
typedef struct mplb_node {
  double state[13];  /* stored coord = first discoverer's state (graph_search.h:84-88) */
  double g, h;
  int32_t key[16];   /* key[15] = count */
  int32_t opened, closed;
  int32_t parent;    /* best predecessor node index (-1 for start) under recoverTraj's rule */
  int32_t action;    /* index into U of the edge parent -> this */
} mplb_node;

typedef struct mplb_map mplb_map;
typedef struct mplb_planner mplb_planner;

const char *mplb_last_error(void);
int mplb_device_count(void);
/* cumulative count of this library's kernel launches in the calling process (bench `gpu_launches`). */
int64_t mplb_launch_count(void);

/* ---- MapUtil<Dim>, include/mpl_collision/map_util.h */
/* setMap (map_util.h:84-90): deep-copies host data (int8, x fastest) and uploads it to the current device. */
int mplb_map_create(int dim, const int32_t *ndim, const double *origin, double res, const int8_t *data, mplb_map **out);
/* Same, but `dev_data` already lives on the current device (e.g. the receive buffer of an NCCL broadcast);
 * it is copied device-to-device on `stream` (a cudaStream_t passed as void*, NULL = default stream). */
int mplb_map_create_from_device(int dim, const int32_t *ndim, const double *origin, double res, const void *dev_data,
                                void *stream, mplb_map **out);
int mplb_map_free_unknown(mplb_map *m);                    /* freeUnknown, map_util.h:259-276 */
int mplb_map_dilate(mplb_map *m, const int32_t *ns, int n);/* dilate, map_util.h:221-257; ns = n rows of Dim ints */
int mplb_map_get_info(const mplb_map *m, int32_t *dim, int32_t *ndim, double *origin, double *res); /* getDim/getOrigin/getRes */
int mplb_map_get_data(const mplb_map *m, int8_t *out, size_t cap);                                   /* getMap, map_util.h:25 */
void mplb_map_destroy(mplb_map *m);

/* ---- PlannerBase<Dim,Coord> / MapPlanner<Dim>, include/mpl_planner/common/planner_base.h, planner/map_planner.h */
int mplb_planner_create(int dim, int verbose, mplb_planner **out); /* MapPlanner ctor, src/mpl_planner/map_planner.cpp:6-11 */
void mplb_planner_destroy(mplb_planner *p);
int mplb_planner_set_map(mplb_planner *p, mplb_map *m);            /* setMapUtil, map_planner.cpp:14-18 (shared, not copied) */

enum mplb_param {
  MPLB_V_MAX = 0,   /* setVmax   planner_base.h:179  default -1 (env_base.h:380) — must be > 0 here */
  MPLB_A_MAX = 1,   /* setAmax   :185 */
  MPLB_J_MAX = 2,   /* setJmax   :191 */
  MPLB_YAW_MAX = 3, /* setYawmax :197 default -1: semi-FOV of validate_yaw (primitive.h:503-525), <= 0 disables it */
  MPLB_DT = 4,      /* setDt     :209 default 1.0 */
  MPLB_W = 5,       /* setW      :215 default 10 */
  MPLB_EPSILON = 6, /* setEpsilon:227 default 1 */
  MPLB_MAX_NUM = 7, /* setMaxNum :241 default -1 */
  MPLB_TOL_POS = 8, /* setTol    :255-265 */
  MPLB_TOL_VEL = 9,
  MPLB_TOL_ACC = 10,
  MPLB_T_MAX = 11,  /* setTmax   :203 (accepted, ignored exactly like env_map::is_goal does, env_map.h:25-45) */
  MPLB_POTENTIAL_WEIGHT = 12, /* setPotentialWeight map_planner.cpp:30-33, default 0.1 (env_map.h:196) */
  MPLB_GRADIENT_WEIGHT = 13,  /* setGradientWeight  map_planner.cpp:35-38, default 0.0 (env_map.h:197) */
  MPLB_WYAW = 14,   /* setWyaw   :221 default 1.0 (env_base.h:372): weight of the heading cost env_map.h:121-128 */
  MPLB_MEM_FRACTION = 100, /* fraction of free device memory the search arenas may take (default 0.6) */
  MPLB_MAX_SLOTS = 101,    /* tuning: cap on concurrently resident plans (CTAs); 0 = all resident CTAs */
  MPLB_EXACT_PREDS = 102,  /* predecessor lists of graph_search.h:100-102 kept per node and resolved by recoverTraj with the
                              final g values: -1 (default) = exactly where a running best predecessor could differ (epsilon > 1,
                              a prior-trajectory heuristic, VEL control with v_max below the control bound), 0 = never,
                              1 = always */
  MPLB_ARENA_BYTES = 103,  /* upper bound in bytes on the search-arena budget (0 = unset, the default): the budget is
                              min(MPLB_MEM_FRACTION of the free memory, this).  Like MPLB_MEM_FRACTION it makes the next
                              batch measure the budget again */
  MPLB_LPA_INIT_NODES = 104, /* LPA*: node capacity of a session when it allocates (first plan, and the first plan after
                                mplb_planner_reset); default 65 536.  Any whole number in [MPLB_LPA_MIN_CAP, MPLB_LPA_MAX_INIT],
                                powers of two or not; other values fail with MPLB_ERR_ARG.  The arrays double when a plan
                                needs more, so this decides when growth happens and nothing else: results do not depend on it */
  MPLB_LPA_INIT_PREDS = 105  /* LPA*: predecessor-record capacity at allocation; default 2^20; same range and rules */
};
#define MPLB_LPA_MIN_CAP 128        /* smallest accepted MPLB_LPA_INIT_NODES / MPLB_LPA_INIT_PREDS */
#define MPLB_LPA_MAX_INIT (1 << 28) /* largest accepted one */
int mplb_planner_set_param(mplb_planner *p, int key, double value);
/* setU (planner_base.h:246): n rows of udim doubles, udim = Dim, or Dim + 1 when the last entry is a yaw rate
 * (primitive.h:217); the row index is the action id. */
int mplb_planner_set_controls(mplb_planner *p, const double *U, int n, int udim);

/* ---- cost shaping of env_map (SURVEY section 8f.1): search region and potential map, env_map.h:104-128.
 * Both are per-planner state like ENV_->search_region_ / potential_map_ and stay set until replaced or cleared.
 * Shaped plans take control sets of up to 128 rows (|U| > 32 runs on the shaped MAXU = 4 kernels) and need positive dynamic
 * bounds for every derivative of the control order; the map may be scrubbed of unknown cells or not (either works). */
/* env_base::set_search_region (env_base.h:301-303): one byte (0/1) per map cell, x fastest.  NULL or n = 0 clears. */
int mplb_planner_set_search_region(mplb_planner *p, const uint8_t *in_region, size_t n);
/* MapPlanner::setSearchRegion (map_planner.cpp:46-95): tunnel of half-width `radius` (Dim doubles, setSearchRadius
 * map_planner.cpp:41-43) around the polyline `path` (npts rows of 3 doubles); dense = the path is already cell-dense. */
int mplb_planner_set_search_region_path(mplb_planner *p, const double *path, int npts, int dense, const double *radius);
/* env_base::get_search_region (env_base.h:365): returns the cell count (0 when no region is set), fills out[0..cap). */
int64_t mplb_planner_get_search_region(mplb_planner *p, uint8_t *out, size_t cap);
/* env_map::set_potential_map (env_map.h:182): one int8 per map cell.  NULL or n = 0 clears. */
int mplb_planner_set_potential_map(mplb_planner *p, const int8_t *pot, size_t n);
/* MapPlanner::createMask + updatePotentialMap (map_planner.cpp:286-391): stamps the radial mask of height H_MAX = 100
 * and exponent `pow` (map_planner.h:104,113) around every cell > 0 inside pos +- range (whole map when range is all
 * zero), REWRITES THE PLANNER'S MAP with the result (like map_util_->setMap(dmap)) and installs it as this planner's
 * potential map.  radius/range: 3 doubles (radius[0] = xy radius, radius[2] = z half-height in 3D). */
int mplb_planner_update_potential_map(mplb_planner *p, const double *pos, const double *radius, const double *range,
                                      double pow);

/* setPriorTrajectory (planner_base.h:249-252 -> env_map::set_prior_trajectory, env_map.h:187-225, heuristic env_base.h:46-53):
 * n_seg primitives given by their coefficient rows cx, cy, cz, cyaw (6 doubles each, highest order first, as
 * toPrimitiveROSMsg lays them out: coeffs[n_seg][4][6]) and durations seg_t[n_seg]; control = the prior's Control flags.
 * While a prior is installed the requested goals are ignored (env_base.h:295-298) and the goal is the prior's end point.
 * n_seg = 0 clears.  The prior is assumed collision free (traverse_trajectory = 0) and cannot be combined with a potential map. */
int mplb_planner_set_prior_trajectory(mplb_planner *p, int n_seg, const double *coeffs, const double *seg_t, int control);

/* plan (planner_base.h:275-325).  Returns MPLB_OK when the call itself worked; the reference's bool is
 * (out->status == MPLB_PLAN_OK || out->status == MPLB_PLAN_START_IS_GOAL).  The search state of this plan
 * stays on the device until the next plan/plan_batch on this handle, for the getters below. */
int mplb_plan(mplb_planner *p, const mplb_waypoint *start, const mplb_waypoint *goal, mplb_result *out);

/* Batch of independent plans on one map (north-star extension; each entry behaves exactly like mplb_plan).
 * HOST buffers: starts/goals [n]; results [n]; actions [n*max_seg] int32 (trajectory action ids, -1 padded;
 * may be NULL); seg_states [n*max_seg*13] doubles (stored coord of each segment's parent node, the argument
 * of env_base::forward_action, env_base.h:228-231; may be NULL).  Plans whose n_seg > max_seg report the
 * true n_seg and only the first max_seg entries. */
int mplb_plan_batch(mplb_planner *p, const mplb_waypoint *starts, const mplb_waypoint *goals, int n,
                    mplb_result *results, int32_t *actions, double *seg_states, int max_seg);
/* Same with DEVICE buffers on the planner's device; asynchronous launches are ordered on `stream`
 * (cudaStream_t as void*, NULL = default) and the call returns after the batch has completed. */
int mplb_plan_batch_device(mplb_planner *p, const void *d_starts, const void *d_goals, int n, void *d_results,
                           void *d_actions, void *d_seg_states, int max_seg, void *stream);

/* ---- wire output (SURVEY section 8f.4): toTrajectoryROSMsg (planning_ros_utils/include/planning_ros_utils/
 * primitive_ros_utils.h:11-33,36-55,78-113) followed by the ROS 1 serialisation of planning_ros_msgs/Trajectory
 * (std_msgs/Header header; Primitive[] primitives {float64[] cx, cy, cz, cyaw; float64 t}; LambdaSeg[] lambda = empty),
 * for every plan of a batch, written by the GPU.  Inputs are the outputs of mplb_plan_batch(_device) with the same
 * max_seg (results, actions and seg_states are all required).  Plan i's message goes to out + i*stride and its byte
 * length to len[i]; failed plans give a message with zero primitives (the reference's empty traj_); len[i] = 0 marks a
 * plan whose trajectory was truncated (n_seg > max_seg) or does not fit in `stride`.  z is the height written into cz
 * for 2D planners (primitive_ros_utils.h:12,18); header fields as in map_planner_node.cpp:55-57,207. */
size_t mplb_trajectory_msg_size(int n_seg, const char *frame_id); /* bytes of one serialised message */
int mplb_serialize_trajectories_device(mplb_planner *p, const void *d_results, const void *d_actions, const void *d_seg_states,
                                       int n, int max_seg, double z, uint32_t seq, uint32_t stamp_sec, uint32_t stamp_nsec,
                                       const char *frame_id, void *d_out, size_t stride, void *d_len, void *stream);
int mplb_serialize_trajectories(mplb_planner *p, const mplb_result *results, const int32_t *actions, const double *seg_states,
                                int n, int max_seg, double z, uint32_t seq, uint32_t stamp_sec, uint32_t stamp_nsec,
                                const char *frame_id, uint8_t *out, size_t stride, uint32_t *len);

/* ---- trajectory post-processing (SURVEY section 8f.4): TrajSolver<Dim>(control, yaw_control) with setWaypoints + setDts,
 * then solve() (include/mpl_traj_solver/traj_solver.h:12-109 over PolySolver<Dim>::solve, src/mpl_traj_solver/poly_solver.cpp:23-221
 * and PolyTraj::toPrimitives, src/mpl_traj_solver/poly_traj.cpp:75-92) for a BATCH of independent waypoint lists, one CTA each.
 * This is the refinement map_planner_node.cpp:216-227 applies to a planned trajectory (waypoints = traj.getWaypoints() with
 * the interior ones set to Control::VEL, dts = traj.getSegmentTimes(), TrajSolver3D(Control::JRK)).
 *   control      MPLB_CONTROL_VEL / ACC / JRK (+ the xYAW variants): minimum velocity / acceleration / jerk spline
 *                (PolySolver(0,1) / (1,2) / (2,3)); SNP has no solver in the reference ("only works up to third order") and
 *                gives empty trajectories here too (n_segs = 0)
 *   yaw_control  MPLB_CONTROL_VEL / ACC / JRK: order of the 1-D yaw spline (traj_solver.h:31-36, 86-103)
 *   wp_offsets   n_traj + 1 ints, wp_offsets[0] = 0: trajectory i owns waypoints wp_offsets[i] .. wp_offsets[i+1]-1; the
 *                `control` field of a waypoint says which of its derivatives are fixed (use_pos .. use_jrk); its yaw is the
 *                yaw key frame
 *   dts          one duration per segment, concatenated: trajectory i owns max(W_i - 1, 0) entries (TrajSolver::setDts)
 *   coefs        per segment, same concatenation: (dim + 1) rows (the axes, then yaw) of six Primitive coefficients, highest
 *                order first — Trajectory::segs[s].pr(a).coeff() / pr_yaw().coeff(), i.e. the cx, cy, [cz,] cyaw rows of
 *                planning_ros_msgs/Primitive
 *   n_segs       (may be NULL) segments of trajectory i's result: W_i - 1, or 0 where the reference returns an empty
 *                Trajectory (fewer than two waypoints, solver not initialised)
 * Host buffers; the _device variant takes wps / dts / coefs in HBM (wp_offsets and n_segs stay host arrays) and orders its
 * work on `stream`, returning once the solve has completed.  The _device variant also takes a sub-range of a larger list:
 * wp_offsets[0] may be any value, and offsets are then relative to it — d_wps points at waypoint wp_offsets[0], while d_dts and
 * d_coefs start at that sub-range's first segment (the host variant requires wp_offsets[0] = 0).  Both variants write every
 * coefficient slot of the range: the slots of trajectories they do not solve (solver not initialised) are zeroed.
 * FP64, every operation in the reference's order with Eigen's unblocked partial-pivot LU restated (DESIGN.md section 4.11
 * states what that pins, the shared-memory / global-scratch split, and the measured accuracy).  A call whose work space in
 * global scratch would exceed 8 GiB (about 7 800 waypoints for 3-D JRK with a JRK yaw) fails with MPLB_ERR_NOMEM. */
int mplb_traj_solve_batch(int dim, int control, int yaw_control, int n_traj, const int32_t *wp_offsets, const mplb_waypoint *wps,
                          const double *dts, double *coefs, int32_t *n_segs);
int mplb_traj_solve_batch_device(int dim, int control, int yaw_control, int n_traj, const int32_t *wp_offsets, const void *d_wps,
                                 const void *d_dts, void *d_coefs, int32_t *n_segs, void *stream);

/* What the last trajectory solve issued by the calling host thread launched (mplb_traj_solve_batch(_device) or
 * mplb_refine_trajectories(_device)); all zero after a call that launched nothing or failed.  One solve is a pair of CTAs per
 * trajectory, position axes and yaw, and each CTA keeps its work space in shared memory when it fits smem_bytes and in
 * global scratch otherwise, so the two CTAs of one trajectory can differ. */
typedef struct mplb_traj_solve_stats {
  int32_t n_traj;       /* trajectories solved (CTA pairs launched) */
  int32_t max_wp;       /* largest waypoint count among them */
  int32_t pos_shared;   /* position CTAs whose work space was in shared memory */
  int32_t pos_global;   /* ... in global scratch */
  int32_t yaw_shared;   /* yaw CTAs in shared memory */
  int32_t yaw_global;   /* yaw CTAs in global scratch */
  int64_t smem_bytes;   /* dynamic shared memory per CTA of the launch */
  int64_t global_bytes; /* global scratch the launch used (0 when every CTA fit in shared memory) */
} mplb_traj_solve_stats;
int mplb_traj_solve_last_stats(mplb_traj_solve_stats *out);

/* The refinement step of map_planner_node.cpp:216-227 for a whole batch without leaving the device: for every successful plan of
 * mplb_plan_batch(_device) (same max_seg; results, actions and seg_states are all required) the waypoints of its trajectory
 * (Trajectory::getWaypoints, trajectory.h:277-289: the stored coord of every segment's parent and the last primitive evaluated at
 * its duration), the interior ones re-flagged Control::VEL, the two ends keeping plan_control (the control flags the batch was planned
 * with), the planner's dt as every segment time, then TrajSolver<Dim>(control, yaw_control)::solve.  coefs: n * max_seg segments of
 * (dim + 1) rows x 6 coefficients (plan i at i * max_seg; zero where nothing was refined); n_segs (HOST, may be NULL): refined segments
 * per plan, 0 for failed or truncated plans.  A gather kernel (one thread per waypoint) followed by the batched solve. */
int mplb_refine_trajectories_device(mplb_planner *p, const void *d_results, const void *d_actions, const void *d_seg_states, int n,
                                    int max_seg, int plan_control, int control, int yaw_control, void *d_coefs, int32_t *n_segs,
                                    void *stream);
int mplb_refine_trajectories(mplb_planner *p, const mplb_result *results, const int32_t *actions, const double *seg_states, int n,
                             int max_seg, int plan_control, int control, int yaw_control, double *coefs, int32_t *n_segs);

/* ---- LPA* incremental replanning (SURVEY section 8f.3; mpl_test_node/src/map_replanner_node.cpp:107-241 is the caller).
 * The search state of a planner with LPA* enabled stays on the device between plans; each call below is the member of the
 * same name.  Occupancy maps with or without a potential map (mplb_planner_set_potential_map /
 * mplb_planner_update_potential_map, MPLB_POTENTIAL_WEIGHT / MPLB_GRADIENT_WEIGHT) and the *xYAW controls (control rows of
 * Dim + 1 entries, MPLB_YAW_MAX / MPLB_WYAW) replan like the plain map; a search region or a prior trajectory makes mplb_plan
 * fail with MPLB_ERR_ARG while LPA* is on.  Stored edge costs are never recomputed when the potential map is replaced, and
 * updateClearedNodes restores an edge as J + w dt without potential or heading terms, both as the reference.  Where the reference iterates its hash map (getSubStateSpace re-pushing
 * the open set, getLinkedNodes filling the voxel -> edge lists) the order is INSERTION order; Boost leaves it unspecified, and
 * it only decides the order among exact key ties (DESIGN.md section 4.12). */
/* PlannerBase::setLPAstar (planner_base.h:170-176): from now on mplb_plan runs GraphSearch::LPAstar (graph_search.h:194-365)
 * on the persistent state space; the per-plan outcome uses the same mplb_result record: pops = expand_iteration of this call, pop_hash =
 * over the nodes whose successors were generated in this call, cost = goal g - start_g_ as graph_search.h:362.  One outcome is
 * not the reference's: a plan that begins with an empty priority queue reports MPLB_PLAN_QUEUE_EMPTY where the reference reads
 * pq_.top() of an empty heap. */
int mplb_planner_set_lpastar(mplb_planner *p, int on);
/* PlannerBase::reset (planner_base.h:164-167): drops the state space; the next plan starts from scratch. */
int mplb_planner_reset(mplb_planner *p);
/* MapUtil::setMap with an edited copy of getMap(), as add/clearCloudCallback do (map_replanner_node.cpp:181-196,221-229):
 * n cells (rows of 3 ints, the third ignored in 2D) receive `value`; cells outside the grid are ignored; the occupancy bit-bricks are
 * rebuilt. */
int mplb_map_set_cells(mplb_map *m, const int32_t *cells3, int n, int value);
/* Same with the n cell rows in device memory, read on `stream` (a cudaStream_t as void*, NULL = default); returns once the
 * cells and the bricks are written. */
int mplb_map_set_cells_device(mplb_map *m, const void *d_cells3, int n, int value, void *stream);
/* MapUtil::setMap again on a map of unchanged geometry: the whole int8 grid is replaced in place, so planners that share the
 * map (setMapUtil keeps a shared pointer in the reference) see the new cells without being re-pointed. */
int mplb_map_set_data(mplb_map *m, const int8_t *data);
/* StateSpace::getSubStateSpace (state_space.h:116-204) through PlannerBase::getSubStateSpace (planner_base.h:155): the node
 * best_child_[time_step] of the last trajectory becomes the root.  Returns hm_.size() afterwards (>= 0) or an error. */
int mplb_get_sub_state_space(mplb_planner *p, int time_step);
/* MapPlanner::getLinkedNodes (map_planner.cpp:125-158): rebuilds the voxel -> (node, predecessor index) table from every
 * stored edge and returns the number of linked points; pts3 (may be NULL) receives min(count, cap) rows of 3 doubles. */
int mplb_get_linked_nodes(mplb_planner *p, double *pts3, int cap);
/* MapPlanner::updateBlockedNodes / updateClearedNodes (map_planner.cpp:160-185 -> StateSpace::increaseCost / decreaseCost,
 * state_space.h:207-240) for n changed cells, against the table of the LAST mplb_get_linked_nodes call (like lhm_).  The map
 * must already hold the new values (mplb_map_set_cells).  Returns the number of (node, predecessor) pairs visited, or an error. */
int mplb_update_blocked_nodes(mplb_planner *p, const int32_t *cells3, int n);
int mplb_update_cleared_nodes(mplb_planner *p, const int32_t *cells3, int n);
/* Many replanners in one launch (one CTA each; e.g. one per robot): every planner must have LPA* enabled and live on the same
 * device; entry i behaves exactly like mplb_plan(planners[i], &starts[i], &goals[i], &results[i]), including the retained
 * trajectory of any length for mplb_get_actions / mplb_get_seg_states.  A session that has to grow stops before the pop that
 * could overflow; the host doubles its arrays and relaunches the batch, in which finished sessions return at once. */
int mplb_lpa_plan_batch(mplb_planner **planners, int n, const mplb_waypoint *starts, const mplb_waypoint *goals, mplb_result *results);
/* ---- a fleet cycle's output on the device (DESIGN.md section 4.12.3, "The cycle's output on the device").
 * mplb_lpa_plan_batch_device: mplb_lpa_plan_batch with DEVICE starts / goals [n] and results [n] on the planners' device, ordered on
 * `stream` (cudaStream_t as void*, NULL = default); returns after the batch has completed.  Entry i behaves exactly like
 * mplb_lpa_plan_batch for planner i (record, state space, growth and resume, the retained trajectory of mplb_get_actions /
 * mplb_get_seg_states, which a failed plan leaves as it was).  Nothing is read back for the caller: bindings that keep a host-side
 * record of the last plan (the Python and C++ result() / getTraj() / getTrajCost()) still show the last plan made through the host
 * calls, while mplb_get_actions / mplb_get_seg_states and the mplb_lpa_get_* dumps show this one.  Plan i's trajectory goes to d_actions[i*max_seg ..] and
 * d_seg_states[(i*max_seg ..)*13], the layout of mplb_plan_batch_device: the true n_seg is reported, only the first max_seg rows are
 * written, action rows past the trajectory (all of them for a failed plan) are -1 and seg-state rows past it are not written.
 * d_actions / d_seg_states may be NULL.  Fails with no planner touched on a null argument, a planner listed twice, LPA* off, planners
 * on different devices or max_seg < 0.  The host work of a call does not grow with n. */
int mplb_lpa_plan_batch_device(mplb_planner **planners, int n, const void *d_starts, const void *d_goals, void *d_results,
                               void *d_actions, void *d_seg_states, int max_seg, void *stream);
/* The next starts of map_replanner_node.cpp:243-253 (start = traj.getWaypoints()[1] after getSubStateSpace): for the plan-batch
 * layout above (same planners, same order, max_seg >= 1), d_waypoints[i] = Trajectory::getWaypoints()[d_index[i]]
 * (trajectory.h:277-289) of plan i as an mplb_waypoint: waypoint j < n_seg is segment j's stored parent coord, waypoint n_seg the
 * last primitive evaluated at dt in the reference's term order; t is the running sum 0 + dt + ... + dt of getWaypoints, control
 * the plan's control flags.  d_index: int32 [n] (device); d_ok: int32 [n] (device), 1 where a waypoint was written, 0 (and
 * d_waypoints[i] untouched) where the plan failed, n_seg > max_seg or d_index[i] is outside [0, n_seg].  The output can be passed
 * to mplb_lpa_plan_batch_device as the next cycle's starts.  Returns after the kernel has completed. */
int mplb_lpa_trajectory_waypoints_device(mplb_planner **planners, int n, const void *d_results, const void *d_actions,
                                         const void *d_seg_states, int max_seg, const void *d_index, void *d_waypoints, void *d_ok,
                                         void *stream);
/* mplb_serialize_trajectories_device (toTrajectoryROSMsg, map_planner_node / map_replanner_node.cpp:124-130,158-164) and
 * mplb_refine_trajectories_device for the plan-batch layout above: entry i is read with planner i's own dim, control order, yaw
 * flag, controls and dt of its last LPA* plan, so one call serves a fleet of differently configured robots and no A* batch is
 * needed.  Bytes, lengths, coefficient rows and n_segs are those the A* forms give for the same rows and configuration (frame,
 * header, z, stride, truncation and len = 0 rules unchanged; refine: plan_control is each plan's own, every planner of one call
 * must plan in the same dim, and control / yaw_control are the solver orders of the whole call).  Both fail before writing
 * anything on a null argument, a planner listed twice, a planner without LPA* or without a plan, or planners on different
 * devices, and return after their work has completed. */
int mplb_lpa_serialize_trajectories_device(mplb_planner **planners, int n, const void *d_results, const void *d_actions,
                                           const void *d_seg_states, int max_seg, double z, uint32_t seq, uint32_t stamp_sec,
                                           uint32_t stamp_nsec, const char *frame_id, void *d_out, size_t stride, void *d_len,
                                           void *stream);
int mplb_lpa_refine_trajectories_device(mplb_planner **planners, int n, const void *d_results, const void *d_actions,
                                        const void *d_seg_states, int max_seg, int control, int yaw_control, void *d_coefs,
                                        int32_t *n_segs, void *stream);
/* The rest of a replan cycle for many replanners per call.  Entry i leaves planners[i] exactly as the single call of the same
 * member would, and reports what that call returns.  Every call checks all of its arguments first and fails with no planner
 * touched when one is null, a planner appears twice, a planner has LPA* off or has not planned, the planners live on
 * different devices, or (sub_state_space) a time step is out of range.  The kernels take one session per block over a
 * contiguous context array, so the launches and synchronisations of a call do not grow with n (DESIGN.md section 4.12.2).
 *   get_linked_nodes_batch      MapPlanner::getLinkedNodes (map_planner.cpp:125-158) per entry: counts[i] = its linked points;
 *                               pts3 (may be NULL) receives the first `cap` rows of all points, entry 0's first
 *   update_nodes_batch          updateBlockedNodes (blocked = 1) / updateClearedNodes (blocked = 0), map_planner.cpp:160-185:
 *                               entry i's cells are rows offsets[i] .. offsets[i+1]-1 of cells3 (rows of 3 ints; offsets has
 *                               n + 1 entries, an empty range is allowed); visited[i] = the pairs it visited
 *   update_nodes_batch_device   the same with the cell rows in device memory (offsets and visited stay host arrays)
 *   sub_state_space_batch       PlannerBase::getSubStateSpace(time_steps[i]) (planner_base.h:155): sizes[i] = hm_.size()
 *                               afterwards, 0 for a planner without a trajectory, or MPLB_ERR_STATE where the sweep met a
 *                               successor no longer in the state space (the other entries complete; the call returns that error) */
int mplb_lpa_get_linked_nodes_batch(mplb_planner **planners, int n, int32_t *counts, double *pts3, int64_t cap);
int mplb_lpa_update_nodes_batch(mplb_planner **planners, int n, int blocked, const int32_t *cells3, const int64_t *offsets,
                                int32_t *visited);
int mplb_lpa_update_nodes_batch_device(mplb_planner **planners, int n, int blocked, const void *d_cells3, const int64_t *offsets,
                                       int32_t *visited);
int mplb_lpa_sub_state_space_batch(mplb_planner **planners, int n, const int32_t *time_steps, int32_t *sizes);
/* State dumps (parity artefacts and getCloseSet / getOpenSet material): hm_ in iteration order, pq_ in its array order,
 * best_child_ (start .. goal).  Two-call pattern: cap = 0 returns the size. */
typedef struct mplb_lpa_node {
  int32_t key[16];   /* lattice ints, key[15] = count */
  double state[13];  /* the State's coord: pos3 vel3 acc3 jrk3 yaw */
  double g, rhs, h;
  int32_t opened, closed, n_succ, n_pred;
  uint64_t succ_hash, pred_hash; /* order-dependent, over (key hash of the other end, action id, cost bits) of the stored lists */
} mplb_lpa_node;
typedef struct mplb_lpa_heap_entry {
  double fval;       /* the stored key: min(g, rhs) + eps * h at push time (state_space.h:270-272) */
  uint64_t key_hash; /* of the node's lattice key */
} mplb_lpa_heap_entry;
int mplb_lpa_get_nodes(mplb_planner *p, mplb_lpa_node *out, int cap);
int mplb_lpa_get_heap(mplb_planner *p, mplb_lpa_heap_entry *out, int cap);
int mplb_lpa_get_best_child(mplb_planner *p, mplb_lpa_node *out, int cap); /* succ_hash / pred_hash left 0 */
/* Capacity of the session's device arrays (read-only diagnostics; DESIGN.md section 4.12).  cap_nodes: node records (and the
 * successor, iteration-order, heap and best_child_ arrays sized with them); cap_pred: predecessor records; tsize: key-table slots;
 * n_nodes_physical: node records in use, including those a getSubStateSpace dropped from hm_ (they keep their id and are reset
 * in place if a plan reaches their key again), so it never shrinks between resets; grows: doublings since the session allocated
 * (before a pop that could overflow, or before a plan whose new start node would not fit).  getSubStateSpace may also enlarge
 * the predecessor pool to (records its sweep can append) + |U|, which is not a power of two and is not counted in grows.  Any
 * pointer may be NULL.  Fails with MPLB_ERR_STATE before the first LPA* plan. */
int mplb_lpa_get_capacity(mplb_planner *p, int32_t *cap_nodes, int32_t *cap_pred, int32_t *tsize, int32_t *n_nodes_physical,
                          int32_t *grows);

/* Result getters of the retained single plan (two-call pattern: pass cap = 0 to get the size). */
int mplb_get_actions(mplb_planner *p, int32_t *actions, int cap);      /* returns n_seg; recoverTraj graph_search.h:369-455 */
int mplb_get_seg_states(mplb_planner *p, double *states13, int cap);   /* returns n_seg */
int mplb_get_nodes(mplb_planner *p, mplb_node *nodes, int cap);        /* returns n_nodes; hm_ iteration (unordered) */
int mplb_get_pop_log(mplb_planner *p, int32_t *node_ids, int cap);     /* returns pops; expanded_nodes_ order, env_map.h:154 */
int mplb_get_open(mplb_planner *p, int32_t *node_ids, int cap);        /* returns n_open; pq_ iteration */

/* env_map::get_succ (env_map.h:147-172) for n arbitrary states: rows [n * |U|]. HOST buffers. */
int mplb_expand(mplb_planner *p, const mplb_waypoint *states, int n, mplb_prim_trace *rows);

/* The search kernel's filtered collision sampler on n arbitrary states (plain map only, like mplb_expand): for every
 * state and every control whose primitive needs sampling, one row per sample time, in no particular order.  Returns
 * the number of rows (may exceed cap; only the first cap are written, rows may be NULL with cap = 0).  use_fast and
 * fast_delta (either may be NULL) receive the configuration's filter switch and guard band in cells.  HOST buffers. */
int mplb_probe_samples(mplb_planner *p, const mplb_waypoint *states, int n, mplb_sample_probe *rows, int cap,
                       int32_t *use_fast, double *fast_delta);

/* The configuration the search kernel would run for start waypoints of this control flag, on the planner's map and
 * settings (parity artefact, read-only; shaped and yaw configurations included): key_bits = bits the packed lattice key
 * spans, key_wide = 1 when that is more than 96 (hash-table slots then also compare the row's full second key word),
 * use_fast = 1 when collision samples go through the filtered granule sampler, 0 when every control is sampled on the
 * exact path.  Any output may be NULL.  Returns MPLB_OK, or the error planning with this configuration would return. */
int mplb_planner_key_layout(mplb_planner *p, int32_t control, int32_t *key_bits, int32_t *key_wide, int32_t *use_fast);

/* Correctly rounded sin/cos as the yaw branch evaluates them (primitive.h:520, env_map.h:125), computed on the device:
 * x, s, c are HOST arrays of n doubles, |x| < 2^20.  Parity artefact: tests compare it with the oracle and mpmath. */
int mplb_sincos_cr(const double *x, int n, double *s, double *c);

/* Timing/diagnostics of the last batch on this planner: ms = device time of the search kernels (CUDA events on
 * the launch stream), launches = kernels launched, tiers = arena tiers used. Any pointer may be NULL. */
int mplb_last_batch_stats(mplb_planner *p, double *kernel_ms, int32_t *launches, int32_t *tiers);

/* One arena tier pass of the last A* batch (read-only diagnostics; DESIGN.md section 3, "Tiers").  A batch starts with
 * every plan in one tier; plans that outgrow a tier's capacity run again from scratch in a larger one.  A pass that finds no
 * tier fitting the arena budget launches nothing and marks its plans MPLB_PLAN_NOMEM (nomem = 1). */
typedef struct mplb_tier_info {
  int32_t cap;          /* node / heap capacity per plan */
  int32_t slots;        /* plans resident at once (CTAs launched); for a NOMEM pass the slots the budget would have allowed */
  int32_t n_work;       /* plans this pass ran (or marked NOMEM) */
  int32_t n_overflow;   /* of those, plans that outgrew `cap` and go to the next pass */
  int32_t hcap;         /* heap entries kept in shared memory per plan */
  int32_t load_inv;     /* hash-table load factor bound 1 / load_inv */
  int32_t tsize_max;    /* largest hash table per plan (slots) */
  int32_t log_cap;      /* predecessor records per plan (0 unless in predecessor-log mode) */
  int64_t stride_bytes; /* arena bytes per slot */
  int32_t nomem;        /* 1: nothing launched, the pass only marked its plans MPLB_PLAN_NOMEM */
  int32_t ordered;      /* 1: plans are taken from the longest-first work list, 0: in query order */
  int32_t resident;     /* CTAs of the search kernel that fit the device at once */
  int32_t reserved;
} mplb_tier_info;
/* Two-call pattern: returns the number of passes of the last batch and fills rows[0 .. min(count, cap)). */
int mplb_last_batch_tiers(mplb_planner *p, mplb_tier_info *rows, int cap);

/* ---- multi-GPU: one process per GPU, the batch sharded by query (query i -> rank i mod N), NCCL over NVLink.
 * Exactly two collectives exist on this path: one broadcast of the voxel grid per map and one gather of result records
 * (and action rows) per batch.  The caller distributes the 128-byte id of rank 0 to the other ranks by whatever means it
 * has (a ROS parameter, a file, MPI, torch.distributed) — the only out-of-band step, like ncclGetUniqueId itself. */
#define MPLB_COMM_ID_BYTES 128
typedef struct mplb_comm mplb_comm;
int mplb_comm_unique_id(uint8_t *id128);                                     /* rank 0: ncclGetUniqueId */
int mplb_comm_create(const uint8_t *id128, int rank, int nranks, mplb_comm **out); /* every rank, current device: ncclCommInitRank */
void mplb_comm_destroy(mplb_comm *c);
int mplb_comm_rank(const mplb_comm *c);
int mplb_comm_size(const mplb_comm *c);
/* MapUtil::setMap on every rank from the root's host grid: ONE ncclBroadcast of the int8 cells (plus a 64-byte header);
 * non-root ranks pass NULL for ndim / origin / data.  Every rank receives its own mplb_map. */
int mplb_comm_broadcast_map(mplb_comm *c, int root, int dim, const int32_t *ndim, const double *origin, double res,
                            const int8_t *data, mplb_map **out);
/* plan_batch over all ranks.  Every rank passes the SAME full query list (host); rank r plans queries r, r + N, ...;
 * the root receives results[n] (and actions[n * max_seg] when not NULL) in query order through one grouped
 * ncclSend/ncclRecv gather.  The other ranks' result pointers may be NULL. */
int mplb_plan_batch_sharded(mplb_planner *p, mplb_comm *c, const mplb_waypoint *starts, const mplb_waypoint *goals, int n,
                            mplb_result *results, int32_t *actions, int max_seg, int root);
/* Device-resident variant: this rank's stripe (n_local plans, device buffers sized for `per` = ceil(n / N) records) is
 * planned and gathered into the root's internal gather buffer; mplb_comm_unstripe then copies the gathered batch to host
 * buffers in query order (root only). */
int mplb_plan_stripe_gather_device(mplb_planner *p, mplb_comm *c, const void *d_starts, const void *d_goals, int n_local, int per,
                                   void *d_results, void *d_actions, int max_seg, int root, void *stream);
int mplb_comm_unstripe(mplb_comm *c, int n, int per, int max_seg, mplb_result *results, int32_t *actions);
/* The same two calls split in halves, so that a caller can keep ONE batch in flight per planner: *_begin enqueues the
 * copies, the ordering kernels and the search launch and returns without waiting; *_end completes the batch (larger arena
 * tiers for overflowed plans, the gather, the copy back).  A launch ends with its longest plan; two planners sharing one map
 * and alternating batches overlap that drain with the start of the next batch (bench.py does this, DESIGN.md section 6).
 * The host buffers given to mplb_plan_batch_sharded_begin are copied before it returns. */
int mplb_plan_stripe_begin(mplb_planner *p, const void *d_starts, const void *d_goals, int n_local, void *d_results, void *d_actions,
                           int max_seg, void *stream);
int mplb_plan_stripe_end(mplb_planner *p, mplb_comm *c, int per, int root);
int mplb_plan_batch_sharded_begin(mplb_planner *p, mplb_comm *c, const mplb_waypoint *starts, const mplb_waypoint *goals, int n,
                                  int max_seg);
int mplb_plan_batch_sharded_end(mplb_planner *p, mplb_comm *c, int n, mplb_result *results, int32_t *actions, int root);

/* ---- a fleet of LPA* replanners over all ranks (DESIGN.md section 6.1): robot i of R lives on rank i mod N, as the queries of
 * mplb_plan_batch_sharded, and every rank holds a replica of the shared map (mplb_comm_broadcast_map).  A cycle is the
 * single-device fleet cycle of section 4.12.2 with two calls distributed: every rank calls both, with the same value / max_seg /
 * root; getLinkedNodes, updateBlocked/ClearedNodes and getSubStateSpace stay rank-local (mplb_lpa_*_batch on the local robots).
 *
 * mplb_map_set_cells_device on every replica with the concatenation c_0 || c_1 || ... || c_{R-1} of all robots' edits.  This
 * rank's n_local robots (its robots rank, rank + N, ... in order) own rows offsets_local[k] .. offsets_local[k+1]-1 of d_cells3
 * (device rows of 3 ints, read once the work on `stream` (a cudaStream_t as void*, NULL = default) has completed; offsets_local
 * is a host array of n_local + 1 entries).  One grouped ncclSend / ncclRecv exchange of a header and one of rows rebuild the
 * concatenation in global robot order on every rank, independent of arrival order, in d_all_cells3 (device, `cap` rows of 3
 * ints) with its R + 1 offsets in d_all_offsets (device int64), and every replica applies it.  Returns the concatenation's row
 * count T.  Every rank passes the same cap: T <= cap means applied on every rank; T > cap means nothing was exchanged or
 * applied anywhere (grow to T on every rank and call again).  With d_all_offsets = NULL on every rank the call is a size query:
 * it returns T and applies nothing.  Every rank returns the same verdict: an argument error on any rank (null arguments, bad
 * offsets, the map off the communicator's device), caps that differ, a size query on some ranks only, or robots per rank that do
 * not follow the striping make every rank fail with MPLB_ERR_ARG.  Returns after the replica is written. */
int64_t mplb_fleet_map_edit(mplb_comm *c, mplb_map *m, const void *d_cells3, const int64_t *offsets_local, int n_local, int value,
                            void *d_all_cells3, void *d_all_offsets, int64_t cap, void *stream);
/* mplb_lpa_plan_batch on this rank's n_local robots (grow-and-relaunch rounds included), then the gather of
 * mplb_plan_batch_sharded: the root receives results[n_total] and, when max_seg > 0, actions[n_total * max_seg] (the first
 * max_seg actions of each successful plan, -1 padded; -1 rows for the others) in robot order.  Every argument is checked before
 * any planner changes, and their verdicts are exchanged first (one small grouped exchange) so that every rank fails alike: null
 * arguments, a planner listed twice, a planner not on the communicator's device, n_local other than the number of robots the
 * striping gives this rank, LPA* off, n_total or max_seg differing between ranks.  On the other ranks results may be NULL; when it is not, it
 * receives their own n_local records in local order (actions is not written there). */
/* The scan and merge of mplb_fleet_map_edit for a caller that moves the payloads with its own transport (MPI,
 * torch.distributed): d_payloads holds the N ranks' payloads back to back (device int32 words; rank r's is payload_words[r]
 * words: the per-robot row counts of its stripe_count robots of n_total, then their rows of 3 ints).  Writes the robot-ordered
 * concatenation and its n_total + 1 offsets as mplb_fleet_map_edit does and returns its row count T (nothing written when
 * T > cap); counts that do not add up to a payload's rows fail with MPLB_ERR_ARG.  Ordered on `stream`; returns when done. */
int64_t mplb_fleet_merge_device(const void *d_payloads, const int64_t *payload_words, int nranks, int n_total, void *d_all_cells3,
                                void *d_all_offsets, int64_t cap, void *stream);
int mplb_fleet_plan(mplb_comm *c, mplb_planner **planners_local, int n_local, int n_total, const mplb_waypoint *starts_local,
                    const mplb_waypoint *goals_local, mplb_result *results, int32_t *actions, int max_seg, int root);

/* ---- VoxelGrid: the map builder of planning_ros_utils (include/planning_ros_utils/voxel_grid.h, src/mapping_utils/
 * voxel_grid.cpp, cited vg:<line>), the map store of mpl_test_node/src/cloud_to_map.cpp and map_replanner_node.cpp.  Both of
 * its int8 grids (map_ and inflated_map_) live on the device, x fastest, so a grid hands its map to an mplb_map without
 * leaving the device.  Every member gives the reference's result bit for bit (DESIGN.md section 4.13).  Where the reference
 * is undefined this library defines:
 *   - a point whose quotient (pt - origin) / res is NaN or beyond int32 is outside (cast<int> is undefined there);
 *   - clear_columns ignores a column outside the grid (clear(nx, ny), vg:31-33, does not check);
 *   - allocate fails with MPLB_ERR_ARG and changes nothing when a truncated dimension or origin is negative (dimensions
 *     only) or beyond int32, or when the grid would have more than 2^31 - 1 cells.
 * Host point buffers are rows of 3 doubles; device point buffers are rows of 3 floats (fp32 = 1) or doubles, widened to
 * double as the reference's vec_Vec3f does.  Calls are synchronous; `stream` (a cudaStream_t as void*, NULL = default)
 * orders the reads of a caller's device buffers. */
typedef struct mplb_voxel_grid mplb_voxel_grid;
/* VoxelGrid(origin, dim, res) (vg:3-10): the empty grid, then allocate(dim, origin) */
int mplb_voxel_grid_create(const double *origin, const double *dim_m, float res, mplb_voxel_grid **out);
void mplb_voxel_grid_destroy(mplb_voxel_grid *g);
/* allocate (vg:129-172): changed = 0 and nothing happens when the truncated geometry is unchanged; otherwise map_ is shifted
 * by the integer origins and inflated_map_ is RESET to the shifted map_ (changed = 1).  changed may be NULL. */
int mplb_voxel_grid_allocate(mplb_voxel_grid *g, const double *dim_m, const double *origin, int32_t *changed);
/* dim_ (3 ints), origin_ (3 ints), origin_d_ (3 doubles), res_; any pointer may be NULL */
int mplb_voxel_grid_get_info(const mplb_voxel_grid *g, int32_t *dim, int32_t *origin_i, double *origin_d, float *res);
int mplb_voxel_grid_clear(mplb_voxel_grid *g); /* clear() (vg:12-16): both grids free */
/* addCloud(pts) (vg:174-180): every inside point's cell of map_ becomes 100 */
int mplb_voxel_grid_add_cloud(mplb_voxel_grid *g, const double *pts, int64_t n);
int mplb_voxel_grid_add_cloud_device(mplb_voxel_grid *g, const void *d_pts, int64_t n, int fp32, void *stream);
/* addCloud(pts, ns) (vg:182-199): ns = n_ns rows of 3 ints.  Returns the length of the new_obs list (>= 0) or an error;
 * new_obs receives its first min(count, cap) cells as rows of 3 ints, in the reference's order.  A call emits a
 * cell at most once, so count <= the grid's cell count and a buffer of that many rows always suffices. */
int64_t mplb_voxel_grid_add_cloud_inflated(mplb_voxel_grid *g, const double *pts, int64_t n, const int32_t *ns, int n_ns,
                                           int32_t *new_obs, int64_t cap);
/* Same with device points (fp32 or fp64) and a device new_obs buffer; ns stays a host array */
int64_t mplb_voxel_grid_add_cloud_inflated_device(mplb_voxel_grid *g, const void *d_pts, int64_t n, int fp32, const int32_t *ns,
                                                  int n_ns, void *d_new_obs, int64_t cap, void *stream);
/* Points per internal pass of the inflated insertion (0 = the default, 2^22 candidate cells per pass, about 134 MB of scratch).  The passes run
 * one after another, which is exactly the sequential order, so this changes memory use and nothing else. */
int mplb_voxel_grid_set_chunk_points(mplb_voxel_grid *g, int64_t points);
int mplb_voxel_grid_decay(mplb_voxel_grid *g); /* decay() (vg:214-225): every cell > 0 of both grids is decremented */
/* n cells (rows of 3 ints) of map_: column = 1 is fill(nx, ny) (vg:35-39, the z of a row is ignored), column = 0 is
 * fill(nx, ny, nz) (vg:41-45); cells outside are ignored like the reference does */
int mplb_voxel_grid_fill(mplb_voxel_grid *g, const int32_t *cells3, int n, int column);
int mplb_voxel_grid_clear_columns(mplb_voxel_grid *g, const int32_t *cells3, int n); /* clear(nx, ny), vg:31-33, z ignored */
/* the same two with the n cell rows in device memory, read on `stream` */
int mplb_voxel_grid_fill_device(mplb_voxel_grid *g, const void *d_cells3, int n, int column, void *stream);
int mplb_voxel_grid_clear_columns_device(mplb_voxel_grid *g, const void *d_cells3, int n, void *stream);
/* getCloud (vg:18-29) / getLocalCloud (vg:47-69): centres of the cells > 0 of map_ / inflated_map_ (the local box), x outermost
 * and z innermost.  Return the number of points and write the first min(count, cap) rows of 3 doubles. */
int64_t mplb_voxel_grid_get_cloud(mplb_voxel_grid *g, double *pts, int64_t cap);
int64_t mplb_voxel_grid_get_local_cloud(mplb_voxel_grid *g, const double *pos, const double *ori, const double *dim,
                                        double *pts, int64_t cap);
/* getMap / getInflatedMap (vg:71-127) data: 100 where the cell is > 0, else 0, x fastest; cap >= the cell count */
int mplb_voxel_grid_get_map(mplb_voxel_grid *g, int inflated, int8_t *out, size_t cap);
/* setMap(map_util, getMap()) without leaving the device: m must be 3D with the grid's dims, origin origin_d_ and res
 * (double)res_ (MPLB_ERR_ARG otherwise).  Its cells are rewritten in place and its bricks rebuilt, as by mplb_map_set_data, so
 * planners sharing m see the change. */
int mplb_voxel_grid_write_map(mplb_voxel_grid *g, int inflated, mplb_map *m);
/* a new mplb_map of the grid's geometry holding getMap / getInflatedMap, built device to device */
int mplb_voxel_grid_create_map(mplb_voxel_grid *g, int inflated, mplb_map **out);
/* MapUtil cell values for n cells (rows of 3 ints, the third ignored in 2D): the int8 value, or INT32_MIN outside the map
 * (the material of isFree / isOccupied / isUnknown, map_util.h:44-80) */
int mplb_map_get_cells(const mplb_map *m, const int32_t *cells3, int n, int32_t *values);
/* MapUtil::rayTrace (map_util.h:117-134) for n_rays rays, and the cell selection of the replanner node's edits
 * (map_replanner_node.cpp:199-229), on the device.  Ray i goes from p1s[i] to p2s[i] (rows of 3 doubles; a 2D map reads the
 * first two) and traces exactly rayTrace's cells: points n = 1 .. max_diff - 1, up to the first point outside the map, a point
 * whose cell equals the previous point's dropped.  For every traced cell pn in trace order and every stencil offset ns[k] in
 * the order given (n_ns rows of 3 ints, the third ignored in 2D; ns = NULL with n_ns = 0 is the single offset 0), the
 * candidate pn + ns[k] is kept
 *   MPLB_TRACE_ALL       always (with the offset 0 alone: rayTrace itself),
 *   MPLB_TRACE_FREE      when it is inside the map and 0 <= value < 100 (isFree, map_util.h:44,57-62),
 *   MPLB_TRACE_OCCUPIED  when it is inside the map and value == 100 (isOccupied, map_util.h:48,64-69),
 * with the map's values at the call.  Duplicates from overlapping stencils stay, as in the node's new_obs list.  Returns the total
 * count (or an error) and writes the first min(count, cap) cells as rows of 3 ints (the third 0 in 2D); offsets (may be NULL)
 * receives n_rays + 1 entries, ray i owning rows offsets[i] .. offsets[i+1]-1.  An endpoint that is not finite, or a ray whose
 * q / 0.8 (its longest axis in cells over 0.8) is 2^31 or more, where the reference's (int) cast is undefined, fails the call
 * with MPLB_ERR_ARG, and so does a call with more than 2^31 - 1 candidates to examine (n_rays x max(n_ns, 1) x the points a ray
 * can have inside the map, about 1.25 x its longest side in cells).  The _device variant takes the endpoints, cells and offsets in device memory (ns stays a host array) and
 * orders its work on `stream`; the count is its one read-back. */
enum { MPLB_TRACE_ALL = 0, MPLB_TRACE_FREE = 1, MPLB_TRACE_OCCUPIED = 2 };
int64_t mplb_map_trace_cells(const mplb_map *m, const double *p1s, const double *p2s, int n_rays, const int32_t *ns, int n_ns,
                             int select, int32_t *cells3, int64_t cap, int64_t *offsets);
int64_t mplb_map_trace_cells_device(const mplb_map *m, const void *d_p1s, const void *d_p2s, int n_rays, const int32_t *ns, int n_ns,
                                    int select, void *d_cells3, int64_t cap, void *d_offsets, void *stream);

#ifdef __cplusplus
}
#endif
#endif
