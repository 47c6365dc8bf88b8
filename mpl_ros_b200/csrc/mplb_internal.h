/* mplb_internal.h — host helpers the translation units of libmplb.so share (not part of the ABI). */
#ifndef MPLB_INTERNAL_H
#define MPLB_INTERNAL_H
#include <stdint.h>
#if defined(__GNUC__)
#define MPLB_HIDDEN __attribute__((visibility("hidden")))
#else
#define MPLB_HIDDEN
#endif
/* records `msg` for mplb_last_error() and returns `code` */
MPLB_HIDDEN int mplb_internal_fail(int code, const char *msg);
/* adds to the counter behind mplb_launch_count() */
MPLB_HIDDEN void mplb_internal_count_launches(int n);

/* ---- what the LPA* unit (mplb_lpa.cu) needs from the planner / map objects of mplb.cu */
struct mplb_planner;
struct mplb_result;
struct mplb_waypoint;
struct MplbLpaHostCfg {
  int dim, nU, max_num, device, verbose, has_map;
  int shaped; /* potential map / search region / prior trajectory / yaw controls installed: not available under LPA* */
  int lpa_init_nodes, lpa_init_preds; /* MPLB_LPA_INIT_NODES / MPLB_LPA_INIT_PREDS */
  double v_max, a_max, j_max, dt, w, eps, tol_pos, tol_vel, tol_acc;
  int nd[3];
  double origin[3];
  double res;
  const int8_t *d_grid; /* the map's int8 cells on the planner's device */
  const double *U;      /* host, nU rows of 3 */
  const double *Uyaw;   /* host, nU yaw rates, or NULL when the control rows carry none */
};
MPLB_HIDDEN int mplb_internal_planner_cfg(mplb_planner *p, MplbLpaHostCfg *out);
/* the retained single plan the getters mplb_get_actions / mplb_get_seg_states serve */
MPLB_HIDDEN void mplb_internal_set_retained(mplb_planner *p, const mplb_result *res, const int *actions, const double *segs13, int n_seg);
/* implemented by mplb_lpa.cu, called by mplb.cu */
MPLB_HIDDEN int mplb_internal_lpa_enabled(mplb_planner *p);
MPLB_HIDDEN int mplb_internal_lpa_plan(mplb_planner *p, const mplb_waypoint *start, const mplb_waypoint *goal, mplb_result *out);
MPLB_HIDDEN void mplb_internal_lpa_drop(mplb_planner *p);

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
#endif
