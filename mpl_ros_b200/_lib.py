"""ctypes loader for libmplb.so (the C ABI declared in include/mplb.h).

The library is built in-tree by __graft_entry__.build() / mpl_ros_b200.build.build_lib().  There is no
fallback of any kind: if the shared object is missing or a CUDA call fails, an exception is raised.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libmplb.so")

WAYPOINT_DTYPE = np.dtype([("pos", "f8", 3), ("vel", "f8", 3), ("acc", "f8", 3), ("jrk", "f8", 3),
                           ("yaw", "f8"), ("t", "f8"), ("control", "i4"), ("enable_t", "i4")], align=True)
RESULT_DTYPE = np.dtype([("status", "i4"), ("n_seg", "i4"), ("cost", "f8"), ("pops", "i4"), ("n_nodes", "i4"),
                         ("n_open", "i4"), ("n_closed", "i4"), ("n_prims", "i8"), ("n_samples", "i8"),
                         ("n_valid", "i8"), ("pop_hash", "u8"), ("closed_hash", "u8"), ("device_ms", "f8")], align=True)
TRACE_DTYPE = np.dtype([("verdict", "i4"), ("n", "i4"), ("n_tested", "i4"), ("block_idx", "i4"), ("cost", "f8"),
                        ("succ", "f8", 13), ("key", "i4", 16)], align=True)
PROBE_DTYPE = np.dtype([("state", "i4"), ("control", "i4"), ("k", "i4"), ("sure", "i4"), ("cell_fast", "i4", 3),
                        ("cell_exact", "i4", 3), ("t", "f8"), ("w", "f8", 3)], align=True)
NODE_DTYPE = np.dtype([("state", "f8", 13), ("g", "f8"), ("h", "f8"), ("key", "i4", 16), ("opened", "i4"),
                       ("closed", "i4"), ("parent", "i4"), ("action", "i4")], align=True)
LPA_NODE_DTYPE = np.dtype([("key", "i4", 16), ("state", "f8", 13), ("g", "f8"), ("rhs", "f8"), ("h", "f8"), ("opened", "i4"),
                           ("closed", "i4"), ("n_succ", "i4"), ("n_pred", "i4"), ("succ_hash", "u8"), ("pred_hash", "u8")], align=True)
LPA_HEAP_DTYPE = np.dtype([("fval", "f8"), ("key_hash", "u8")], align=True)
TIER_DTYPE = np.dtype([("cap", "i4"), ("slots", "i4"), ("n_work", "i4"), ("n_overflow", "i4"), ("hcap", "i4"), ("load_inv", "i4"),
                       ("tsize_max", "i4"), ("log_cap", "i4"), ("stride_bytes", "i8"), ("nomem", "i4"), ("ordered", "i4"),
                       ("resident", "i4"), ("reserved", "i4")], align=True)
TRAJ_STATS_DTYPE = np.dtype([("n_traj", "i4"), ("max_wp", "i4"), ("pos_shared", "i4"), ("pos_global", "i4"), ("yaw_shared", "i4"),
                             ("yaw_global", "i4"), ("smem_bytes", "i8"), ("global_bytes", "i8")], align=True)
assert WAYPOINT_DTYPE.itemsize == 120 and RESULT_DTYPE.itemsize == 80 and TIER_DTYPE.itemsize == 56
assert TRAJ_STATS_DTYPE.itemsize == 40

# every symbol include/mplb.h declares: (restype, argtypes)
_VP, _I, _D = C.c_void_p, C.c_int, C.c_double
SYMBOLS = {
    "mplb_last_error": (C.c_char_p, []),
    "mplb_device_count": (_I, []),
    "mplb_launch_count": (C.c_int64, []),
    "mplb_map_create": (_I, [_I, _VP, _VP, _D, _VP, _VP]),
    "mplb_map_create_from_device": (_I, [_I, _VP, _VP, _D, _VP, _VP, _VP]),
    "mplb_map_free_unknown": (_I, [_VP]),
    "mplb_map_dilate": (_I, [_VP, _VP, _I]),
    "mplb_map_get_info": (_I, [_VP, _VP, _VP, _VP, _VP]),
    "mplb_map_get_data": (_I, [_VP, _VP, C.c_size_t]),
    "mplb_map_destroy": (None, [_VP]),
    "mplb_planner_create": (_I, [_I, _I, _VP]),
    "mplb_planner_destroy": (None, [_VP]),
    "mplb_planner_set_map": (_I, [_VP, _VP]),
    "mplb_planner_set_param": (_I, [_VP, _I, _D]),
    "mplb_planner_set_controls": (_I, [_VP, _VP, _I, _I]),
    "mplb_planner_set_search_region": (_I, [_VP, _VP, C.c_size_t]),
    "mplb_planner_set_search_region_path": (_I, [_VP, _VP, _I, _I, _VP]),
    "mplb_planner_get_search_region": (C.c_int64, [_VP, _VP, C.c_size_t]),
    "mplb_planner_set_potential_map": (_I, [_VP, _VP, C.c_size_t]),
    "mplb_planner_update_potential_map": (_I, [_VP, _VP, _VP, _VP, _D]),
    "mplb_planner_set_prior_trajectory": (_I, [_VP, _I, _VP, _VP, _I]),
    "mplb_plan": (_I, [_VP, _VP, _VP, _VP]),
    "mplb_plan_batch": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _I]),
    "mplb_plan_batch_device": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _VP, _I, _VP]),
    "mplb_get_actions": (_I, [_VP, _VP, _I]),
    "mplb_get_seg_states": (_I, [_VP, _VP, _I]),
    "mplb_get_nodes": (_I, [_VP, _VP, _I]),
    "mplb_get_pop_log": (_I, [_VP, _VP, _I]),
    "mplb_get_open": (_I, [_VP, _VP, _I]),
    "mplb_expand": (_I, [_VP, _VP, _I, _VP]),
    "mplb_probe_samples": (_I, [_VP, _VP, _I, _VP, _I, _VP, _VP]),
    "mplb_planner_key_layout": (_I, [_VP, _I, _VP, _VP, _VP]),
    "mplb_last_batch_stats": (_I, [_VP, _VP, _VP, _VP]),
    "mplb_last_batch_tiers": (_I, [_VP, _VP, _I]),
    "mplb_comm_unique_id": (_I, [_VP]),
    "mplb_comm_create": (_I, [_VP, _I, _I, _VP]),
    "mplb_comm_destroy": (None, [_VP]),
    "mplb_comm_rank": (_I, [_VP]),
    "mplb_comm_size": (_I, [_VP]),
    "mplb_comm_broadcast_map": (_I, [_VP, _I, _I, _VP, _VP, _D, _VP, _VP]),
    "mplb_plan_batch_sharded": (_I, [_VP, _VP, _VP, _VP, _I, _VP, _VP, _I, _I]),
    "mplb_plan_stripe_gather_device": (_I, [_VP, _VP, _VP, _VP, _I, _I, _VP, _VP, _I, _I, _VP]),
    "mplb_comm_unstripe": (_I, [_VP, _I, _I, _I, _VP, _VP]),
    "mplb_plan_stripe_begin": (_I, [_VP, _VP, _VP, _I, _VP, _VP, _I, _VP]),
    "mplb_plan_stripe_end": (_I, [_VP, _VP, _I, _I]),
    "mplb_plan_batch_sharded_begin": (_I, [_VP, _VP, _VP, _VP, _I, _I]),
    "mplb_plan_batch_sharded_end": (_I, [_VP, _VP, _I, _VP, _VP, _I]),
    "mplb_sincos_cr": (_I, [_VP, _I, _VP, _VP]),
    "mplb_planner_set_lpastar": (_I, [_VP, _I]),
    "mplb_planner_reset": (_I, [_VP]),
    "mplb_map_set_cells": (_I, [_VP, _VP, _I, _I]),
    "mplb_map_set_data": (_I, [_VP, _VP]),
    "mplb_get_sub_state_space": (_I, [_VP, _I]),
    "mplb_get_linked_nodes": (_I, [_VP, _VP, _I]),
    "mplb_update_blocked_nodes": (_I, [_VP, _VP, _I]),
    "mplb_update_cleared_nodes": (_I, [_VP, _VP, _I]),
    "mplb_lpa_plan_batch": (_I, [_VP, _I, _VP, _VP, _VP]),
    "mplb_lpa_get_nodes": (_I, [_VP, _VP, _I]),
    "mplb_lpa_get_heap": (_I, [_VP, _VP, _I]),
    "mplb_lpa_get_best_child": (_I, [_VP, _VP, _I]),
    "mplb_lpa_get_capacity": (_I, [_VP, _VP, _VP, _VP, _VP, _VP]),
    "mplb_refine_trajectories_device": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _VP, _VP, _VP]),
    "mplb_refine_trajectories": (_I, [_VP, _VP, _VP, _VP, _I, _I, _I, _I, _I, _VP, _VP]),
    "mplb_traj_solve_batch": (_I, [_I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "mplb_traj_solve_batch_device": (_I, [_I, _I, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "mplb_traj_solve_last_stats": (_I, [_VP]),
    "mplb_trajectory_msg_size": (C.c_size_t, [_I, C.c_char_p]),
    "mplb_serialize_trajectories_device": (_I, [_VP, _VP, _VP, _VP, _I, _I, _D, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p,
                                                _VP, C.c_size_t, _VP, _VP]),
    "mplb_serialize_trajectories": (_I, [_VP, _VP, _VP, _VP, _I, _I, _D, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p,
                                         _VP, C.c_size_t, _VP]),
    "mplb_voxel_grid_create": (_I, [_VP, _VP, C.c_float, _VP]),
    "mplb_voxel_grid_destroy": (None, [_VP]),
    "mplb_voxel_grid_allocate": (_I, [_VP, _VP, _VP, _VP]),
    "mplb_voxel_grid_get_info": (_I, [_VP, _VP, _VP, _VP, _VP]),
    "mplb_voxel_grid_clear": (_I, [_VP]),
    "mplb_voxel_grid_add_cloud": (_I, [_VP, _VP, C.c_int64]),
    "mplb_voxel_grid_add_cloud_device": (_I, [_VP, _VP, C.c_int64, _I, _VP]),
    "mplb_voxel_grid_add_cloud_inflated": (C.c_int64, [_VP, _VP, C.c_int64, _VP, _I, _VP, C.c_int64]),
    "mplb_voxel_grid_add_cloud_inflated_device": (C.c_int64, [_VP, _VP, C.c_int64, _I, _VP, _I, _VP, C.c_int64, _VP]),
    "mplb_voxel_grid_set_chunk_points": (_I, [_VP, C.c_int64]),
    "mplb_voxel_grid_decay": (_I, [_VP]),
    "mplb_voxel_grid_fill": (_I, [_VP, _VP, _I, _I]),
    "mplb_voxel_grid_clear_columns": (_I, [_VP, _VP, _I]),
    "mplb_voxel_grid_get_cloud": (C.c_int64, [_VP, _VP, C.c_int64]),
    "mplb_voxel_grid_get_local_cloud": (C.c_int64, [_VP, _VP, _VP, _VP, _VP, C.c_int64]),
    "mplb_voxel_grid_get_map": (_I, [_VP, _I, _VP, C.c_size_t]),
    "mplb_voxel_grid_write_map": (_I, [_VP, _I, _VP]),
    "mplb_voxel_grid_create_map": (_I, [_VP, _I, _VP]),
    "mplb_map_get_cells": (_I, [_VP, _VP, _I, _VP]),
    "mplb_map_set_cells_device": (_I, [_VP, _VP, _I, _I, _VP]),
    "mplb_voxel_grid_fill_device": (_I, [_VP, _VP, _I, _I, _VP]),
    "mplb_voxel_grid_clear_columns_device": (_I, [_VP, _VP, _I, _VP]),
    "mplb_map_trace_cells": (C.c_int64, [_VP, _VP, _VP, _I, _VP, _I, _I, _VP, C.c_int64, _VP]),
    "mplb_map_trace_cells_device": (C.c_int64, [_VP, _VP, _VP, _I, _VP, _I, _I, _VP, C.c_int64, _VP, _VP]),
    "mplb_lpa_get_linked_nodes_batch": (_I, [_VP, _I, _VP, _VP, C.c_int64]),
    "mplb_lpa_update_nodes_batch": (_I, [_VP, _I, _I, _VP, _VP, _VP]),
    "mplb_lpa_update_nodes_batch_device": (_I, [_VP, _I, _I, _VP, _VP, _VP]),
    "mplb_lpa_sub_state_space_batch": (_I, [_VP, _I, _VP, _VP]),
    "mplb_fleet_map_edit": (C.c_int64, [_VP, _VP, _VP, _VP, _I, _I, _VP, _VP, C.c_int64, _VP]),
    "mplb_fleet_merge_device": (C.c_int64, [_VP, _VP, _I, _I, _VP, _VP, C.c_int64, _VP]),
    "mplb_fleet_plan": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _I, _I]),
    "mplb_lpa_plan_batch_device": (_I, [_VP, _I, _VP, _VP, _VP, _VP, _VP, _I, _VP]),
    "mplb_lpa_trajectory_waypoints_device": (_I, [_VP, _I, _VP, _VP, _VP, _I, _VP, _VP, _VP, _VP]),
    "mplb_lpa_serialize_trajectories_device": (_I, [_VP, _I, _VP, _VP, _VP, _I, _D, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p,
                                                    _VP, C.c_size_t, _VP, _VP]),
    "mplb_lpa_refine_trajectories_device": (_I, [_VP, _I, _VP, _VP, _VP, _I, _I, _I, _VP, _VP, _VP]),
}
TRACE_ALL, TRACE_FREE, TRACE_OCCUPIED = 0, 1, 2  # mplb_map_trace_cells selections

PARAM = dict(v_max=0, a_max=1, j_max=2, yaw_max=3, dt=4, w=5, epsilon=6, max_num=7, tol_pos=8, tol_vel=9,
             tol_acc=10, t_max=11, potential_weight=12, gradient_weight=13, wyaw=14, mem_fraction=100, max_slots=101, exact_preds=102,
             arena_bytes=103, lpa_init_nodes=104, lpa_init_preds=105)

_LIB = None


class MplbError(RuntimeError):
    pass


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise MplbError("libmplb.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "— there is no CPU fallback" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the ABI lost a symbol
            fn.restype = res
            fn.argtypes = args
        _LIB = L
    return _LIB


def check(rc):
    if rc < 0:
        raise MplbError("mplb error %d: %s" % (rc, lib().mplb_last_error().decode()))
    return rc


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)
