"""mpl_ros_b200 — H100-native drop-in for the A* hot path of sikang/mpl_ros.

Public surface (mirrors the reference's class names, see planner.py): MapUtil / OccMapUtil / VoxelMapUtil,
Waypoint, Primitive, Trajectory, MapPlanner / OccMapPlanner / VoxelMapPlanner, TrajSolver, VoxelGrid (voxel_grid.py).  The compute lives in
libmplb.so (hand-written sm_90a CUDA behind the C ABI of include/mplb.h); importing this package does not
load it, the first call does, and it raises if the library or a CUDA device is missing.
"""
from . import maps  # noqa: F401
from .planner import (ACC, ACCxYAW, JRK, JRKxYAW, SNP, SNPxYAW, VEL, VELxYAW, MapPlanner, MapUtil, MplbError, OccMapPlanner, OccMapUtil, Primitive,  # noqa: F401
                      TRACE_ALL, TRACE_FREE, TRACE_OCCUPIED, Trajectory, VoxelMapPlanner, VoxelMapUtil, Waypoint, waypoints_array)
from .traj_solver import TrajSolver, TrajSolver2D, TrajSolver3D  # noqa: F401,E402
from .voxel_grid import VoxelGrid  # noqa: F401,E402
