"""CPU-side checks of a fleet cycle's device output: libmplb.so exports mplb_lpa_plan_batch_device,
mplb_lpa_trajectory_waypoints_device, mplb_lpa_serialize_trajectories_device and mplb_lpa_refine_trajectories_device with the
arity include/mplb.h declares, and the Python and C++ bindings have their members."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CALLS = ("mplb_lpa_plan_batch_device", "mplb_lpa_trajectory_waypoints_device", "mplb_lpa_serialize_trajectories_device",
         "mplb_lpa_refine_trajectories_device")
MEMBERS = ("planLPABatchDevice", "trajectoryWaypointsBatch", "serializeLPABatch", "refineLPABatch")


def test_device_cycle_exports_are_present():
    from mpl_ros_b200.build import build_lib
    from mpl_ros_b200 import _lib
    build_lib()
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "mplb.h")).read()
    for name in CALLS:
        assert hasattr(L, name), name
        decl = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\);", hdr)
        assert decl, name
        assert decl.group(1).count(",") + 1 == len(_lib.SYMBOLS[name][1]), name


def test_bindings_have_the_members():
    import mpl_ros_b200 as mp
    for m in MEMBERS:
        assert callable(getattr(mp.MapPlanner, m)), m
    hpp = open(os.path.join(ROOT, "include", "mpl_b200", "map_planner.hpp")).read()
    for m in MEMBERS:
        assert re.search(r"static bool " + m + r"\(", hpp), m
