"""CPU-side checks of the sharded fleet's entry points: libmplb.so exports mplb_fleet_map_edit and mplb_fleet_plan with the
signatures include/mplb.h declares, and the bindings know them."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLEET = ("mplb_fleet_map_edit", "mplb_fleet_merge_device", "mplb_fleet_plan")


def test_fleet_exports_are_present():
    from mpl_ros_b200.build import build_lib
    from mpl_ros_b200 import _lib
    build_lib()
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "mplb.h")).read()
    for name in FLEET:
        assert hasattr(L, name), name
        decl = re.search(r"\b(int64_t|int)\s+" + name + r"\s*\(([^;]*)\);", hdr)
        assert decl, name
        assert decl.group(2).count(",") + 1 == len(_lib.SYMBOLS[name][1]), name
    assert re.search(r"int64_t\s+mplb_fleet_map_edit", hdr)
