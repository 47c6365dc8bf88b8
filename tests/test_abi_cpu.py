"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/mplb.h
declares; no compute call is made (there is no GPU here and no CPU fallback to call)."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from mpl_ros_b200.build import build_lib
    from mpl_ros_b200 import _lib
    build_lib()
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "mplb.h")).read()
    declared = set(re.findall(r"\b(mplb_[a-z_]+)\s*\(", hdr))
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    for name in declared:
        assert hasattr(L, name), name


def test_struct_layouts_match_header():
    from mpl_ros_b200 import _lib
    import oracle
    assert _lib.WAYPOINT_DTYPE.itemsize == 120 and _lib.RESULT_DTYPE.itemsize == 80
    assert _lib.TRACE_DTYPE.itemsize == 4 * 4 + 8 + 13 * 8 + 16 * 4
    assert _lib.PROBE_DTYPE.itemsize == 4 * 4 + 6 * 4 + 8 + 3 * 8
    # the oracle mirrors the same layouts so tests can share buffers
    assert oracle.WAYPOINT_DTYPE == _lib.WAYPOINT_DTYPE and oracle.RESULT_DTYPE == _lib.RESULT_DTYPE


def test_traj_solve_stats_layout():
    """mplb_traj_solve_stats: six int32 counters, then two int64 byte counts (include/mplb.h)."""
    from mpl_ros_b200 import _lib
    d = _lib.TRAJ_STATS_DTYPE
    assert d.itemsize == 40 and d.fields["smem_bytes"][1] == 24 and d.fields["global_bytes"][1] == 32
    hdr = open(os.path.join(ROOT, "include", "mplb.h")).read()
    body = hdr[hdr.index("typedef struct mplb_traj_solve_stats"):hdr.index("} mplb_traj_solve_stats;")]
    assert re.findall(r"int(?:32|64)_t (\w+);", body) == list(d.names)


def test_no_device_is_a_loud_error():
    """Without a CUDA device the planner must fail, not fall back."""
    import pytest
    import mpl_ros_b200 as mp
    from mpl_ros_b200 import _lib
    if _lib.lib().mplb_device_count() > 0:
        pytest.skip("a GPU is visible")
    with pytest.raises(mp.MplbError):
        mp.VoxelMapPlanner(False)


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "mpl_ros_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".hpp")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "oracle/" not in src and "mpl_oracle" not in src, f


def test_device_memory_has_one_owner():
    """Every device allocation of libmplb goes through DevBuf in mplb_internal.h, which frees what it owns, and every CUDA
    error is reported by its one macro: no unit allocates or frees raw device memory or defines an error macro of its own."""
    csrc = os.path.join(ROOT, "mpl_ros_b200", "csrc")
    devbuf = 0
    for f in sorted(os.listdir(csrc)):
        if not f.endswith((".cu", ".cuh", ".h")):
            continue
        src = open(os.path.join(csrc, f)).read()
        devbuf += len(re.findall(r"\bstruct\s+(?:\w+\s+)?DevBuf\b\s*\{", src))
        if f == "mplb_internal.h":
            continue
        assert not re.search(r"\bcuda(?:Malloc|Free)\s*\(", src), f
        for name, body in re.findall(r"#define\s+(\w+)((?:[^\n]*\\\n)*[^\n]*)", src):
            assert not re.search(r"\bcudaError_t\b|\bcudaGetErrorString\b", body), (f, name)
    assert devbuf == 1
