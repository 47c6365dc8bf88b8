#!/usr/bin/env python3
"""Diagnostics: build libmplb with -DMPLB_PHASE_TIMING into a separate .so, run the bench batch once and print
the clock64() cycle accumulators of thread 0 (search warp).  The TOTAL cycles per pop is reliable; the per-phase
split is only indicative (clock64 is not ordered with barriers) — use the barrier-stall samples of an ncu capture for
phase durations.  Not part of the product."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from mpl_ros_b200 import build as B  # noqa: E402

out = os.path.join(ROOT, "mpl_ros_b200", os.environ.get("MPLB_PROF_SO", "libmplb_prof.so"))
if "--build-only" in sys.argv or not os.path.exists(out):
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")] + B.NVCC_FLAGS + ["-DMPLB_PHASE_TIMING=" + os.environ.get("MPLB_PT", "1")] + os.environ.get("MPLB_DEFS", "").split() + ["-o", out] + [os.path.join(B.CSRC, u) for u in B.UNITS])
    if "--build-only" in sys.argv:
        sys.exit(0)
from mpl_ros_b200 import _lib  # noqa: E402
_lib.LIB_PATH = out
import mpl_ros_b200 as mp  # noqa: E402
from mpl_ros_b200 import maps  # noqa: E402
from mpl_ros_b200 import workloads as W  # noqa: E402

# usage: phase_timing.py [max_slots] [--c5 N_QUERIES]  (default: the first 1024 queries of the C2 list)
c5 = "--c5" in sys.argv
spec = W.C5 if c5 else W.C2
nq = int(sys.argv[sys.argv.index("--c5") + 1]) if c5 else 1024
m = W.c5_map() if c5 else W.c2_map()
mu = mp.VoxelMapUtil(); mu.setMap(m.origin, m.dim, m.data, m.res); mu.freeUnknown()
pl = mp.VoxelMapPlanner(False); pl.setMapUtil(mu)
P = spec["params"]
pl.setVmax(P["v_max"]); pl.setAmax(P["a_max"]); pl.setDt(P["dt"]); pl.setU(W.controls(spec)); pl.setTol(P["tol_pos"])
if "max_num" in P:
    pl.setMaxNum(int(os.environ.get("MPLB_MAX_NUM", P["max_num"])))
if c5:
    pl.setMemFraction(0.85)
S, G = (W.c5_queries if c5 else W.c2_queries)(m, nq)
s, g = mp.waypoints_array(nq), mp.waypoints_array(nq)
W.fill(s, g, S, G, spec["control"])
if len(sys.argv) > 1 and sys.argv[1].isdigit():
    pl.setMaxSlots(int(sys.argv[1]))
    print('max_slots', sys.argv[1])
for _ in range(1 if c5 else 2):
    res, _, _ = pl.plan_batch(s, g, max_seg=64)
print("kernel_ms", pl.last_batch_stats())
ph16 = np.zeros((len(s), 16), dtype=np.int64)
L = _lib.lib()
L.mplb_debug_phase_cycles.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
assert L.mplb_debug_phase_cycles(pl._h, ph16.ctypes.data_as(C.c_void_p), len(s)) == 0
ph = ph16[:, :8]
dbg = ph16[:, 8:]
print('dbg per pop', (dbg.sum(axis=0) / res['pops'].sum()).astype(int).tolist())
print('per pop: decide cycles %.0f  store cycles %.0f  granules evaluated %.1f  hazards %.4f  exact samples %.3f' % tuple(dbg[:, k].sum() / res['pops'].sum() for k in (0, 1, 2, 3, 4)))
names = ["P1 (miss path only) + bar1", "P2 probe issue + h + resolve", "P2 (unused)", "P2 wait at bar 2", "P3 relax: decide+stores",
         "P3 relax: heap ops", "P3 terminate+pop", "loop top (barrier C + checks)"]
pops = res["pops"].astype(np.float64)
tot = ph.sum()
print("total pops", int(pops.sum()), "cycles/pop (all plans)", tot / pops.sum())
for k, nm in enumerate(names):
    print("%-28s %6.1f%%  %8.0f cyc/pop" % (nm, 100.0 * ph[:, k].sum() / tot, ph[:, k].sum() / pops.sum()))
big = np.argsort(-pops)[:5]
for i in big:
    print("plan", i, "pops", int(pops[i]), "cycles/pop", ph[i].sum() / pops[i], (ph[i] / pops[i]).astype(int).tolist())
