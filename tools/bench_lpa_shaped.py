"""LPA* replanning with a potential map and with yaw controls on the GPU: the time of one replan after a map edit (block the
cells around the middle of the trajectory, getLinkedNodes, updateBlockedNodes, then the timed plan) for plain, potential and yaw
replanners on corridor (tests/lpa_shaped_flow.py settings), single (median of REPS fresh replanners) and as a batch of 64 in one
mplb_lpa_plan_batch.  Each timed call ends in a device synchronise (the library synchronises before returning).  Prints the card's
name and power limit, then one JSON object.  Run on a machine with the GPU:  python tools/bench_lpa_shaped.py"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpl_ros_b200 as mp  # noqa: E402
from mpl_ros_b200 import _lib  # noqa: E402
import lpa_flow  # noqa: E402
import lpa_shaped_flow as F  # noqa: E402
from test_gpu_lpa_shaped import GpuMap, GpuPlanner  # noqa: E402

REPS = 5
KINDS = {"plain": "corridor_plain", "potential": "corridor_pot_grad", "yaw": "corridor_yaw"}
F.FLOWS.setdefault("corridor_plain", dict(config="corridor", control=F.ACC, params={}))


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def prepared(kind):
    """a replanner after its first plan, with cells blocked across the middle of its trajectory and reported"""
    f = F.FLOWS[kind]
    m, mp_, pl, dim, start, goal = F.build(kind, GpuMap, GpuPlanner)
    if f.get("pot"):
        pl.update_potential_map(np.r_[start, 0.0])
    s = F.waypoints(start, f["control"], f.get("start_yaw", 0.0))
    g = F.waypoints(goal, f["control"], 0.0)
    r = pl.lpa_plan(s, g)
    assert int(r["status"]) == 0, (kind, r)
    path = pl.lpa_best_child_states()[:, :3]
    pl.lpa_get_linked_nodes()
    cells = lpa_flow.cells_on_path(m, dim, path[len(path) // 2:len(path) // 2 + 1], 2)
    mp_.set_cells(cells, 100)
    pl.lpa_update_blocked_nodes(cells)
    return pl, s, g


def single(kind):
    t, pops = [], 0
    for _ in range(REPS):
        pl, s, g = prepared(kind)
        t0 = time.perf_counter()
        r = pl.lpa_plan(s, g)
        t.append(time.perf_counter() - t0)
        pops = int(r["pops"])
    return dict(replan_ms_median=float(np.median(t)) * 1e3, replan_ms_min=min(t) * 1e3, replan_pops=pops)


def batch(kind, n=64):
    items = [prepared(kind) for _ in range(n)]
    s, g = mp.waypoints_array(n), mp.waypoints_array(n)
    for i, (pl, si, gi) in enumerate(items):
        for f in ("pos", "vel", "acc", "jrk", "yaw", "control"):
            s[f][i], g[f][i] = si[f][0], gi[f][0]
    res = np.zeros(n, dtype=_lib.RESULT_DTYPE)
    handles = (C.c_void_p * n)(*[it[0].pl._h for it in items])
    t0 = time.perf_counter()
    _lib.check(_lib.lib().mplb_lpa_plan_batch(handles, n, _lib.ptr(s), _lib.ptr(g), _lib.ptr(res)))
    dt = time.perf_counter() - t0
    return dict(batch=n, replan_ms=dt * 1e3, pops_total=int(res["pops"].sum()), ok=int((res["status"] == 0).sum()))


def main():
    print("card: " + card(), flush=True)
    prepared("corridor_plain")  # warm-up: module load, first allocations
    out = {}
    for tag, kind in KINDS.items():
        out[tag] = dict(single=single(kind), batch64=batch(kind))
    print(json.dumps(dict(card=card(), lpa_replan_after_edit=out)))


if __name__ == "__main__":
    main()
