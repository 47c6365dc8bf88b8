"""One replan cycle of a fleet of N LPA* replanners (map_replanner_node.cpp's add-cloud callback for every robot), timed two ways:
the batched calls (getLinkedNodesBatch, updateBlockedNodesBatch, planLPABatch, getSubStateSpaceBatch) and the same calls looped
one planner at a time.  Every robot has its own map; its edit is the node's: trace a ray across the middle of its trajectory on
the device, keep the isFree cells of a 3 x 3 stencil, write them as obstacles (mplb_map_set_cells_device).  The cycle is then
getLinkedNodes, updateBlockedNodes, plan, getSubStateSpace(1) (start = the next waypoint), plan.

For N in (1, 8, 64, 256) on the skir and simple configurations the two modes run CYCLES cycles each, alternating in one process,
and must leave identical states (hm_ dump, heap, best_child_ of every planner).  Each call ends in a device synchronise (the
library synchronises before returning).  Prints the card's name and power limit, then one JSON line per (config, N) with the
median ms per cycle and the kernel launches per cycle (mplb_launch_count) of both modes.
Run on a machine with the GPU:  python tools/bench_lpa_fleet.py [--sizes 1,8,64,256] [--cycles 4]"""
import argparse
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
from helpers import fill_waypoints, load_config  # noqa: E402

NS3 = np.array([(x, y, 0) for x in range(-1, 2) for y in range(-1, 2)], dtype=np.int32)


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


class Robot:
    def __init__(self, cfg, k):
        m, dim, params, U, start, goal = load_config(cfg)
        self.dim = dim
        self.mu = mp.MapUtil(dim)
        self.mu.setMap(m.origin, m.dim, m.data, m.res)
        self.mu.freeUnknown()
        self.pl = mp.MapPlanner(dim)
        self.pl.setMapUtil(self.mu)
        for key, v in params.items():
            (self.pl.setDt if key == "dt" else lambda x, key=key: self.pl._set(key, x))(v)
        self.pl.setU(U)
        self.pl.setLPAInitNodes(4096)  # arrays double as needed: results do not depend on it, memory for 512 replanners does
        self.pl.setLPAInitPreds(65536)
        self.pl.setLPAstar(True)
        self.s, self.g = mp.waypoints_array(1), mp.waypoints_array(1)
        fill_waypoints(self.s, start, mp.ACC)
        fill_waypoints(self.g, goal, mp.ACC)
        self.k = k

    def edit(self):
        """the node's add-cloud edit on the device: ray across the trajectory's middle, isFree cells of the stencil -> 100"""
        import torch
        best = self.pl.lpaBestChild()["state"][:, :3]
        if len(best) < 4:
            return
        a, b = best[len(best) // 3].copy(), best[2 * len(best) // 3].copy()
        d1, d2 = torch.tensor(a[None], device="cuda"), torch.tensor(b[None], device="cuda")
        cap = 4096
        dc = torch.zeros((cap, 3), dtype=torch.int32, device="cuda")
        vp = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        n = _lib.check(_lib.lib().mplb_map_trace_cells_device(self.mu._h, vp(d1), vp(d2), 1, _lib.ptr(NS3), len(NS3), mp.TRACE_FREE,
                                                             vp(dc), cap, None, None))
        self.cells = dc[:min(n, cap)].cpu().numpy()
        _lib.check(_lib.lib().mplb_map_set_cells_device(self.mu._h, vp(dc), min(n, cap), 100, None))


def cycle(robots, batched):
    pls = [r.pl for r in robots]
    for r in robots:
        r.edit()
    cells = [getattr(r, "cells", np.zeros((0, 3), dtype=np.int32)) for r in robots]
    if batched:
        mp.MapPlanner.getLinkedNodesBatch(pls)
        mp.MapPlanner.updateBlockedNodesBatch(pls, cells)
        mp.MapPlanner.planLPABatch(pls, [r.s[0] for r in robots], [r.g[0] for r in robots])
    else:
        for r, c in zip(robots, cells):
            r.pl.getLinkedNodes()
            r.pl.updateBlockedNodes(c)
            r.pl.plan(r.s, r.g)
    nxt = []
    for r in robots:
        st = r.pl.lpaBestChild()["state"]
        w = None
        if len(st) > 2:
            w = mp.waypoints_array(1)
            w["pos"][0], w["vel"][0], w["acc"][0], w["control"] = st[1, 0:3], st[1, 3:6], st[1, 6:9], mp.ACC
        nxt.append(w)
    if batched:
        mp.MapPlanner.getSubStateSpaceBatch(pls, [1 if w is not None else 0 for w in nxt])
    else:
        for r, w in zip(robots, nxt):
            r.pl.getSubStateSpace(1 if w is not None else 0)
    for r, w in zip(robots, nxt):
        if w is not None:
            r.s = w
    if batched:
        mp.MapPlanner.planLPABatch(pls, [r.s[0] for r in robots], [r.g[0] for r in robots])
    else:
        for r in robots:
            r.pl.plan(r.s, r.g)


def state(r):
    return (r.pl.lpaNodes().tobytes(), r.pl.lpaHeap().tobytes(), r.pl.lpaBestChild().tobytes())


def run(cfg, n, cycles):
    sets = {mode: [Robot(cfg, i) for i in range(n)] for mode in ("batched", "looped")}
    for mode, rs in sets.items():  # the first plan (an A*-sized search) is not part of the cycle
        mp.MapPlanner.planLPABatch([r.pl for r in rs], [r.s[0] for r in rs], [r.g[0] for r in rs])
    t = {m: [] for m in sets}
    launches = {m: [] for m in sets}
    L = _lib.lib()
    for c in range(cycles):
        for mode in (("batched", "looped") if c % 2 == 0 else ("looped", "batched")):
            l0 = L.mplb_launch_count()
            t0 = time.perf_counter()
            cycle(sets[mode], mode == "batched")
            t[mode].append((time.perf_counter() - t0) * 1e3)
            launches[mode].append(int(L.mplb_launch_count() - l0))
        for a, b in zip(sets["batched"], sets["looped"]):
            assert state(a) == state(b), (cfg, n, c)
    return {m: dict(ms_per_cycle=float(np.median(t[m])), ms_min=float(min(t[m])), launches_per_cycle=float(np.median(launches[m])))
            for m in sets}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64,256")
    ap.add_argument("--cycles", type=int, default=4)
    ap.add_argument("--configs", default="skir,simple")
    a = ap.parse_args()
    cd = card()
    print("card: " + cd, flush=True)
    run("skir", 1, 1)  # warm-up: module load, first allocations
    for cfg in a.configs.split(","):
        for n in (int(x) for x in a.sizes.split(",")):
            print(json.dumps(dict(card=cd, config=cfg, replanners=n, cycles=a.cycles, **run(cfg, n, a.cycles))), flush=True)


if __name__ == "__main__":
    main()
