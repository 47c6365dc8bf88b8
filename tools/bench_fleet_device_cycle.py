"""A fleet replan cycle whose output stays on the device, against the same cycle with today's per-robot readback.

The cycle is tools/bench_lpa_fleet.py's (the node's device ray-trace edit, getLinkedNodes, updateBlockedNodes, plan,
getSubStateSpace(1), plan from the next waypoint), with the node's output step after each plan: the planning_ros_msgs/Trajectory
wire bytes of every robot.  Two modes alternate in one process, each cycle ending in a device synchronise:
  host    planLPABatch, then per robot getActions / getSegStates, the message built on the host and the next start built from the
          retained trajectory (getWaypoints()[1], t = dt)
  device  planLPABatchDevice, serializeLPABatch, trajectoryWaypointsBatch (index 1) as the next cycle's device starts, and one
          read of the records to choose getSubStateSpace's time steps
Both modes must leave identical states (hm_ dump, heap, best_child_ of every planner) and identical messages.  Prints the card's
name and power limit, then one JSON line per (config, N) with the median ms per cycle and the kernel launches per cycle.
Run on a machine with the GPU:  python tools/bench_fleet_device_cycle.py [--sizes 1,8,64,256] [--cycles 4]"""
import argparse
import json
import os
import struct
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mpl_ros_b200 as mp  # noqa: E402
from mpl_ros_b200 import _lib  # noqa: E402
from bench_lpa_fleet import Robot, card, state  # noqa: E402

MAX_SEG = 512
RES, WP = _lib.RESULT_DTYPE, _lib.WAYPOINT_DTYPE


def message(dim, control, actions, seg_states, U, dt):
    """toTrajectoryROSMsg + ROS 1 serialisation on the host (z = 0, frame "map", seq 0, stamp 0)"""
    order = {1: 1, 3: 2, 7: 3, 15: 4}[control & 15]
    b = struct.pack("<IIII", 0, 0, 0, 3) + b"map" + struct.pack("<I", len(actions))
    for a, st in zip(actions, seg_states):
        for ax in range(3):
            c = [0.0] * 6
            if ax < dim:
                for d in range(order):
                    c[5 - d] = st[d * 3 + ax]
                c[5 - order] = U[a][ax]
            b += struct.pack("<I", 6) + struct.pack("<6d", *c)
        b += struct.pack("<I", 6) + struct.pack("<6d", *([0.0] * 6))
        b += struct.pack("<d", dt)
    return b + struct.pack("<I", 0)


class Fleet:
    def __init__(self, cfg, n, device):
        self.robots = [Robot(cfg, i) for i in range(n)]
        self.pls = [r.pl for r in self.robots]
        self.device = device
        self.msgs = []
        mp.MapPlanner.planLPABatch(self.pls, [r.s[0] for r in self.robots], [r.g[0] for r in self.robots])  # not timed
        if device:
            s = np.concatenate([r.s for r in self.robots])
            g = np.concatenate([r.g for r in self.robots])
            self.d_s = torch.from_numpy(s.view(np.uint8).copy()).cuda()
            self.d_g = torch.from_numpy(g.view(np.uint8).copy()).cuda()
            self.res = torch.zeros(n * RES.itemsize, dtype=torch.uint8, device="cuda")
            self.act = torch.zeros((n, MAX_SEG), dtype=torch.int32, device="cuda")
            self.seg = torch.zeros((n, MAX_SEG, 13), dtype=torch.float64, device="cuda")
            self.stride = int(_lib.lib().mplb_trajectory_msg_size(MAX_SEG, b"map"))
            self.out = torch.zeros(n * self.stride, dtype=torch.uint8, device="cuda")
            self.len = torch.zeros(n, dtype=torch.int32, device="cuda")
            self.ok = torch.zeros(n, dtype=torch.int32, device="cuda")

    def plan(self):
        if self.device:
            mp.MapPlanner.planLPABatchDevice(self.pls, self.d_s, self.d_g, self.res, self.act, self.seg, MAX_SEG)
            mp.MapPlanner.serializeLPABatch(self.pls, self.res, self.act, self.seg, MAX_SEG, self.out, self.stride, self.len)
        else:
            mp.MapPlanner.planLPABatch(self.pls, [r.s[0] for r in self.robots], [r.g[0] for r in self.robots])
            self.msgs = []
            for r in self.robots:
                ok = int(r.pl.result()["status"]) == 0
                a, s = (r.pl.getActions(), r.pl.getSegStates()) if ok else ([], [])
                self.msgs.append(message(r.dim, mp.ACC, a, s, r.pl.U_, r.pl.dt_))

    def messages(self):
        if not self.device:
            return self.msgs
        ln = self.len.cpu().numpy()
        out = self.out.cpu().numpy().reshape(len(self.robots), self.stride)
        return [out[i, :ln[i]].tobytes() for i in range(len(self.robots))]

    def next_starts(self):
        """getSubStateSpace(1) and start = getWaypoints()[1] where the trajectory has two segments or more"""
        if self.device:
            res = self.res.cpu().numpy().view(RES)
            assert (res["n_seg"][res["status"] == 0] <= MAX_SEG).all()
            adv = [int(r["status"]) == 0 and int(r["n_seg"]) >= 2 for r in res]
            idx = torch.tensor([1 if a else -1 for a in adv], dtype=torch.int32, device="cuda")
            mp.MapPlanner.trajectoryWaypointsBatch(self.pls, self.res, self.act, self.seg, MAX_SEG, idx, self.d_s, self.ok)
        else:
            adv = []
            for r in self.robots:
                ok = int(r.pl.result()["status"]) == 0 and len(r.pl.getActions()) >= 2
                adv.append(ok)
                if ok:
                    st = r.pl.getSegStates()[1]
                    w = mp.waypoints_array(1)
                    w["pos"][0], w["vel"][0], w["acc"][0], w["jrk"][0], w["yaw"][0] = st[0:3], st[3:6], st[6:9], st[9:12], st[12]
                    w["t"], w["control"] = 0.0 + r.pl.dt_, mp.ACC
                    r.s = w
        mp.MapPlanner.getSubStateSpaceBatch(self.pls, [1 if a else 0 for a in adv])

    def cycle(self):
        for r in self.robots:
            r.edit()
        cells = [getattr(r, "cells", np.zeros((0, 3), dtype=np.int32)) for r in self.robots]
        mp.MapPlanner.getLinkedNodesBatch(self.pls)
        mp.MapPlanner.updateBlockedNodesBatch(self.pls, cells)
        self.plan()
        m1 = self.messages()
        self.next_starts()
        self.plan()
        torch.cuda.synchronize()
        return m1


def run(cfg, n, cycles):
    fl = {m: Fleet(cfg, n, m == "device") for m in ("host", "device")}
    t = {m: [] for m in fl}
    launches = {m: [] for m in fl}
    L = _lib.lib()
    for c in range(cycles):
        msgs = {}
        for mode in (("host", "device") if c % 2 == 0 else ("device", "host")):
            l0 = L.mplb_launch_count()
            t0 = time.perf_counter()
            msgs[mode] = fl[mode].cycle()
            t[mode].append((time.perf_counter() - t0) * 1e3)
            launches[mode].append(int(L.mplb_launch_count() - l0))
        assert msgs["host"] == msgs["device"], (cfg, n, c)
        assert fl["host"].messages() == fl["device"].messages(), (cfg, n, c)
        for a, b in zip(fl["host"].robots, fl["device"].robots):
            assert state(a) == state(b), (cfg, n, c)
    return {m: dict(ms_per_cycle=float(np.median(t[m])), ms_min=float(min(t[m])), launches_per_cycle=float(np.median(launches[m])))
            for m in fl}


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
