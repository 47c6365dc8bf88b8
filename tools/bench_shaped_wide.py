"""Batches of the two node configurations that plan on the |U| > 32 cost-shaping kernels, on the fixture maps:
  - node3d_yaw81: map_planner_node with use_3d and use_yaw (81 rows, ACCxYAW, yaw_max -1, u_yaw 0.3) on levine;
  - distmap81:    distance_map_planner_node's set with num = 4 (81 rows, ACC) on corridor, with the potential map of
                  updatePotentialMap (radius 1 m, weight 0.5) installed.
Per configuration: plans/s and primitive expansions/s over the batch's kernel time (mplb_last_batch_stats, median of
STEPS timed batches after WARMUP), p50 / p95 of the per-plan device ms, resident slots and the heap top
(mplb_last_batch_tiers).  The CPU arm plans a sample of the same queries with the reference's own sources
(oracle/_ref/libmplref.so, built by build()) on every host core, as bench.py --impl reference does, and checks that they
agree with the GPU's records.  Prints the card's name and power limit, then one JSON object.
Both configurations stop at MaxExpandStep 2000 (setMaxNum), so that the unreachable queries among the random pairs do not
exhaust the whole map and the batch time measures planning rather than a few map-wide searches.
Run on a machine with the GPU:  python tools/bench_shaped_wide.py [--n 1024] [--cpu-sample 16]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
import mpl_ros_b200 as mp  # noqa: E402
from mpl_ros_b200 import maps  # noqa: E402
from oracle import ref  # noqa: E402

STEPS, WARMUP = 5, 2


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def yaw_rows(U, u_yaw):
    return np.array([list(r) + [y] for r in U for y in (-u_yaw, 0.0, u_yaw)])


def configs():
    lv = maps.load_fixture("levine")
    cor = maps.load_fixture("corridor")
    return {
        "node3d_yaw81": dict(m=lv, dim=3, U=yaw_rows(maps.make_U(1.0, 1, 3), 0.3), control=mp.ACCxYAW,
                             params=dict(v_max=2.0, a_max=1.0, dt=1.0, tol_pos=0.5, yaw_max=-1.0, max_num=2000), pot=None),
        "distmap81": dict(m=cor, dim=2, U=maps.make_U(0.5, 4, 2), control=mp.ACC,
                          params=dict(v_max=1.0, a_max=1.0, dt=1.0, tol_pos=0.5, epsilon=1.0, max_num=2000),
                          pot=dict(radius=[1.0, 1.0], weight=0.5)),
    }


def waypoints(make, pos, control, dim):
    w = make(len(pos))
    w["pos"][:, :dim] = pos
    w["control"] = control
    return w


def gpu_planner(c):
    mu = mp.MapUtil(c["dim"])
    mu.setMap(c["m"].origin, c["m"].dim, c["m"].data, c["m"].res)
    mu.freeUnknown()
    pl = mp.MapPlanner(c["dim"], False)
    pl.setMapUtil(mu)
    setters = dict(v_max="setVmax", a_max="setAmax", dt="setDt", yaw_max="setYawmax", epsilon="setEpsilon",
                   max_num="setMaxNum")
    for k, v in c["params"].items():
        if k != "tol_pos":
            getattr(pl, setters[k])(v)
    pl.setTol(c["params"]["tol_pos"])
    pl.setU(c["U"])
    pl._keep = mu
    return pl


def run_gpu(c, S, G):
    pl = gpu_planner(c)
    if c["pot"]:
        pl.setPotentialRadius(c["pot"]["radius"])
        pl.setPotentialWeight(c["pot"]["weight"])
        pl.updatePotentialMap(S[0])
    s, g = waypoints(mp.waypoints_array, S, c["control"], c["dim"]), waypoints(mp.waypoints_array, G, c["control"], c["dim"])
    ms = []
    for k in range(WARMUP + STEPS):
        res, _, _ = pl.plan_batch(s, g)
        if k >= WARMUP:
            ms.append(pl.last_batch_stats()["kernel_ms"])
    tiers = pl.last_batch_tiers()
    t = float(np.median(ms)) * 1e-3
    n = len(S)
    return res, dict(plans=n, ok=int((res["status"] == 0).sum()), kernel_ms=t * 1e3, plans_per_s=n / t,
                     prim_expansions_per_s=float(res["n_prims"].sum()) / t,
                     device_ms_p50=float(np.percentile(res["device_ms"], 50)),
                     device_ms_p95=float(np.percentile(res["device_ms"], 95)),
                     resident=int(tiers[0]["resident"]), slots=int(tiers[0]["slots"]), hcap=int(tiers[0]["hcap"]),
                     tiers=len(tiers))


def run_cpu(c, S, G, gpu_res):
    if not ref.available():
        return dict(skipped="oracle/_ref/libmplref.so was not built")
    rm = ref.RefMap(c["m"].origin, c["m"].dim, c["m"].data, c["m"].res)
    rm.free_unknown()
    rp = ref.RefPlanner(c["dim"])
    rp.set_map(rm)
    for k, v in c["params"].items():
        rp.set_param(k, v)
    rp.set_controls(c["U"])
    if c["pot"]:
        rp.set_vec("potential_radius", list(c["pot"]["radius"]) + [0.0] * (3 - len(c["pot"]["radius"])))
        rp.set_param("potential_weight", c["pot"]["weight"])
        rp.update_potential_map(np.r_[S[0], np.zeros(3 - c["dim"])])
    s, g = waypoints(oracle.make_waypoints, S, c["control"], c["dim"]), waypoints(oracle.make_waypoints, G, c["control"], c["dim"])
    nth = os.cpu_count() or 1
    t0 = time.perf_counter()
    res = rp.plan_batch(s, g, nthreads=nth)
    t = time.perf_counter() - t0
    same = all(res["pops"][i] == gpu_res["pops"][i] and res["cost"][i] == gpu_res["cost"][i] for i in range(len(S))
               if gpu_res["status"][i] == 0)
    return dict(plans=len(S), threads=nth, seconds=t, plans_per_s=len(S) / t,
                prim_expansions_per_s=float(res["n_prims"].sum()) / t, agrees_with_gpu=bool(same))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--cpu-sample", type=int, default=16)
    a = ap.parse_args()
    print("card: " + card(), flush=True)
    out = dict(card=card())
    for name, c in configs().items():
        S, G = maps.sample_queries(c["m"], a.n, seed=1)
        res, g = run_gpu(c, S, G)
        k = min(a.cpu_sample, a.n)
        out[name] = dict(gpu=g, cpu_reference=run_cpu(c, S[:k], G[:k], res[:k]))
        print(name, json.dumps(out[name]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
