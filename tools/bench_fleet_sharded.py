"""Replan-cycle time of a fleet of R LPA* replanners on ONE shared map, sharded over N GPUs (mplb_fleet_map_edit,
mplb_fleet_plan through mpl_ros_b200.dist.ShardedFleet; DESIGN.md section 6.1).  Robot i lives on rank i mod N.

A cycle is the shared-map fleet cycle: every robot traces its edit on its rank's replica (a ray across the middle of its
trajectory, the isFree cells of a 3 x 3 stencil), the edits are exchanged and every replica applies all of them in robot
order, then getLinkedNodes, updateBlockedNodes (every robot receives the whole concatenation), plan (gathered to rank 0) and
getSubStateSpace(1).  Start / goal pairs are drawn with a fixed seed from the configuration's free cells.

For each configuration and R, the N = 1 and N = 2 runs alternate (REPS times each, one process per rank, N = 2 only where two
GPUs are visible).  Rank 0 times every cycle with a host clock; each library call returns after its device work is complete.
Prints the card's name and power limit, then one JSON line per (config, R, N): median ms per cycle and the bytes that crossed
between GPUs per cycle (counts and rows of the edit exchange, result records and action rows of the gather).
Run on a machine with the GPUs:  python tools/bench_fleet_sharded.py [--sizes 64,256] [--cycles 3] [--reps 2]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
NS3 = np.array([(x, y, 0) for x in range(-1, 2) for y in range(-1, 2)], dtype=np.int32)
MAX_SEG = 64


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        return q.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def exchanged_bytes(nloc, rows, world):
    """bytes that cross between GPUs in one cycle: every rank's payload (4 B per robot count, 12 B per cell row) to the N - 1
    others plus the (rows, robots, cap) header, and the gather of per = ceil(R / N) records of 80 B and action rows of
    4 * MAX_SEG B from the N - 1 non-root ranks"""
    if world == 1:
        return 0
    R = sum(nloc)
    per = (R + world - 1) // world
    edit = sum((4 * n + 12 * k + 24) * (world - 1) for n, k in zip(nloc, rows))
    return int(edit + (world - 1) * per * (80 + 4 * MAX_SEG))


def worker(rank, world, cfg, R, cycles, idfile, out):
    import torch
    torch.cuda.set_device(rank)
    torch.zeros(1, device="cuda")
    import mpl_ros_b200 as mp
    from mpl_ros_b200 import dist as md, maps
    from helpers import fill_waypoints, load_config
    if rank == 0:
        with open(idfile + ".tmp", "wb") as f:
            f.write(md.Comm.unique_id())
        os.replace(idfile + ".tmp", idfile)
    while not os.path.exists(idfile):
        time.sleep(0.05)
    comm = md.Comm(open(idfile, "rb").read(), rank, world)
    m, dim, params, U, start, goal = load_config(cfg)
    mu = comm.broadcast_map(dim, m.origin, m.dim, m.res, m.data, 0) if rank == 0 else comm.broadcast_map(0)
    mu.freeUnknown()
    S, G = maps.sample_queries(m, R, seed=21, min_dist=1.5, max_dist=5.0)
    idx = md.shard_indices(R, rank, world)
    pls, s, g = [], [], []
    for i in idx:
        pl = mp.MapPlanner(dim)
        pl.setMapUtil(mu)
        for key, v in params.items():
            (pl.setDt if key == "dt" else lambda x, key=key: pl._set(key, x))(v)
        pl.setU(U)
        pl.setLPAInitNodes(4096)
        pl.setLPAInitPreds(65536)
        pl.setLPAstar(True)
        a, b = mp.waypoints_array(1), mp.waypoints_array(1)
        fill_waypoints(a, S[i][:dim], mp.ACC)
        fill_waypoints(b, G[i][:dim], mp.ACC)
        pls.append(pl); s.append(a); g.append(b)
    fleet = md.ShardedFleet(pls, R, mu, comm=comm, device=torch.device("cuda", rank))
    fleet.plan([w[0] for w in s], [w[0] for w in g], max_seg=MAX_SEG)  # the first plans (A*-sized searches) are not timed
    times, nbytes = [], []
    for _ in range(cycles):
        t0 = time.perf_counter()
        lists = []
        for pl in pls:
            best = pl.lpaBestChild()["state"][:, :dim]
            c = np.zeros((0, 3), dtype=np.int32)
            if len(best) >= 4:
                c, _ = mu.traceCells(best[len(best) // 3][None], best[2 * len(best) // 3][None], NS3[:, :dim], mp.TRACE_FREE)
            lists.append(c)
        rows = [len(c) for c in lists]
        fleet.map_edit(lists, 100)
        fleet.links()
        fleet.update(True)
        fleet.plan([w[0] for w in s], [w[0] for w in g], max_seg=MAX_SEG)
        ts = []
        for k, pl in enumerate(pls):
            st = pl.lpaBestChild()["state"]
            ts.append(1 if len(st) > 2 else 0)
            if len(st) > 2:
                w = mp.waypoints_array(1)
                w["pos"][0], w["vel"][0], w["acc"][0], w["control"] = st[1, 0:3], st[1, 3:6], st[1, 6:9], mp.ACC
                s[k] = w
        fleet.sub_state_space(ts)
        times.append((time.perf_counter() - t0) * 1e3)
        nbytes.append((len(idx), sum(rows)))
    np.save(out + ".rank%d.npy" % rank, np.array([len(idx), sum(r for _, r in nbytes)], dtype=np.int64))
    if rank == 0:
        np.save(out, np.array(times))


def run(cfg, R, world, cycles):
    import torch.multiprocessing as tmp
    d = tempfile.mkdtemp(prefix="fleet_bench_")
    out = os.path.join(d, "times.npy")
    tmp.spawn(worker, args=(world, cfg, R, cycles, os.path.join(d, "id"), out), nprocs=world, join=True)
    t = np.load(out)
    per_rank = [np.load(out + ".rank%d.npy" % r) for r in range(world)]
    nb = exchanged_bytes([int(x[0]) for x in per_rank], [int(x[1]) // cycles for x in per_rank], world)
    return float(np.median(t)), float(t.min()), nb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="64,256")
    ap.add_argument("--configs", default="skir,simple")
    ap.add_argument("--cycles", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    import torch
    worlds = [1, 2] if torch.cuda.device_count() >= 2 else [1]
    cd = card()
    print("card: " + cd + ("" if 2 in worlds else "  (one GPU visible: N = 2 not measured)"), flush=True)
    for cfg in a.configs.split(","):
        for R in (int(x) for x in a.sizes.split(",")):
            got = {w: [] for w in worlds}
            for rep in range(a.reps):
                for w in (worlds if rep % 2 == 0 else worlds[::-1]):
                    got[w].append(run(cfg, R, w, a.cycles))
            for w in worlds:
                print(json.dumps(dict(card=cd, config=cfg, robots=R, gpus=w, cycles=a.cycles * a.reps,
                                      ms_per_cycle=float(np.median([x[0] for x in got[w]])), ms_min=float(min(x[1] for x in got[w])),
                                      bytes_per_cycle=got[w][0][2])), flush=True)


if __name__ == "__main__":
    main()
