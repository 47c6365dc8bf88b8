"""A sharded fleet's output on the device: every rank runs mplb_lpa_plan_batch_device, mplb_lpa_serialize_trajectories_device and
mplb_lpa_trajectory_waypoints_device on its own robots, the planners mplb_fleet_plan serves, with no collective of their own.  With a
communicator of one, and with two ranks where the box has two GPUs, the messages, records and next starts of every robot equal
those of the single-device fleet, through a cycle of plan, next start, getSubStateSpace and plan from the device starts."""
import os
import sys
import time

import numpy as np
import pytest

import mpl_ros_b200 as mp
from mpl_ros_b200 import _lib, dist as mdist
from test_gpu_fleet_sharded import ROOT, Reference, Sharded, robot_specs, state

pytestmark = pytest.mark.gpu
MAX_SEG = 256
RES, WP = _lib.RESULT_DTYPE, _lib.WAYPOINT_DTYPE


def device_cycle(pls, starts, goals):
    """plan, messages, next starts (getWaypoints()[1] where the plan has two segments or more), getSubStateSpace, plan, messages:
    returns what a rank would publish, as host arrays for the comparison"""
    import torch
    n = len(pls)
    out = {}
    d_s = torch.from_numpy(np.concatenate(starts).view(np.uint8).copy()).cuda()
    d_g = torch.from_numpy(np.concatenate(goals).view(np.uint8).copy()).cuda()
    res = torch.zeros(n * RES.itemsize, dtype=torch.uint8, device="cuda")
    act = torch.zeros((n, MAX_SEG), dtype=torch.int32, device="cuda")
    seg = torch.zeros((n, MAX_SEG, 13), dtype=torch.float64, device="cuda")
    stride = int(_lib.lib().mplb_trajectory_msg_size(MAX_SEG, b"map"))
    msg = torch.zeros(n * stride, dtype=torch.uint8, device="cuda")
    ln = torch.zeros(n, dtype=torch.int32, device="cuda")
    ok = torch.zeros(n, dtype=torch.int32, device="cuda")
    for step in range(2):
        mp.MapPlanner.planLPABatchDevice(pls, d_s, d_g, res, act, seg, MAX_SEG)
        mp.MapPlanner.serializeLPABatch(pls, res, act, seg, MAX_SEG, msg, stride, ln, seq=step)
        r = res.cpu().numpy().view(RES)
        lens = ln.cpu().numpy()
        m = msg.cpu().numpy().reshape(n, stride)
        out["res%d" % step] = r.copy()
        out["msg%d" % step] = [m[i, :lens[i]].tobytes() for i in range(n)]
        if step == 0:
            adv = [int(x["status"]) == 0 and int(x["n_seg"]) >= 2 for x in r]
            idx = torch.tensor([1 if a else -1 for a in adv], dtype=torch.int32, device="cuda")
            mp.MapPlanner.trajectoryWaypointsBatch(pls, res, act, seg, MAX_SEG, idx, d_s, ok)
            out["next"] = d_s.cpu().numpy().view(WP).copy()
            out["ok"] = ok.cpu().numpy().copy()
            mp.MapPlanner.getSubStateSpaceBatch(pls, [1 if a else 0 for a in adv])
    return out


def compare(ref, got, robots):
    """got: the cycle of `robots` (global indices, in that order) against the single-device cycle ref"""
    for k, i in enumerate(robots):
        for step in range(2):
            assert got["res%d" % step][k].tobytes() == ref["res%d" % step][i].tobytes(), (step, i)
            assert got["msg%d" % step][k] == ref["msg%d" % step][i], (step, i)
            assert len(got["msg%d" % step][k]) > 0 or int(ref["res%d" % step][i]["status"]) != 0
        assert got["next"][k].tobytes() == ref["next"][i].tobytes() and got["ok"][k] == ref["ok"][i], i


@pytest.mark.parametrize("kind", ["skir", "corridor"])
def test_rank_local_device_calls_with_a_comm_of_one(kind):
    import torch
    m, dim, specs = robot_specs(kind)
    ref = Reference(m, dim, specs, with_oracle=False)
    ref.plan()
    comm = mdist.Comm(mdist.Comm.unique_id(), 0, 1)
    sh = Sharded(comm, m, dim, specs, torch.device("cuda", 0))
    sh.plan(MAX_SEG)  # mplb_fleet_plan through the shared plan path
    for a, b in zip(ref.rob, sh.rob):
        assert state(a) == state(b)
    want = device_cycle(ref.pls(), ref.s, ref.g)
    got = device_cycle([r.pl for r in sh.rob], sh.s, sh.g)
    compare(want, got, sh.idx)
    assert sum(want["ok"]) > 0 and any(len(x) for x in want["msg1"])
    for a, b in zip(ref.rob, sh.rob):
        assert state(a) == state(b)


def _rank_worker(rank, world, idfile, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    torch.cuda.set_device(rank)
    torch.zeros(1, device="cuda")
    from mpl_ros_b200 import dist as md
    if rank == 0:
        with open(idfile + ".tmp", "wb") as f:
            f.write(md.Comm.unique_id())
        os.replace(idfile + ".tmp", idfile)
    while not os.path.exists(idfile):
        time.sleep(0.05)
    comm = md.Comm(open(idfile, "rb").read(), rank, world)
    m, dim, specs = robot_specs("skir")
    sh = Sharded(comm, m, dim, specs, torch.device("cuda", rank))
    sh.plan(MAX_SEG)
    got = device_cycle([r.pl for r in sh.rob], sh.s, sh.g)
    np.savez(os.path.join(out_dir, "rank%d.npz" % rank), res0=got["res0"], res1=got["res1"], next=got["next"], ok=got["ok"],
             msg0=np.array(got["msg0"], dtype=object), msg1=np.array(got["msg1"], dtype=object), idx=np.array(sh.idx))


def test_two_ranks_equal_the_single_device_fleet(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as tmp
    m, dim, specs = robot_specs("skir")
    ref = Reference(m, dim, specs, with_oracle=False)
    ref.plan()
    want = device_cycle(ref.pls(), ref.s, ref.g)
    tmp.spawn(_rank_worker, args=(2, str(tmp_path / "nccl_id"), str(tmp_path)), nprocs=2, join=True)
    for r in range(2):
        z = np.load(str(tmp_path / ("rank%d.npz" % r)), allow_pickle=True)
        got = {k: z[k] for k in ("res0", "res1", "next", "ok")}
        got["msg0"], got["msg1"] = list(z["msg0"]), list(z["msg1"])
        compare(want, got, list(z["idx"]))
