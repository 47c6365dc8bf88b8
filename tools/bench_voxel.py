"""Times the GPU VoxelGrid (mplb_voxel.cu) against the reference's own voxel_grid.cpp on the CPU (oracle/_ref/libvoxelref.so,
where built) and prints one JSON line.  Device times are CUDA events around each call after a warm-up call of the same shape;
every call synchronises before it returns, so an event pair brackets the whole call.  CPU times are wall-clock, one run.

Workloads: the levine /cloud fixture points (tests/golden/voxel_grid.npz) tiled and jittered from a seed to 1 M and 10 M
points on levine's grid; addCloud, addCloud(pts, ns) with the replanner node's 5x5x1 ns and with a 5x5x5 ns, setMap through
write_map on levine's grid and on a 1024^3 grid, getCloud.

usage: python tools/bench_voxel.py [--sizes 1000000,10000000] [--reps 5] [--no-ref]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
NS_NODE = np.array([(x, y, 0) for x in range(-2, 3) for y in range(-2, 3)], dtype=np.int32)
NS_CUBE5 = np.array([(x, y, z) for x in range(-2, 3) for y in range(-2, 3) for z in range(-2, 3)], dtype=np.int32)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
        return name, power
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e, "unknown"


def cloud(z, n, seed=0):
    base = z["levine_pts"].astype(np.float32)
    rs = np.random.RandomState(seed)
    reps = -(-n // len(base))
    pts = np.concatenate([base + rs.normal(0, 0.03, base.shape).astype(np.float32) for _ in range(reps)])[:n]
    return np.ascontiguousarray(pts)


def ev_time(torch, fn, reps):
    fn()  # warm-up of this shape
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def cpu_time(fn):
    t = time.perf_counter()
    fn()
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-ref", action="store_true")
    a = ap.parse_args()
    import torch
    import mpl_ros_b200 as mp
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    ref = None
    if not a.no_ref:
        from oracle import voxel as ov
        if os.path.exists(ov._RVX):
            ref = ov.RefVoxelGrid
    z = np.load(os.path.join(ROOT, "tests", "golden", "voxel_grid.npz"))
    args = (z["levine_origin"], z["levine_dim"], float(z["levine_res"]))
    name, power = card()
    out = dict(tool="bench_voxel", gpu=name, power_limit=power, unit="ms", reps=a.reps, grid=[int(x) for x in mp.VoxelGrid(*args).info()[0]],
               rows=[])

    def row(what, n, gpu_ms, ref_ms=None, **kw):
        r = dict(op=what, points=n, gpu_ms=round(gpu_ms, 4), ref_cpu_ms=None if ref_ms is None else round(ref_ms, 2), **kw)
        if ref_ms is not None:
            r["speedup"] = round(ref_ms / gpu_ms, 1)
        out["rows"].append(r)
        print(json.dumps(r), file=sys.stderr)

    for n in [int(s) for s in a.sizes.split(",")]:
        pts = cloud(z, n)
        t = torch.from_numpy(pts).cuda()
        g = mp.VoxelGrid(*args)
        gm = ev_time(torch, lambda: g.addCloudDevice(t), a.reps)
        rm = None
        p64 = pts.astype(np.float64)
        if ref is not None:
            rg = ref(*args)
            rm = cpu_time(lambda: rg.add_cloud(p64))
        row("add_cloud", n, gm, rm, input="device fp32")
        for ns_name, ns in (("5x5x1", NS_NODE), ("5x5x5", NS_CUBE5)):
            obs = torch.empty((min(n * len(ns), 200_000_000), 3), dtype=torch.int32, device="cuda")  # rows beyond it are counted

            def ins():
                g2 = mp.VoxelGrid(*args)  # a fresh grid each time: the first insertion is the expensive one
                return g2.addCloudDevice(t, ns=ns, out=obs)
            gm = ev_time(torch, ins, a.reps)
            count = ins()
            rm = None
            if ref is not None and n <= 1_000_000:
                rg = ref(*args)
                rm = cpu_time(lambda: rg.add_cloud_inflated(p64, ns))
            row("add_cloud_inflated", n, gm, rm, ns=ns_name, new_obs=int(count), note="includes grid creation")
        del t
        torch.cuda.empty_cache()

    g = mp.VoxelGrid(*args)
    g.addCloud(z["levine_pts"].astype(np.float64))
    dim, _, ori_d, res = g.info()
    mu = mp.VoxelMapUtil()
    mu.setMap(ori_d, dim, np.zeros(int(np.prod(dim)), dtype=np.int8), float(res))
    row("write_map", 0, ev_time(torch, lambda: g.writeMap(mu), a.reps), grid="levine %s" % list(map(int, dim)))
    rm = None
    if ref is not None:
        rg = ref(*args)
        rg.add_cloud(z["levine_pts"].astype(np.float64))
        rm = cpu_time(lambda: rg.get_cloud())
    row("get_cloud", 0, ev_time(torch, lambda: g.getCloud(), a.reps), rm, cloud=len(g.getCloud()), grid="levine")
    if ref is not None:
        rm = cpu_time(lambda: rg.get_map())
        row("get_map_host_bytes", 0, ev_time(torch, lambda: g.getMapData(), a.reps), rm, grid="levine")
    del g, mu
    big = mp.VoxelGrid((0.0, 0.0, 0.0), (102.45, 102.45, 102.45), 0.1)  # 1024^3 cells at float(0.1)
    bd = big.info()[0]
    if int(np.prod(bd.astype(np.int64))) > 0:
        mb = mp.VoxelMapUtil()
        mb.setMap(big.info()[2], bd, np.zeros(int(np.prod(bd.astype(np.int64))), dtype=np.int8), float(big.info()[3]))
        row("write_map", 0, ev_time(torch, lambda: big.writeMap(mb), a.reps), grid="%s" % list(map(int, bd)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
