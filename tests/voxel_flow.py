"""The replanner node's flow (mpl_test_node/src/map_replanner_node.cpp:175-259,326-331 with launch/map_replanner_node/test.launch)
over any VoxelGrid + map + LPA* planner triple: start-up from the simple bag's /cloud (every 16th point, tests/golden/voxel_grid.npz),
plan; add_cloud.sh (ray of the two points, the 5 x 5 isFree cells filled as columns, setMap(getMap()), updateBlockedNodes),
replan; clear_cloud.sh (the ray's isOccupied columns cleared, setMap, updateClearedNodes), replan; subtree (getSubStateSpace(1),
start = the trajectory's next waypoint), replan.  Used by tools/make_golden_voxel.py on the reference's own sources and by the
oracle and GPU tests, which compare with what it recorded.

An implementation is `edit(add, p1, p2) -> cells`: the node's callback up to the planner call, including the map update the
planner sees; `grid` (oracle method names) and `planner` (the LpaMixin call shapes of tests/lpa_flow.py) come with it."""
import numpy as np

import lpa_flow
import oracle

CONTROL = 3  # start.use_pos, use_vel (map_replanner_node.cpp:374-378): Control::ACC
# setTol(0.5, 1, 1) in the node; tol_acc is left unset because an ACC-control state carries no acceleration to test and the
# library refuses the setting there
PARAMS = dict(v_max=2.0, a_max=1.0, j_max=1.0, dt=1.0, tol_pos=0.5, tol_vel=1.0)


def controls():
    from mpl_ros_b200 import maps
    return maps.make_U(1.0, 1, 3, use_3d=False)  # u_max 1, num 1, use_3d false (map_replanner_node.cpp:401-412)


def geometry(z):
    return z["simple_origin"], z["simple_dim"], float(z["simple_res"])


def configure(pl):
    for k, v in PARAMS.items():
        pl.set_param(k, v)
    pl.set_controls(controls())
    pl._lpa_control = CONTROL


def run(z, grid, planner, edit):
    """returns (snapshots for lpa_flow.digest, per-edit records: cells, map bits after the edit, update count)"""
    st = z["replanner_start"]
    s, g = oracle.make_waypoints(1), oracle.make_waypoints(1)
    s["pos"][0], s["vel"][0], s["acc"][0] = st[0:3], st[3:6], st[6:9]
    g["pos"][0] = z["replanner_goal"]
    s["control"] = g["control"] = CONTROL
    snaps, edits = [], []
    res = planner.lpa_plan(s, g)
    snaps.append(lpa_flow.snapshot(planner, res))
    for name, add in (("add_cloud", True), ("clear_cloud", False)):
        linked = planner.lpa_get_linked_nodes()  # visualizeGraph after every plan
        p = z["replanner_" + name].astype(np.float64)
        cells = edit(add, p[0], p[-1])
        n = (planner.lpa_update_blocked_nodes if add else planner.lpa_update_cleared_nodes)(cells)
        edits.append(dict(cells=cells, map=np.packbits(grid.get_map() == 100), updated=int(n)))
        snaps.append(lpa_flow.snapshot(planner, None, linked))
        res = planner.lpa_plan(s, g)
        snaps.append(lpa_flow.snapshot(planner, res))
    nxt = planner.lpa_waypoint(1)
    planner.lpa_get_sub_state_space(1)
    snaps.append(lpa_flow.snapshot(planner, None))
    res = planner.lpa_plan(nxt, g)
    snaps.append(lpa_flow.snapshot(planner, res))
    return snaps, edits


def oracle_cells_edit(grid, values, apply_map, origin, dim, res):
    """the node's callbacks with the oracle's rayTrace; `values(cells)` reads the planner's map (isFree: 0 <= v < 100,
    isOccupied: v == 100, outside never), `apply_map()` is setMap(map_util, grid.getMap())"""
    from oracle import voxel as ov
    ns = np.array([(x, y, 0) for x in range(-2, 3) for y in range(-2, 3)], dtype=np.int32)

    def edit(add, p1, p2):
        pns = ov.ray_trace(origin, dim, res, p1, p2)
        if add:
            cand = (pns[:, None, :] + ns[None, :, :]).reshape(-1, 3)
            v = values(cand)
            cells = cand[(v >= 0) & (v < 100)]
            grid.fill(cells, True)
        else:
            cells = pns[values(pns) == 100]
            grid.clear_columns(cells)
        apply_map()
        return cells
    return edit


def set_map_cells(m, old, new, dim):
    """setMap with new cells of unchanged geometry on an oracle / reference map: the cells that differ are written"""
    for v in (0, 100):
        idx = np.flatnonzero((old != new) & (new == v))
        if len(idx):
            cells = np.stack([idx % dim[0], (idx // dim[0]) % dim[1], idx // (dim[0] * dim[1])], axis=1).astype(np.int32)
            m.set_cells(cells, v)


def host_flow(z, G, Map, Planner, ref_mu=None):
    """the flow on host implementations: G a grid class, Map / Planner the oracle's or the reference's; with ref_mu (the
    reference's MapUtil class) the edits are the reference's own callbacks, otherwise the oracle's restatement"""
    g = G(*geometry(z))
    g.add_cloud(z["simple_pts"].astype(np.float64))
    dim, _, ori_d, res = g.info()
    cur = {"map": g.get_map()}
    m = Map(ori_d, dim, cur["map"], float(res))
    m.free_unknown()
    pl = Planner(3)
    pl.set_map(m)
    configure(pl)

    def sync():
        new = g.get_map()
        set_map_cells(m, cur["map"], new, dim)
        cur["map"] = new

    if ref_mu is not None:
        mu = ref_mu(ori_d, dim, float(res), cur["map"])

        def edit(add, p1, p2):
            cells = mu.node_edit(g, add, p1, p2)
            sync()
            return cells
    else:
        def values(cells):
            inside = np.all((cells >= 0) & (cells < dim), axis=1)
            v = np.full(len(cells), np.iinfo(np.int32).min, dtype=np.int64)
            c = cells[inside].astype(np.int64)
            v[inside] = cur["map"][c[:, 0] + dim[0] * c[:, 1] + dim[0] * dim[1] * c[:, 2]]
            return v
        edit = oracle_cells_edit(g, values, sync, ori_d, dim, float(res))
    return run(z, g, pl, edit)


def check(snaps, edits, z):
    """compare with the reference's run recorded in the fixture"""
    d = lpa_flow.digest(snaps)
    gold = z["flow_digest"]
    assert len(d) == len(gold)
    for f in gold.dtype.names:
        assert np.array_equal(d[f], gold[f]), f
    for k, e in enumerate(edits):
        assert np.array_equal(e["cells"], z["flow_cells_%d" % k]), k
        assert np.array_equal(e["map"], z["flow_map_%d" % k]), k
        assert e["updated"] == int(z["flow_updated"][k]), k
