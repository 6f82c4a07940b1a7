"""Frontiers on the costmap (include/tloam_b200.h "Frontiers"; k_fr_* in libtloam_b200_frontier.so).
tests/frontier_oracle.py is the bit-for-bit numpy restatement.

CPU: the frontier-cell rule against a literal loop at every code class, free_max 0 / 252 and the grid's edges; the
components against scipy.ndimage.label and a literal explore_lite-style search, on random grids, diagonal-only chains,
spirals and a component touching every edge; the approach tie rule, the centroid bits, the cost formula, the filter
boundary and the order; the symbols, the new library's kernels, the digests of every other library, the shim's driver.
GPU: labels, frontiers and cells equal the restatement on host grids of shapes on and off the tile size, adversarial
components, a seq-00-shaped grid (labels also equal scipy's) and the ray-cast drive before and after a correction; a room
whose nearer door is behind a wall; repeat searches; the status codes; nothing else changes; the shim."""
import ctypes as C
import json
import os
import struct
import subprocess

import numpy as np
import pytest

import frontier_oracle as fo
import plan_oracle as po
import sass_digest
from test_distance import SEQ00, random_grid
from test_global_map_intensity import same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_frontier_default_config", "tloam_b200_frontier_search", "tloam_b200_frontier_download",
               "tloam_b200_frontier_cells", "tloam_b200_frontier_labels"]
KERNELS = ("k_fr_tile", "k_fr_border", "k_fr_flatten", "k_fr_compact", "k_fr_stats",
           "k_gmm_hist", "k_gmm_offsets", "k_gmm_scatter", "k_gmm_head_count", "k_gmm_head_scatter")
CODES = np.array([0, 1, 100, 251, 252, 253, 254, 255], dtype=np.uint8)


def scipy_labels(F):
    """scipy.ndimage.label with the 3 x 3 structure, renumbered from 0 in order of each label's first cell"""
    from scipy import ndimage
    S, k = ndimage.label(F, structure=np.ones((3, 3)))
    vals, first = np.unique(S.ravel(), return_index=True)
    first = first[vals > 0]
    rank = np.empty(k + 1, dtype=np.int64)
    rank[0] = -1
    rank[1 + np.argsort(np.argsort(first))] = np.arange(k)
    out = np.where(S > 0, rank[S], 0xFFFFFFFF).astype(np.uint32)
    return out, k


def spiral(n):
    """one-cell-wide square rings one inside the other, each joined to the next: a winding path of True cells"""
    g = np.zeros((n, n), dtype=bool)
    lo, hi = 0, n - 1
    while lo <= hi:
        g[lo, lo:hi + 1] = True
        g[lo:hi + 1, hi] = True
        g[hi, lo:hi + 1] = True
        g[lo + 2:hi + 1, lo] = True
        if lo + 2 <= hi:
            g[lo + 2, lo:lo + 3] = True
        lo, hi = lo + 2, hi - 2
    return g


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1), (1, 9), (7, 1), (5, 6), (23, 17)])
def test_frontier_cell_rule_matches_a_literal_loop(shape):
    rng = np.random.default_rng(shape[0] * 31 + shape[1])
    for free_max in (0, 1, 100, 252):
        c = rng.choice(CODES, shape)
        F = fo.frontier_cells(c, free_max)
        H, W = shape
        for j in range(H):
            for i in range(W):
                want = c[j, i] == 255 and any(0 <= i + di < W and 0 <= j + dj < H and c[j + dj, i + di] <= free_max
                                              for di, dj in ((1, 0), (-1, 0), (0, 1), (0, -1)))
                assert F[j, i] == want, (free_max, i, j)
    c = np.full((3, 3), 255, dtype=np.uint8)
    c[1, 1] = 252
    assert fo.frontier_cells(c, 252).tolist() == [[False, True, False], [True, False, True], [False, True, False]]
    assert not fo.frontier_cells(c, 251).any()


def test_components_match_scipy_and_a_literal_search():
    rng = np.random.default_rng(3)
    grids = [rng.random(s) < p for s, p in (((1, 1), 1.0), ((1, 40), 0.6), ((40, 1), 0.6), ((33, 65), 0.35),
                                            ((64, 64), 0.45), ((97, 70), 0.5))]
    diag = np.zeros((20, 20), dtype=bool)
    diag[np.arange(20), np.arange(20)] = True                      # diagonal-only chains
    diag[np.arange(19), 19 - np.arange(19)] = True
    diag[0, 5] = diag[1, 6] = diag[2, 7] = True
    edges = np.zeros((12, 15), dtype=bool)                         # one component touching every edge
    edges[0, :] = edges[:, 0] = edges[-1, :] = edges[:, -1] = True
    edges[6, 1:9] = True
    grids += [diag, edges, spiral(31), spiral(40)]
    for F in grids:
        L, k = fo.components(F)
        B, kb = fo.bfs_components(F)
        S, ks = scipy_labels(F)
        assert k == kb == ks and np.array_equal(L, B) and np.array_equal(L, S)
    assert fo.components(edges)[1] == 1 and fo.components(spiral(31))[1] == 1


def tiny_case():
    """a 4 x 5 grid with known frontiers: codes, potential"""
    c = np.array([[255, 255, 0, 255, 255],
                  [255, 254, 0, 0, 255],
                  [0, 0, 0, 254, 255],
                  [255, 255, 254, 254, 255]], dtype=np.uint8)
    P = np.full(c.shape, po.INF, dtype=np.uint64)
    P[c <= 252] = 700
    return c, P


def test_approach_ties_go_to_the_lowest_index_and_the_centroid_and_cost_are_the_formula():
    c, P = tiny_case()
    out = fo.search(c, P, (1.0, -2.0), 0.25, min_frontier_size=0.0)
    L = out["labels"]
    assert out["components"] == 3 and out["cells"] == 6
    assert L[0, 1] == L[1, 0] == 0 and L[0, 3] == L[1, 4] == 1 and L[3, 0] == L[3, 1] == 2
    assert (L == fo.NONE).sum() == 20 - 6 and L[0, 0] == L[0, 4] == L[2, 4] == fo.NONE
    fr = out["frontiers"]
    by_id = {int(fr["id"][k]): k for k in range(len(fr["id"]))}
    k0 = by_id[0]
    # frontier 0's free 4-neighbours (2, 0) and (0, 2) tie at P = 700: the lower index, 2, wins
    assert (fr["approach_i"][k0], fr["approach_j"][k0]) == (2, 0)
    k1 = by_id[1]
    assert fr["size"][k1] == 2 and (fr["sum_i"][k1], fr["sum_j"][k1]) == (3 + 4, 0 + 1)
    assert (fr["min_i"][k1], fr["min_j"][k1], fr["max_i"][k1], fr["max_j"][k1]) == (3, 0, 4, 1)
    assert fr["centroid_x"][k1].tobytes() == np.float64(1.0 + (7 / 2 + 0.5) * 0.25).tobytes()
    assert fr["centroid_y"][k1].tobytes() == np.float64(-2.0 + (1 / 2 + 0.5) * 0.25).tobytes()
    d = (700.0 / (70.0 * 50.0)) * 0.25
    assert fr["distance"][k1] == d and fr["cost"][k1] == 3.0 * d - 1.0 * (2.0 * 0.25)
    costs = fr["cost"][fr["status"] == 0]
    assert (np.diff(costs) >= 0).all()
    P2 = P.copy()
    P2[2, 0] = P2[2, 1] = po.INF                                   # frontier 2's only free neighbours: unreachable
    P2[0, 2] = 700
    out2 = fo.search(c, P2, (1.0, -2.0), 0.25, min_frontier_size=0.0)
    f2 = out2["frontiers"]
    assert f2["status"].tolist()[-1] == 1 and f2["id"].tolist()[-1] == 2 and np.isinf(f2["cost"][-1])
    assert out2["reachable"] == 2


def test_filter_keeps_the_boundary_and_the_order_breaks_ties_by_id():
    c = np.zeros((3, 9), dtype=np.uint8)
    c[0, :] = 255
    c[0, 2] = c[0, 5] = 254                                        # frontiers of 2, 2 and 3 cells along row 0
    P = np.full(c.shape, 7000, dtype=np.uint64)
    out = fo.search(c, P, (0.0, 0.0), 0.25, min_frontier_size=0.5)
    fr = out["frontiers"]
    assert out["components"] == 3 and fr["id"].tolist() == [2, 0, 1]     # the largest first, then equal costs by id
    assert fr["size"].tolist() == [3, 2, 2]
    out = fo.search(c, P, (0.0, 0.0), 0.25, min_frontier_size=0.5000001)
    assert out["frontiers"]["id"].tolist() == [2]
    out = fo.search(c, P, (0.0, 0.0), 0.25, min_frontier_size=0.5, gain_scale=0.0)
    assert out["frontiers"]["id"].tolist() == [0, 1, 2]           # equal costs: by id
    assert out["offsets"].tolist() == [0, 2, 4, 7] and out["ij"][:, 1].tolist() == [0] * 7
    assert out["ij"][:, 0].tolist() == [0, 1, 3, 4, 6, 7, 8]


def test_config_limits():
    assert fo.config_valid(0, 0.0, 0.0, 0.0) and fo.config_valid(252, 1e9, 1e9, 1e9)
    assert not fo.config_valid(253, 0.5, 3.0, 1.0) and not fo.config_valid(252, -1e-300, 3.0, 1.0)
    assert not fo.config_valid(252, np.inf, 3.0, 1.0) and not fo.config_valid(252, 0.5, np.nan, 1.0)
    assert not fo.config_valid(252, 0.5, 3.0, -1.0)


# ---- the library ------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_frontier_library_holds_only_its_kernels_for_sm90a_without_stack():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.FRONTIER_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.FRONTIER_LIB], capture_output=True, text=True,
                         check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.FRONTIER_LIB], capture_output=True, text=True,
                         check=True).stdout
    usage = [l for l in res.splitlines() if "REG:" in l]
    assert len(usage) == len(KERNELS) and all("STACK:0 " in l for l in usage), usage


def test_every_other_library_keeps_its_sass():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_frontier.json")))
    assert len(want) == 19 and "libtloam_b200_frontier.so" not in want and "libtloam_b200_greg.so" in want
    for lib in want:
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


def test_frontier_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "frontier_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
GRID_CFG = dict(inscribed_radius=0.3, inflation_radius=1.0)        # at 0.25 m: codes 0, 1 .. 252, 253, 254 and 255
BARE = dict(inscribed_radius=0.0, inflation_radius=0.0)            # codes 0, 254 and 255 only
ORIGIN, RES = (-3.25, 7.5), 0.25


def passable(costs, rng):
    t = po.cell_costs(costs)
    j, i = np.argwhere(t > 0)[rng.integers(0, int((t > 0).sum()))]
    return int(i), int(j)


def search_and_check(r, f, p, plan_cfg=None, **cfg):
    """frontier_search against the restatement: info, labels, every kept frontier's fields and cells"""
    c = fo.config(**cfg)
    nc = (plan_cfg or {}).get("neutral_cost", 50)
    want = fo.search(f.costs, p.potential, f.origin, f.resolution, neutral_cost=nc, **c)
    info, got = r.frontier_search(**cfg)
    H, W = f.costs.shape
    assert (info["width"], info["height"], (info["goal_i"], info["goal_j"])) == (W, H, p.goal)
    assert (info["origin_x"], info["origin_y"], info["resolution"]) == (f.origin[0], f.origin[1], f.resolution)
    assert (info["cells"], info["components"], info["kept"], info["reachable"]) == \
        (want["cells"], want["components"], len(want["frontiers"]["id"]), want["reachable"])
    assert np.array_equal(r.frontier_labels(), want["labels"])
    wf = want["frontiers"]
    g = {"id": [q.id for q in got], "size": [q.size for q in got], "sum_i": [q.sums[0] for q in got],
         "sum_j": [q.sums[1] for q in got], "min_i": [q.bbox[0] for q in got], "min_j": [q.bbox[1] for q in got],
         "max_i": [q.bbox[2] for q in got], "max_j": [q.bbox[3] for q in got],
         "centroid_x": [q.centroid[0] for q in got], "centroid_y": [q.centroid[1] for q in got],
         "approach_i": [q.approach[0] for q in got], "approach_j": [q.approach[1] for q in got],
         "approach_x": [q.approach_xy[0] for q in got], "approach_y": [q.approach_xy[1] for q in got],
         "approach_potential": [q.approach_potential for q in got], "status": [q.status for q in got],
         "distance": [q.distance for q in got], "cost": [q.cost for q in got]}
    for k in fo.FIELDS:
        if wf[k].dtype.kind == "f":
            assert same_bits(np.array(g[k], dtype=np.float64), wf[k]), k
        else:
            assert [int(v) for v in g[k]] == [int(v) for v in wf[k]], k
    ij = np.concatenate([q.cells for q in got]) if got else np.zeros((0, 2), dtype=np.int32)
    xy = np.concatenate([q.xy for q in got]) if got else np.zeros((0, 2))
    assert np.array_equal(ij, want["ij"]) and same_bits(xy, fo.centres(want["ij"], f.origin, f.resolution))
    assert [len(q.cells) for q in got] == np.diff(want["offsets"]).tolist()
    return info, got, want


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1), (1, 777), (513, 1), (31, 31), (32, 32), (33, 33), (64, 64), (65, 65),
                                   (129, 257)])
def test_gpu_host_grids_are_the_restatement(shape):
    import tloam_b200
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    g = random_grid(shape, rng, 0.04, 0.3)
    if g.size == 1:
        g[0, 0] = 0
    r = tloam_b200.LocalRegistration()
    for cfg in (GRID_CFG, BARE):
        f = r.distance_build(g, ORIGIN, RES, **cfg)
        goal = passable(f.costs, rng)
        p = r.plan_build(po.centres([goal], ORIGIN, RES)[0])
        search_and_check(r, f, p)
        search_and_check(r, f, p, free_max=0, min_frontier_size=0.0)
        search_and_check(r, f, p, min_frontier_size=0.75, potential_scale=0.5, gain_scale=7.0)
        p = r.plan_build(po.centres([goal], ORIGIN, RES)[0], neutral_cost=1, cost_factor=259)
        search_and_check(r, f, p, plan_cfg=dict(neutral_cost=1), free_max=100, min_frontier_size=0.0)
    r.close()


def serpentine_unknown(H=200, W=200, x0=16, x1=48):
    """a one-cell unknown corridor folding along rows 1, 3, 5 ... from column x0 to x1, joined at alternating ends,
    inside free space: one frontier that crosses the tile edges at 32, 64 ... again and again"""
    g = np.zeros((H, W), dtype=np.int8)
    rows = list(range(1, H - 1, 2))
    for k, j in enumerate(rows):
        g[j, x0:x1 + 1] = -1
        if k + 1 < len(rows):
            g[j + 1, x1 if k % 2 == 0 else x0] = -1
    return g


def adversarial_grids():
    out = {"serpentine": serpentine_unknown(), "serpentine_x": serpentine_unknown().T.copy()}
    g = np.zeros((130, 130), dtype=np.int8)                        # a diagonal staircase across tile corners
    for k in range(130):
        g[k, k] = -1
        g[k, 129 - k] = -1
    out["staircase"] = g
    g = np.full((100, 161), -1, dtype=np.int8)                     # one component spanning the grid
    g[1:-1:3, 1:-1] = 0
    out["spanning"] = g
    g = np.zeros((97, 131), dtype=np.int8)                         # single isolated cells
    g[::2, ::2] = -1
    out["singles"] = g
    g = np.where(np.add.outer(np.arange(66), np.arange(70)) % 2 == 0, -1, 0).astype(np.int8)
    out["checkerboard"] = g                                        # diagonal-only, one component
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["serpentine", "serpentine_x", "staircase", "spanning", "singles", "checkerboard"])
def test_gpu_adversarial_components_are_the_restatement(name):
    import tloam_b200
    g = adversarial_grids()[name]
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, (0.0, 0.0), 0.1, **BARE)
    assert set(np.unique(f.costs).tolist()) <= {0, 254, 255}
    p = r.plan_build(po.centres([passable(f.costs, np.random.default_rng(1))], (0.0, 0.0), 0.1)[0])
    info, got, want = search_and_check(r, f, p, min_frontier_size=0.0)
    S, k = scipy_labels(fo.frontier_cells(f.costs))
    assert np.array_equal(r.frontier_labels(), S) and info["components"] == k
    if name in ("serpentine", "serpentine_x", "spanning", "checkerboard"):
        assert info["components"] == 1
    if name == "singles":
        assert info["components"] == info["cells"] == (97 // 2 + 1) * (131 // 2 + 1)
    r.close()


@pytest.mark.gpu
def test_gpu_seq00_shaped_grid_labels_are_scipys_and_frontiers_the_restatement():
    import tloam_b200
    rng = np.random.default_rng(0)
    g = random_grid(SEQ00, rng, p_obstacle=0.002, p_unknown=0.3)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, (-270.3, -310.7), 0.1, **GRID_CFG)
    p = r.plan_build(po.centres([passable(f.costs, rng)], f.origin, f.resolution)[0])
    info, got, want = search_and_check(r, f, p)
    S, k = scipy_labels(fo.frontier_cells(f.costs))
    assert np.array_equal(want["labels"], S) and info["components"] == k and k > 10000
    r.close()


def room_with_two_doors():
    """a 60 x 60 room at 0.1 m in unknown space, doors in its west and east walls; a wall inside the room west of the
    robot, open only at its south end, so the west door is nearer in a straight line and farther by path"""
    g = np.full((70, 70), -1, dtype=np.int8)
    g[5:65, 5:65] = 100
    g[6:64, 6:64] = 0
    g[30:37, 5] = -1                                               # the west door, 7 cells
    g[30:37, 64] = -1                                              # the east door
    g[6:60, 20] = 100                                              # the inner wall, open at rows 60 .. 63
    robot = (28, 33)                                               # 8 cells east of the inner wall
    return g, robot


@pytest.mark.gpu
def test_gpu_room_ranks_the_door_with_the_shorter_path_first_and_routes_to_it():
    import tloam_b200
    g, robot = room_with_two_doors()
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, (0.0, 0.0), 0.1, **BARE)
    robot_xy = po.centres([robot], (0.0, 0.0), 0.1)[0]
    p = r.plan_build(robot_xy)
    info, got, _ = search_and_check(r, f, p)
    assert info["kept"] == 2 and info["reachable"] == 2
    east, west = got
    assert east.bbox[0] == 64 and west.bbox[0] == 5
    # by straight line the west door is the nearer one, by path the east one
    dw = np.hypot(*(np.array(west.centroid) - robot_xy))
    de = np.hypot(*(np.array(east.centroid) - robot_xy))
    assert dw < de and east.distance < west.distance and east.cost < west.cost
    (path,) = r.plan_paths([east.approach_xy])
    route = path.cells[::-1]
    assert path.status == 0 and path.cost == east.approach_potential
    assert tuple(route[0]) == robot and tuple(route[-1]) == east.approach
    t = po.cell_costs(f.costs)
    assert (t[route[:, 1], route[:, 0]] > 0).all()
    for (i0, j0), (i1, j1) in zip(route[:-1], route[1:]):           # the reversed path is a path: no corner is cut
        assert max(abs(i1 - i0), abs(j1 - j0)) == 1
        if i0 != i1 and j0 != j1:
            assert t[j0, i1] > 0 and t[j1, i0] > 0
    r.close()


@pytest.mark.gpu
def test_gpu_occupancy_drive_frontiers_are_the_restatement_before_and_after_a_correction():
    import pose_graph_oracle as pgo
    import tloam_b200
    from test_occupancy import COARSE, ray_frames
    from test_pose_graph import loop_result
    frames = ray_frames(10)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 20)
    r.global_map_correction_enable()
    r.occupancy_enable(**COARSE)
    r.pose_graph_enable()
    O = []
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
        r.pose_graph_add_node(pose)
        O.append(pose)
    r.occupancy_build()
    f = r.distance_build()
    robot = O[-1][:2, 3]
    p = r.plan_build(robot)
    before, got, _ = search_and_check(r, f, p)
    assert before["reachable"] > 0 and got[0].status == 0
    (path,) = r.plan_paths([got[0].approach_xy])
    assert path.status == 0 and tuple(path.cells[-1]) == p.goal
    r.pose_graph_add_loop(loop_result(1, 5, pgo.inv_mul(O[1], O[5]) @ pgo.exp4([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(6))
    r.occupancy_build()
    f2 = r.distance_build()
    p2 = r.plan_build(robot)
    after, _, _ = search_and_check(r, f2, p2)
    assert after["components"] > 0
    r.close()


@pytest.mark.gpu
def test_gpu_repeated_searches_give_the_same_bits():
    import tloam_b200
    rng = np.random.default_rng(33)
    g = random_grid((300, 421), rng, 0.03, 0.3)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, ORIGIN, RES, **GRID_CFG)
    r.plan_build(po.centres([passable(f.costs, rng)], ORIGIN, RES)[0])
    out = []
    for _ in range(3):
        info, got = r.frontier_search()
        out.append((info, got, r.frontier_labels()))
    for info, got, lab in out[1:]:
        assert info == out[0][0] and np.array_equal(lab, out[0][2])
        for a, b in zip(got, out[0][1]):
            assert (a.id, a.cost.hex(), a.approach, a.size) == (b.id, b.cost.hex(), b.approach, b.size)
            assert np.array_equal(a.cells, b.cells) and same_bits(a.xy, b.xy)
    r.close()


@pytest.mark.gpu
def test_gpu_frontier_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.FrontierConfig()
    L.tloam_b200_frontier_default_config(C.byref(cfg))
    assert (cfg.free_max, cfg.min_frontier_size, cfg.potential_scale, cfg.gain_scale) == (252, 0.5, 3.0, 1.0)
    info = _lib.FrontierInfo()
    assert L.tloam_b200_frontier_search(h, C.byref(cfg), C.byref(info)) == _lib.ERR_NOT_READY     # no field
    assert L.tloam_b200_frontier_download(h, None, 1 << 30) == _lib.ERR_NOT_READY
    assert L.tloam_b200_frontier_cells(h, None, None, None, 1 << 30) == _lib.ERR_NOT_READY
    assert L.tloam_b200_frontier_labels(h, None, 1 << 30) == _lib.ERR_NOT_READY
    g = np.zeros((4, 6), dtype=np.int8)
    g[:, 4:] = -1
    g[0, 3] = 100
    r.distance_build(g, (0.0, 0.0), 1.0, **BARE)
    assert L.tloam_b200_frontier_search(h, C.byref(cfg), None) == _lib.ERR_NOT_READY               # no plan
    r.plan_build((0.5, 0.5))
    assert L.tloam_b200_frontier_search(None, C.byref(cfg), None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_frontier_search(h, None, None) == _lib.ERR_INVALID_ARG
    for field, bad in (("free_max", 253), ("min_frontier_size", -0.1), ("min_frontier_size", np.inf),
                       ("potential_scale", np.nan), ("potential_scale", -1.0), ("gain_scale", -np.inf)):
        c = _lib.FrontierConfig()
        L.tloam_b200_frontier_default_config(C.byref(c))
        setattr(c, field, bad)
        assert L.tloam_b200_frontier_search(h, C.byref(c), None) == _lib.ERR_INVALID_ARG, field
    c = _lib.FrontierConfig(252, 0.0, 0.0, 0.0)
    assert L.tloam_b200_frontier_search(h, C.byref(c), C.byref(info)) == _lib.OK
    # column 4 below row 0 (row 0's west neighbour is lethal); the approach (3, 1), since (3, 0) closes its diagonal
    assert (info.cells, info.components, info.kept, info.reachable, info.goal_i, info.goal_j) == (3, 1, 1, 1, 0, 0)
    assert L.tloam_b200_frontier_download(h, None, 0) == _lib.ERR_INVALID_ARG
    rec = (_lib.FrontierRecord * 1)()
    assert L.tloam_b200_frontier_download(h, rec, 1) == _lib.OK
    assert (rec[0].size, rec[0].approach_i, rec[0].approach_j, rec[0].min_j, rec[0].max_j) == (3, 3, 1, 1, 3)
    assert rec[0].approach_potential == (po.SIDE + po.DIAG + po.SIDE) * 50
    assert L.tloam_b200_frontier_cells(h, None, None, None, 2) == _lib.ERR_INVALID_ARG
    ij = (C.c_int * 6)()
    assert L.tloam_b200_frontier_cells(h, None, ij, None, 3) == _lib.OK and list(ij) == [4, 1, 4, 2, 4, 3]
    assert L.tloam_b200_frontier_labels(h, None, 23) == _lib.ERR_INVALID_ARG
    lab = (C.c_uint * 24)()
    assert L.tloam_b200_frontier_labels(h, lab, 24) == _lib.OK
    assert [lab[j * 6 + 4] for j in range(4)] == [0xFFFFFFFF, 0, 0, 0] and lab[5] == 0xFFFFFFFF
    r.distance_build(g, (0.0, 0.0), 1.0, **BARE)                    # a new field: the plan is stale
    assert L.tloam_b200_frontier_search(h, C.byref(c), None) == _lib.ERR_NOT_READY
    assert L.tloam_b200_frontier_labels(h, lab, 24) == _lib.OK      # the refused search kept the last one
    assert L.tloam_b200_frontier_search(h, C.byref(c), None) == _lib.ERR_NOT_READY
    r.plan_build((0.5, 0.5))
    assert L.tloam_b200_frontier_search(h, C.byref(c), None) == _lib.OK
    assert L.tloam_b200_frontier_download(None, rec, 1) == _lib.ERR_INVALID_ARG
    r.close()


@pytest.mark.gpu
def test_gpu_search_changes_nothing_else():
    """a search leaves the distance field, the plan, its kept paths, the map and the launch counts of later appends as they
    are, and a later distance build or plan leaves the search's results"""
    from test_occupancy import COARSE, host_run, ray_frames
    import tloam_b200
    frames = ray_frames(10)
    plain, l_plain = host_run(frames[:8], True)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 20)
    r.occupancy_enable(**COARSE)
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
    g0 = r.occupancy_build()
    map0 = r.global_map()
    f = r.distance_build()
    p = r.plan_build(frames[5][1][:2, 3])
    t = po.cell_costs(f.costs)
    starts = po.centres(np.argwhere(t > 0)[::53][:, ::-1], f.origin, f.resolution)
    paths = r.plan_paths(starts)
    info, got = r.frontier_search()
    lab = r.frontier_labels()
    P = np.zeros(p.potential.size, dtype=np.uint64)
    assert r._L.tloam_b200_plan_download(r._h, P.ctypes.data_as(C.POINTER(C.c_ulonglong)), P.size) == 0
    assert np.array_equal(P.reshape(p.potential.shape), p.potential)
    m = sum(len(q.cells) for q in paths)
    ij = np.zeros((m, 2), dtype=np.int32)
    assert r._L.tloam_b200_plan_path_cells(r._h, ij.ctypes.data_as(C.POINTER(C.c_int)), None, m) == 0
    assert np.array_equal(ij, np.concatenate([q.cells for q in paths]))
    f1 = r.distance_build()
    assert same_bits(f1.signed, f.signed) and np.array_equal(f1.costs, f.costs) and np.array_equal(f1.values, f.values)
    assert np.array_equal(r.occupancy_build().cells, g0.cells) and same_bits(r.global_map(), map0)
    launches = []
    for scan, pose, inten in frames[6:8]:
        n0 = r.launch_count()
        r.global_map_append(scan, pose, intensity=inten)
        launches.append(r.launch_count() - n0)
    assert launches == l_plain[6:8] and same_bits(r.global_map(), plain.global_map())
    r.distance_build(np.zeros((3, 3), dtype=np.int8), (0.0, 0.0), 1.0)
    r.plan_build((0.5, 0.5))                                        # another field and plan: the search stays
    assert np.array_equal(r.frontier_labels(), lab)
    rec = (tloam_b200._lib.FrontierRecord * max(len(got), 1))()
    assert r._L.tloam_b200_frontier_download(r._h, rec, len(got)) == 0
    assert [rec[k].id for k in range(len(got))] == [q.id for q in got]
    mc = sum(q.size for q in got)
    cij = np.zeros((mc, 2), dtype=np.int32)
    assert r._L.tloam_b200_frontier_cells(r._h, None, cij.ctypes.data_as(C.POINTER(C.c_int)), None, mc) == 0
    assert np.array_equal(cij, np.concatenate([q.cells for q in got]))
    r.close()
    plain.close()


@pytest.mark.gpu
def test_gpu_frontier_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("frontier_driver", "front_end_b200.hpp")
    d = os.path.dirname(exe)
    in_path, out_path = os.path.join(d, "frontier_in.bin"), os.path.join(d, "frontier_out.bin")
    g, robot = room_with_two_doors()
    g[20:45, 5] = g[20:45, 64] = -1                                 # doors wide enough for the driver's 0.3 m inscribed
    rng = np.random.default_rng(8)
    g = np.where((g == 0) & (rng.random(g.shape) < 0.03), -1, g).astype(np.int8)     # unknown specks in the room too
    origin, res = (-1.5, 2.25), 0.1
    robot_xy = po.centres([robot], origin, res)[0]
    with open(in_path, "wb") as fh:
        fh.write(struct.pack("QQ3d", g.shape[1], g.shape[0], origin[0], origin[1], res) + g.tobytes())
        fh.write(struct.pack("2d", *robot_xy))
    run = subprocess.run([exe, in_path, out_path], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    r = tloam_b200.LocalRegistration()
    r.distance_build(g, origin, res, inscribed_radius=0.3, inflation_radius=1.0)
    r.plan_build(robot_xy)
    info, got = r.frontier_search()
    cells, comps, kept, reach = (int(v) for v in run.stdout.split())
    assert (cells, comps, kept, reach) == (info["cells"], info["components"], info["kept"], info["reachable"])
    blob = open(out_path, "rb").read()
    o = 0
    for q in got:
        fid, status, size, ap = struct.unpack_from("<QqQQ", blob, o)
        o += 32
        v = np.frombuffer(blob, dtype=np.float64, count=6, offset=o)
        o += 48
        xy = np.frombuffer(blob, dtype=np.float64, count=2 * size, offset=o).reshape(-1, 2)
        o += 16 * size
        assert (fid, status, size, ap) == (q.id, q.status, q.size, q.approach_potential)
        assert same_bits(v, [q.cost, q.distance, q.centroid[0], q.centroid[1], q.approach_xy[0], q.approach_xy[1]])
        assert same_bits(xy, q.xy)
    (m,) = struct.unpack_from("<Q", blob, o)
    o += 8
    route = np.frombuffer(blob, dtype=np.float64, count=2 * m, offset=o).reshape(-1, 2)
    o += 16 * m
    assert o == len(blob) and got and got[0].status == 0 and m > 1
    (path,) = r.plan_paths([got[0].approach_xy])
    assert same_bits(route, path.xy[::-1])
    r.close()
