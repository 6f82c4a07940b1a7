"""Path planning on the costmap (include/tloam_b200.h "Path planning"; k_plan_* in libtloam_b200_plan.so).
tests/plan_oracle.py is the bit-for-bit numpy restatement.

CPU: the heapq potential against a brute-force Bellman-Ford on tiny grids and against scipy's csgraph Dijkstra up to 512 x
512, the Bellman certificate's acceptance and rejections, the cell-cost rule at every code and the config limits, the path
rule (exact descent, no corner cutting, a pinned path on a symmetric grid, every status), the symbols, the new library's
kernels, the digests of every other library, the shim's driver.  GPU: the potential and the paths equal the restatement
on host grids of shapes on and off the tile size, a serpentine maze, a 2 048 x 2 048 grid (scipy), a seq-00-shaped grid
(the certificate) and the ray-cast drive's occupancy build, before and after a correction; repeat builds; snapshots and
refusals; nothing else changes; the status codes; the shim."""
import ctypes as C
import json
import os
import struct
import subprocess

import numpy as np
import pytest

import plan_oracle as po
import sass_digest
from test_distance import SEQ00, random_grid
from test_global_map_intensity import same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_plan_default_config", "tloam_b200_plan_build", "tloam_b200_plan_download",
               "tloam_b200_plan_paths", "tloam_b200_plan_path_cells"]
KERNELS = ("k_plan_init", "k_plan_round", "k_plan_count", "k_plan_length", "k_plan_walk")
TILE = 32
INF = int(po.INF)


def random_costs(shape, rng, p_lethal=0.15, p_unknown=0.1):
    """costmap codes of every kind: 0 .. 252, 253, 254 and 255"""
    c = rng.integers(0, 253, shape)
    c = np.where(rng.random(shape) < 0.5, 0, c)
    u = rng.random(shape)
    c = np.where(u < p_lethal, rng.choice([253, 254], shape), c)
    c = np.where((u >= p_lethal) & (u < p_lethal + p_unknown), 255, c)
    return c.astype(np.uint8)


def passable_cell(t, rng):
    j, i = np.argwhere(t > 0)[rng.integers(0, int((t > 0).sum()))]
    return int(i), int(j)


# ---------------------------------------------------------------------------------------------------------------------
def test_potential_matches_the_brute_force_on_tiny_grids():
    rng = np.random.default_rng(1)
    cases = [(np.array([[7]], dtype=np.uint16), (0, 0)),
             (po.cell_costs(random_costs((1, 9), rng, 0.2)), None), (po.cell_costs(random_costs((8, 1), rng, 0.2)), None)]
    only_goal = np.zeros((4, 5), dtype=np.uint16)                  # every cell impassable but the goal
    only_goal[2, 3] = 50
    cases.append((only_goal, (3, 2)))
    isolated = np.full((5, 5), 60, dtype=np.uint16)                # the goal walled in by impassable cells
    isolated[1:4, 1:4] = 0
    isolated[2, 2] = 60
    cases.append((isolated, (2, 2)))
    for shape in ((3, 4), (6, 5), (7, 7)):
        for allow in (0, 1):
            cases.append((po.cell_costs(random_costs(shape, rng, 0.25), allow_unknown=allow), None))
    for t, goal in cases:
        if t.max() == 0:
            continue
        goal = goal or passable_cell(t, rng)
        P = po.potential(t, goal)
        assert np.array_equal(P, po.brute(t, goal)), (t, goal)
        assert po.bellman_holds(P, t, goal)
    P = po.potential(only_goal, (3, 2))
    assert P[2, 3] == 0 and (P[only_goal == 0] == po.INF).all()
    P = po.potential(isolated, (2, 2))
    assert P[2, 2] == 0 and (np.delete(P.ravel(), 12) == po.INF).all()


@pytest.mark.parametrize("shape", [(8, 8), (37, 53), (128, 128), (512, 512)])
@pytest.mark.parametrize("allow_unknown", [0, 1])
def test_potential_matches_scipy(shape, allow_unknown):
    rng = np.random.default_rng(shape[0] + allow_unknown)
    t = po.cell_costs(random_costs(shape, rng), allow_unknown=allow_unknown)
    goal = passable_cell(t, rng)
    P = po.potential(t, goal)
    assert np.array_equal(P, po.scipy_potential(t, goal))
    assert (P != po.INF).sum() > 1


def test_bellman_certificate_accepts_the_potential_and_rejects_every_fault():
    rng = np.random.default_rng(5)
    t = po.cell_costs(random_costs((40, 60), rng, 0.1, 0.0))
    t[20, :] = 0                                                   # a wall: the rows below cannot reach the goal
    goal = (5, 5)
    t[goal[1], goal[0]] = 50
    P = po.potential(t, goal)
    assert po.bellman_holds(P, t, goal)
    fin = np.argwhere((P != po.INF) & (P != 0))
    for k in range(20):
        j, i = fin[rng.integers(0, len(fin))]
        for delta in (1, -1):
            Q = P.copy()
            Q[j, i] = np.uint64(int(Q[j, i]) + delta)
            assert not po.bellman_holds(Q, t, goal)
    pocket = np.argwhere((P == po.INF) & (t > 0))
    assert len(pocket) and (pocket[:, 0] > 20).all()
    Q = P.copy()
    Q[pocket[0][0], pocket[0][1]] = 10 ** 6                        # a finite value where the goal cannot be reached
    assert not po.bellman_holds(Q, t, goal)
    Q = P.copy()
    Q[goal[1], goal[0]] = 1
    assert not po.bellman_holds(Q, t, goal)


def test_cell_cost_rule_at_every_code_and_the_config_limits():
    codes = np.arange(256, dtype=np.uint8)
    for neutral, factor in ((50, 3), (1, 0), (1, 259), (65535, 0), (100, 259)):
        for allow in (0, 1):
            t = po.cell_costs(codes, neutral, factor, allow)
            want = [neutral + factor * c if c <= 252 else (neutral + factor * 252 if c == 255 and allow else 0)
                    for c in range(256)]
            assert t.tolist() == want and t.dtype == np.uint16
    assert po.config_valid(1, 0, 0) and po.config_valid(65535, 0, 1) and po.config_valid(1, 260, 1)
    assert po.config_valid(65535 - 252 * 259, 259, 0) and not po.config_valid(65536 - 252 * 259, 259, 0)
    assert not po.config_valid(0, 3, 1) and not po.config_valid(50, 3, 2) and not po.config_valid(1, 261, 0)


def test_paths_descend_by_exactly_each_steps_cost():
    rng = np.random.default_rng(7)
    t = po.cell_costs(random_costs((90, 70), rng, 0.2))
    goal = passable_cell(t, rng)
    P = po.potential(t, goal)
    starts = np.argwhere(P != po.INF)[:, ::-1][rng.integers(0, int((P != po.INF).sum()), 200)]
    for status, cost, cells in po.paths(P, t, starts):
        assert status == 0 and cost == int(P[cells[0, 1], cells[0, 0]]) and tuple(cells[-1]) == goal
        for (i0, j0), (i1, j1) in zip(cells[:-1], cells[1:]):
            k = po.DIAG if i0 != i1 and j0 != j1 else po.SIDE
            assert max(abs(i1 - i0), abs(j1 - j0)) == 1
            assert int(P[j0, i0]) - int(P[j1, i1]) == k * int(t[j1, i1])


def test_paths_never_cut_a_corner_between_lethal_cells():
    t = np.full((6, 6), 50, dtype=np.uint16)
    t[2, 2] = t[3, 3] = 0                                          # corner-touching: the gap (2, 3)-(3, 2) is closed
    t[:, 4:] = 0
    t[4:, :] = 0
    P = po.potential(t, (3, 2))
    (status, cost, cells), = po.paths(P, t, [(2, 3)])
    assert status == 0 and cost == int(P[3, 2])
    steps = {(tuple(a), tuple(b)) for a, b in zip(cells[:-1], cells[1:])}
    assert ((2, 3), (3, 2)) not in steps and len(cells) > 2
    assert po.bellman_holds(P, t, (3, 2))


def test_neighbour_order_pins_the_path_on_a_symmetric_grid():
    t = np.full((5, 5), 50, dtype=np.uint16)
    t[2, 1:4] = 0                                                  # a wall across the middle, mirror-symmetric in x
    P = po.potential(t, (2, 0))
    assert np.array_equal(P, P[:, ::-1])
    (status, cost, cells), = po.paths(P, t, [(2, 4)])
    assert status == 0 and cost == int(P[4, 2])
    # at the start (+1, 0), (-1, 0) and the diagonals (+1, -1), (-1, -1) tie and (+1, 0) comes first, so the path goes
    # round the right end; at (4, 1) the side move (-1, 0) ties with the diagonal (-1, -1) and comes first
    assert cells.tolist() == [[2, 4], [3, 4], [4, 3], [4, 2], [4, 1], [3, 1], [2, 0]]


def test_every_status_is_produced():
    t = np.full((4, 6), 50, dtype=np.uint16)
    t[:, 3] = 0
    P = po.potential(t, (0, 0))
    ij, ok = po.cells_of([[0.5, 0.5], [3.5, 1.5], [5.5, 2.5], [np.nan, 0.0], [-0.01, 1.0], [6.0, 1.0], [0.2, 0.3]],
                         (0.0, 0.0), 1.0, t.shape)
    out = po.paths(P, t, ij, ok)
    assert [s for s, _, _ in out] == [0, 2, 3, 1, 1, 1, 0]
    assert out[0][2].tolist() == [[0, 0]] and out[0][1] == 0 and out[2][1] == INF and len(out[2][2]) == 0
    assert po.centres([[0, 0], [5, 3]], (-1.0, 2.0), 0.1).tolist() == [[-1.0 + 0.5 * 0.1, 2.0 + 0.5 * 0.1],
                                                                      [-1.0 + 5.5 * 0.1, 2.0 + 3.5 * 0.1]]


# ---- the library ------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_plan_library_holds_only_its_kernels_for_sm90a_without_stack():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.PLAN_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.PLAN_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.PLAN_LIB], capture_output=True, text=True,
                         check=True).stdout
    usage = [l for l in res.splitlines() if "REG:" in l]
    assert len(usage) == len(KERNELS) and all("STACK:0 " in l for l in usage), usage


def test_every_other_library_keeps_its_sass():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_plan.json")))
    assert len(want) == 17 and "libtloam_b200_plan.so" not in want and "libtloam_b200_dist.so" in want
    for lib in want:
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


def test_plan_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "plan_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
GRID_CFG = dict(inscribed_radius=0.3, inflation_radius=1.0)        # at 0.25 m: codes 0, 1 .. 252, 253, 254 and 255
ORIGIN, RES = (-3.25, 7.5), 0.25


def centre(cell, origin=ORIGIN, res=RES):
    return po.centres([cell], origin, res)[0]


def plan_and_check(r, f, goal, starts=(), exact=True, **cfg):
    """plan_build at the centre of cell goal and plan_paths from the centres of starts against the restatement"""
    c = po.config(**cfg)
    t = po.cell_costs(f.costs, **c)
    p = r.plan_build(centre(goal, f.origin, f.resolution), **cfg)
    assert p.goal == tuple(goal) and p.origin == f.origin and p.resolution == f.resolution
    assert p.potential.shape == f.costs.shape
    if exact:
        assert np.array_equal(p.potential, po.potential(t, goal))
    else:
        assert po.bellman_holds(p.potential, t, goal)
    assert p.reachable == int((p.potential != po.INF).sum()) and p.rounds >= 1 and p.tiles >= p.rounds
    xy = po.centres(starts, f.origin, f.resolution) if len(starts) else np.zeros((0, 2))
    got = r.plan_paths(xy)
    ij, ok = po.cells_of(xy, f.origin, f.resolution, f.costs.shape)
    want = po.paths(p.potential, t, ij, ok)
    assert len(got) == len(want)
    for g, (status, cost, cells) in zip(got, want):
        assert (g.status, g.cost) == (status, cost) and np.array_equal(g.cells, cells)
        assert same_bits(g.xy, po.centres(cells, f.origin, f.resolution).reshape(-1, 2))
    return p, got, t


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1, 1), (1, 777), (513, 1), (31, 31), (32, 32), (33, 33), (64, 64), (65, 65),
                                   (255, 257)])
def test_gpu_host_grids_are_the_restatement(shape):
    import tloam_b200
    rng = np.random.default_rng(shape[0] * 1000 + shape[1])
    g = random_grid(shape, rng, 0.04, 0.15)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, ORIGIN, RES, **GRID_CFG)
    for allow in (0, 1):
        t = po.cell_costs(f.costs, allow_unknown=allow)
        if not t.any():
            continue
        goal = passable_cell(t, rng)
        starts = [tuple(x) for x in np.argwhere(np.ones(shape))[rng.integers(0, g.size, 64)][:, ::-1]] + [goal]
        plan_and_check(r, f, goal, starts, allow_unknown=allow)
        plan_and_check(r, f, goal, starts, neutral_cost=1, cost_factor=259, allow_unknown=allow)
        plan_and_check(r, f, goal, starts, neutral_cost=65535, cost_factor=0, allow_unknown=allow)
    r.close()


def serpentine(H=200, W=200, x0=16, x1=48):
    """one-cell corridors along rows 1, 3, 5, ... from column x0 to x1 (across the tile boundary at 32), joined at
    alternating ends; everything else an obstacle.  Returns the grid, the corridor's first and last cell"""
    g = np.full((H, W), 100, dtype=np.int8)
    rows = list(range(1, H - 1, 2))
    for k, j in enumerate(rows):
        g[j, x0:x1 + 1] = 0
        if k + 1 < len(rows):
            g[j + 1, x1 if k % 2 == 0 else x0] = 0
    last = (x1 if len(rows) % 2 == 1 else x0, rows[-1])
    return g, (x0, rows[0]), last


def distinct_tile_runs(cells):
    """the fewest runs of pairwise-distinct tiles the path's tile sequence splits into"""
    runs, seen, prev = 1, set(), None
    for i, j in cells:
        tile = (i // TILE, j // TILE)
        if tile == prev:
            continue
        if tile in seen:
            runs += 1
            seen = set()
        seen.add(tile)
        prev = tile
    return runs


@pytest.mark.gpu
def test_gpu_serpentine_maze_is_exact_and_takes_a_round_per_fold():
    """A block relaxes each of its tiles once per round, and a cell that falls on a tile's edge reaches the next tile
    through the next round's worklist or, when that tile is staged later in the same round, at once; either way the
    front passes through any one tile at most once per round.  So the rounds are at least the number of runs of
    distinct tiles along the path, which on this maze is about the number of folds."""
    import tloam_b200
    g, first, last = serpentine()
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, (0.0, 0.0), 0.1, inscribed_radius=0.0, inflation_radius=0.0)
    assert set(np.unique(f.costs).tolist()) == {0, 254}
    p, paths, t = plan_and_check(r, f, first, [last, first])
    cells = paths[0].cells
    assert len(cells) == int((g == 0).sum()) and paths[1].cells.tolist() == [list(first)]
    crossings = sum(1 for a, b in zip(cells[:-1], cells[1:]) if (a[0] // TILE, a[1] // TILE) != (b[0] // TILE, b[1] // TILE))
    runs = distinct_tile_runs(cells[::-1].tolist())
    assert crossings >= 99 and runs >= 49                          # about one run per two folds
    assert p.rounds >= runs, (p.rounds, runs, crossings)
    r.close()


@pytest.mark.gpu
def test_gpu_goal_on_a_tile_corner_reaches_the_tiles_around_it():
    """the goal's only passable neighbours lie in the three other tiles at its corner: the goal never falls, so those
    tiles must be relaxed from the start"""
    import tloam_b200
    for gi, gj in ((31, 31), (32, 32), (31, 32), (32, 31), (31, 5), (5, 32)):
        g = np.zeros((70, 66), dtype=np.int8)
        ti, tj = gi // TILE, gj // TILE
        for dj in (-1, 0, 1):
            for di in (-1, 0, 1):
                i, j = gi + di, gj + dj
                if (di or dj) and i // TILE == ti and j // TILE == tj:
                    g[j, i] = 100                                  # every neighbour inside the goal's tile is lethal
        r = tloam_b200.LocalRegistration()
        f = r.distance_build(g, (0.0, 0.0), 1.0, inscribed_radius=0.0, inflation_radius=0.0)
        p, _, _ = plan_and_check(r, f, (gi, gj), [(0, 0), (65, 69)])
        assert p.reachable > 60 * 60, (gi, gj)
        r.close()


@pytest.mark.gpu
def test_gpu_2048_square_equals_scipy():
    import tloam_b200
    rng = np.random.default_rng(2048)
    g = random_grid((2048, 2048), rng, 0.02, 0.2)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, ORIGIN, RES, **GRID_CFG)
    t = po.cell_costs(f.costs)
    goal = passable_cell(t, rng)
    p = r.plan_build(centre(goal))
    assert np.array_equal(p.potential, po.scipy_potential(t, goal)) and p.reachable > 2048 * 1024
    r.close()


@pytest.mark.gpu
def test_gpu_seq00_shaped_grid_passes_the_certificate_and_its_paths_are_the_rule():
    import tloam_b200
    rng = np.random.default_rng(0)
    g = random_grid(SEQ00, rng, p_obstacle=0.002, p_unknown=0.3)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, (-270.3, -310.7), 0.1, **GRID_CFG)
    t = po.cell_costs(f.costs)
    goal = passable_cell(t, rng)
    starts = [tuple(x) for x in np.argwhere(np.ones(SEQ00, dtype=bool)[::97, ::97])[:1024][:, ::-1] * 97]
    p, paths, _ = plan_and_check(r, f, goal, starts, exact=False)
    assert p.reachable > SEQ00[0] * SEQ00[1] // 4 and sum(q.status == 0 for q in paths) > 256
    r.close()


def occupancy_drive(frames, correction=False):
    import tloam_b200
    from test_occupancy import COARSE
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 20)
    if correction:
        r.global_map_correction_enable()
    r.occupancy_enable(**COARSE)
    return r


@pytest.mark.gpu
def test_gpu_occupancy_drive_plans_exactly_and_follows_a_correction():
    import pose_graph_oracle as pgo
    from test_occupancy import ray_frames
    from test_pose_graph import loop_result
    frames = ray_frames(10)
    r = occupancy_drive(frames, correction=True)
    r.pose_graph_enable()
    O = []
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
        r.pose_graph_add_node(pose)
        O.append(pose)
    r.occupancy_build()
    f = r.distance_build()
    goal_xy, start_xy = O[0][:2, 3], O[-1][:2, 3]
    before = r.plan_build(goal_xy)
    t = po.cell_costs(f.costs)
    assert np.array_equal(before.potential, po.potential(t, before.goal))
    (path,) = r.plan_paths([start_xy])
    assert path.status == 0 and tuple(path.cells[-1]) == before.goal
    assert (t[path.cells[:, 1], path.cells[:, 0]] > 0).all()
    r.pose_graph_add_loop(loop_result(1, 5, pgo.inv_mul(O[1], O[5]) @ pgo.exp4([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(6))
    r.occupancy_build()
    f2 = r.distance_build()
    after = r.plan_build(goal_xy)
    t2 = po.cell_costs(f2.costs)
    assert np.array_equal(after.potential, po.potential(t2, after.goal))
    assert after.potential.shape != before.potential.shape or not np.array_equal(after.potential, before.potential)
    (path,) = r.plan_paths([start_xy])
    assert path.status == 0 and (t2[path.cells[:, 1], path.cells[:, 0]] > 0).all()
    r.close()


@pytest.mark.gpu
def test_gpu_repeated_builds_give_the_same_bits():
    import tloam_b200
    rng = np.random.default_rng(33)
    g = random_grid((300, 421), rng, 0.03, 0.2)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(g, ORIGIN, RES, **GRID_CFG)
    goal = passable_cell(po.cell_costs(f.costs), rng)
    starts = po.centres(np.argwhere(np.ones((300, 421)))[::997][:, ::-1], ORIGIN, RES)
    out = []
    for _ in range(3):
        p = r.plan_build(centre(goal))
        out.append((p.potential, r.plan_paths(starts)))
    for P, paths in out[1:]:
        assert np.array_equal(P, out[0][0])
        assert all(np.array_equal(a.cells, b.cells) and a.cost == b.cost for a, b in zip(paths, out[0][1]))
    r.close()


def download_potential(r, n):
    P = np.zeros(n, dtype=np.uint64)
    assert r._L.tloam_b200_plan_download(r._h, P.ctypes.data_as(C.POINTER(C.c_ulonglong)), n) == 0
    return P


def download_cells(r, m):
    ij, xy = np.zeros((m, 2), dtype=np.int32), np.zeros((m, 2))
    assert r._L.tloam_b200_plan_path_cells(r._h, ij.ctypes.data_as(C.POINTER(C.c_int)),
                                           xy.ctypes.data_as(C.POINTER(C.c_double)), m) == 0
    return ij, xy


@pytest.mark.gpu
def test_gpu_plan_is_a_snapshot_and_changes_nothing_else():
    """a later distance build and a refused plan build keep the potential and the paths; plan calls leave the distance
    field, the occupancy cells, the map and the launch counts of later appends as they are"""
    from test_occupancy import host_run, ray_frames
    frames = ray_frames(10)
    plain, l_plain = host_run(frames[:8], True)
    r = occupancy_drive(frames)
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
    g0 = r.occupancy_build()
    map0 = r.global_map()
    f = r.distance_build()
    t = po.cell_costs(f.costs)
    goal = passable_cell(t, np.random.default_rng(2))
    p = r.plan_build(centre(goal, f.origin, f.resolution))
    starts = po.centres(np.argwhere(t > 0)[::53][:, ::-1], f.origin, f.resolution)
    paths = r.plan_paths(starts)
    m = sum(len(q.cells) for q in paths)
    assert m > len(paths) and np.array_equal(p.potential, po.potential(t, goal))
    f1 = r.distance_build()
    assert same_bits(f1.signed, f.signed) and np.array_equal(f1.costs, f.costs) and np.array_equal(f1.values, f.values)
    assert np.array_equal(r.occupancy_build().cells, g0.cells) and same_bits(r.global_map(), map0)
    launches = []
    for scan, pose, inten in frames[6:8]:
        n0 = r.launch_count()
        r.global_map_append(scan, pose, intensity=inten)
        launches.append(r.launch_count() - n0)
    assert launches == l_plain[6:8] and same_bits(r.global_map(), plain.global_map())
    r.occupancy_build()
    r.distance_build(np.zeros((3, 3), dtype=np.int8), (0.0, 0.0), 1.0)   # another field: the plan stays
    assert np.array_equal(download_potential(r, p.potential.size).reshape(p.potential.shape), p.potential)
    ij, xy = download_cells(r, m)
    assert np.array_equal(ij, np.concatenate([q.cells for q in paths]))
    assert same_bits(xy, np.concatenate([q.xy for q in paths]))
    with pytest.raises(tloam_b200_error()):
        r.plan_build((100.0, 100.0))                               # outside the new field: refused
    assert np.array_equal(download_potential(r, p.potential.size).reshape(p.potential.shape), p.potential)
    assert np.array_equal(download_cells(r, m)[0], ij)
    r.close()
    plain.close()


def tloam_b200_error():
    import tloam_b200
    return tloam_b200.RegistrationError


@pytest.mark.gpu
def test_gpu_plan_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.PlanConfig()
    L.tloam_b200_plan_default_config(C.byref(cfg))
    assert (cfg.neutral_cost, cfg.cost_factor, cfg.allow_unknown) == (50, 3, 1)
    info = _lib.PlanInfo()
    xy = np.array([0.5, 0.5])
    dp = xy.ctypes.data_as(C.POINTER(C.c_double))
    off = (C.c_size_t * 2)()
    st = (C.c_int * 1)()
    cost = (C.c_ulonglong * 1)()
    assert L.tloam_b200_plan_build(h, C.byref(cfg), 0.5, 0.5, C.byref(info)) == _lib.ERR_NOT_READY   # no distance build
    assert L.tloam_b200_plan_download(h, None, 1 << 30) == _lib.ERR_NOT_READY
    assert L.tloam_b200_plan_paths(h, dp, 1, off, st, cost) == _lib.ERR_NOT_READY
    assert L.tloam_b200_plan_path_cells(h, None, None, 1 << 30) == _lib.ERR_NOT_READY
    g = np.zeros((4, 6), dtype=np.int8)
    g[:, 3] = 100                                                  # column 3 lethal; columns 4, 5 cut off
    g[0, 5] = -1                                                   # unknown
    r.distance_build(g, (0.0, 0.0), 1.0, inscribed_radius=0.0, inflation_radius=0.0)
    assert L.tloam_b200_plan_build(None, C.byref(cfg), 0.5, 0.5, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_plan_build(h, None, 0.5, 0.5, None) == _lib.ERR_INVALID_ARG
    for field, bad in (("neutral_cost", 0), ("cost_factor", 261), ("allow_unknown", 2), ("allow_unknown", -1)):
        c = _lib.PlanConfig()
        L.tloam_b200_plan_default_config(C.byref(c))
        setattr(c, field, bad)
        assert L.tloam_b200_plan_build(h, C.byref(c), 0.5, 0.5, None) == _lib.ERR_INVALID_ARG, field
    c = _lib.PlanConfig(65535 - 252 * 260, 260, 0)                 # at the limit: allowed
    assert L.tloam_b200_plan_build(h, C.byref(c), 0.5, 0.5, None) == _lib.OK
    c = _lib.PlanConfig(65536 - 252 * 260, 260, 0)
    assert L.tloam_b200_plan_build(h, C.byref(c), 0.5, 0.5, None) == _lib.ERR_INVALID_ARG
    for gx, gy in ((np.nan, 0.5), (0.5, np.inf), (-0.01, 0.5), (6.0, 0.5), (0.5, 4.0), (3.5, 0.5)):   # bad / lethal goals
        assert L.tloam_b200_plan_build(h, C.byref(cfg), gx, gy, None) == _lib.ERR_INVALID_ARG, (gx, gy)
    c0 = _lib.PlanConfig(50, 3, 0)
    assert L.tloam_b200_plan_build(h, C.byref(c0), 5.5, 0.5, None) == _lib.ERR_INVALID_ARG   # unknown, allow_unknown 0
    assert L.tloam_b200_plan_build(h, C.byref(cfg), 5.5, 0.5, C.byref(info)) == _lib.OK      # unknown, allow_unknown 1
    assert (info.goal_i, info.goal_j, info.width, info.height, info.reachable) == (5, 0, 6, 4, 8)
    assert L.tloam_b200_plan_build(h, C.byref(cfg), 0.5, 0.5, C.byref(info)) == _lib.OK
    assert (info.goal_i, info.goal_j, info.reachable, info.rounds, info.tiles) == (0, 0, 12, 1, 1)
    assert L.tloam_b200_plan_download(h, None, 23) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_plan_download(h, None, 24) == _lib.OK
    assert L.tloam_b200_plan_path_cells(h, None, None, 0) == _lib.ERR_NOT_READY    # a new build drops the paths
    assert L.tloam_b200_plan_paths(h, None, 1, off, st, cost) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_plan_paths(h, None, (1 << 24) + 1, None, None, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_plan_paths(h, None, 0, off, None, None) == _lib.OK and off[0] == 0
    starts = np.array([[2.5, 3.5], [3.5, 0.5], [4.5, 1.5], [np.nan, 0.0], [9.0, 0.0]])
    offs = (C.c_size_t * 6)()
    sts = (C.c_int * 5)()
    costs = (C.c_ulonglong * 5)()
    assert L.tloam_b200_plan_paths(h, starts.ctypes.data_as(C.POINTER(C.c_double)), 5, offs, sts, costs) == _lib.OK
    assert list(sts) == [0, 2, 3, 1, 1] and list(offs) == [0, 4, 4, 4, 4, 4] and costs[0] == (2 * po.DIAG + po.SIDE) * 50
    assert list(costs)[1:] == [INF] * 4
    assert L.tloam_b200_plan_path_cells(h, None, None, 3) == _lib.ERR_INVALID_ARG
    ij = (C.c_int * 8)()
    assert L.tloam_b200_plan_path_cells(h, ij, None, 4) == _lib.OK and list(ij) == [2, 3, 2, 2, 1, 1, 0, 0]
    assert L.tloam_b200_plan_path_cells(None, ij, None, 4) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_plan_download(None, None, 24) == _lib.ERR_INVALID_ARG
    r.close()


@pytest.mark.gpu
def test_gpu_plan_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("plan_driver", "front_end_b200.hpp")
    d = os.path.dirname(exe)
    in_path, out_path = os.path.join(d, "plan_in.bin"), os.path.join(d, "plan_out.bin")
    rng = np.random.default_rng(8)
    grid = random_grid((90, 133), rng, 0.03, 0.15)
    r = tloam_b200.LocalRegistration()
    f = r.distance_build(grid, ORIGIN, RES, **GRID_CFG)
    goal = centre(passable_cell(po.cell_costs(f.costs), rng))
    starts = np.column_stack([rng.uniform(ORIGIN[0] - 1, ORIGIN[0] + 34, 200), rng.uniform(ORIGIN[1] - 1, ORIGIN[1] + 23, 200)])
    with open(in_path, "wb") as fh:
        fh.write(struct.pack("QQ3d", 133, 90, ORIGIN[0], ORIGIN[1], RES) + grid.tobytes())
        fh.write(struct.pack("2d", *goal) + struct.pack("Q", len(starts)) + starts.tobytes())
    run = subprocess.run([exe, in_path, out_path], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    p = r.plan_build(goal)
    paths = r.plan_paths(starts)
    r.close()
    w, h, reachable = (int(v) for v in run.stdout.split())
    assert (h, w) == p.potential.shape and reachable == p.reachable
    blob = open(out_path, "rb").read()
    n = w * h
    assert np.array_equal(np.frombuffer(blob, dtype=np.uint64, count=n).reshape(h, w), p.potential)
    o = 8 * n
    for q in paths:
        status, cost, m = struct.unpack_from("<qQQ", blob, o)
        o += 24
        xy = np.frombuffer(blob, dtype=np.float64, count=2 * m, offset=o).reshape(-1, 2)
        o += 16 * m
        assert (status, cost) == (q.status, q.cost) and same_bits(xy, q.xy)
    assert o == len(blob)
