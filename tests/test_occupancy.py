"""The occupancy grid of the global map (include/tloam_b200.h "Occupancy grid"; k_occ_* in libtloam_b200_occ.so): a 2D scan
per appended frame, and free and hit counts per cell at the frames' current poses.  tests/occupancy_oracle.py is the
bit-for-bit numpy restatement.

CPU: the restatement against its literal transcription (rows on sector boundaries, at min_range / max_range, at z_lo /
z_hi, NaN and Inf rows, three distinct rows at one rho in every sector, a cell whose rho_c + free_margin equals e_j, hits on the grid's edge and outside it,
an empty map, the extent limit), the value rule and the PGM / YAML writer through map_server's reading rule, the quality
on the ray-cast drive at the true poses and with drifting odometry, the symbols, the new library's kernels, the digests of
every other library, the shim's driver.  GPU: every scan, count, value, the origin, the size and dropped equal the
restatement bit for bit (host appends with and without intensity, ties in rho, packed appends, the chained mapping loop, a grown
frame table, a reset, a refused append, a correction); the grid changes no map bit and, off, no launch count; the status
codes; the shim."""
import ctypes as C
import functools
import json
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import occupancy_oracle as oo
import sass_digest
import scan_context_oracle as sco
from test_global_map_intensity import same_bits
from test_map_dynamic import pose_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_occupancy_default_config", "tloam_b200_occupancy_enable", "tloam_b200_occupancy_build",
               "tloam_b200_occupancy_download", "tloam_b200_occupancy_scans_download"]
KERNELS = ("k_occ_clear", "k_occ_bin", "k_occ_pick", "k_occ_final", "k_occ_extent", "k_occ_free", "k_occ_hits",
           "k_occ_value")
# the GPU tests' grid: coarse enough for the restatement to run in a moment, the ray-cast world's 360 azimuths
COARSE = dict(resolution=0.25, n_cols=360, z_lo=-1.2, z_hi=0.5, min_range=3.0, max_range=30.0, free_margin=0.1)
SMALL = [oo.config(resolution=1.0, n_cols=7, z_lo=-1.0, z_hi=0.5, min_range=1.0, max_range=8.0, free_margin=0.3),
         oo.config(resolution=0.5, n_cols=24, z_lo=-0.5, z_hi=1.0, min_range=0.5, max_range=6.0, free_margin=0.0),
         oo.config(resolution=0.7, n_cols=1, z_lo=-2.0, z_hi=-0.5, min_range=2.0, max_range=9.0, free_margin=0.5)]


def edge_scan(cfg, rng, n=400):
    """a seeded sensor-frame cloud with the edge rows of the definition"""
    D = sco.boundaries(cfg["n_cols"])
    r = rng.uniform(0.5 * cfg["min_range"], 1.1 * cfg["max_range"], n)
    az = rng.uniform(0, 2 * np.pi, n)
    z = rng.uniform(cfg["z_lo"] - 1.0, cfg["z_hi"] + 1.0, n)
    p = np.stack([r * np.cos(az), r * np.sin(az), z], axis=1)
    lo, hi = cfg["min_range"], cfg["max_range"]
    extra = [[np.nan, 1.0, 0.0], [np.inf, 0.0, 0.0], [2.0, -np.inf, 0.0], [3.0, 1.0, np.nan], [lo, 0.0, cfg["z_lo"]],
             [hi, 0.0, cfg["z_hi"]], [-lo, 0.0, cfg["z_hi"]], [0.0, -hi, cfg["z_lo"]], [np.nextafter(hi, np.inf), 0.0, 0.0],
             [np.nextafter(lo, 0.0), 0.0, 0.0], [0.0, lo, np.nextafter(cfg["z_lo"], -np.inf)],
             [0.0, 0.5 * (lo + hi), np.nextafter(cfg["z_hi"], np.inf)]]
    for k in range(len(D)):                                        # exactly on every sector boundary
        rr = rng.uniform(lo, hi)
        extra.append([D[k, 0] * rr, D[k, 1] * rr, 0.5 * (cfg["z_lo"] + cfg["z_hi"])])
        extra.append([D[k, 0] * rr, D[k, 1] * rr, cfg["z_lo"] - 0.3])
    return np.concatenate([p, np.array(extra)])


def tie_scan(cfg, rng):
    """(scan, the obstacle every sector must keep, the one the highest index would give): per sector three distinct band
    rows at one (x, y), so at one rho bit for bit, with a farther band row and a floor row, all rows shuffled; the tied row
    of lowest index must win"""
    n, lo, hi = cfg["n_cols"], cfg["min_range"], cfg["max_range"]
    zs = np.linspace(cfg["z_lo"], cfg["z_hi"], 5)[1:4]
    rows, tied = [], []
    for j in range(n):
        a = 2.0 * np.pi * (j + 0.5) / n
        rho = rng.uniform(lo + 0.3 * (hi - lo), lo + 0.6 * (hi - lo))
        x, y = rho * math.cos(a), rho * math.sin(a)
        for z in zs:
            tied.append(len(rows))
            rows.append([x, y, z])
        rows.append([1.2 * x, 1.2 * y, zs[0]])                     # farther, in the band
        rows.append([1.1 * x, 1.1 * y, cfg["z_lo"] - 0.5])         # the floor
    rows = np.array(rows)
    order = rng.permutation(len(rows))
    scan = rows[order]
    where = np.argsort(order)                                      # new index of every original row
    want, last = np.full((n, 3), np.nan), np.full((n, 3), np.nan)
    for j in range(n):
        want[j] = rows[min(tied[3 * j:3 * j + 3], key=lambda t: where[t])]
        last[j] = rows[max(tied[3 * j:3 * j + 3], key=lambda t: where[t])]
    return scan, want, last


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(len(SMALL)))
def test_scan2d_matches_the_literal_transcription(k):
    cfg = SMALL[k]
    scan = edge_scan(cfg, np.random.default_rng(40 + k))
    ob, fl = oo.scan2d(scan, cfg)
    lob, lfl = oo.scan2d_literal(scan, cfg)
    assert same_bits(ob, lob) and same_bits(fl, lfl)
    assert (~np.isnan(ob[:, 0])).sum() >= min(cfg["n_cols"], 5) and (~np.isnan(fl)).any()
    assert np.isnan(oo.scan2d(np.zeros((0, 3)), cfg)[0]).all()


@pytest.mark.parametrize("k", range(len(SMALL)))
def test_obstacle_ties_go_to_the_lowest_row_index(k):
    cfg = SMALL[k]
    scan, want, last = tie_scan(cfg, np.random.default_rng(60 + k))
    ob, _ = oo.scan2d(scan, cfg)
    lob, _ = oo.scan2d_literal(scan, cfg)
    assert same_bits(ob, want) and same_bits(lob, want)
    assert not (want == last).all(axis=1).any()                    # the highest index would give another row everywhere


@pytest.mark.parametrize("k", range(len(SMALL)))
def test_build_matches_the_literal_transcription(k):
    """three frames, one tilted (roll and pitch), with hand-made obstacles past the window so that hits fall on the grid's
    last cells and outside it (dropped); a captured scan cannot drop a hit, since |P o - t| <= W - resolution"""
    cfg = SMALL[k]
    rng = np.random.default_rng(50 + k)
    poses = [pose_of(0.3, -0.2, 0.4), pose_of(4.1, 2.7, -1.3, 0.2), pose_of(-2.0, 5.5, 2.9)]
    c, s = math.cos(0.3), math.sin(0.3)
    poses[1] = poses[1] @ np.array([[1, 0, 0, 0], [0, c, -s, 0], [0, s, c, 0], [0, 0, 0, 1.0]]) @ \
        np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1.0]])
    scans = [oo.scan2d(edge_scan(cfg, rng), cfg) for _ in poses]
    far = scans[2][0].copy()
    W = oo.window(cfg)
    far[: min(3, len(far))] = [[W + 3.0, 0.0, 0.0], [-(W + 0.4), 0.1, 0.0], [0.0, W - 0.01, 0.0]][: min(3, len(far))]
    scans[2] = (far, scans[2][1])
    got, want = oo.build(scans, poses, cfg), oo.build_literal(scans, poses, cfg)
    for key in ("origin", "width", "height", "dropped"):
        assert got[key] == want[key], key
    for key in ("occupied", "free", "cells"):
        assert np.array_equal(got[key], want[key]), key
    assert got["dropped"] > 0 and got["free"].sum() > 0 and got["occupied"].sum() > 0


def test_free_margin_equality_counts_free():
    """a cell whose rho_c + free_margin equals e_j bit for bit is free; the next cell out is not"""
    cfg = oo.config(resolution=0.5, n_cols=8, min_range=1.0, max_range=10.0, free_margin=0.1)
    W, r = oo.window(cfg), cfg["resolution"]
    ox = r * math.floor((0.0 - W) / r)
    ty = ox + (40 + 0.5) * r                                       # the frame on a row of cell centres: d1 = 0
    d0 = (ox + (float(30) + 0.5) * r) - 0.0                        # cell 30 of that row
    assert d0 > cfg["min_range"]
    e = d0 + cfg["free_margin"]
    ob = np.full((8, 3), np.nan)
    ob[0] = [e, 0.0, 0.0]                                          # sector 0, rho = sqrt(e e) = e
    P = pose_of(0.0, ty, 0.0)
    g = oo.build([(ob, np.full(8, np.nan))], [P], cfg)
    lg = oo.build_literal([(ob, np.full(8, np.nan))], [P], cfg)
    assert np.array_equal(g["free"], lg["free"])
    jy = int(round((ty - g["origin"][1]) / r - 0.5))
    i = int(round((0.0 + d0 - g["origin"][0]) / r - 0.5))
    assert g["free"][jy, i] == 1 and g["free"][jy, i + 1] == 0


def test_empty_map_and_the_extent_limit():
    cfg = oo.config()
    g = oo.build([], [], cfg)
    assert (g["width"], g["height"], g["dropped"]) == (0, 0, 0) and g["cells"].shape == (0, 0)
    ob, fl = np.full((cfg["n_cols"], 3), np.nan), np.full(cfg["n_cols"], np.nan)
    far = [pose_of(0.0, 0.0, 0.0), pose_of(3000.0, 3000.0, 0.0)]     # 60 k x 60 k cells > 2^28
    assert oo.build([(ob, fl)] * 2, far, cfg) is None
    near = [pose_of(0.0, 0.0, 0.0), pose_of(1000.0, 0.0, 0.0)]
    ox, oy, w, h = oo.grid_extent(near, cfg)
    assert w * h <= oo.MAX_CELLS and ox <= -oo.window(cfg) and oy <= -oo.window(cfg)


def test_value_rule():
    occ = np.array([0, 0, 1, 1, 2, 1, 65, 35, 3, 0], dtype=np.uint32)
    free = np.array([0, 5, 0, 1, 1, 2, 35, 65, 0, 4_000_000_000], dtype=np.uint32)
    want = [-1 if o + f == 0 else (100 * int(o) + (int(o) + int(f)) // 2) // (int(o) + int(f)) for o, f in zip(occ, free)]
    assert oo.values(occ, free).tolist() == want == [-1, 0, 100, 50, 67, 33, 65, 35, 100, 0]


def read_map_server(stem):
    """map_server's trinary reading rule (negate 0): p = (255 - v) / 255, > occupied_thresh -> 100, < free_thresh -> 0,
    else -1; image row 0 is the map's last row"""
    with open(stem + ".yaml") as f:
        y = dict(line.split(": ", 1) for line in f.read().splitlines() if ": " in line)
    with open(stem + ".pgm", "rb") as f:
        data = f.read()
    head, o = [], 0
    while len(head) < 4:
        end = data.index(b"\n", o)
        line = data[o:end]
        o = end + 1
        if not line.startswith(b"#"):
            head += line.split()
    assert head[0] == b"P5" and head[3] == b"255"
    w, h = int(head[1]), int(head[2])
    img = np.frombuffer(data, dtype=np.uint8, count=w * h, offset=o).reshape(h, w)[::-1]
    p = (255.0 - img) / 255.0
    occ_t, free_t = float(y["occupied_thresh"]), float(y["free_thresh"])
    out = np.where(p > occ_t, 100, np.where(p < free_t, 0, -1)).astype(np.int8)
    origin = [float(v) for v in y["origin"].strip("[]").split(",")]
    return out, origin, float(y["resolution"]), y["image"]


def test_pgm_writer_round_trips_through_map_servers_rule(tmp_path):
    import tloam_b200
    rng = np.random.default_rng(7)
    grid = rng.integers(-1, 101, (37, 53)).astype(np.int8)
    grid[0, :4] = [25, 26, 64, 65]
    stem = str(tmp_path / "map")
    tloam_b200.save_occupancy_map(stem, grid, (-12.5, 3.25), 0.1)
    got, origin, res, image = read_map_server(stem)
    want = np.where(grid >= 65, 100, np.where((grid >= 0) & (grid <= 25), 0, -1))
    assert np.array_equal(got, want)
    assert origin[:2] == [-12.5, 3.25] and res == 0.1 and image == "map.pgm"
    assert got[0, :4].tolist() == [0, -1, -1, 100]


# ---- quality on the ray-cast drive ------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def drive_scans():
    from test_loop_closure import cast, make_world, route
    world = make_world()
    return [cast(world, x, y, yaw, seed=k) for k, (x, y, yaw) in enumerate(route())]


def true_poses():
    from test_loop_closure import route
    return [pose_of(x, y, yaw) for x, y, yaw in route()]


def footprints():
    """(every box and pole, the boxes the route does not drive through): a box the sensor stands in is invisible to the
    ray cast from there, so the cells inside it are seen free"""
    from test_loop_closure import make_world, route
    c, h, poles = make_world()
    R = np.array([(x, y) for x, y, _ in route()])
    crossed = np.array([((np.abs(R[:, 0] - c[k, 0]) < h[k, 0]) & (np.abs(R[:, 1] - c[k, 1]) < h[k, 1])).any()
                        for k in range(len(c))])
    return (c, h, poles), (c[~crossed], h[~crossed], poles)


def footprint_distance(xy, world):
    """(distance to the nearest box footprint or pole disk, depth inside one: negative inside)"""
    c, h, poles = world
    d, depth = np.full(len(xy), np.inf), np.full(len(xy), np.inf)
    for k in range(len(c)):
        ax, ay = np.abs(xy[:, 0] - c[k, 0]) - h[k, 0], np.abs(xy[:, 1] - c[k, 1]) - h[k, 1]
        d = np.minimum(d, np.hypot(np.maximum(ax, 0.0), np.maximum(ay, 0.0)))
        depth = np.minimum(depth, np.where((ax < 0) & (ay < 0), np.maximum(ax, ay), np.inf))
    for px, py, _ in poles:
        rr = np.hypot(xy[:, 0] - px, xy[:, 1] - py) - 0.25
        d = np.minimum(d, np.maximum(rr, 0.0))
        depth = np.minimum(depth, np.where(rr < 0, rr, np.inf))
    return d, depth


def grid_quality(g, res):
    from scipy.spatial import cKDTree
    from test_loop_closure import route
    h, w = g["cells"].shape
    jj, ii = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    xy = np.column_stack([g["origin"][0] + (ii.ravel() + 0.5) * res, g["origin"][1] + (jj.ravel() + 0.5) * res])
    v = g["cells"].ravel().astype(np.int64)
    every, seen = footprints()
    d, _ = footprint_distance(xy, every)
    _, depth = footprint_distance(xy, seen)
    occ, free = v >= 65, (v >= 0) & (v <= 20)
    R = np.array([(x, y) for x, y, _ in route()])
    path = np.concatenate([np.linspace(R[k], R[k + 1], 41) for k in range(len(R) - 1)])
    near = (cKDTree(path).query(xy)[0] <= 1.0) & (d > 0.5)
    return dict(occupied=int(occ.sum()), precision=float((d[occ] <= 0.15).mean()),
                free_in_footprint=float((depth[free] <= -0.1).sum() / free.sum()), route_free=float(free[near].mean()))


def test_quality_of_the_defaults_on_the_ray_cast_drive():
    """the whole route (118 frames, 16 beams, 720 azimuths) at the true poses with the defaults.  Measured: 100 % of the
    6 805 occupied cells within 0.15 m of a footprint, 0.004 % of the free cells inside a footprint shrunk by 0.1 m, 100 %
    of the cells within 1 m of the route and 0.5 m from obstacles free"""
    cfg = oo.config()
    g = oo.build([oo.scan2d(s, cfg) for s in drive_scans()], true_poses(), cfg)
    q = grid_quality(g, cfg["resolution"])
    print(q)
    assert g["dropped"] == 0 and q["occupied"] > 5000
    assert q["precision"] >= 0.99 and q["free_in_footprint"] <= 0.0005 and q["route_free"] >= 0.99


def test_drift_blurs_the_grid_and_the_true_poses_restore_it():
    """the same scans at odometry drifting 2 cm and 0.05 degrees per frame: the occupied precision falls (measured 72.5 %);
    rebuilt at the true poses (what a loop correction gives) it is back (100 %)"""
    cfg = oo.config()
    scans = [oo.scan2d(s, cfg) for s in drive_scans()]
    truth = true_poses()
    step = pose_of(0.02, 0.0, math.radians(0.05))
    drift, acc = [], np.eye(4)
    for T in truth:
        drift.append(T @ acc)
        acc = acc @ step
    bad = grid_quality(oo.build(scans, drift, cfg), cfg["resolution"])
    good = grid_quality(oo.build(scans, truth, cfg), cfg["resolution"])
    print(bad, good)
    assert bad["precision"] <= 0.8 and good["precision"] >= 0.99


# ---- the library ------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_occ_library_holds_only_its_kernels_for_sm90a_without_spills():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.OCC_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.OCC_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.OCC_LIB], capture_output=True, text=True,
                         check=True).stdout
    usage = [l for l in res.splitlines() if "REG:" in l]
    assert len(usage) == len(KERNELS) and all("STACK:0 " in l for l in usage), usage


def test_every_other_library_keeps_its_sass():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_occupancy.json")))
    assert len(want) == 15 and "libtloam_b200_occ.so" not in want
    for lib in want:
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


def test_occupancy_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "occupancy_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def ray_frames(n, n_az=360):
    """(scan, pose, intensity) of the route's first n frames, a NaN row in frame 3"""
    from test_loop_closure import cast, make_world, route
    world = make_world()
    out = []
    for k, (x, y, yaw) in enumerate(route()[:n]):
        scan = cast(world, x, y, yaw, n_az=n_az, seed=k)
        if k == 3:
            scan[5] = [np.nan, 0.0, 0.0]
        out.append((scan, pose_of(x, y, yaw), np.random.default_rng(k).uniform(0, 100, len(scan))))
    return out


def assert_grid(r, scans, poses, cfg=COARSE):
    """the device's scans and grid against the restatement of scans (sensor-frame rows per map frame) at the build poses"""
    c = oo.config(**cfg)
    ob, fl, rec = r.occupancy_scans()
    assert ob.shape == (len(scans), c["n_cols"], 3)
    for k, s in enumerate(scans):
        wo, wf = oo.scan2d(s, c)
        assert same_bits(ob[k], wo) and same_bits(fl[k], wf), k
    g = r.occupancy_build()
    want = oo.build(list(zip(ob, fl)), poses, c)
    assert g.origin == want["origin"] and g.cells.shape == (want["height"], want["width"])
    assert g.dropped == want["dropped"] == 0 and g.frames == len(scans)
    assert np.array_equal(g.occupied, want["occupied"]) and np.array_equal(g.free, want["free"])
    assert np.array_equal(g.cells, want["cells"])
    return g, rec


def host_run(frames, occupancy, intensity=True, packed=False, capacity=1 << 20):
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=capacity)
    if occupancy:
        r.occupancy_enable(**COARSE)
    launches = []
    for scan, pose, inten in frames:
        n0 = r.launch_count()
        if packed:
            rec = np.zeros(len(scan), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("intensity", "<f4")])
            for j, name in enumerate("xyz"):
                rec[name] = scan[:, j]
            rec["intensity"] = inten
            r.global_map_append_packed(rec, pose)
        else:
            r.global_map_append(scan, pose, intensity=inten if intensity else None)
        launches.append(r.launch_count() - n0)
    return r, launches


@pytest.mark.gpu
@pytest.mark.parametrize("intensity", [True, False])
def test_gpu_host_appends_are_the_restatement(intensity):
    """scans, counts, values, origin, size and dropped equal the restatement; the map and its tables are the bits of the
    grid off; four more launches per append"""
    frames = ray_frames(12)
    on, l_on = host_run(frames, True, intensity)
    off, l_off = host_run(frames, False, intensity)
    assert same_bits(on.global_map(), off.global_map()) and np.array_equal(on.global_map_frames(), off.global_map_frames())
    assert same_bits(on.registered_scan(), off.registered_scan())
    if intensity:
        assert same_bits(on.global_map_intensity(), off.global_map_intensity())
    assert [a - b for a, b in zip(l_on, l_off)] == [4] * len(frames)
    g, rec = assert_grid(on, [f[0] for f in frames], [f[1] for f in frames])
    assert all(same_bits(a, b[1]) for a, b in zip(rec, frames))
    print(f"{g.cells.shape}, occupied {(g.cells >= 65).sum()}, free {((g.cells >= 0) & (g.cells <= 20)).sum()}")
    assert (g.cells >= 65).sum() > 100
    on.close()
    off.close()


@pytest.mark.gpu
def test_gpu_obstacle_ties_go_to_the_lowest_row_index():
    """three distinct rows at one rho in every sector, shuffled differently per append: k_occ_pick keeps the lowest row"""
    import tloam_b200
    c = oo.config(**COARSE)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.occupancy_enable(**COARSE)
    wants = []
    for k in range(4):
        scan, want, _ = tie_scan(c, np.random.default_rng(70 + k))
        r.global_map_append(scan, pose_of(0.5 * k, 0.0, 0.0))
        wants.append(want)
    ob, _, _ = r.occupancy_scans()
    for k, want in enumerate(wants):
        assert same_bits(ob[k], want), k
    r.close()


@pytest.mark.gpu
def test_gpu_packed_appends_are_the_restatement():
    """the packed rows are the float32 values widened: the restatement reads those"""
    frames = ray_frames(6)
    r, _ = host_run(frames, True, packed=True)
    widened = [scan.astype(np.float32).astype(np.float64) for scan, _, _ in frames]
    assert_grid(r, widened, [f[1] for f in frames])
    r.close()


@pytest.mark.gpu
def test_gpu_chained_mapping_loop_is_the_restatement():
    """process_raw_scan -> scan_match -> global_map_append_frame chained: the recorded poses are get_result's, and the
    odometry and the map are the bits of the grid off"""
    import tloam_b200
    from test_global_map import with_nonfinite
    from test_process_cloud import FE, moved
    from tloam_b200 import synth
    scan0 = synth.raw_scan()
    scans = [with_nonfinite(scan0, 90)] + [with_nonfinite(moved(scan0, np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k]),
                                                                100 + k), 200 + k) for k in range(1, 6)]

    def run(occupancy):
        r = tloam_b200.LocalRegistration(fitness_thres=0.3)
        r.enable_global_map()
        if occupancy:
            r.occupancy_enable(**COARSE)
        poses = []
        for k, scan in enumerate(scans):
            r.process_raw_scan(scan, feature=FE)
            if k == 0:
                r.submap_init_frame()
                continue
            r.scan_matching_predicted_async()
            r.submap_update_frame_chained()
            r.global_map_append_frame()
            poses.append(r.get_result())
        return r, poses

    on, p_on = run(True)
    off, p_off = run(False)
    assert all(np.array_equal(a, b) for a, b in zip(p_on, p_off))
    assert same_bits(on.global_map(), off.global_map())
    _, rec = assert_grid(on, scans[1:], p_on)
    assert all(same_bits(a, b) for a, b in zip(rec, p_on))
    on.close()
    off.close()


@pytest.mark.gpu
def test_gpu_frame_table_growth_and_refusal():
    """1 100 small appends grow the frame table (1 024 slots) with the records; a refused append leaves no record"""
    import tloam_b200
    from tloam_b200 import _lib
    frames = ray_frames(3)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.occupancy_enable(**COARSE)
    rng = np.random.default_rng(5)
    scans, poses = [], []
    for k in range(1100):
        s = frames[k % 3][0][rng.choice(len(frames[k % 3][0]), 60, replace=False)]
        P = pose_of(0.01 * k, -0.02 * k, 0.003 * k)
        r.global_map_append(s, P)
        scans.append(s)
        poses.append(P)
        if k == 700:                                               # refused: spans more than 2^21 voxels
            r.global_map_append(np.vstack([s, [[3.0e6, 0.0, 0.0]]]), pose_of(5.0, 5.0, 1.0))
            with pytest.raises(tloam_b200.RegistrationError) as e:
                r.global_map_size()
            assert e.value.status == _lib.ERR_VOXEL_RANGE
    assert r.global_map_size()[1] == 1100 and r.global_map_capacity()[1] > 0
    assert_grid(r, scans, poses)
    r.close()


@pytest.mark.gpu
def test_gpu_reset_keeps_the_grid_on():
    import tloam_b200
    frames = ray_frames(5)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.occupancy_enable(**COARSE)
    for scan, pose, _ in frames:
        r.global_map_append(scan, pose)
    r.reset_global_map()
    g = r.occupancy_build()
    assert g.cells.shape == (0, 0) and g.frames == 0
    r.global_map_append(np.zeros((0, 3)), frames[0][1])           # an empty append takes a slot with an empty scan
    for scan, pose, _ in frames[1:3]:
        r.global_map_append(scan, pose)
    ob, fl, _ = r.occupancy_scans()
    assert np.isnan(ob[0]).all() and np.isnan(fl[0]).all()
    assert_grid(r, [np.zeros((0, 3))] + [f[0] for f in frames[1:3]], [f[1] for f in frames[:3]])
    r.close()


@pytest.mark.gpu
def test_gpu_build_after_a_correction_follows_the_corrected_poses():
    import tloam_b200
    import pose_graph_oracle as pgo
    from test_pose_graph import loop_result
    frames = ray_frames(10)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_correction_enable()
    r.occupancy_enable(**COARSE)
    r.pose_graph_enable()
    O = []
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
        r.pose_graph_add_node(pose)
        O.append(pose)
    before = r.occupancy_build()
    r.pose_graph_add_loop(loop_result(1, 5, pgo.inv_mul(O[1], O[5]) @ pgo.exp4([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(6))
    for scan, pose, inten in frames[6:]:
        r.global_map_append(scan, pose, intensity=inten)
    _, P = r.global_map_frame_poses()
    assert not same_bits(P[3], O[3])
    g, rec = assert_grid(r, [f[0] for f in frames], list(P))
    assert same_bits(rec[3], O[3])                                 # the record keeps the append's pose
    ob, fl, _ = r.occupancy_scans()
    at_odometry = oo.build(list(zip(ob, fl)), list(rec), oo.config(**COARSE))
    assert at_odometry["occupied"].shape != g.occupied.shape or not np.array_equal(at_odometry["occupied"], g.occupied)
    assert before.frames == 6
    r.close()


@pytest.mark.gpu
def test_gpu_grid_off_keeps_the_launch_counts():
    """a handle whose grid was turned off by enable_global_map launches what a handle that never had it launches"""
    import tloam_b200
    frames = ray_frames(4)
    plain, l_plain = host_run(frames, False)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.occupancy_enable(**COARSE)
    r.enable_global_map()
    launches = []
    for scan, pose, inten in frames:
        n0 = r.launch_count()
        r.global_map_append(scan, pose, intensity=inten)
        launches.append(r.launch_count() - n0)
    assert launches == l_plain and same_bits(r.global_map(), plain.global_map())
    with pytest.raises(tloam_b200.RegistrationError):
        r.occupancy_build()
    r.close()
    plain.close()


@pytest.mark.gpu
def test_gpu_occupancy_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.OccupancyConfig()
    L.tloam_b200_occupancy_default_config(C.byref(cfg))
    assert (cfg.resolution, cfg.n_cols, cfg.z_lo, cfg.z_hi, cfg.min_range, cfg.max_range, cfg.free_margin) == \
        (0.1, 1024, -1.2, 0.5, 3.0, 30.0, 0.1)
    info = _lib.OccupancyInfo()
    d = np.zeros(4)
    assert L.tloam_b200_occupancy_enable(None, C.byref(cfg)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_occupancy_enable(h, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_occupancy_enable(h, C.byref(cfg)) == _lib.ERR_NOT_READY                   # mapping off
    assert L.tloam_b200_occupancy_build(h, C.byref(info)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_occupancy_download(h, None, None, None, 0) == _lib.ERR_NOT_READY
    assert L.tloam_b200_occupancy_scans_download(h, 0, 0, None, None) == _lib.ERR_NOT_READY
    r.enable_global_map()
    assert L.tloam_b200_occupancy_build(h, C.byref(info)) == _lib.ERR_NOT_READY                  # grid off
    assert L.tloam_b200_occupancy_scans_download(h, 0, 0, None, None) == _lib.ERR_NOT_READY
    for field, bad in (("resolution", 0.0), ("resolution", float("nan")), ("n_cols", 0), ("n_cols", 4097),
                       ("z_lo", 0.5), ("z_hi", float("inf")), ("min_range", 0.0), ("max_range", 2.0),
                       ("free_margin", -0.1), ("free_margin", float("nan"))):
        c = _lib.OccupancyConfig()
        L.tloam_b200_occupancy_default_config(C.byref(c))
        setattr(c, field, bad)
        assert L.tloam_b200_occupancy_enable(h, C.byref(c)) == _lib.ERR_INVALID_ARG, (field, bad)
    frames = ray_frames(3)
    r.global_map_append(frames[0][0], frames[0][1])
    assert L.tloam_b200_occupancy_enable(h, C.byref(cfg)) == _lib.ERR_NOT_READY                  # not empty
    r.reset_global_map()
    r.occupancy_enable(**COARSE)
    assert L.tloam_b200_occupancy_download(h, None, None, None, 0) == _lib.ERR_NOT_READY          # no build yet
    assert L.tloam_b200_occupancy_build(h, None) == _lib.OK                                      # empty: 0 x 0
    assert L.tloam_b200_occupancy_download(h, None, None, None, 0) == _lib.OK
    for scan, pose, _ in frames:
        r.global_map_append(scan, pose)
    assert L.tloam_b200_occupancy_scans_download(h, 3, 1, _dp(d), None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_occupancy_scans_download(h, 3, 0, None, None) == _lib.OK
    assert L.tloam_b200_occupancy_build(h, C.byref(info)) == _lib.OK and info.width * info.height > 0
    assert L.tloam_b200_occupancy_download(h, None, None, None, info.width * info.height - 1) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_occupancy_download(h, None, None, None, info.width * info.height) == _lib.OK
    far = pose_of(1.0e5, 1.0e5, 0.0)                               # the extent passes 2^28 cells
    r.global_map_append(frames[0][0], far)
    assert L.tloam_b200_occupancy_build(h, C.byref(info)) == _lib.ERR_VOXEL_RANGE
    assert L.tloam_b200_occupancy_download(h, None, None, None, 1 << 30) == _lib.ERR_NOT_READY   # a refused build leaves none
    r.enable_global_map()                                          # turns it off
    assert L.tloam_b200_occupancy_build(h, C.byref(info)) == _lib.ERR_NOT_READY
    r.close()


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


@pytest.mark.gpu
def test_gpu_occupancy_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("occupancy_driver", "front_end_b200.hpp")
    frames = ray_frames(6)
    path = os.path.join(os.path.dirname(exe), "occupancy_raw.bin")
    out_path = os.path.join(os.path.dirname(exe), "occupancy_out.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(frames)))
        for p, T, _ in frames:
            fh.write(np.ascontiguousarray(T.ravel(order="F")).tobytes() + struct.pack("Q", len(p)))
            fh.write(np.ascontiguousarray(p, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path, out_path, repr(COARSE["resolution"]), str(COARSE["n_cols"]), repr(COARSE["max_range"])],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    w, h = (int(s) for s in res.stdout.split())
    r, _ = host_run(frames, True, intensity=False)
    g = r.occupancy_build()
    r.close()
    with open(out_path, "rb") as fh:
        blob = fh.read()
    ox, oy, res_ = struct.unpack_from("3d", blob, 0)
    (dropped,) = struct.unpack_from("Q", blob, 24)
    cells = np.frombuffer(blob, dtype=np.int8, offset=32).reshape(h, w)
    assert (ox, oy) == g.origin and res_ == COARSE["resolution"] and dropped == g.dropped
    assert np.array_equal(cells, g.cells)
