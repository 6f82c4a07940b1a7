"""The distance field and costmap of an occupancy grid (include/tloam_b200.h "Distance field and costmap"; k_dist_* in
libtloam_b200_dist.so).  tests/distance_oracle.py is the bit-for-bit numpy restatement.

CPU: the restatement against a brute force (1 x 1, 1 x N, N x 1, borders, ties, no obstacle, all obstacle) and against
scipy.ndimage.distance_transform_edt up to the seq-00 shape, the cost rule against InflationLayer::computeCost at its edges,
the publisher table, the query at its edges, the symbols, the new library's kernels, the digests of every other library,
the shim's driver.  GPU: sq, sd, costs and values equal the restatement and sq equals scipy, from host grids and from the
occupancy build (also after a correction); the build changes no occupancy cell, map bit or append launch count; the
query's bits; the status codes; the shim."""
import ctypes as C
import json
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import distance_oracle as do
import sass_digest
from test_global_map_intensity import same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_distance_default_config", "tloam_b200_distance_build", "tloam_b200_distance_build_grid",
               "tloam_b200_distance_download", "tloam_b200_distance_query"]
KERNELS = ("k_dist_bands", "k_dist_cols", "k_dist_rows", "k_dist_cost", "k_dist_query")
SEQ00 = (6238, 5528)                                               # (height, width) of the seq-00-shaped occupancy grid


def random_grid(shape, rng, p_obstacle=0.2, p_unknown=0.2):
    """cells of every class: obstacles (65 .. 100), free (0 .. 25), unknown (-1 and 26 .. 64)"""
    u = rng.random(shape)
    g = rng.integers(0, 26, shape)
    g = np.where(u < p_obstacle, rng.integers(65, 101, shape), g)
    unk = np.where(rng.random(shape) < 0.5, -1, rng.integers(26, 65, shape))
    g = np.where((u >= p_obstacle) & (u < p_obstacle + p_unknown), unk, g)
    return g.astype(np.int8)


def scipy_sq(grid):
    from scipy.ndimage import distance_transform_edt as edt
    ob = do.obstacles(grid)
    return np.where(ob, np.round(edt(ob) ** 2), np.round(edt(~ob) ** 2)).astype(np.uint32)


def edge_grids():
    rng = np.random.default_rng(3)
    out = [np.array([[100]], dtype=np.int8), np.array([[0]], dtype=np.int8), np.array([[-1]], dtype=np.int8)]
    for shape in ((1, 13), (11, 1), (7, 9), (16, 5)):
        for p in (0.0, 0.15, 0.6, 1.0):
            out.append(random_grid(shape, rng, p))
    b = np.zeros((9, 12), dtype=np.int8)                           # obstacles only on the border
    b[0, :] = b[-1, :] = b[:, 0] = b[:, -1] = 100
    out.append(b)
    t = np.zeros((9, 9), dtype=np.int8)                            # ties: cells equidistant from two obstacles
    t[4, 0] = t[4, 8] = t[0, 4] = t[8, 4] = 100
    out.append(t)
    return out


# ---------------------------------------------------------------------------------------------------------------------
def test_restatement_matches_the_brute_force():
    for k, g in enumerate(edge_grids()):
        assert np.array_equal(do.squared(g).astype(np.int64), do.brute(g)), k
    assert (do.squared(np.zeros((4, 6), dtype=np.int8)) == do.INF).all()
    assert (do.squared(np.full((4, 6), 100, dtype=np.int8)) == do.INF).all()


@pytest.mark.parametrize("shape", [(2, 2), (3, 50), (61, 47), (257, 129), SEQ00])
def test_restatement_matches_scipy(shape):
    g = random_grid(shape, np.random.default_rng(shape[0]), p_obstacle=0.25 if shape != SEQ00 else 0.3)
    assert np.array_equal(do.squared(g), scipy_sq(g))


def test_cost_rule_matches_inflation_layers_compute_cost():
    for res, cfg in ((0.1, do.config()), (0.05, do.config(inscribed_radius=0.3, inflation_radius=0.55, cost_scaling_factor=10.0)),
                     (0.25, do.config(inscribed_radius=0.0, inflation_radius=1.0, cost_scaling_factor=0.0))):
        t = do.cost_table(cfg, res)
        Rc = do.cell_radius(cfg, res)
        assert len(t) == Rc * Rc + 1
        want = [do.compute_cost_literal(math.sqrt(s), res, cfg["inscribed_radius"], cfg["cost_scaling_factor"])
                for s in range(len(t))]
        assert t.tolist() == want
        # sq = R_c^2 is inflated, R_c^2 + 1 is not; unknown cells inside and outside the inscribed radius
        H = 2 * Rc + 3
        g = np.zeros((1, H), dtype=np.int8)
        g[0, 0] = 100
        g[0, 1:] = 0
        sq = do.squared(g)
        c = do.costs(sq, g, cfg, res)
        assert c[0, 0] == 254 and c[0, Rc] == t[Rc * Rc] and c[0, Rc + 1] == 0
        gu = g.copy()
        gu[0, 1:] = -1
        cu = do.costs(sq, gu, cfg, res)
        inside = [x for x in range(1, H) if x * x <= Rc * Rc and t[x * x] == 253]
        assert all(cu[0, x] == 253 for x in inside)
        assert all(cu[0, x] == 255 for x in range(1, H) if x not in inside)
    # dist * res exactly the inscribed radius: 253; the next cell out decays
    cfg = do.config(inscribed_radius=0.5, inflation_radius=2.0)
    t = do.cost_table(cfg, 0.25)
    assert 2 * 0.25 == 0.5 and t[4] == 253 and t[5] == do.compute_cost_literal(math.sqrt(5), 0.25, 0.5, 3.0) < 253


def test_publisher_table_is_the_literal_loop():
    want = [0] * 256
    want[253], want[254], want[255] = 99, 100, -1
    for i in range(1, 253):
        want[i] = 1 + (97 * (i - 1)) // 251
    assert do.values(np.arange(256, dtype=np.uint8)).tolist() == want
    assert (want[1], want[252], want[128]) == (1, 98, 50)


def test_query_restatement_at_its_edges():
    rng = np.random.default_rng(9)
    g = random_grid((6, 8), rng, 0.3)
    f = do.field(g, (-1.5, 2.25), 0.5)
    sd = f["signed"]
    ox, oy, r = -1.5, 2.25, 0.5
    centres = np.array([[ox + (i + 0.5) * r, oy + (j + 0.5) * r] for j in range(6) for i in range(8)])
    d, gr = do.query(sd, (ox, oy), r, centres)
    assert np.array_equal(d, sd.ravel().astype(np.float64))
    d, gr = do.query(sd, (ox, oy), r, [[ox + 7.5 * r, oy + 5.5 * r], [ox + 7.5 * r, oy + 0.5 * r]])   # u = width - 1
    assert d[0] == sd[5, 7] and d[1] == sd[0, 7] and np.isfinite(gr).all()
    d, gr = do.query(sd, (ox, oy), r, [[ox + 0.49 * r, oy + r], [ox + 8 * r, oy + r], [np.nan, oy], [ox + r, oy + 5.6 * r]])
    assert np.isnan(d).all() and np.isnan(gr).all()
    d, gr = do.query(do.field(np.zeros((4, 4), dtype=np.int8), (0, 0), 1.0)["signed"], (0, 0), 1.0, [[1.0, 1.0]])
    assert np.isnan(d).all() and np.isnan(gr).all()
    d, gr = do.query(sd, (ox, oy), r, [[ox + 1.25 * r, oy + 2.75 * r]])
    a, b = 0.75, 0.25
    s00, s10, s01, s11 = (float(sd[2, 0]), float(sd[2, 1]), float(sd[3, 0]), float(sd[3, 1]))
    assert d[0] == (1 - b) * ((1 - a) * s00 + a * s10) + b * ((1 - a) * s01 + a * s11)
    assert gr[0, 0] == ((1 - b) * (s10 - s00) + b * (s11 - s01)) / r


# ---- the library ------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_dist_library_holds_only_its_kernels_for_sm90a_without_stack():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.DIST_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.DIST_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.DIST_LIB], capture_output=True, text=True,
                         check=True).stdout
    usage = [l for l in res.splitlines() if "REG:" in l]
    assert len(usage) == len(KERNELS) and all("STACK:0 " in l for l in usage), usage


def test_every_other_library_keeps_its_sass():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_distance.json")))
    assert len(want) == 16 and "libtloam_b200_dist.so" not in want and "libtloam_b200_occ.so" in want
    for lib in want:
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


def test_distance_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "distance_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def assert_field(f, want, scipy=True):
    assert f.sq.shape == want["sq"].shape and f.obstacles == want["obstacles"]
    assert f.origin == want["origin"] and f.resolution == want["resolution"]
    assert np.array_equal(f.sq, want["sq"]) and same_bits(f.signed, want["signed"])
    assert np.array_equal(f.costs, want["costs"]) and np.array_equal(f.values, want["values"])
    if scipy and 0 < f.obstacles < f.sq.size:
        assert np.array_equal(f.sq, scipy_sq(want["grid"]))


def host_field(r, g, origin=(-3.25, 7.5), res=0.1, **cfg):
    f = r.distance_build(g, origin, res, **cfg)
    want = do.field(g, origin, res, do.config(**cfg))
    want["grid"] = g
    return f, want


@pytest.mark.gpu
def test_gpu_host_grids_are_the_restatement():
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    for k, g in enumerate(edge_grids()):
        f, want = host_field(r, g, res=0.25, inscribed_radius=0.3, inflation_radius=1.0)
        assert_field(f, want), k
    rng = np.random.default_rng(11)
    for shape in ((1, 1), (1, 777), (513, 1), (37, 91), (255, 257), (1023, 65)):
        g = random_grid(shape, rng, 0.02)
        f, want = host_field(r, g)
        assert_field(f, want)
    for fill in (0, 100, -1):                                      # no obstacle / all obstacle / all unknown
        g = np.full((33, 45), fill, dtype=np.int8)
        f, want = host_field(r, g)
        assert_field(f, want)
        assert np.isinf(f.signed).all()
    r.close()


@pytest.mark.gpu
def test_gpu_seq00_shaped_grid_is_the_restatement_and_scipy():
    import tloam_b200
    g = random_grid(SEQ00, np.random.default_rng(0), p_obstacle=0.01, p_unknown=0.3)
    r = tloam_b200.LocalRegistration()
    f, want = host_field(r, g, origin=(-270.3, -310.7), res=0.1)
    assert_field(f, want)
    xy = np.column_stack([np.random.default_rng(1).uniform(-275, 290, 200_000), np.random.default_rng(2).uniform(-315, 320, 200_000)])
    d, gr = r.distance_query(xy)
    wd, wg = do.query(f.signed, f.origin, f.resolution, xy)
    assert same_bits(d, wd) and same_bits(gr, wg) and np.isfinite(d).sum() > 100_000
    r.close()


@pytest.mark.gpu
def test_gpu_query_bits():
    import tloam_b200
    rng = np.random.default_rng(21)
    g = random_grid((40, 57), rng, 0.05)
    r = tloam_b200.LocalRegistration()
    f, _ = host_field(r, g, origin=(1.5, -2.0), res=0.2)
    ox, oy, res = 1.5, -2.0, 0.2
    centres = np.array([[ox + (i + 0.5) * res, oy + (j + 0.5) * res] for j in range(40) for i in range(57)])
    edges = [[ox + 56.5 * res, oy + 39.5 * res], [ox + 0.5 * res, oy + 0.5 * res], [ox + 56.5 * res, oy + 3.3 * res],
             [ox + 0.4 * res, oy + 3.0], [ox + 57.0 * res, oy + 1.0], [np.nan, 0.0], [np.inf, 0.0], [ox + 2.0, -1e300]]
    xy = np.vstack([centres, edges, np.column_stack([rng.uniform(ox - 1, ox + 12.5, 5000), rng.uniform(oy - 1, oy + 9, 5000)])])
    d, gr = r.distance_query(xy)
    wd, wg = do.query(f.signed, f.origin, f.resolution, xy)
    assert same_bits(d, wd) and same_bits(gr, wg)
    assert np.allclose(d[:len(centres)], f.signed.ravel(), rtol=1e-12, atol=1e-12)   # centres: a, b are 0 up to rounding
    d0, g0 = r.distance_query(np.zeros((0, 2)))
    assert d0.shape == (0,) and g0.shape == (0, 2)
    r.distance_build(np.zeros((5, 5), dtype=np.int8), (0, 0), 1.0)   # no obstacle: infinite field, NaN everywhere
    d, gr = r.distance_query(xy[:100])
    assert np.isnan(d).all() and np.isnan(gr).all()
    r.distance_build(np.zeros((1, 5), dtype=np.int8), (0, 0), 1.0)   # one row: no cell square to interpolate in
    assert np.isnan(r.distance_query([[2.5, 0.5]])[0]).all()
    r.close()


def occupancy_handle(frames, correction=False):
    import tloam_b200
    from test_occupancy import COARSE
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 20)
    if correction:
        r.global_map_correction_enable()
    r.occupancy_enable(**COARSE)
    return r


@pytest.mark.gpu
def test_gpu_occupancy_build_is_the_restatement_and_changes_nothing():
    """the field of the occupancy build of the ray-cast drive equals the restatement of the downloaded cells; the build
    leaves the occupancy grid, the map and the launch counts of later appends as they are"""
    from test_occupancy import COARSE, host_run, ray_frames
    frames = ray_frames(12)
    r = occupancy_handle(frames)
    plain, l_plain = host_run(frames[:8], True)
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
    g0 = r.occupancy_build()
    map0 = r.global_map()
    f = r.distance_build()
    want = do.field(g0.cells, g0.origin, COARSE["resolution"])
    want["grid"] = g0.cells
    assert_field(f, want)
    assert f.obstacles > 100 and (f.costs == 253).any() and (f.values == 99).any()
    g1 = r.occupancy_build()
    assert np.array_equal(g1.cells, g0.cells) and same_bits(r.global_map(), map0)
    launches = []
    for scan, pose, inten in frames[6:8]:
        n0 = r.launch_count()
        r.global_map_append(scan, pose, intensity=inten)
        launches.append(r.launch_count() - n0)
    assert launches == l_plain[6:8] and same_bits(r.global_map(), plain.global_map())
    r.occupancy_build()                                            # the field is a snapshot: a later build leaves it
    sd = np.zeros(f.sq.size, dtype=np.float32)
    assert r._L.tloam_b200_distance_download(r._h, sd.ctypes.data_as(C.POINTER(C.c_float)), None, None, None, sd.size) == 0
    assert same_bits(sd.reshape(f.sq.shape), f.signed)
    r.close()
    plain.close()


@pytest.mark.gpu
def test_gpu_build_after_a_correction_follows_the_corrected_grid():
    import pose_graph_oracle as pgo
    from test_occupancy import COARSE, ray_frames
    from test_pose_graph import loop_result
    frames = ray_frames(10)
    r = occupancy_handle(frames, correction=True)
    r.pose_graph_enable()
    O = []
    for scan, pose, inten in frames[:6]:
        r.global_map_append(scan, pose, intensity=inten)
        r.pose_graph_add_node(pose)
        O.append(pose)
    r.occupancy_build()
    before = r.distance_build()
    r.pose_graph_add_loop(loop_result(1, 5, pgo.inv_mul(O[1], O[5]) @ pgo.exp4([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(6))
    g = r.occupancy_build()
    f = r.distance_build()
    want = do.field(g.cells, g.origin, COARSE["resolution"])
    want["grid"] = g.cells
    assert_field(f, want)
    assert f.sq.shape != before.sq.shape or not np.array_equal(f.sq, before.sq)
    r.reset_global_map()                                           # an empty grid: a 0 x 0 field
    r.occupancy_build()
    e = r.distance_build()
    assert e.sq.shape == (0, 0) and e.obstacles == 0
    assert np.isnan(r.distance_query([[0.0, 0.0]])[0]).all()
    r.close()


@pytest.mark.gpu
def test_gpu_distance_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    from test_occupancy import COARSE
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.DistanceConfig()
    L.tloam_b200_distance_default_config(C.byref(cfg))
    assert (cfg.inscribed_radius, cfg.inflation_radius, cfg.cost_scaling_factor) == (0.9, 3.0, 3.0)
    info = _lib.DistanceInfo()
    g = np.zeros((4, 5), dtype=np.int8)
    g[1, 2] = 100
    gp = g.ctypes.data_as(C.POINTER(C.c_byte))
    xy = np.zeros(2)
    dp = xy.ctypes.data_as(C.POINTER(C.c_double))
    assert L.tloam_b200_distance_download(h, None, None, None, None, 1 << 30) == _lib.ERR_NOT_READY   # no build yet
    assert L.tloam_b200_distance_query(h, dp, 1, None, None) == _lib.ERR_NOT_READY
    assert L.tloam_b200_distance_build(h, C.byref(cfg), C.byref(info)) == _lib.ERR_NOT_READY           # mapping off
    r.enable_global_map()
    assert L.tloam_b200_distance_build(h, C.byref(cfg), C.byref(info)) == _lib.ERR_NOT_READY           # grid off
    r.occupancy_enable(**COARSE)
    assert L.tloam_b200_distance_build(h, C.byref(cfg), C.byref(info)) == _lib.ERR_NOT_READY           # not built
    assert L.tloam_b200_distance_build(None, C.byref(cfg), None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_distance_build(h, None, None) == _lib.ERR_INVALID_ARG
    for field, bad in (("inscribed_radius", -0.1), ("inscribed_radius", 3.5), ("inflation_radius", float("inf")),
                       ("cost_scaling_factor", -1.0), ("cost_scaling_factor", float("nan")), ("inflation_radius", 410.0)):
        c = _lib.DistanceConfig()
        L.tloam_b200_distance_default_config(C.byref(c))
        setattr(c, field, bad)
        assert L.tloam_b200_distance_build_grid(h, C.byref(c), gp, 5, 4, 0.0, 0.0, 0.1, None) == _lib.ERR_INVALID_ARG, field
    c = _lib.DistanceConfig()
    L.tloam_b200_distance_default_config(C.byref(c))
    c.inflation_radius = 409.6                                     # R_c = 4096 at 0.1 m: allowed
    assert L.tloam_b200_distance_build_grid(h, C.byref(c), gp, 5, 4, 0.0, 0.0, 0.1, None) == _lib.OK
    for args in ((None, 5, 4, 0.0, 0.0, 0.1), (gp, 0, 4, 0.0, 0.0, 0.1), (gp, 5, 0, 0.0, 0.0, 0.1),
                 (gp, 5, 4, float("nan"), 0.0, 0.1), (gp, 5, 4, 0.0, float("inf"), 0.1), (gp, 5, 4, 0.0, 0.0, 0.0),
                 (gp, 5, 4, 0.0, 0.0, float("nan")), (gp, 1 << 15, (1 << 13) + 1, 0.0, 0.0, 0.1)):
        assert L.tloam_b200_distance_build_grid(h, C.byref(cfg), *args, None) == _lib.ERR_INVALID_ARG, args
    big = np.zeros(1 << 17, dtype=np.int8)                         # 1 x 2^17 cells: (2^17 - 1)^2 > 2^32
    bp = big.ctypes.data_as(C.POINTER(C.c_byte))
    assert L.tloam_b200_distance_build_grid(h, C.byref(cfg), bp, 1 << 17, 1, 0.0, 0.0, 0.1, None) == _lib.ERR_VOXEL_RANGE
    edge = np.zeros(65536, dtype=np.int8)                          # 65536 x 1: (65535)^2 < 2^32 - 1
    edge[7] = 100
    ep = edge.ctypes.data_as(C.POINTER(C.c_byte))
    assert L.tloam_b200_distance_build_grid(h, C.byref(cfg), ep, 1, 65536, 0.0, 0.0, 0.1, C.byref(info)) == _lib.OK
    sq = np.zeros(65536, dtype=np.uint32)
    assert L.tloam_b200_distance_download(h, None, sq.ctypes.data_as(C.POINTER(C.c_uint)), None, None, 65536) == _lib.OK
    assert sq[65535] == (65535 - 7) ** 2 and sq[7] == 1 and sq[0] == 49
    assert L.tloam_b200_distance_download(h, None, None, None, None, 65535) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_distance_query(h, None, 1, None, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_distance_query(h, dp, 1, None, None) == _lib.OK
    # a refused build keeps the last field
    assert L.tloam_b200_distance_build_grid(h, C.byref(cfg), bp, 1 << 17, 1, 0.0, 0.0, 0.1, None) == _lib.ERR_VOXEL_RANGE
    assert L.tloam_b200_distance_download(h, None, None, None, None, 65536) == _lib.OK
    r.close()


@pytest.mark.gpu
def test_gpu_distance_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    from test_occupancy import COARSE, host_run, ray_frames
    exe = build_driver("distance_driver", "front_end_b200.hpp")
    frames = ray_frames(6)
    d = os.path.dirname(exe)
    raw_path, grid_path, out_path = (os.path.join(d, n) for n in ("distance_raw.bin", "distance_grid.bin", "distance_out.bin"))
    with open(raw_path, "wb") as fh:
        fh.write(struct.pack("Q", len(frames)))
        for p, T, _ in frames:
            fh.write(np.ascontiguousarray(T.ravel(order="F")).tobytes() + struct.pack("Q", len(p)))
            fh.write(np.ascontiguousarray(p, dtype=np.float64).tobytes())
    rng = np.random.default_rng(4)
    grid = random_grid((71, 103), rng, 0.03)
    origin, res = (-4.0, 2.5), 0.15
    xy = np.column_stack([rng.uniform(-4.5, 12.0, 3000), rng.uniform(2.0, 13.5, 3000)])
    with open(grid_path, "wb") as fh:
        fh.write(struct.pack("QQ3d", 103, 71, origin[0], origin[1], res) + grid.tobytes())
        fh.write(struct.pack("Q", len(xy)) + xy.tobytes())
    run = subprocess.run([exe, raw_path, grid_path, out_path, repr(COARSE["resolution"]), str(COARSE["n_cols"]),
                          repr(COARSE["max_range"])], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    shapes = [tuple(int(v) for v in line.split()) for line in run.stdout.split("\n") if line.strip()]
    r, _ = host_run(frames, True, intensity=False)
    r.occupancy_build()
    fields = [r.distance_build()]
    fields.append(r.distance_build(grid, origin, res))
    qd, qg = r.distance_query(xy)
    r.close()
    blob = open(out_path, "rb").read()
    o = 0
    for (w, h, nob), f in zip(shapes, fields):
        n = w * h
        assert (h, w) == f.sq.shape and nob == f.obstacles
        sd = np.frombuffer(blob, dtype=np.float32, count=n, offset=o).reshape(h, w)
        costs = np.frombuffer(blob, dtype=np.uint8, count=n, offset=o + 4 * n).reshape(h, w)
        values = np.frombuffer(blob, dtype=np.int8, count=n, offset=o + 5 * n).reshape(h, w)
        o += 6 * n
        assert same_bits(sd, f.signed) and np.array_equal(costs, f.costs) and np.array_equal(values, f.values)
    dd = np.frombuffer(blob, dtype=np.float64, count=len(xy), offset=o)
    gg = np.frombuffer(blob, dtype=np.float64, count=2 * len(xy), offset=o + 8 * len(xy)).reshape(-1, 2)
    assert same_bits(dd, qd) and same_bits(gg, qg)
