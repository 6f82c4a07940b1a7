"""The terrain map (include/tloam_b200.h "Terrain"; k_ter_* in libtloam_b200_terrain.so): per cell the ground reference,
elevation, step, slope, roughness and a traversability value, from the global map or a host cloud.
tests/terrain_oracle.py is the bit-for-bit numpy restatement.

CPU: the restatement against its literal per-cell transcription (every layer and value, -0.0 / +0.0, ties, grid edges and
corners, windows with no known cell, one row, all rows in one cell, non-finite rows), G and step against scipy's
minimum / maximum filters, the plane fit against numpy.linalg.lstsq and the determinant / min_fit rule, the threshold
boundaries, the combination table, the 2^28 limit, the quality on a ray-cast terrain world, and the kerb / driveway
route; the symbols, the new library's kernels, the digests of every other library, the shim's driver.  GPU: every layer,
count and value equals the restatement bit for bit (host clouds, the world through the device map, static rows, after a
correction, combined with the occupancy grid); the costmap of the values; the route on the device; repeat builds,
status codes, nothing else changes, the shim."""
import ctypes as C
import functools
import json
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import distance_oracle as do
import plan_oracle as po
import sass_digest
import terrain_oracle as to
from test_frontier import search_and_check
from test_global_map_intensity import same_bits
from test_loop_closure import ELEV, SENSOR_Z
from test_map_dynamic import pose_of

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_terrain_default_config", "tloam_b200_terrain_build", "tloam_b200_terrain_build_cloud",
               "tloam_b200_terrain_download", "tloam_b200_distance_build_terrain"]
KERNELS = ("k_ter_bounds", "k_ter_low", "k_ter_ground", "k_ter_high", "k_ter_layers")
LAYERS = ("ground", "elevation", "step", "slope", "roughness", "points", "values")
COUNTS = ("used", "skipped", "dropped", "overhang", "known", "lethal")
# a small config for the literal transcription: every window a few cells wide
SMALL = to.config(resolution=0.25, ground_radius=0.5, step_radius=0.25, slope_radius=0.5, min_fit=4)


def random_cloud(n, seed, span=(3.0, 2.0)):
    """a seeded cloud with overhangs, signed zeros, exact ties and a non-finite row"""
    rng = np.random.default_rng(seed)
    p = np.column_stack([rng.uniform(0, span[0], n), rng.uniform(0, span[1], n), rng.normal(0, 0.2, n)])
    p[rng.random(n) < 0.05, 2] = 3.0
    p[rng.random(n) < 0.1, 2] = 0.0
    p[rng.random(n) < 0.1, 2] = -0.0
    if n > 4:
        p[1] = [np.nan, 0.0, 0.0]
        p[2, 1] = np.inf
        p[3] = p[4]
    return p


def assert_same(got, want, counts=True):
    for k in LAYERS:
        assert same_bits(np.asarray(got[k]), np.asarray(want[k])), k
    if counts:
        for k in COUNTS:
            assert got[k] == want[k], (k, got[k], want[k])


# ---- the restatement -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_the_literal_transcription(seed):
    rng = np.random.default_rng(100 + seed)
    cfg = dict(SMALL, min_points=int(rng.integers(1, 3)), min_fit=int(rng.integers(3, 7)))
    p = random_cloud(int(rng.integers(30, 300)), seed)
    assert_same(to.build(p, cfg), to.build_literal(p, cfg))


def test_edge_cases_match_the_literal_transcription():
    """one row; every row in one cell; a grid of one row of cells; isolated known cells (windows with no other known cell);
    rows exactly on cell faces; only non-finite rows"""
    clouds = [np.array([[0.3, 0.4, -0.0]]),
              np.array([[0.1, 0.1, z] for z in (0.0, -0.0, 0.5, 2.9, 0.5)]),
              np.array([[0.25 * k, 0.0, 0.05 * k] for k in range(12)]),
              np.array([[0.0, 0.0, 0.0], [2.0, 2.0, 1.0], [0.0, 2.0, -1.0], [2.0, 0.0, 0.3]]),
              np.array([[0.25, 0.5, 0.1], [0.5, 0.25, -0.1], [0.75, 0.75, 0.0], [1.0, 1.0, 0.2]]),
              np.array([[np.nan, 0.0, 0.0], [0.0, np.inf, 0.0]])]
    for k, p in enumerate(clouds):
        got, want = to.build(p, SMALL), to.build_literal(p, SMALL)
        assert_same(got, want)
        assert (got["width"], got["height"]) == (want["width"], want["height"]), k
    assert to.build(clouds[-1], SMALL)["width"] == 0


def test_signed_zeros_order_minus_below_plus():
    """-0.0 orders below +0.0: the least z of a cell of both is -0.0, the elevation +0.0, and the step their difference"""
    p = np.array([[0.1, 0.1, 0.0], [0.1, 0.1, -0.0], [0.4, 0.1, -0.0]])
    t = to.build(p, SMALL)
    assert math.copysign(1.0, t["low"][0, 0]) == -1.0 and math.copysign(1.0, t["elevation"][0, 0]) == 1.0
    assert math.copysign(1.0, t["ground"][0, 0]) == -1.0 and t["step"][0, 0] == 0.0
    assert to.geometry(np.array([[-0.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), 0.2)[0] == 0.0
    assert math.copysign(1.0, to.geometry(np.array([[-0.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), 0.2)[0]) == -1.0


def test_ground_and_step_are_scipy_window_filters():
    from scipy.ndimage import maximum_filter, minimum_filter
    cfg = to.config(resolution=0.1, ground_radius=0.3, step_radius=0.2)
    p = random_cloud(3000, 7, span=(4.0, 3.0))
    t = to.build(p, cfg)
    rg, rs, _ = t["radii"]
    low = np.where(np.isnan(t["low"]), np.inf, t["low"])
    assert np.array_equal(minimum_filter(low, size=2 * rg + 1, mode="constant", cval=np.inf), t["ground"])
    known = t["points"] >= cfg["min_points"]
    e = t["elevation"]
    hi = maximum_filter(np.where(known, e, -np.inf), size=2 * rs + 1, mode="constant", cval=-np.inf)
    lo = minimum_filter(np.where(known, e, np.inf), size=2 * rs + 1, mode="constant", cval=np.inf)
    assert np.array_equal(np.where(known, hi - lo, np.nan), t["step"], equal_nan=True)
    assert known.sum() > 100 and t["overhang"] > 0


def test_plane_fit_is_least_squares_and_the_determinant_rule():
    rng = np.random.default_rng(3)
    E = rng.normal(0, 0.1, (9, 11))
    E[rng.random(E.shape) < 0.3] = np.nan
    rp, res = 2, 0.2
    slope, rough = to.plane_fit(E, rp, 4, res)
    checked = 0
    for j in range(E.shape[0]):
        for i in range(E.shape[1]):
            if np.isnan(E[j, i]):
                assert np.isnan(slope[j, i])
                continue
            pts = [(ii - i, jj - j, E[jj, ii] - E[j, i]) for jj in range(max(0, j - rp), min(E.shape[0], j + rp + 1))
                   for ii in range(max(0, i - rp), min(E.shape[1], i + rp + 1)) if not np.isnan(E[jj, ii])]
            A = np.array([[u, v, 1.0] for u, v, _ in pts])
            w = np.array([x for _, _, x in pts])
            if len(pts) < 4 or np.linalg.matrix_rank(A) < 3:
                assert np.isnan(slope[j, i]) and np.isnan(rough[j, i])
                continue
            (a, b, d), *_ = np.linalg.lstsq(A, w, rcond=None)
            assert abs(slope[j, i] - math.hypot(a, b) / res) <= 1e-12
            assert abs(rough[j, i] - np.abs(w - A @ [a, b, d]).max()) <= 1e-12
            checked += 1
    assert checked > 40
    line = np.full((5, 5), np.nan)
    line[2, :] = [0.0, 0.1, 0.2, 0.3, 0.4]                         # collinear: D == 0 whatever min_fit
    s, r = to.plane_fit(line, 2, 1, res)
    assert np.isnan(s).all() and np.isnan(r).all()
    diag = np.full((5, 5), np.nan)
    for k in range(5):
        diag[k, k] = 0.1 * k
    assert np.isnan(to.plane_fit(diag, 2, 1, res)[0]).all()
    plane = np.fromfunction(lambda j, i: 0.02 * i - 0.01 * j, (5, 5))
    s, r = to.plane_fit(plane, 2, 25, res)
    assert np.isfinite(s[2, 2]) and np.isnan(s[0, 0])                # 25 cells only at the centre
    assert abs(s[2, 2] - math.hypot(0.02, 0.01) / res) < 1e-12


def test_threshold_boundaries_and_the_combination_table():
    cfg = to.config(max_step=0.25, max_roughness=0.5)
    step = np.array([0.25, np.nextafter(0.25, 1.0), 0.0, 0.0, 0.0, np.nan, 0.0])
    slope = np.array([0.0, 0.0, 0.3, np.nextafter(0.3, 1.0), 0.0, np.nan, np.nan])
    rough = np.array([0.0, 0.0, 0.0, 0.0, np.nextafter(0.5, 1.0), np.nan, 0.5])
    known = np.array([True] * 7)
    assert to.classify(step, slope, rough, known, cfg, 0.3).tolist() == [0, 100, 0, 100, 100, 0, 0]
    assert to.classify(step, slope, rough, ~known, cfg, 0.3).tolist() == [-1] * 7
    # a slope exactly at the tangent bound is traversable; with the bound one double lower it is lethal
    E = np.fromfunction(lambda j, i: 0.05 * i, (5, 5))
    s, _ = to.plane_fit(E, 1, 3, 0.2)
    assert abs(s[2, 2] - 0.25) < 1e-12
    kn = np.ones(1, dtype=bool)
    assert to.classify(np.zeros(1), s[2:3, 2], np.zeros(1), kn, cfg, s[2, 2])[0] == 0
    assert to.classify(np.zeros(1), s[2:3, 2], np.zeros(1), kn, cfg, np.nextafter(s[2, 2], 0.0))[0] == 100
    o = np.arange(-1, 101)
    for t in (-1, 0, 100):
        want = [100 if (t == 100 or v >= 65) else (0 if (t == 0 or 0 <= v <= 25) else -1) for v in o]
        assert to.combine(np.full(len(o), t), o).tolist() == want


def test_the_grid_limit():
    r = 0.2
    side = math.sqrt(float(to.MAX_CELLS)) * r
    assert to.geometry(np.array([[0.0, 0.0, 0.0], [side - 1.5 * r, side - 1.5 * r, 0.0]]), r) is not None
    assert to.geometry(np.array([[0.0, 0.0, 0.0], [side + r, side + r, 0.0]]), r) is None
    assert to.build(np.array([[0.0, 0.0, 0.0], [1.0e5, 0.0, 0.0], [0.0, 1.0e5, 0.0]]), to.config()) is None


# ---- a ray-cast terrain world ----------------------------------------------------------------------------------------
KERB = 0.15
DRIVE = (30.0, 35.0)                      # the driveway's x range; its ramp rises KERB over y 4 .. 4 + KERB / 0.08
RAMP = (50.0, 54.0, -14.0, -8.0)          # x0, x1, y0, y1 of the steep ramp, rising 0.35 per m towards -y
DITCH = (10.0, 40.0, 10.0, 13.0)          # x0, x1, y0, y1; floor 0.5 m below the sidewalk
DECK = (70.0, 76.0, 4.5, 5.0)             # the overpass deck's x range and z range, spanning y -16 .. 16
# boxes, pillars, the side walls and the end walls: (cx, cy, hx, hy, z top)
BOXES = np.array([[44.0, 9.5, 0.6, 0.6, KERB + 1.0], [22.0, -10.0, 1.0, 0.8, KERB + 0.6], [62.0, 10.0, 1.5, 1.0, KERB + 1.4],
                  [84.0, -10.5, 0.8, 1.2, KERB + 0.8], [73.0, 9.0, 0.3, 0.3, 4.5], [73.0, -9.0, 0.3, 0.3, 4.5],
                  [40.0, 16.5, 60.0, 0.5, 3.0], [40.0, -16.5, 60.0, 0.5, 3.0], [-6.0, 0.0, 0.5, 16.0, 3.0],
                  [94.0, 0.0, 0.5, 16.0, 3.0]])


def height(x, y):
    """the ground's height at (x, y): road |y| < 4 at 0, sidewalks at KERB, the driveway ramp, the steep ramp and the
    ditch"""
    z = np.where(np.abs(y) < 4.0, 0.0, KERB)
    dl = KERB / 0.08
    drive = (x >= DRIVE[0]) & (x < DRIVE[1]) & (y >= 4.0) & (y < 4.0 + dl)
    z = np.where(drive, 0.08 * (y - 4.0), z)
    ramp = (x >= RAMP[0]) & (x < RAMP[1]) & (y >= RAMP[2]) & (y < RAMP[3])
    z = np.where(ramp, KERB + 0.35 * (RAMP[3] - y), z)
    plat = (x >= RAMP[0]) & (x < RAMP[1]) & (y < RAMP[2]) & (y > -16.0)
    z = np.where(plat, KERB + 0.35 * (RAMP[3] - RAMP[2]), z)
    ditch = (x >= DITCH[0]) & (x < DITCH[1]) & (y >= DITCH[2]) & (y < DITCH[3])
    return np.where(ditch, KERB - 0.5, z)


def _boxes_t(o, d):
    """first hit of rays o + t d with the boxes, the pillars and the deck (inf for none)"""
    lo = np.column_stack([BOXES[:, 0] - BOXES[:, 2], BOXES[:, 1] - BOXES[:, 3], np.full(len(BOXES), -1.0)])
    hi = np.column_stack([BOXES[:, 0] + BOXES[:, 2], BOXES[:, 1] + BOXES[:, 3], BOXES[:, 4]])
    lo = np.vstack([lo, [DECK[0], -16.0, DECK[2]]])
    hi = np.vstack([hi, [DECK[1], 16.0, DECK[3]]])
    with np.errstate(divide="ignore", invalid="ignore"):
        t1 = (lo[None] - o[None, None]) / d[:, None, :]
        t2 = (hi[None] - o[None, None]) / d[:, None, :]
        tn = np.nanmax(np.minimum(t1, t2), axis=2)
        tf = np.nanmin(np.maximum(t1, t2), axis=2)
    return np.where((tn <= tf) & (tn > 0), tn, np.inf).min(axis=1)


def cast(x, y, yaw, n_az=360, seed=0, t_max=30.0, dt=0.1):
    """the scan (sensor frame) of a 16-beam sensor SENSOR_Z above the ground at (x, y) heading yaw"""
    az = (np.arange(n_az) + 0.5) * (2 * np.pi / n_az)
    el, a = np.meshgrid(ELEV, az, indexing="ij")
    d = np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.sin(el)], axis=-1).reshape(-1, 3)
    c, s = math.cos(yaw), math.sin(yaw)
    dw = d @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]).T
    o = np.array([x, y, float(height(np.array(x), np.array(y))) + SENSOR_Z])
    tb = _boxes_t(o, dw)
    th = np.full(len(dw), np.inf)
    ts = np.arange(0.3, t_max, dt)
    for k in range(0, len(ts), 200):
        T = ts[k:k + 200]
        p = o[None, None] + T[None, :, None] * dw[:, None, :]
        below = p[..., 2] <= height(p[..., 0], p[..., 1])
        first = np.where(below.any(axis=1), T[np.argmax(below, axis=1)], np.inf)
        th = np.where(np.isinf(th), first, th)
    # refine the ground hits by bisection over the last step
    lo_t, hi_t = th - dt, th.copy()
    hit = np.isfinite(th)
    for _ in range(10):
        mid = 0.5 * (lo_t + hi_t)
        p = o + mid[:, None] * dw
        below = p[:, 2] <= height(p[:, 0], p[:, 1])
        hi_t = np.where(hit & below, mid, hi_t)
        lo_t = np.where(hit & ~below, mid, lo_t)
    t = np.minimum(np.where(hit, hi_t, np.inf), tb)
    keep = np.isfinite(t) & (t < t_max)
    rng = np.random.default_rng(seed)
    pw = dw[keep] * t[keep, None] + rng.normal(0, 0.01, (int(keep.sum()), 3))
    return pw @ np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])     # back to the sensor frame


def route():
    return [(2.0 * k, -1.0, 0.0) for k in range(45)]


@functools.lru_cache(maxsize=1)
def scans():
    return [cast(x, y, yaw, seed=k) for k, (x, y, yaw) in enumerate(route())]


def map_of_world(voxel=0.1):
    """the global-map restatement of the drive at the true poses: each frame's voxel down-sample, concatenated"""
    import global_map_oracle as gmo
    from oracle import pyoracle
    poses = [pose_of(x, y, yaw) for x, y, yaw in route()]
    return gmo.global_map(pyoracle, [gmo.transform(s, p) for s, p in zip(scans(), poses)], voxel)[0]


def regions(t):
    """(edge cells by kind, traversable cells): the edge cells lie within one cell of a kerb, a ditch edge or a box
    edge, or inside the steep ramp; the traversable ones are road and driveway cells at least 2 cells beyond the reach
    of the step and slope windows (max(rs, rp) cells) from every edge"""
    h, w = t["values"].shape
    r = t["resolution"]
    jj, ii = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    x, y = t["origin"][0] + (ii + 0.5) * r, t["origin"][1] + (jj + 0.5) * r
    kerb = (np.abs(np.abs(y) - 4.0) < r) & ~((y > 0) & (x > DRIVE[0] - r) & (x < DRIVE[1] + r)) & (x > 1) & (x < 88)
    ditch = (x > DITCH[0] + r) & (x < DITCH[1] - r) & ((np.abs(y - DITCH[2]) < r) | (np.abs(y - DITCH[3]) < r))
    ramp = (x > RAMP[0] + 2 * r) & (x < RAMP[1] - 2 * r) & (y > RAMP[2] + 2 * r) & (y < RAMP[3] - 2 * r)
    box = np.zeros_like(kerb)
    for cx, cy, hx, hy, _ in BOXES[:6]:
        box |= np.abs(np.maximum(np.abs(x - cx) - hx, np.abs(y - cy) - hy)) < r
    m = (max(t["radii"][1:]) + 2) * r
    road = np.abs(y) < 4.0 - m
    drive = (x > DRIVE[0] + m) & (x < DRIVE[1] - m) & (y > 4.0) & (y < 4.0 + KERB / 0.08)
    return dict(kerb=kerb, ditch=ditch, ramp=ramp, box=box), (road | drive) & (x > 0) & (x < 88)


def test_quality_of_the_defaults_on_the_terrain_world():
    """the drive (45 frames, 16 beams) mapped at voxel 0.1 m at the true poses, the terrain at the defaults.  Targets set
    before measuring: >= 95 % of the known edge cells lethal, >= 99 % of the known traversable cells traversable.
    Measured: 96.0 % of 2 575 edge cells (kerbs 100 %, ditch edges 78.6 %, steep ramp 91.1 %, box edges 99.2 %) and
    100 % of 13 274 road, driveway and under-overpass cells; the 0.2 m step radius first proposed (one cell) gave 69.4 %"""
    t = to.build(map_of_world(), to.config())
    edges, trav = regions(t)
    v = t["values"]
    e = (edges["kerb"] | edges["ditch"] | edges["ramp"] | edges["box"]) & (v >= 0)
    ok = trav & (v >= 0)
    print({k: float((v[m & (v >= 0)] == 100).mean()) for k, m in edges.items()}, e.sum(), ok.sum())
    assert e.sum() > 2000 and ok.sum() > 10000 and t["overhang"] > 1000
    assert (v[e] == 100).mean() >= 0.95 and (v[ok] == 0).mean() >= 0.99


def occupancy_of_world():
    """the occupancy grid restatement of the drive at the true poses (the occupancy defaults, 360 azimuths)"""
    import occupancy_oracle as oo
    cfg = oo.config(n_cols=360)
    return oo.build([oo.scan2d(s, cfg) for s in scans()], [pose_of(x, y, yaw) for x, y, yaw in route()], cfg), cfg


START, GOAL = (20.0, -1.5), (20.0, 6.5)


def route_on(values, origin, res):
    """the plan from START to GOAL on the costmap of the values (distance and plan defaults): its cells' centres"""
    f = do.field(values, origin, res)
    t = po.cell_costs(f["costs"])
    g, _ = po.cells_of([GOAL], origin, res, values.shape)
    s, _ = po.cells_of([START], origin, res, values.shape)
    P = po.potential(t, (int(g[0, 0]), int(g[0, 1])))
    status, _, cells = po.paths(P, t, s)[0]
    return status, po.centres(cells, origin, res), f


def crosses_kerb_outside_the_driveway(xy):
    """(the path crosses y = 4 outside the driveway, it crosses inside it)"""
    crossing = (xy[:-1, 1] < 4.0) != (xy[1:, 1] < 4.0)
    x = 0.5 * (xy[:-1, 0] + xy[1:, 0])
    inside = (x >= DRIVE[0]) & (x <= DRIVE[1])
    return bool((crossing & ~inside).any()), bool((crossing & inside).any())


def test_the_combined_terrain_routes_over_the_driveway():
    """start on the road, goal on the sidewalk, the distance and plan defaults: on the occupancy grid alone the plan
    crosses the kerb; on the terrain combined with it the plan reaches the sidewalk only over the driveway"""
    og, ocfg = occupancy_of_world()
    status, xy, _ = route_on(og["cells"], og["origin"], ocfg["resolution"])
    assert status == 0 and crosses_kerb_outside_the_driveway(xy) == (True, False)
    grid = (og["origin"][0], og["origin"][1], ocfg["resolution"], og["width"], og["height"])
    t = to.build(map_of_world(), to.config(combine_occupancy=1), grid=grid, occupancy=og["cells"])
    status, xy, _ = route_on(t["values"], og["origin"], ocfg["resolution"])
    assert status == 0 and crosses_kerb_outside_the_driveway(xy) == (False, True)


# ---- the library ------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_terrain_library_holds_only_its_kernels_for_sm90a_without_spills():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.TERRAIN_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.TERRAIN_LIB], capture_output=True, text=True,
                         check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.TERRAIN_LIB], capture_output=True, text=True,
                         check=True).stdout
    usage = [l for l in res.splitlines() if "REG:" in l]
    assert len(usage) == len(KERNELS) and all("STACK:0 " in l for l in usage), usage


def test_every_other_library_keeps_its_sass():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_terrain.json")))
    assert len(want) == 20 and "libtloam_b200_terrain.so" not in want and "libtloam_b200_frontier.so" in want
    for lib in want:
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


def test_terrain_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "terrain_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def as_dict(t):
    """a TerrainMap in the restatement's keys"""
    d = dict(t.info)
    d.update(values=t.values, ground=t.ground, elevation=t.elevation, step=t.step, slope=t.slope, roughness=t.roughness,
             points=t.points)
    return d


def assert_device(t, want):
    assert want is not None
    assert t.origin == want["origin"] and t.values.shape == (want["height"], want["width"])
    assert same_bits(np.array(t.origin), np.array(want["origin"])) and t.radii == want["radii"]
    assert_same(as_dict(t), want)
    assert t.info["rows"] == want["used"] + want["skipped"] + want["dropped"]


@pytest.mark.gpu
def test_gpu_host_clouds_are_the_restatement():
    """grids from 1 x 1 to 129 x 257 and larger, the small and the default windows"""
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    cases = [(np.array([[0.05, 0.05, 0.3]]), SMALL), (random_cloud(40, 1, (0.2, 0.2)), SMALL),
             (random_cloud(5000, 2, (129 * 0.25 - 0.01, 257 * 0.25 - 0.01)), SMALL),
             (random_cloud(20000, 3, (40.0, 30.0)), to.config()),
             (random_cloud(30000, 4, (20.0, 50.0)), to.config(resolution=0.1)),
             (random_cloud(3000, 6, (5.0, 5.0)), dict(SMALL, min_fit=(1 << 31) + 5)),   # compared unsigned: no fit
             (np.array([[np.nan, 0.0, 0.0]]), SMALL), (np.zeros((0, 3)), to.config())]
    shapes = []
    for p, cfg in cases:
        t = r.terrain_build(p, **cfg)
        assert_device(t, to.build(p, cfg))
        if cfg["min_fit"] > 1 << 31:
            assert t.info["known"] > 100 and np.isnan(t.slope).all() and np.isnan(t.roughness).all()
        shapes.append(t.values.shape)
    print(shapes)
    assert (1, 1) in shapes and any(h >= 257 and w >= 129 for h, w in shapes)
    r.close()


def device_world(dynamic=False, occupancy=False, correction=False, n=None):
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(voxel=0.1)
    if dynamic:
        r.global_map_dynamic_enable()
    if occupancy:
        r.occupancy_enable(n_cols=360)
    if correction:
        r.global_map_correction_enable()
        r.pose_graph_enable()
    for (x, y, yaw), s in zip(route()[:n], scans()[:n]):
        r.global_map_append(s, pose_of(x, y, yaw))
        if correction:
            r.pose_graph_add_node(pose_of(x, y, yaw))
    return r


@pytest.mark.gpu
def test_gpu_world_through_the_device_map_is_the_restatement():
    """all rows, the static rows and the combined grid after an occupancy build; repeat builds give the same bits; the
    costmap of the values is distance_build_grid's; the plan over it takes the driveway"""
    r = device_world(dynamic=True, occupancy=True)
    rows = r.global_map()
    cfg = to.config()
    t = r.terrain_build()
    assert_device(t, to.build(rows, cfg))
    again = r.terrain_build()
    assert_same(as_dict(again), as_dict(t))
    st = r.terrain_build(static_only=1)
    xyz, _ = r.global_map_static()
    assert_device(st, to.build(xyz, cfg))
    g = r.occupancy_build()
    grid = (g.origin[0], g.origin[1], g.resolution, g.cells.shape[1], g.cells.shape[0])
    c = r.terrain_build(combine_occupancy=1)
    want = to.build(rows, to.config(combine_occupancy=1), grid=grid, occupancy=g.cells)
    assert c.combined and c.resolution == g.resolution
    assert_device(c, want)
    f = r.distance_build_terrain()
    h = r.distance_build(c.values, c.origin, c.resolution)
    for k in ("signed", "sq", "costs", "values"):
        assert same_bits(getattr(f, k), getattr(h, k)), k
    r.distance_build_terrain()
    P = r.plan_build(GOAL)
    path = r.plan_paths([START])[0]
    assert path.status == 0 and crosses_kerb_outside_the_driveway(path.xy) == (False, True)
    fd = do.field(c.values, c.origin, c.resolution)
    t_ = po.cell_costs(fd["costs"])
    gi, _ = po.cells_of([GOAL], c.origin, c.resolution, c.values.shape)
    assert np.array_equal(P.potential, po.potential(t_, (int(gi[0, 0]), int(gi[0, 1]))))
    assert np.array_equal(f.costs, fd["costs"])
    info, got, _ = search_and_check(r, f, P)                       # the frontiers on it: the restatement's
    assert info["kept"] > 0
    r.close()


@pytest.mark.gpu
def test_gpu_terrain_follows_a_correction_and_stays_a_snapshot():
    import pose_graph_oracle as pgo
    from test_pose_graph import loop_result
    r = device_world(correction=True, n=12)
    before = r.terrain_build()
    O = [pose_of(x, y, yaw) for x, y, yaw in route()[:12]]
    r.pose_graph_add_loop(loop_result(1, 9, pgo.inv_mul(O[1], O[9]) @ pgo.exp4([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(12))
    rows = r.global_map()
    after = r.terrain_build()
    assert_device(after, to.build(rows, to.config()))
    assert not same_bits(after.values, before.values) or after.origin != before.origin
    r.close()


@pytest.mark.gpu
def test_gpu_terrain_status_codes_and_nothing_else_changes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.TerrainConfig()
    L.tloam_b200_terrain_default_config(C.byref(cfg))
    info = _lib.TerrainInfo()
    dcfg = _lib.DistanceConfig()
    L.tloam_b200_distance_default_config(C.byref(dcfg))
    assert L.tloam_b200_terrain_build(None, C.byref(cfg), C.byref(info)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_terrain_build(h, None, C.byref(info)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_terrain_build(h, C.byref(cfg), C.byref(info)) == _lib.ERR_NOT_READY          # mapping off
    assert L.tloam_b200_terrain_download(h, None, None, None, None, None, None, None, 0) == _lib.ERR_NOT_READY
    assert L.tloam_b200_distance_build_terrain(h, C.byref(dcfg), None) == _lib.ERR_NOT_READY
    for field, bad in (("resolution", 0.0), ("resolution", float("nan")), ("clearance", -1.0), ("max_slope", 1.6),
                       ("step_radius", 3.5), ("slope_radius", float("inf")), ("ground_radius", 300.0), ("min_points", 0),
                       ("min_fit", 0), ("static_only", 1), ("max_roughness", -0.1)):
        c = _lib.TerrainConfig()
        L.tloam_b200_terrain_default_config(C.byref(c))
        setattr(c, field, bad)
        assert L.tloam_b200_terrain_build_cloud(h, C.byref(c), None, 0, None) == _lib.ERR_INVALID_ARG, (field, bad)
    c = _lib.TerrainConfig()
    L.tloam_b200_terrain_default_config(C.byref(c))
    c.combine_occupancy = 1
    assert L.tloam_b200_terrain_build_cloud(h, C.byref(c), None, 0, None) == _lib.ERR_NOT_READY
    p = random_cloud(500, 9)
    first = r.terrain_build(p)
    far = np.array([[0.0, 0.0, 0.0], [1.0e5, 1.0e5, 0.0]])
    with pytest.raises(tloam_b200.RegistrationError) as e:
        r.terrain_build(far)
    assert e.value.status == _lib.ERR_VOXEL_RANGE
    n = first.values.size
    assert L.tloam_b200_terrain_download(h, None, None, None, None, None, None, None, n - 1) == _lib.ERR_INVALID_ARG
    values = np.zeros(first.values.shape, dtype=np.int8)
    assert L.tloam_b200_terrain_download(h, values.ctypes.data_as(C.POINTER(C.c_byte)), None, None, None, None, None,
                                         None, n) == _lib.OK
    assert np.array_equal(values, first.values)                                    # a refused build keeps the last
    r.close()
    # nothing else changes: the map, the occupancy grid, the last distance field and plan as they stand (downloaded,
    # not rebuilt), and the launch counts of the other calls against a handle that never built a terrain
    r, plain = device_world(occupancy=True, n=6), device_world(occupancy=True, n=6)
    for q in (r, plain):
        shape = q.occupancy_build().cells.shape
        q.distance_build()
        q.plan_build(START)
    before = held_state(r, shape)
    assert same_state(before, held_state(plain, shape))
    n0 = r.launch_count()
    r.terrain_build(combine_occupancy=1)
    assert r.launch_count() - n0 == 5                                            # k_ter_low, _ground x 2, _high, _layers
    assert same_state(held_state(r, shape), before)
    deltas = []
    for q in (r, plain):                                           # an append, then each build, counted on its own
        counts = [q.launch_count()]
        q.global_map_append(scans()[6], pose_of(*route()[6]))
        counts.append(q.launch_count())
        shape = q.occupancy_build().cells.shape
        counts.append(q.launch_count())
        q.distance_build()
        counts.append(q.launch_count())
        q.plan_build(START)
        counts.append(q.launch_count())
        deltas.append(np.diff(counts).tolist())
    assert deltas[0] == deltas[1] and min(deltas[0]) > 0
    assert same_state(held_state(r, shape), held_state(plain, shape))
    r.close()
    plain.close()


def held_state(r, shape):
    """the map, the occupancy grid, the distance field and the plan the handle holds (all on one grid of `shape`),
    downloaded without a rebuild"""
    L, h = r._L, r._h
    n = shape[0] * shape[1]
    cells, occ, free = np.zeros(shape, np.int8), np.zeros(shape, np.uint32), np.zeros(shape, np.uint32)
    sd, sq, costs, values = np.zeros(shape, np.float32), np.zeros(shape, np.uint32), np.zeros(shape, np.uint8), \
        np.zeros(shape, np.int8)
    P = np.zeros(shape, np.uint64)
    ptr = lambda a, t: a.ctypes.data_as(C.POINTER(t))                       # noqa: E731
    assert L.tloam_b200_occupancy_download(h, ptr(cells, C.c_byte), ptr(occ, C.c_uint), ptr(free, C.c_uint), n) == 0
    assert L.tloam_b200_distance_download(h, ptr(sd, C.c_float), ptr(sq, C.c_uint), ptr(costs, C.c_ubyte),
                                          ptr(values, C.c_byte), n) == 0
    assert L.tloam_b200_plan_download(h, ptr(P, C.c_ulonglong), n) == 0
    return dict(map=r.global_map(), cells=cells, occupied=occ, free=free, sd=sd, sq=sq, costs=costs, values=values, P=P)


def same_state(a, b):
    return all(same_bits(a[k], b[k]) if a[k].dtype.kind == "f" else np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.gpu
def test_gpu_terrain_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("terrain_driver", "front_end_b200.hpp")
    rng = np.random.default_rng(5)
    p = np.column_stack([rng.uniform(0, 30.0, 20000), rng.uniform(0, 20.0, 20000), rng.normal(0, 0.005, 20000)])
    p[p[:, 1] > 12.0, 2] += 0.15                                   # a kerb across the cloud
    goal = (5.0, 5.0)
    path = os.path.join(os.path.dirname(exe), "terrain_in.bin")
    out_path = os.path.join(os.path.dirname(exe), "terrain_out.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p).tobytes() + struct.pack("2d", *goal))
    res = subprocess.run([exe, path, out_path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    w, h, known, lethal, reachable = (int(s) for s in res.stdout.split())
    r = tloam_b200.LocalRegistration()
    t = r.terrain_build(p)
    f = r.distance_build_terrain()
    P = r.plan_build(goal)
    r.close()
    blob = open(out_path, "rb").read()
    n = w * h
    origin = struct.unpack_from("2d", blob, 0)
    values = np.frombuffer(blob, dtype=np.int8, count=n, offset=16).reshape(h, w)
    elevation = np.frombuffer(blob, dtype=np.float64, count=n, offset=16 + n).reshape(h, w)
    slope = np.frombuffer(blob, dtype=np.float64, count=n, offset=16 + 9 * n).reshape(h, w)
    costs = np.frombuffer(blob, dtype=np.uint8, count=n, offset=16 + 17 * n).reshape(h, w)
    assert origin == t.origin and (h, w) == t.values.shape and (known, lethal) == (t.info["known"], t.info["lethal"])
    assert np.array_equal(values, t.values) and same_bits(elevation, t.elevation) and same_bits(slope, t.slope)
    assert np.array_equal(costs, f.costs) and reachable == P.reachable
