"""Loop closure (include/tloam_b200.h "Loop closure", k_sc_bin / k_sc_finish / k_sc_search / k_sc_reduce in
libtloam_b200_loop.so): a Scan Context descriptor per added frame and an exact search over every earlier frame at every
column shift.  tests/scan_context_oracle.py is the CPU restatement; its vectorised form is pinned here to a literal
per-row / per-column transcription.  The sector comes from a table of boundary directions, not from atan2, so no row is
exempted near a sector boundary: descriptors and distances are compared bit for bit.

CPU: the two oracle forms, the rotation convention of shift and yaw, the symbols, the new library's kernels, the shim.
GPU: descriptors and searches against the oracle, a revisit in a ray-cast world, the scan loop_add_frame reads, the
odometry loop's bits with detection on, determinism and growth, status codes, the shim against the Python mirror."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import sass_digest
import scan_context_oracle as sco
from tloam_b200 import synth
from test_global_map import with_nonfinite
from test_global_map_intensity import same_bits
from test_packed_scan import sorted_rows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_loop_default_config", "tloam_b200_loop_enable", "tloam_b200_loop_reset", "tloam_b200_loop_add_frame",
               "tloam_b200_loop_add", "tloam_b200_loop_result", "tloam_b200_loop_size", "tloam_b200_loop_descriptor_download"]
CONFIGS = [sco.config(), sco.config(n_ring=7, n_sector=13, max_radius=30.0, lidar_height=-0.5),
           sco.config(n_ring=3, n_sector=2, max_radius=12.0), sco.config(n_ring=5, n_sector=1, max_radius=20.0),
           sco.config(n_ring=1, n_sector=97, max_radius=50.0, lidar_height=0.0)]


def random_cloud(n, seed, spread=60.0):
    """rows around the sensor, some beyond 80 m, a few at r = 0, non-finite rows, rows on sector-boundary directions"""
    rng = np.random.default_rng(seed)
    p = np.column_stack([rng.uniform(-spread, spread, n), rng.uniform(-spread, spread, n), rng.uniform(-3.0, 4.0, n)])
    p[:5, :2] = 0.0                                                # r = 0
    p[5, :2] = [-0.0, 0.0]
    p[6:9] = [[90.0, 1.0, 0.0], [0.0, -85.0, 1.0], [80.0, 0.0, 2.0]]   # beyond max_radius, and exactly on it
    p[9:13] = [[np.nan, 1.0, 1.0], [1.0, np.inf, 0.0], [2.0, 2.0, -np.inf], [np.nan] * 3]
    for k, S in enumerate((60, 13, 2, 97)):                           # rows on boundary directions of the configurations above
        t = 2.0 * math.pi * np.arange(1, S) / S
        m = min(len(t), 8)
        p[20 + 8 * k:20 + 8 * k + m, :2] = np.column_stack([np.cos(t[:m]), np.sin(t[:m])]) * 10.0
    p[60:70, 1] = 0.0                                              # on the x axis, both signs of x
    p[60:65, 0] *= -1
    return p


def flat(desc):
    return np.concatenate([np.ravel(x) for x in desc])


def assert_same_descriptor(got, want):
    for g, w, name in zip(got, want, ("bins", "ring key", "column norms")):
        assert g.shape == w.shape and same_bits(g, w), name


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_oracle_descriptor_matches_the_literal_transcription(k):
    cfg = CONFIGS[k]
    clouds = [random_cloud(3000, 10 + k), random_cloud(2000, 20 + k, spread=150.0)]
    neg = random_cloud(1500, 30 + k, spread=20.0)
    neg[:, 2] = -np.abs(neg[:, 2]) - 3.0                           # every maximum negative
    half = random_cloud(1500, 40 + k)
    half = half[~(half[:, 1] > 0)]                                 # the upper half-plane empty: empty columns
    clouds += [neg, half, np.zeros((0, 3))]
    for p in clouds:
        want = sco.descriptor_literal(p, cfg)
        assert_same_descriptor(sco.descriptor(p, cfg), want)
    bins = sco.descriptor(neg, cfg)[0]
    assert (bins < 0).any() and not (bins > 0).any()
    if cfg["n_sector"] > 2:
        assert (sco.descriptor(half, cfg)[2] == 0).any()


@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_oracle_distances_match_the_literal_transcription(k):
    cfg = CONFIGS[k]
    S = cfg["n_sector"]
    descs = [sco.descriptor(random_cloud(2000, 50 + k + 7 * i), cfg) for i in range(3)]
    half = random_cloud(1500, 60 + k)
    descs.append(sco.descriptor(half[~(half[:, 1] > 0)], cfg))     # empty columns
    descs.append(sco.descriptor(np.zeros((0, 3)), cfg))            # no column at all: distance 1.0
    table = sco.distances(descs[0], descs)
    assert table.shape == (len(descs), S)
    for j in range(len(descs)):
        for s in range(S):
            assert same_bits(np.array(table[j, s]), np.array(sco.distance_literal(descs[0], descs[j], s))), (j, s)
    assert np.all(table[-1] == 1.0)


def test_oracle_search_breaks_ties_by_candidate_then_shift():
    cfg = sco.config()
    p = random_cloud(3000, 70)
    d = sco.descriptor(p, cfg)
    other = sco.descriptor(random_cloud(3000, 71), cfg)
    descs = [other, d, d, other, d]                                # frames 1 and 2 tie exactly with the query (frame 4)
    j, s, dist, table = sco.query(descs, 4, 2, chunk=2)
    assert table.shape == (3, 60) and (j, s) == (1, 0) and dist == table[1, 0] == table[2, 0] and dist < 1e-12
    assert sco.query(descs, 1, 2)[0] == -1 and sco.query(descs, 2, 2)[:2] == (0, int(np.argmin(table[0])))


def sector_centred_cloud(cfg, seed):
    """rows at the centre of their bin (azimuth and range), so that a rotation by whole sectors moves no row across a bin"""
    rng = np.random.default_rng(seed)
    R, S = cfg["n_ring"], cfg["n_sector"]
    n = 4000
    ring = rng.integers(0, R, n)
    sector = rng.integers(0, S, n)
    r = (ring + 0.5) * cfg["max_radius"] / R
    a = (sector + 0.5) * 2 * np.pi / S
    return np.column_stack([r * np.cos(a), r * np.sin(a), rng.uniform(-1.5, 3.0, n)])


def rz(a):
    return np.array([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]])


@pytest.mark.parametrize("k", [0, 1, 7, 29, 30, 31, 59])
def test_rotation_by_whole_sectors_gives_the_shift_and_yaw_convention(k):
    """query = candidate rotated by k sectors about z (p_query = Rz(alpha) p_cand): shift k, distance 0 up to the rounding of
    cos = (a . a) / (|a| |a|), yaw = -alpha wrapped to (-pi, pi], and Rz(yaw) takes the query's rows back onto the candidate's"""
    cfg = sco.config()
    cand = sector_centred_cloud(cfg, 80 + k)
    alpha = k * 2 * math.pi / 60
    q = cand @ rz(alpha).T
    a, b = sco.descriptor(q, cfg), sco.descriptor(cand, cfg)
    assert np.array_equal(a[0], np.roll(b[0], k, axis=1))
    j, s, dist, table = sco.query([b, a], 1, 1)
    assert (j, s) == (0, k) and abs(dist) < 1e-12 and np.sort(table[0])[1] > 0.01
    yaw = sco.yaw_of(s, 60)
    assert -math.pi < yaw <= math.pi and math.isclose(math.remainder(yaw + alpha, 2 * math.pi), 0.0, abs_tol=1e-12)
    assert np.allclose(q @ rz(yaw).T, cand, atol=1e-9)


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_loop_library_holds_only_the_four_kernels_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.LOOP_LIB))
    kernels = ("k_sc_bin", "k_sc_finish", "k_sc_search", "k_sc_reduce")
    assert len(names) == 4 and [sum(f"{len(k)}{k}E" in m for m in names) for k in kernels] == [1, 1, 1, 1]
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.LOOP_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


def test_loop_driver_compiles_warning_free():
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("loop_driver", "front_end_b200.hpp"))
    src = os.path.join(ROOT, "tests", "mock", "loop_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- a ray-cast world with a revisit ------------------------------------------------------------------------------------
ELEV = np.radians(np.linspace(-24.0, 2.0, 16))
SENSOR_Z = 1.73


def make_world(seed=3):
    """seeded boxes and poles, with nothing periodic in their placement"""
    rng = np.random.default_rng(seed)
    nb = 140
    c = np.column_stack([rng.uniform(-70, 150, nb), rng.uniform(-70, 130, nb), np.zeros(nb)])
    h = np.column_stack([rng.uniform(1.0, 6.0, nb), rng.uniform(1.0, 6.0, nb), rng.uniform(1.0, 5.0, nb)])
    c[:, 2] = h[:, 2] - SENSOR_Z
    poles = np.column_stack([rng.uniform(-70, 150, 120), rng.uniform(-70, 130, 120), rng.uniform(2.0, 8.0, 120)])
    return c, h, poles


def cast(world, x, y, yaw, n_az=720, seed=0):
    """the scan (sensor frame) of a 16-beam sensor at (x, y, SENSOR_Z) heading yaw: first returns within 80 m"""
    c, hw, poles = world
    az = (np.arange(n_az) + 0.5) * (2 * np.pi / n_az)
    el, a = np.meshgrid(ELEV, az, indexing="ij")
    d = np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.sin(el)], axis=-1).reshape(-1, 3)
    dw = d @ rz(yaw).T
    o = np.array([x, y, 0.0])                                      # the world with the sensor's height removed
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(dw[:, 2] < -1e-9, -SENSOR_Z / dw[:, 2], np.inf)
        t1 = (c[None, :, :] - hw[None, :, :] - o) / dw[:, None, :]
        t2 = (c[None, :, :] + hw[None, :, :] - o) / dw[:, None, :]
        tn = np.nanmax(np.minimum(t1, t2), axis=2)
        tf = np.nanmin(np.maximum(t1, t2), axis=2)
        tb = np.where((tn <= tf) & (tn > 0), tn, np.inf).min(axis=1)
        A = dw[:, 0] ** 2 + dw[:, 1] ** 2
        ox, oy = o[0] - poles[:, 0], o[1] - poles[:, 1]
        B = dw[:, 0:1] * ox[None, :] + dw[:, 1:2] * oy[None, :]
        disc = B * B - A[:, None] * (ox * ox + oy * oy - 0.25 ** 2)[None, :]
        tp = (-B - np.sqrt(np.maximum(disc, 0.0))) / A[:, None]
        zp = tp * dw[:, 2:3]
        tp = np.where((disc > 0) & (tp > 0) & (zp > -SENSOR_Z) & (zp < poles[None, :, 2] - SENSOR_Z), tp, np.inf).min(axis=1)
    t = np.minimum(np.minimum(t, tb), tp)
    keep = np.isfinite(t) & (t < 80.0)
    rng = np.random.default_rng(seed)
    return d[keep] * t[keep, None] + rng.normal(0, 0.01, (int(keep.sum()), 3))


# leg 1 east along y = 0 (2 m steps), leg 2 north, leg 3 west, then a straight leg heading -97 deg that ends 0.4 m / 0.3 m
# off frame REVISIT_OF's place
REVISIT_OF = 10
RETURN_YAW = math.radians(-97.0)


def route():
    poses = [(2.0 * k, 0.0, 0.0) for k in range(40)]
    poses += [(80.0, 2.0 * k, math.pi / 2) for k in range(1, 31)]
    poses += [(80.0 - 2.0 * k, 60.0, math.pi) for k in range(1, 23)]
    end = np.array([2.0 * REVISIT_OF + 0.4, 0.3])
    step = 2.0 * np.array([math.cos(RETURN_YAW), math.sin(RETURN_YAW)])
    poses += [(float(end[0] - k * step[0]), float(end[1] - k * step[1]), RETURN_YAW) for k in range(25, -1, -1)]
    return poses


def route_scans():
    world = make_world()
    return route(), [cast(world, x, y, yaw, seed=k) for k, (x, y, yaw) in enumerate(route())]


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_gpu_descriptors_are_the_oracles(k):
    """HDL-64E and VLP-16 scans with NaN / Inf rows and the random clouds above, through loop_add"""
    import tloam_b200
    cfg = CONFIGS[k]
    r = tloam_b200.LocalRegistration()
    r.loop_enable(**cfg)
    clouds = [with_nonfinite(synth.raw_scan(), 7), with_nonfinite(synth.vlp16_raw_scan(), 9), random_cloud(5000, 90 + k),
              np.zeros((0, 3))]
    for i, p in enumerate(clouds):
        r.loop_add(p)
        assert_same_descriptor(r.loop_descriptor(i), sco.descriptor(p, cfg))
    assert r.loop_size() == len(clouds)
    r.close()


def database_clouds(n, seed):
    """n small clouds; every 7th repeats an earlier one (exact ties between candidates), every 11th is a rotated earlier one"""
    out = []
    rng = np.random.default_rng(seed)
    for i in range(n):
        if i >= 7 and i % 7 == 0:
            out.append(out[int(rng.integers(0, i))].copy())
        elif i >= 11 and i % 11 == 0:
            with np.errstate(invalid="ignore"):                    # the non-finite rows stay non-finite
                out.append(out[int(rng.integers(0, i))] @ rz(rng.uniform(0, 2 * np.pi)).T)
        else:
            out.append(random_cloud(1200, 1000 * seed + i, spread=float(rng.uniform(20, 90))))
    return out


def check_database(n, exclude_recent, seed, **extra):
    import tloam_b200
    cfg = sco.config(exclude_recent=exclude_recent)
    clouds = database_clouds(n, seed)
    descs = [sco.descriptor(p, cfg) for p in clouds]
    r = tloam_b200.LocalRegistration()
    r.loop_enable(**cfg, **extra)
    results = []
    for i, p in enumerate(clouds):
        r.loop_add(p)
        got = r.loop_result()
        j, s, dist, _ = sco.query(descs, i, exclude_recent)
        assert (got.query, got.candidate, got.shift) == (i, j, s), (i, got, j, s)
        assert same_bits(np.array(got.distance), np.array(dist)), (i, got.distance, dist)
        assert got.is_loop == (j >= 0 and dist < cfg["dist_threshold"])
        assert got.yaw == (sco.yaw_of(s, 60) if j >= 0 else 0.0)
        results.append(got)
    r.close()
    return results


@pytest.mark.gpu
@pytest.mark.parametrize("n,exclude_recent", [(1, 50), (51, 50), (320, 50), (40, 0), (30, 3)])
def test_gpu_search_is_the_oracles_exhaustive_search(n, exclude_recent):
    res = check_database(n, exclude_recent, seed=n)
    assert all((x.candidate >= 0) == (x.query >= exclude_recent) for x in res)
    if exclude_recent == 0:                                        # a frame (or an earlier exact copy) is its own best match
        assert all(x.candidate <= x.query and x.shift == 0 and abs(x.distance) < 1e-12 for x in res)
    if n > 100:
        assert any(x.is_loop for x in res) and any(not x.is_loop for x in res if x.candidate >= 0)


@pytest.mark.gpu
def test_gpu_revisit_in_a_ray_cast_world():
    """the route returns to frame REVISIT_OF's place with a 97 deg different heading and a 0.5 m offset: the return frame
    finds a frame of the revisit window with is_loop and the yaw within a sector of the heading difference; frames whose
    place no earlier eligible frame is near report no loop; no query ever sees one of the 50 newest frames"""
    import tloam_b200
    poses, scans = route_scans()
    r = tloam_b200.LocalRegistration()
    r.loop_enable()
    res = []
    for p in scans:
        r.loop_add(p)
        res.append(r.loop_result())
    xy = np.array([p[:2] for p in poses])
    for i, x in enumerate(res):
        assert x.query == i
        if i < 50:
            assert x.candidate == -1 and not x.is_loop
            continue
        assert 0 <= x.candidate <= i - 50
        near = np.linalg.norm(xy[:i - 49] - xy[i], axis=1).min()
        if near > 20.0:
            assert not x.is_loop, (i, x, near)
    last = res[-1]
    window = np.flatnonzero(np.linalg.norm(xy[:len(xy) - 50] - xy[-1], axis=1) < 4.0)
    assert REVISIT_OF in window and last.is_loop and last.candidate in window, (last, window)
    want = math.remainder(RETURN_YAW - poses[last.candidate][2], 2 * math.pi)   # p_cand = Rz(psi_query - psi_cand) p_query
    assert abs(math.remainder(last.yaw - want, 2 * math.pi)) <= 2 * math.pi / 60 + 1e-12, (last.yaw, want)
    print(f"revisit: frame {last.query} -> {last.candidate} shift {last.shift} yaw {math.degrees(last.yaw):.1f} deg "
          f"(true {math.degrees(want):.1f}) distance {last.distance:.4f}")
    r.close()


def process_packed(r, arr, time=None):
    from test_process_cloud import FE
    if time is None:
        return r.process_raw_scan_packed(arr, feature=FE)
    return r.process_raw_scan_packed(arr, feature=FE, deskew=True, frame_period=0.1)


@pytest.mark.gpu
def test_gpu_add_frame_reads_the_scan_the_global_map_would():
    """after process_raw_scan, _packed and _timed: loop_add_frame's descriptor is the descriptor of the scan
    global_map_append_frame appends (read back as the registered scan at pose I): raw, or corrected when timed"""
    import scipy.linalg
    import tloam_b200
    from test_deskew import XI_SEED, hat, pack_timed, scan_times
    from test_packed_scan import f32_scan
    from test_process_cloud import FE
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.loop_enable(exclude_recent=0)
    raw = with_nonfinite(synth.raw_scan(), 7)
    f = f32_scan(raw)
    arr, _ = pack_timed(f, scan_times(len(f), 5), "velodyne_xyzirt22")
    steps = [lambda: r.process_raw_scan(raw, feature=FE), lambda: process_packed(r, arr),
             lambda: r.process_raw_scan(raw, feature=FE, time=scan_times(len(raw), 6), frame_period=0.1),
             lambda: process_packed(r, arr, time=True)]
    cfg = sco.config(exclude_recent=0)
    descs = []
    for k, step in enumerate(steps):
        r.set_pose_history(np.eye(4), scipy.linalg.expm(hat(XI_SEED)))
        step()
        r.loop_add_frame()
        r.global_map_append_frame(np.eye(4))
        scan = r.registered_scan()
        got = r.loop_descriptor(k)
        assert_same_descriptor(got, sco.descriptor(scan, cfg))
        if k >= 2:                                                 # the corrected scan, not the raw one
            plain = sco.descriptor(raw if k == 2 else f.astype(np.float64), cfg)
            assert not np.array_equal(got[0], plain[0])
        descs.append(sco.descriptor(scan, cfg))
        j, s, dist, _ = sco.query(descs, k, 0)
        res = r.loop_result()
        assert (res.query, res.candidate, res.shift) == (k, j, s) and same_bits(np.array(res.distance), np.array(dist))
    r.close()


def odometry_loop(scans, loop):
    """process_raw_scan_packed -> (submap_init_frame | scan_match_predicted_async -> submap_update_frame_chained ->
    global_map_append_frame chained) -> [loop_add_frame] -> get_result"""
    import tloam_b200
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()
    if loop:
        r.loop_enable(exclude_recent=2)
    poses, sources, results = [], [], []
    for k, a in enumerate(scans):
        process_packed(r, a)
        if k == 0:
            r.submap_init_frame()
        else:
            r.scan_matching_predicted_async()
            r.submap_update_frame_chained()
            r.global_map_append_frame()
        if loop:
            r.loop_add_frame()
        if k:
            poses.append(r.get_result())
        sources.append([r.source_cloud(c) for c in range(4)])
        if loop:
            results.append(r.loop_result())
    out = dict(poses=poses, sources=sources, submap=[r.submap_cloud(c) for c in range(4)], map=r.global_map(),
               frames=r.global_map_frames(), reg=r.registered_scan(), loop=results)
    if loop:
        out["desc"] = [r.loop_descriptor(k) for k in range(r.loop_size())]
    r.close()
    return out


def assert_same_odometry(a, b):
    assert len(a["poses"]) == len(b["poses"])
    for k in range(len(a["poses"])):
        assert np.array_equal(a["poses"][k], b["poses"][k]), k
    for k in range(len(a["sources"])):
        for c in range(4):
            assert same_bits(a["sources"][k][c], b["sources"][k][c]), (k, c)
    for c in range(4):                                             # the same rows; the submap's voxel emission is unordered
        assert same_bits(sorted_rows(a["submap"][c]), sorted_rows(b["submap"][c])), c
    assert same_bits(a["map"], b["map"]) and np.array_equal(a["frames"], b["frames"]) and same_bits(a["reg"], b["reg"])


@pytest.mark.gpu
def test_gpu_odometry_is_bit_identical_with_detection_on_and_deterministic():
    from test_deskew import loop_scans
    scans = loop_scans()
    off = odometry_loop(scans, False)
    on, again = odometry_loop(scans, True), odometry_loop(scans, True)
    assert len(off["poses"]) == 6
    assert_same_odometry(on, off)
    assert_same_odometry(on, again)
    assert on["loop"] == again["loop"]
    assert all(same_bits(flat(p), flat(q)) for p, q in zip(on["desc"], again["desc"]))
    assert [x.candidate for x in on["loop"][:2]] == [-1, -1] and all(0 <= x.candidate <= x.query - 2 for x in on["loop"][2:])


@pytest.mark.gpu
def test_gpu_grown_database_gives_the_preallocated_bits():
    """capacity 1 (grows at frames 1, 2, 3, 5, 8, ...) against capacity 1024, on the same 60 clouds: results and descriptors"""
    import tloam_b200
    clouds = database_clouds(60, 7)
    runs = []
    for cap in (1, 1024):
        r = tloam_b200.LocalRegistration()
        r.loop_enable(exclude_recent=5, initial_capacity_frames=cap)
        res = []
        for p in clouds:
            r.loop_add(p)
            res.append(r.loop_result())
        runs.append((res, [flat(r.loop_descriptor(k)) for k in range(60)]))
        r.close()
    assert runs[0][0] == runs[1][0]
    assert all(same_bits(a, b) for a, b in zip(runs[0][1], runs[1][1]))


@pytest.mark.gpu
def test_gpu_loop_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    res = _lib.LoopResult()
    n = C.c_size_t(0)
    buf = np.zeros(4096 + 200)
    dp = buf.ctypes.data_as(C.POINTER(C.c_double))
    # before enable: every call NOT_READY
    assert L.tloam_b200_loop_add_frame(h) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_add(h, dp, 1) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_result(h, C.byref(res)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_size(h, C.byref(n)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_descriptor_download(h, 0, dp) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_reset(h) == _lib.ERR_NOT_READY

    def cfg(**kw):
        c = _lib.LoopConfig()
        L.tloam_b200_loop_default_config(C.byref(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    bad = [dict(n_ring=0), dict(n_sector=0), dict(n_ring=-3), dict(n_ring=64, n_sector=65), dict(n_ring=4097, n_sector=1),
           dict(max_radius=0.0), dict(max_radius=-1.0), dict(max_radius=float("nan")), dict(max_radius=float("inf")),
           dict(exclude_recent=-1), dict(lidar_height=float("nan")), dict(lidar_height=float("inf")),
           dict(dist_threshold=float("nan")), dict(dist_threshold=-float("inf"))]
    for kw in bad:
        assert L.tloam_b200_loop_enable(h, C.byref(cfg(**kw))) == _lib.ERR_INVALID_ARG, kw
    assert L.tloam_b200_loop_enable(h, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_add_frame(h) == _lib.ERR_NOT_READY               # still off
    assert L.tloam_b200_loop_enable(h, C.byref(cfg(n_ring=64, n_sector=64, exclude_recent=0))) == _lib.OK   # 4096 bins: valid
    r._loop_shape = (64, 64)
    # enabled: no frame yet
    assert L.tloam_b200_loop_add_frame(h) == _lib.ERR_NOT_READY               # no process_raw_scan yet
    assert L.tloam_b200_loop_result(h, C.byref(res)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_descriptor_download(h, 0, dp) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_add(h, None, 5) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_result(h, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_add(h, None, 0) == _lib.OK                     # an empty frame
    assert L.tloam_b200_loop_result(h, C.byref(res)) == _lib.OK and (res.query, res.candidate, res.distance) == (0, 0, 1.0)
    raw = synth.raw_scan(n_az=400)
    from test_process_cloud import FE
    r.process_raw_scan(raw, feature=FE)
    r.loop_add_frame()
    r.segment_raw_scan(raw)                                                  # the raw scan's buffer may have been reused
    assert L.tloam_b200_loop_add_frame(h) == _lib.ERR_NOT_READY
    assert r.loop_size() == 2 and r.loop_result().query == 1
    r.loop_reset()
    assert r.loop_size() == 0 and L.tloam_b200_loop_result(h, C.byref(res)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_add_frame(h) == _lib.ERR_NOT_READY
    r.loop_add(raw)
    x = r.loop_result()
    assert (x.query, x.candidate, x.shift) == (0, 0, 0) and abs(x.distance) < 1e-12
    r.loop_enable(exclude_recent=1)                                          # a second enable restarts the database
    r.loop_add(raw)
    x = r.loop_result()
    assert r.loop_size() == 1 and (x.candidate, x.shift, x.yaw, x.is_loop) == (-1, 0, 0.0, False) and x.distance == math.inf
    r.close()


@pytest.mark.gpu
def test_gpu_loop_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    from test_process_cloud import FE
    exe = build_driver("loop_driver", "front_end_b200.hpp")
    scans = [synth.raw_scan(seed=s, n_az=900) for s in range(8)]
    scans += [scans[1] @ rz(0.4).T, scans[3]]
    path = os.path.join(os.path.dirname(exe), "loop_raw.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path, "3"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [l.split() for l in res.stdout.strip().split("\n")]
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=3)
    for k, p in enumerate(scans):
        if k % 2 == 0:
            r.process_raw_scan(p, feature=FE)
            r.loop_add_frame()
        else:
            r.loop_add(p)
        x = r.loop_result()
        g = got[k]
        assert (int(g[0]), int(g[1]), int(g[2]), bool(int(g[3]))) == (x.query, x.candidate, x.shift, x.is_loop)
        assert float(g[4]) == x.yaw and float(g[5]) == x.distance
    assert int(got[-1][1]) == 3                                   # an exact repeat of frame 3
    r.close()
