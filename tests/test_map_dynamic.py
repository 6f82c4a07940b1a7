"""Dynamic-point removal for the global map (include/tloam_b200.h "Dynamic-point removal"; k_gmd_* in
libtloam_b200_gmd.so): free-space votes from every appended scan's range image, and the map without the points later scans
looked through.  tests/map_dynamic_oracle.py is the bit-for-bit numpy restatement.

CPU: the restatement against its literal transcription (NaN / Inf rows, rows on column and row boundaries, rows at the
range limits, a window that wraps), the binary-search column against the linear count, the quality on a ray-cast drive with
a passing car and a parked box, the symbols, the new library's kernels, the shim's driver.  GPU: the counters after every
append and the static map equal the restatement bit for bit (host appends with and without intensity, the chained mapping
loop), removal changes no other bit and no launch count when off, growth, status codes, correction, the shim."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import map_correct_oracle as mco
import map_dynamic_oracle as mdo
import sass_digest
import scan_context_oracle as sco
from test_global_map_intensity import same_bits

NEW_SYMBOLS = ["tloam_b200_global_map_dynamic_default_config", "tloam_b200_global_map_dynamic_enable",
               "tloam_b200_global_map_votes_download", "tloam_b200_global_map_static_download"]
KERNELS = ("k_gmd_clear", "k_gmd_bin", "k_gmd_window", "k_gmd_vote", "k_gmd_count", "k_gmd_scatter")

# the ray-cast world's 16-beam sensor (test_loop_closure.ELEV: -24 .. 2 degrees) with every beam in the middle of its row
BEAM = 26.0 / 15.0
VLP = dict(n_rows=16, fov_down=-24.0 - BEAM / 2, fov_up=2.0 + BEAM / 2, n_cols=360)
SMALL = [mdo.config(n_rows=8, fov_down=-25.0, fov_up=5.0, n_cols=24, window_rows=1, window_cols=2, min_range=1.0,
                    max_range=30.0),
         mdo.config(n_rows=5, fov_down=-10.0, fov_up=10.0, n_cols=7, window_rows=0, window_cols=0, margin_abs=0.3,
                    margin_rel=0.1, min_range=2.0, max_range=20.0),
         mdo.config(n_rows=6, fov_down=-30.0, fov_up=3.0, n_cols=40, window_rows=2, window_cols=3, min_range=1.5,
                    max_range=25.0)]


def pose_of(x, y, yaw, z=0.0):
    c, s = math.cos(yaw), math.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    T[:3, 3] = [x, y, z]
    return T


def edge_cloud(cfg, rng, n=600):
    """a seeded cloud in a sensor frame with the edge rows of the definition"""
    D, b = mdo.col_bounds(cfg), mdo.row_bounds(cfg)
    r = rng.uniform(0.7 * cfg["max_range"], 0.9 * cfg["max_range"], n)            # a far wall, and some rows anywhere
    r[::10] = rng.uniform(0.5 * cfg["min_range"], 1.2 * cfg["max_range"], len(r[::10]))
    az = rng.uniform(0, 2 * np.pi, n)
    el = rng.uniform(math.asin(b[0]) - 0.05, math.asin(b[-1]) + 0.05, n)
    p = np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), r * np.sin(el)], axis=1)
    extra = [[np.nan, 1.0, 2.0], [np.inf, 0.0, 0.0], [1.0, -np.inf, 0.0], [0.0, 0.0, np.nan],
             [cfg["min_range"], 0.0, 0.0], [cfg["max_range"], 0.0, 0.0], [-cfg["min_range"], 0.0, 0.0],
             [0.0, -cfg["max_range"], 0.0], [np.nextafter(cfg["max_range"], np.inf), 0.0, 0.0]]
    for k in range(len(D)):                                        # exactly on every column boundary: c y - s x == 0
        rr = rng.uniform(cfg["min_range"], cfg["max_range"])
        extra.append([D[k, 0] * rr, D[k, 1] * rr, 0.0])
        extra.append([D[k, 0], D[k, 1], 0.0])
    for k in range(len(b)):                                        # s == b_k exactly (z = b_k at r = 1 after the nudge)
        x = math.sqrt(max(1.0 - b[k] * b[k], 0.0)) * 5.0
        z = b[k] * 5.0
        for _ in range(200):
            s = z / math.sqrt((x * x + 0.0) + z * z)
            if s == b[k]:
                break
            z = np.nextafter(z, np.inf if s < b[k] else -np.inf)
        extra.append([x, 0.0, z])
    # around column 0 on both sides (the window wraps there)
    for a in (1e-3, -1e-3, 2 * np.pi / cfg["n_cols"] * 0.5, -2 * np.pi / cfg["n_cols"] * 0.5):
        extra.append([8.0 * math.cos(a), 8.0 * math.sin(a), -0.5])
    return np.concatenate([p, np.array(extra)])


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(len(SMALL)))
def test_oracle_matches_the_literal_transcription(k):
    cfg = SMALL[k]
    rng = np.random.default_rng(10 + k)
    scan = edge_cloud(cfg, rng, 3000)
    pose = pose_of(0.7, -0.4, 0.3, 0.1)
    # the map: the scan's rows moved by a small motion (hits), rows pulled towards the sensor (through), a fresh cloud
    fin = scan[np.isfinite(scan).all(axis=1)]
    pts = np.concatenate([mco.transform_points(pose_of(0.05, 0.02, 0.01), fin[:300]), 0.3 * fin[300:500],
                          edge_cloud(cfg, rng, 300)[:300] * 0.6])
    pts = mco.transform_points(pose, pts)
    t, h, img, win = mdo.vote_literal(pts, scan, pose, cfg)
    b, D = mdo.row_bounds(cfg), mdo.col_bounds(cfg)
    vimg = mdo.range_image(scan, cfg, b, D)
    vwin = mdo.window_image(vimg, cfg)
    assert same_bits(vimg, img)
    assert np.array_equal(np.isnan(vwin), np.isnan(win)) and same_bits(vwin[~np.isnan(vwin)], win[~np.isnan(win)])
    vt, vh = mdo.vote(pts, scan, pose, cfg)
    assert np.array_equal(vt, t) and np.array_equal(vh, h)
    assert t.sum() > 0 and h.sum() > 10 and not np.isnan(win).all()


@pytest.mark.parametrize("n_cols", [1, 2, 3, 7, 60, 360, 1024])
def test_binary_search_column_is_the_linear_count(n_cols):
    cfg = mdo.config(n_cols=n_cols, window_cols=0)
    rng = np.random.default_rng(n_cols)
    D = mdo.col_bounds(cfg)
    p = rng.normal(0, 10, (20000, 2))
    p[:50, 1] = 0.0                                                # on the half-plane split
    p[50:60] = 0.0
    on = [[D[k, 0] * s, D[k, 1] * s] for k in range(len(D)) for s in (1.0, 3.7, 1e-3)]
    p = np.concatenate([p, np.array(on).reshape(-1, 2)])
    got = mdo.columns(p[:, 0], p[:, 1], D, n_cols)
    assert np.array_equal(got, mdo.columns_linear(p[:, 0], p[:, 1], D, n_cols))
    # the linear count is scan_context_oracle.rings_sectors' sector
    xyz = np.column_stack([p, np.zeros(len(p))])
    _, _, sector = sco.rings_sectors(xyz, sco.config(n_sector=n_cols, max_radius=1e9))
    assert np.array_equal(got, sector)
    assert got.min() >= 0 and got.max() <= n_cols - 1


def test_binary_search_row_is_the_linear_count():
    cfg = mdo.config()
    b = mdo.row_bounds(cfg)
    rng = np.random.default_rng(4)
    s = np.concatenate([rng.uniform(b[0] - 0.02, b[-1] + 0.02, 20000), b, np.nextafter(b, 2), np.nextafter(b, -2)])
    row, inside = mdo.rows(s, b)
    n = cfg["n_rows"]
    want = np.array([sum(1 for k in range(1, n) if v > b[k]) for v in s])
    assert np.array_equal(inside, (s >= b[0]) & (s <= b[n]))
    assert np.array_equal(row[inside], want[inside])


# ---- quality on the ray-cast drive ------------------------------------------------------------------------------------
CAR_HALF = np.array([2.25, 0.9, 0.75])                             # a 4.5 x 1.8 x 1.5 m car
CLEARANCE = 0.2


def car_at(x, y):
    from test_loop_closure import SENSOR_Z
    return np.array([x, y, CLEARANCE + CAR_HALF[2] - SENSOR_Z])


def drive(cfg, car_of, frames):
    """the route of test_loop_closure with a box per frame (car_of(k): its centre, or None), mapped at the exact poses
    with 1 m voxels; returns (dynamic, car-labelled) per map point.  A map point is car-labelled when a row of its voxel
    lies on the box (within the 0.01 m range noise)."""
    from test_loop_closure import cast, make_world, route
    world = make_world()
    votes = mdo.Votes(cfg)
    pts, labels = np.zeros((0, 3)), np.zeros(0, dtype=bool)
    for k, (x, y, yaw) in enumerate(route()[:frames]):
        box = car_of(k)
        c, h, poles = world
        if box is not None:
            c, h = np.vstack([c, box]), np.vstack([h, CAR_HALF])
        scan = cast((c, h, poles), x, y, yaw, seed=k)
        T = pose_of(x, y, yaw)
        reg = mco.transform_points(T, scan)
        hit = np.zeros(len(reg), dtype=bool) if box is None else np.all(np.abs(reg - box) <= CAR_HALF + 0.1, axis=1)
        if k == 0:                                                 # the mapping loop appends from frame 1
            continue
        key = np.floor((reg - (reg.min(axis=0) - 0.5)) / 1.0).astype(np.int64)
        _, inv = np.unique(key, axis=0, return_inverse=True)
        inv = inv.reshape(-1)
        cnt = np.bincount(inv)
        block = np.stack([np.bincount(inv, reg[:, d]) for d in range(3)], axis=1) / cnt[:, None]
        votes.append(pts, scan, T, len(block))
        pts = np.concatenate([pts, block])
        labels = np.concatenate([labels, np.bincount(inv, hit.astype(float)) > 0])
    return mdo.dynamic(votes.through, votes.hits, cfg), labels


def test_quality_of_the_defaults_on_a_passing_car():
    """an oncoming car in the next lane along the first leg (3 m per frame), the route's first 46 frames.  The window
    keeps the ground: the row below a ground point returns closer.  Measured with the defaults (the HDL-64E's window and
    margins on the 16-beam image): 54.4 % of the car's points dynamic, so the target of 90 % is missed on this sparse
    sensor (DESIGN.md section 6 has why); 0.03 % of the static points, so the target of at most 1 % is met."""
    cfg = mdo.config(**VLP)
    dyn, car = drive(cfg, lambda k: car_at(90.0 - 3.0 * k, 3.5) if k < 40 else None, 46)
    got_car, got_static = dyn[car].mean(), dyn[~car].mean()
    print(f"car {car.sum()} points, {got_car:.3f} dynamic; static {(~car).sum()} points, {got_static:.4f} dynamic")
    assert car.sum() > 100
    assert got_car >= 0.54
    assert got_static <= 0.0015


def test_a_parked_box_that_leaves_ends_dynamic():
    """a box parked beside the first leg for the first half of the drive, then gone: the later frames carve it.
    Measured: 34.2 % of its points end dynamic (the rest sit low, where the row below returns from the ground first);
    none stays dynamic while the box is still there"""
    cfg = mdo.config(**VLP)
    box = car_at(40.0, 6.0)
    half, _ = drive(cfg, lambda k: box, 20)
    dyn, car = drive(cfg, lambda k: box if k < 20 else None, 40)
    print(f"parked box: {car.sum()} points, {dyn[car].mean():.3f} dynamic; static {dyn[~car].mean():.4f}")
    assert car.sum() > 50 and dyn[car].mean() >= 0.34 and dyn[~car].mean() <= 0.0015
    assert not half[car[:len(half)]].any()


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_gmd_library_holds_only_the_new_kernels_for_sm90a():
    """the six kernels, sm_90a only; the only DFMA are those of the correctly rounded division and square root, which
    k_gmd_bin and k_gmd_vote share (one each): the vote's own products and sums are not contracted"""
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.GMD_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.GMD_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    sass = subprocess.run([sass_digest.cuobjdump(), "-sass", build.GMD_LIB], capture_output=True, text=True, check=True).stdout
    dfma, fn = {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            fn = next(k for k in KERNELS if f"{len(k)}{k}E" in line)
            dfma[fn] = 0
        elif fn and "DFMA" in line:
            dfma[fn] += 1
    assert all(dfma[k] == 0 for k in ("k_gmd_clear", "k_gmd_window", "k_gmd_count", "k_gmd_scatter")), dfma
    assert dfma["k_gmd_vote"] == dfma["k_gmd_bin"], dfma


def test_map_dynamic_driver_compiles_warning_free():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "mock", "map_dynamic_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(root, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def ray_cast_frames(n, n_az=360, car=True):
    """(scan, pose, intensity) of the route's first n frames with the passing car"""
    from test_loop_closure import cast, make_world, route
    world = make_world()
    out = []
    for k, (x, y, yaw) in enumerate(route()[:n]):
        c, h, poles = world
        if car:
            c, h = np.vstack([c, car_at(40.0 - 3.0 * k, 3.5)]), np.vstack([h, CAR_HALF])
        scan = cast((c, h, poles), x, y, yaw, n_az=n_az, seed=k)
        if k == 3:
            scan[5] = [np.nan, 0.0, 0.0]
        out.append((scan, pose_of(x, y, yaw), np.random.default_rng(k).uniform(0, 100, len(scan))))
    return out


def host_run(frames, dynamic, cfg=VLP, capacity=1 << 20, intensity=True, per_append=True):
    """host appends; per append the map rows before it and (with removal) the counters after it"""
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=capacity)
    if dynamic:
        r.global_map_dynamic_enable(**cfg)
    maps, votes, regs, launches = [], [], [], []
    for scan, pose, inten in frames:
        if per_append:
            maps.append(r.global_map())
        n0 = r.launch_count()
        r.global_map_append(scan, pose, intensity=inten if intensity else None)
        launches.append(r.launch_count() - n0)
        regs.append(r.registered_scan())
        if dynamic and per_append:
            votes.append(r.global_map_votes())
    out = dict(map=r.global_map(), frames=r.global_map_frames(), regs=regs, launches=launches, maps=maps, votes=votes,
               growths=r.global_map_capacity()[1])
    out["intensity"] = r.global_map_intensity() if r.global_map_has_intensity() else None
    if dynamic:
        out["final"] = r.global_map_votes()
        out["static"] = r.global_map_static()
    r.close()
    return out


def restate(frames, maps, cfg):
    """the restatement's counters after every append, from the map rows the device had before each append"""
    c = mdo.config(**cfg)
    t, h = np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32)
    out = []
    for k, (scan, pose, _) in enumerate(frames):
        m = maps[k]
        t = np.concatenate([t, np.zeros(len(m) - len(t), dtype=np.uint32)])
        h = np.concatenate([h, np.zeros(len(m) - len(h), dtype=np.uint32)])
        if len(m):
            dt, dh = mdo.vote(m, scan, pose, c)
            t, h = t + dt, h + dh
        out.append((t.copy(), h.copy()))
    return out


def assert_votes(got, want):
    for k, ((gt, gh), (wt, wh)) in enumerate(zip(got, want)):
        n = len(wt)
        assert np.array_equal(gt[:n], wt) and np.array_equal(gh[:n], wh), (k, np.nonzero(gt[:n] != wt)[0][:5])
        assert not gt[n:].any() and not gh[n:].any(), k


@pytest.mark.gpu
@pytest.mark.parametrize("intensity", [True, False])
def test_gpu_host_appends_are_the_restatement(intensity):
    """the counters after every host append and the static map (xyz and intensity) equal the restatement bit for bit;
    the map, frame table, intensity and registered scans are the bits of removal off; four more launches per append"""
    frames = ray_cast_frames(14)
    on, off = host_run(frames, True, intensity=intensity), host_run(frames, False, intensity=intensity)
    assert same_bits(on["map"], off["map"]) and np.array_equal(on["frames"], off["frames"])
    assert all(same_bits(a, b) for a, b in zip(on["regs"], off["regs"]))
    assert (on["intensity"] is None) == (not intensity)
    if intensity:
        assert same_bits(on["intensity"], off["intensity"])
    assert [a - b for a, b in zip(on["launches"], off["launches"])] == [4] * len(frames)
    want = restate(frames, on["maps"], VLP)
    assert_votes(on["votes"], want)
    t, h = on["final"]
    assert_votes([(t, h)], want[-1:])
    xyz, inten = mdo.static_map(on["map"], on["intensity"], t, h, mdo.config(**VLP))
    assert same_bits(on["static"][0], xyz)
    if intensity:
        assert same_bits(on["static"][1], inten)
    else:
        assert on["static"][1] is None
    dyn = mdo.dynamic(t, h, mdo.config(**VLP))
    print(f"{len(t)} points, {int(dyn.sum())} dynamic, max through {t.max()}, max hits {h.max()}")
    assert 0 < dyn.sum() < len(t) // 10


@pytest.mark.gpu
def test_gpu_removal_off_keeps_the_launch_counts():
    """a handle whose removal was turned off by enable_global_map launches what a handle that never had it launches"""
    import tloam_b200
    frames = ray_cast_frames(4)
    plain = host_run(frames, False, per_append=False)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_dynamic_enable(**VLP)
    r.enable_global_map()
    launches = []
    for scan, pose, inten in frames:
        n0 = r.launch_count()
        r.global_map_append(scan, pose, intensity=inten)
        launches.append(r.launch_count() - n0)
    assert launches == plain["launches"] and same_bits(r.global_map(), plain["map"])
    with pytest.raises(tloam_b200.RegistrationError):
        r.global_map_votes()
    r.close()


@pytest.mark.gpu
def test_gpu_chained_mapping_loop_is_the_restatement():
    """process_raw_scan -> scan_match_predicted_async -> submap_update_frame_chained -> global_map_append_frame chained:
    the counters after every append equal the restatement at get_result's poses; the odometry, the map and the registered
    scan are the bits of removal off"""
    import tloam_b200
    from test_global_map import with_nonfinite
    from test_process_cloud import FE, moved
    from tloam_b200 import synth
    scan0 = synth.raw_scan()                                       # test_deskew.loop_scans' drive, in FP64
    scans = [with_nonfinite(scan0, 90)] + [with_nonfinite(moved(scan0, np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k]),
                                                                100 + k), 200 + k) for k in range(1, 8)]
    frames = [(s, None, None) for s in scans]
    cfg = dict(n_rows=64, fov_down=-25.0, fov_up=3.0, n_cols=900, min_range=2.0)

    def run(dynamic):
        r = tloam_b200.LocalRegistration(fitness_thres=0.3)
        r.enable_global_map()
        if dynamic:
            r.global_map_dynamic_enable(**cfg)
        poses, maps, votes = [], [], []
        for k, (scan, _, _) in enumerate(frames):
            r.process_raw_scan(scan, feature=FE)
            if k == 0:
                r.submap_init_frame()
                continue
            r.scan_matching_predicted_async()
            r.submap_update_frame_chained()
            maps.append(r.global_map())
            r.global_map_append_frame()
            poses.append(r.get_result())
            if dynamic:
                votes.append(r.global_map_votes())
        out = dict(poses=poses, maps=maps, votes=votes, map=r.global_map(), frames=r.global_map_frames(),
                   reg=r.registered_scan())
        if dynamic:
            out["static"] = r.global_map_static()
        r.close()
        return out

    on, off = run(True), run(False)
    assert all(np.array_equal(a, b) for a, b in zip(on["poses"], off["poses"]))
    assert same_bits(on["map"], off["map"]) and np.array_equal(on["frames"], off["frames"]) and same_bits(on["reg"], off["reg"])
    fr = [(frames[k][0], on["poses"][k - 1], None) for k in range(1, len(frames))]
    want = restate(fr, on["maps"], cfg)
    assert_votes(on["votes"], want)
    t, h = on["votes"][-1]
    print(f"chained: {len(t)} points, through {int(t.sum())}, hits {int(h.sum())}")
    assert h.sum() > 0
    assert same_bits(on["static"][0], mdo.static_map(on["map"], None, t, h, mdo.config(**cfg))[0])


@pytest.mark.gpu
def test_gpu_grown_map_gives_the_preallocated_counters():
    frames = ray_cast_frames(10)
    grown, pre = host_run(frames, True, capacity=1, per_append=False), host_run(frames, True, per_append=False)
    assert grown["growths"] > 0
    assert same_bits(grown["map"], pre["map"])
    for a, b in zip(grown["final"], pre["final"]):
        assert np.array_equal(a, b)
    assert same_bits(grown["static"][0], pre["static"][0]) and same_bits(grown["static"][1], pre["static"][1])


@pytest.mark.gpu
def test_gpu_votes_after_a_correction_see_the_moved_blocks():
    """with correction tracking: appends after global_map_correct vote at P_f = M O_f against the moved blocks, as the
    restatement composed with map_correct_oracle says; the counters of the moved blocks are kept"""
    import tloam_b200
    from test_pose_graph import loop_result
    import pose_graph_oracle as pgo
    frames = ray_cast_frames(10)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_correction_enable()
    r.global_map_dynamic_enable(**VLP)
    r.pose_graph_enable()
    v = mdo.Votes(mdo.config(**VLP))
    O = []
    for k, (scan, pose, inten) in enumerate(frames[:6]):
        before = r.global_map()
        r.global_map_append(scan, pose, intensity=inten)
        r.pose_graph_add_node(pose)
        O.append(pose)
        v.append(before, scan, pose, len(r.global_map()) - len(before))
    r.pose_graph_add_loop(loop_result(1, 5, pgo.inv_mul(O[1], O[5]) @ pgo.exp4([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(6))
    moved = r.global_map()
    t0, h0 = r.global_map_votes()
    assert np.array_equal(t0, v.through) and np.array_equal(h0, v.hits)
    M = r.pose_graph_correction()
    assert not same_bits(M, np.eye(4))
    for scan, pose, inten in frames[6:]:
        before = r.global_map()
        r.global_map_append(scan, pose, intensity=inten)
        v.append(before, scan, mco.append_pose(M, pose), len(r.global_map()) - len(before))
    assert same_bits(r.global_map(0, len(moved)), moved)
    t, h = r.global_map_votes()
    assert np.array_equal(t, v.through) and np.array_equal(h, v.hits)
    r.close()


@pytest.mark.gpu
def test_gpu_map_dynamic_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.GlobalMapDynamicConfig()
    L.tloam_b200_global_map_dynamic_default_config(C.byref(cfg))
    assert (cfg.n_rows, cfg.n_cols, cfg.window_rows, cfg.window_cols, cfg.min_through) == (64, 1024, 1, 2, 3)
    assert (cfg.fov_up, cfg.fov_down, cfg.margin_abs, cfg.margin_rel, cfg.min_range, cfg.max_range) == \
        (2.0, -24.9, 1.0, 0.02, 3.0, 60.0)
    u = np.zeros(4, dtype=np.uint32)
    up = u.ctypes.data_as(C.POINTER(C.c_uint))
    n = C.c_size_t(7)
    assert L.tloam_b200_global_map_dynamic_enable(None, C.byref(cfg)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_dynamic_enable(h, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_dynamic_enable(h, C.byref(cfg)) == _lib.ERR_NOT_READY           # mapping off
    assert L.tloam_b200_global_map_votes_download(h, 0, 0, up, up) == _lib.ERR_NOT_READY
    assert L.tloam_b200_global_map_static_download(h, None, None, 0, C.byref(n)) == _lib.ERR_NOT_READY
    r.enable_global_map()
    assert L.tloam_b200_global_map_votes_download(h, 0, 0, up, up) == _lib.ERR_NOT_READY          # removal off
    assert L.tloam_b200_global_map_static_download(h, None, None, 0, C.byref(n)) == _lib.ERR_NOT_READY
    for field, bad in (("n_rows", 0), ("n_cols", 0), ("fov_up", -30.0), ("fov_down", -91.0), ("fov_up", float("nan")),
                       ("window_rows", 64), ("window_rows", -1), ("window_cols", 512), ("margin_abs", -1.0),
                       ("margin_rel", float("inf")), ("min_range", 0.0), ("max_range", 2.0), ("min_through", 0)):
        c = _lib.GlobalMapDynamicConfig()
        L.tloam_b200_global_map_dynamic_default_config(C.byref(c))
        setattr(c, field, bad)
        assert L.tloam_b200_global_map_dynamic_enable(h, C.byref(c)) == _lib.ERR_INVALID_ARG, (field, bad)
    frames = ray_cast_frames(3)
    r.global_map_append(frames[0][0], frames[0][1])
    assert L.tloam_b200_global_map_dynamic_enable(h, C.byref(cfg)) == _lib.ERR_NOT_READY           # not empty
    r.reset_global_map()
    r.global_map_dynamic_enable(**VLP)
    assert L.tloam_b200_global_map_static_download(h, None, None, 0, C.byref(n)) == _lib.OK and n.value == 0
    for scan, pose, _ in frames:
        r.global_map_append(scan, pose)
    npts = r.global_map_size()[0]
    t, hh = r.global_map_votes()
    assert hh.any()
    assert L.tloam_b200_global_map_votes_download(h, npts, 1, up, up) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_votes_download(h, npts, 0, up, up) == _lib.OK
    assert L.tloam_b200_global_map_votes_download(h, 2, 2, None, None) == _lib.OK
    n = C.c_size_t(0)
    assert L.tloam_b200_global_map_static_download(h, None, None, 0, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert n.value == len(r.global_map_static()[0]) > 0
    r.reset_global_map()                                           # zeroes the counters, keeps removal on
    assert r.global_map_votes()[0].shape == (0,)
    r.global_map_append(frames[0][0], frames[0][1])
    t, hh = r.global_map_votes()
    assert not t.any() and not hh.any()
    r.enable_global_map()                                          # turns it off
    assert L.tloam_b200_global_map_votes_download(h, 0, 0, up, up) == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_map_dynamic_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("map_dynamic_driver", "front_end_b200.hpp")
    frames = ray_cast_frames(8)
    path = os.path.join(os.path.dirname(exe), "map_dynamic_raw.bin")
    out_path = os.path.join(os.path.dirname(exe), "map_dynamic_out.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(frames)))
        for p, T, inten in frames:
            fh.write(np.ascontiguousarray(T.ravel(order="F")).tobytes() + struct.pack("Q", len(p)))
            fh.write(np.ascontiguousarray(p, dtype=np.float64).tobytes() + np.ascontiguousarray(inten).tobytes())
    res = subprocess.run([exe, path, out_path, str(VLP["n_rows"]), str(VLP["n_cols"]), repr(VLP["fov_down"]),
                          repr(VLP["fov_up"])], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    n_pts, n_static = (int(s) for s in res.stdout.split())
    py = host_run(frames, True, per_append=False)
    with open(out_path, "rb") as fh:
        blob = fh.read()
    t = np.frombuffer(blob, dtype=np.uint32, count=n_pts)
    hh = np.frombuffer(blob, dtype=np.uint32, count=n_pts, offset=4 * n_pts)
    o = 8 * n_pts
    (ns,) = struct.unpack_from("Q", blob, o)
    xyz = np.frombuffer(blob, dtype=np.float64, count=3 * ns, offset=o + 8).reshape(-1, 3)
    o += 8 + 24 * ns
    (ni,) = struct.unpack_from("Q", blob, o)
    inten = np.frombuffer(blob, dtype=np.float64, count=ni, offset=o + 8)
    assert n_pts == len(py["map"]) and ns == n_static == len(py["static"][0])
    assert np.array_equal(t, py["final"][0]) and np.array_equal(hh, py["final"][1])
    assert same_bits(xyz, py["static"][0]) and same_bits(inten, py["static"][1])
