"""Localization in a prior map (include/tloam_b200.h "Localization in a prior map"; k_loc_* in libtloam_b200_loc.so): a scan
registered point to plane against a grid-indexed map with a normal per row.  tests/localize_oracle.py is the CPU
restatement.

CPU: the restatement's grid search against brute force and a k-d tree (rows on cell faces, duplicates, radii at cell
multiples, empty neighbourhoods), its normals against the submap verification's, recovery of a known transform, the
prediction, the symbols and the library's kernels.  GPU: the cell table, the normals, the query, every pass's matches and
the result against the restatement; a map of more than 1 M rows; the merged map; the prediction; the status codes."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import localize_oracle as lo
import loop_verify_oracle as lvo
import loop_verify_submap_oracle as lso
import sass_digest
from test_global_map_intensity import same_bits
from test_loop_verify import apply4, se3, structured_cloud

NEW_SYMBOLS = ["tloam_b200_localize_default_config", "tloam_b200_localize_enable", "tloam_b200_localize_set_map",
               "tloam_b200_localize_set_map_merged", "tloam_b200_localize_frame", "tloam_b200_localize",
               "tloam_b200_localize_matches", "tloam_b200_localize_query", "tloam_b200_localize_map_normals",
               "tloam_b200_localize_cells"]
KERNELS = ("k_loc_bounds", "k_loc_keys", "k_gmm_hist", "k_gmm_offsets", "k_gmm_scatter", "k_gmm_head_count",
           "k_gmm_head_scatter", "k_loc_cells", "k_loc_normals", "k_loc_predict", "k_loc_match", "k_loc_reduce", "k_loc_step",
           "k_loc_final")


def brute(P, M, r):
    """the exhaustive scan limited to d2 <= r * r, by (d2, index)"""
    idx, d2 = np.full(len(P), -1, dtype=np.int64), np.full(len(P), np.inf)
    for i, p in enumerate(P):
        d = lso._d2(p[None, :], M)
        ok = np.flatnonzero(d <= r * r)
        if len(ok):
            j = ok[np.lexsort((ok, d[ok]))[0]]
            idx[i], d2[i] = j, d[j]
    return idx, d2


def face_cloud(seed=0):
    """rows on cell faces (integer and half-integer coordinates), exact duplicates and a random part"""
    rng = np.random.default_rng(seed)
    a = rng.integers(-4, 5, (600, 3)).astype(np.float64)
    b = rng.integers(-8, 9, (300, 3)).astype(np.float64) * 0.5
    c = rng.uniform(-4, 4, (600, 3))
    M = np.vstack([a, b, c, a[:50], c[:50]])
    return M


# ---- CPU: the restatement ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("r", [0.5, 1.0, 2.0, 3.0, 0.37])
def test_oracle_grid_search_is_the_exhaustive_scan(r):
    M = face_cloud()
    g = lo.grid(M, 1.0)
    rng = np.random.default_rng(1)
    P = np.vstack([M[::7], M[::11] + rng.choice([-r, r, 0.0], (len(M[::11]), 3)), rng.uniform(-6, 6, (300, 3)),
                   [[50.0, 50.0, 50.0], [-20.0, 0.0, 0.0]]])                 # the last two: empty neighbourhoods
    gi, gd = lo.search(g, P, r)
    bi, bd = brute(P, M, r)
    assert np.array_equal(gi, bi) and same_bits(gd, bd)
    assert (gi[-2:] == -1).all() and np.isinf(gd[-2:]).all()
    dup = np.flatnonzero((gi >= 1500) & (gi < 1550))                         # a duplicate never wins over its original
    assert len(dup) == 0
    dist, _ = cKDTree(M).query(P)
    hit = gi >= 0
    assert np.allclose(np.sqrt(gd[hit]), dist[hit], rtol=0, atol=1e-12) and (dist[~hit] > r * (1 - 1e-12)).all()


def test_oracle_grid_table_orders_rows_by_cell_then_row():
    M = face_cloud(2)
    g = lo.grid(M, 0.5)
    cells = np.floor((M - M.min(0)) / 0.5).astype(np.int64)
    order = np.lexsort((np.arange(len(M)), cells[:, 2], cells[:, 1], cells[:, 0]))
    assert np.array_equal(g["srow"], order)
    assert len(g["ckey"]) == len(np.unique(cells, axis=0)) and g["cstart"][-1] == len(M)
    with pytest.raises(ValueError):
        lo.grid(np.array([[0.0, 0.0, 0.0], [2.0 ** 21, 0.0, 0.0]]), 1.0)
    with pytest.raises(ValueError):
        lo.grid(np.array([[0.0, np.nan, 0.0]]), 1.0)


def test_oracle_normals_are_the_submap_verifications():
    M = np.vstack([structured_cloud(5), face_cloud(3)])
    cfg = lo.config()
    nrm, valid, cnt = lo.normals(lo.grid(M, 1.0), cfg)
    n2, v2, c2, _, _ = lso.normals(M, lso.config())
    assert np.array_equal(cnt, c2) and np.array_equal(valid, v2) and same_bits(nrm, n2)
    nrm3, valid3, cnt3 = lo.normals(lo.grid(M, 0.4), cfg)                  # a finer grid: the same neighbourhoods
    assert np.array_equal(cnt3, c2) and same_bits(nrm3, n2)


def test_oracle_recovers_a_noise_free_transform():
    M = structured_cloud(3)
    T_true = se3([1.5, -0.8, 0.1, 0.01, -0.02, 0.35])
    Q = apply4(np.linalg.inv(T_true), M[::3])
    guess = T_true @ se3([0.6, -0.5, 0.05, 0.0, 0.0, math.radians(2.0)])
    cfg = lo.config()
    g = lo.grid(M, cfg["cell"])
    nrm, valid, _ = lo.normals(g, cfg)
    r = lo.run(Q, g, nrm, valid, guess, cfg)
    err = np.abs(r["T"] - T_true).max()
    assert r["termination"] == lo.CONVERGED and r["accepted"] and err < 1e-9, (r["termination"], err)
    assert r["fitness"] < 1e-18 and len(r["passes"]) == r["iterations"] + 1
    far = lo.run(Q + 500.0, g, nrm, valid, np.eye(4), cfg)
    assert far["termination"] == lo.FEW_INLIERS and not far["accepted"] and far["fitness"] == cfg["corr_dist_coarse"] ** 2
    assert lo.run(np.zeros((0, 3)), g, nrm, valid, guess, cfg)["termination"] == lo.EMPTY


def test_oracle_prediction_is_dead_reckoning_in_the_map_frame():
    L = se3([10.0, -3.0, 0.2, 0.01, 0.02, 0.7])
    Op, On = se3([1.0, 2.0, 0.0, 0.0, 0.0, 0.3]), se3([2.5, 2.4, 0.01, 0.001, -0.002, 0.36])
    G = lo.predict(L, Op, On)
    assert np.abs(G - L @ np.linalg.inv(Op) @ On).max() < 1e-12 and np.array_equal(G[3], [0, 0, 0, 1])
    assert same_bits(lo.predict(L, On, On)[:3, 3], L[:3, 3]) or np.abs(lo.predict(L, On, On) - L).max() < 1e-14
    M = lo.map_odom(G, On)
    assert np.abs(M - G @ np.linalg.inv(On)).max() < 1e-12


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)
    c = _lib.LocalizeConfig()
    _lib.load().tloam_b200_localize_default_config(C.byref(c))
    assert {k: getattr(c, k) for k, _ in c._fields_} == lo.config()


def test_loc_library_holds_only_its_kernels_for_sm90a_and_normals_and_match_do_not_spill():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.LOC_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.LOC_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.LOC_LIB], capture_output=True, text=True, check=True).stdout
    lines = res.splitlines()
    for k in ("k_loc_normals", "k_loc_match"):
        usage = [lines[i + 1] for i, l in enumerate(lines) if f"{len(k)}{k}E" in l]
        assert len(usage) == 1 and " LOCAL:0 " in usage[0] and " STACK:0 " in usage[0], (k, usage)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def handle(**cfg):
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.localize_enable(**cfg)
    return r


def check_index(r, M, cfg, name):
    g = lo.grid(M, cfg["cell"])
    rows, keys, starts = r.localize_cells(len(M))
    assert np.array_equal(rows, g["srow"]) and np.array_equal(keys, g["ckey"]) and np.array_equal(starts, g["cstart"]), name
    nrm, valid, cnt = lo.normals(g, cfg)
    gn, gv, gc = r.localize_map_normals()
    assert np.array_equal(gc, cnt) and np.array_equal(gv, valid), name
    assert same_bits(gn, nrm), name
    return g, nrm, valid


def check_run(r, got, Q, g, nrm, valid, guess, cfg, name):
    want = lo.run(Q, g, nrm, valid, guess, cfg)
    assert (got.iterations, got.termination, got.inliers, got.accepted) == \
        (want["iterations"], want["termination"], want["inliers"], want["accepted"]), (name, got, want)
    if want["termination"] == lo.EMPTY:
        assert got.fitness == math.inf and same_bits(got.T, guess), name
        return want
    assert np.abs(got.T - want["T"]).max() < 1e-9, (name, np.abs(got.T - want["T"]).max())
    for a, b in ((got.fitness, want["fitness"]), (got.rmse, want["rmse"])):
        assert a == b or abs(a - b) <= 1e-9 * abs(b) + 1e-15, (name, a, b)
    assert len(want["passes"]) == got.iterations + 1
    for k, (idx, d2) in enumerate(want["passes"]):
        gi, gd = r.localize_matches(k)
        assert np.array_equal(gi, idx), (name, k)
        if k == 0:
            assert same_bits(gd, d2), name
    print(f"localize {name}: {len(Q)} query rows, {want['iterations']} iterations, termination {want['termination']}, "
          f"fitness {want['fitness']:.4g}")
    return want


@pytest.mark.gpu
def test_gpu_index_normals_and_runs_match_the_restatement():
    from oracle import pyoracle
    pyoracle.build()
    cfg = lo.config()
    M = np.vstack([structured_cloud(3), face_cloud(4) * 3.0])
    r = handle()
    r.localize_set_map(M)
    g, nrm, valid = check_index(r, M, cfg, "structured")
    T_true = se3([1.5, -0.8, 0.1, 0.01, -0.02, 0.35])
    rng = np.random.default_rng(7)
    scan = apply4(np.linalg.inv(T_true), M[::2]) + rng.normal(0, 0.01, (len(M[::2]), 3))
    scan[::97] = np.nan
    for k, guess in enumerate([T_true @ se3([0.6, -0.5, 0.05, 0.0, 0.0, math.radians(2.0)]), T_true,
                               T_true @ se3([-1.0, 0.8, 0.0, 0.0, 0.0, math.radians(-4.0)])]):
        got = r.localize(scan, guess)
        Q = r.localize_query()
        want_q = lvo.keyframe(pyoracle, scan, cfg["voxel"])     # the loop keyframe's down-sample, up to its rounding
        assert Q.shape == want_q.shape and np.abs(np.sort(Q, axis=0) - np.sort(want_q, axis=0)).max() < 1e-9, k
        want = check_run(r, got, Q, g, nrm, valid, guess, cfg, f"guess {k}")
        assert same_bits(got.T_map_odom, lo.map_odom(got.T, np.eye(4))) and same_bits(got.guess, guess)
        if k < 2:
            assert want["accepted"] and np.abs(got.T - T_true).max() < 0.02
    got = r.localize(np.zeros((0, 3)), T_true)
    assert got.termination == lo.EMPTY and not got.accepted and got.n_query_points == 0
    got = r.localize(scan + 500.0, np.eye(4))
    check_run(r, got, r.localize_query(), g, nrm, valid, np.eye(4), cfg, "off the map")
    assert got.termination == lo.FEW_INLIERS


@pytest.mark.gpu
def test_gpu_index_of_the_ray_cast_map():
    from oracle import pyoracle
    from test_loop_closure import cast, make_world, route
    from test_loop_verify import pose4
    pyoracle.build()
    world = make_world()
    first = np.vstack([apply4(pose4(route()[k]), cast(world, *route()[k], seed=k)) for k in range(0, 70, 2)])
    M = lvo.keyframe(pyoracle, first, 0.5)
    r = handle()
    r.localize_set_map(M)
    check_index(r, M, lo.config(), "ray-cast")
    r.close()


@pytest.mark.gpu
def test_gpu_prediction_follows_the_previous_result():
    cfg = lo.config()
    M = structured_cloud(3)
    r = handle()
    r.localize_set_map(M)
    with pytest.raises(Exception):
        r.localize(M[::3])                                          # no guess and no previous localization: NOT_READY
    T_true = se3([1.5, -0.8, 0.1, 0.01, -0.02, 0.35])
    scan = apply4(np.linalg.inv(T_true), M[::3])
    first = r.localize(scan, T_true @ se3([0.3, 0.2, 0.0, 0.0, 0.0, 0.01]))
    second = r.localize(scan)                                       # no frame registered: O_now = O_prev = I
    assert same_bits(second.guess, lo.predict(first.T if first.accepted else first.guess, np.eye(4), np.eye(4)))
    bad = r.localize(scan + 500.0)                                  # rejected: the next guess is this one's guess
    assert not bad.accepted
    third = r.localize(scan)
    assert same_bits(third.guess, lo.predict(bad.guess, np.eye(4), np.eye(4)))


@pytest.mark.gpu
def test_gpu_a_map_of_more_than_a_million_rows():
    cfg = lo.config()
    rng = np.random.default_rng(11)
    n = 1_100_000
    ab = rng.uniform(0, 600, (n, 2))
    M = np.column_stack([ab, 0.3 * np.sin(ab[:, 0] / 7.0) + 0.01 * rng.normal(size=n)])
    r = handle()
    r.localize_set_map(M)
    rows, keys, starts = r.localize_cells(n)
    g = lo.grid(M, cfg["cell"])
    assert np.array_equal(rows, g["srow"]) and np.array_equal(keys, g["ckey"]) and np.array_equal(starts, g["cstart"])
    gn, gv, gc = r.localize_map_normals()
    sub = np.sort(rng.choice(n, 20000, replace=False))              # the restatement on a sample of rows, by the same grid
    nrm, valid, cnt = lo.normals(g, cfg, sub)
    assert np.array_equal(gc[sub], cnt) and np.array_equal(gv[sub], valid) and same_bits(gn[sub], nrm)
    print(f"1.1 M rows: {len(keys)} cells, {gv.mean():.3f} valid, {gc.mean():.1f} neighbours per row")


@pytest.mark.gpu
def test_gpu_set_map_merged_is_set_map_of_the_downloaded_merge():
    cfg = lo.config()
    r = handle()
    r.enable_global_map(voxel=0.3)
    for k in range(3):
        r.global_map_append(structured_cloud(20 + k), pose=se3([0.5 * k, 0.0, 0.0, 0.0, 0.0, 0.05 * k]))
    xyz, _ = r.global_map_merged(0.3)
    r.localize_set_map_merged()
    a = r.localize_cells(len(xyz)), r.localize_map_normals()
    r.localize_set_map(xyz)
    b = r.localize_cells(len(xyz)), r.localize_map_normals()
    for u, v in zip(a[0] + a[1], b[0] + b[1]):
        assert same_bits(np.asarray(u, dtype=np.float64), np.asarray(v, dtype=np.float64))
    check_index(r, xyz, cfg, "merged")


@pytest.mark.gpu
def test_gpu_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    res = _lib.LocalizeResult()
    assert L.tloam_b200_localize(h, None, 0, None, C.byref(res)) == _lib.ERR_NOT_READY        # off
    assert L.tloam_b200_localize_set_map_merged(h) == _lib.ERR_NOT_READY
    cfg = _lib.LocalizeConfig()
    L.tloam_b200_localize_default_config(C.byref(cfg))
    cfg.corr_dist_coarse = 3.5
    assert L.tloam_b200_localize_enable(h, C.byref(cfg)) == _lib.ERR_INVALID_ARG
    r.localize_enable()
    assert L.tloam_b200_localize(h, None, 0, None, C.byref(res)) == _lib.ERR_NOT_READY        # no map
    assert L.tloam_b200_localize_set_map_merged(h) == _lib.ERR_NOT_READY                      # no merge
    bad = np.array([[0.0, 0.0, 0.0], [1.0, np.inf, 0.0]])
    assert L.tloam_b200_localize_set_map(h, bad.ctypes.data_as(C.POINTER(C.c_double)), 2) == _lib.ERR_INVALID_ARG
    wide = np.array([[0.0, 0.0, 0.0], [2.0 ** 21 + 1.0, 0.0, 0.0]])
    assert L.tloam_b200_localize_set_map(h, wide.ctypes.data_as(C.POINTER(C.c_double)), 2) == _lib.ERR_VOXEL_RANGE
    r.localize_set_map(structured_cloud(3))
    shear = np.eye(4)
    shear[0, 1] = 0.5
    g = shear.ravel(order="F").copy()
    assert L.tloam_b200_localize(h, None, 0, g.ctypes.data_as(C.POINTER(C.c_double)), C.byref(res)) == _lib.ERR_BAD_POSE
    assert L.tloam_b200_localize(h, None, 0, None, C.byref(res)) == _lib.ERR_NOT_READY        # the first needs a guess
    assert r.localize(np.zeros((0, 3)), np.eye(4)).termination == lo.EMPTY
    r.localize_set_map(np.zeros((0, 3)))
    assert r.localize(structured_cloud(3), np.eye(4)).termination == lo.EMPTY                # an empty map


# ---- CPU: a second drive through the ray-cast world, against the map of the first -----------------------------------------
# frames 0 .. 49 of test_loop_closure's route (a straight leg and the turn into the second), driven again 0.6 m to the left
# with new noise and an odometry that drifts 2 cm, 0.5 cm and 0.1 deg per frame; every frame after the first from the
# prediction.  DESIGN.md section 4c has the errors and the fitness values this fixes.
SECOND_DRIVE = range(50)
ACCURACY_BOUND = (0.05, math.radians(0.1))


def second_drive(cfg):
    """(per frame: the result, the true pose, the odometry pose) of the second drive, and the prior map"""
    from oracle import pyoracle
    from test_loop_closure import cast, make_world, route
    from test_loop_verify import pose4
    pyoracle.build()
    world = make_world()
    P = [pose4(p) for p in route()]
    first = np.vstack([apply4(P[k], cast(world, *route()[k], seed=k)) for k in SECOND_DRIVE])
    prior = lvo.keyframe(pyoracle, first, 0.5)                      # the first drive's map, merged at 0.5 m
    g = lo.grid(prior, cfg["cell"])
    nrm, valid, _ = lo.normals(g, cfg)
    side = np.eye(4)
    side[1, 3] = 0.6
    truth, odom, out = [], [], []
    drift = se3([0.02, 0.005, 0.0, 0.0, 0.0, math.radians(0.1)])
    for k in SECOND_DRIVE:
        Pk = P[k] @ side
        x, y, yaw = Pk[0, 3], Pk[1, 3], math.atan2(Pk[1, 0], Pk[0, 0])
        scan = cast(world, x, y, yaw, seed=1000 + k)
        O = np.eye(4) if k == 0 else odom[-1] @ np.linalg.inv(truth[-1]) @ Pk @ drift
        if k == 0:
            G = Pk @ se3([0.4, -0.3, 0.0, 0.0, 0.0, math.radians(2.0)])
        else:
            G = lo.predict(out[-1]["T"] if out[-1]["accepted"] else out[-1]["G"], odom[-1], O)
        r = lo.run(lvo.keyframe(pyoracle, scan, cfg["voxel"]), g, nrm, valid, G, cfg)
        r["G"] = G
        truth.append(Pk)
        odom.append(O)
        out.append(r)
    return out, truth, odom, prior


def test_oracle_localizes_a_second_drive_against_the_first_drives_map():
    cfg = lo.config()
    out, truth, odom, prior = second_drive(cfg)
    errs = [lvo.relative_error(r["T"], P) for r, P in zip(out, truth)]
    acc = [r["accepted"] for r in out]
    dead = lvo.relative_error(odom[-1] @ np.linalg.inv(odom[0]) @ truth[0], truth[-1])
    print(f"second drive: {len(prior)} map rows, {sum(acc)} / {len(out)} accepted, max error of an accepted frame "
          f"{max(e[0] for e, a in zip(errs, acc) if a):.4f} m {math.degrees(max(e[1] for e, a in zip(errs, acc) if a)):.4f} deg; "
          f"fitness {min(r['fitness'] for r in out):.4f} .. {max(r['fitness'] for r in out):.4f}; "
          f"iterations {max(r['iterations'] for r in out)}; odometry alone ends {dead[0]:.3f} m {math.degrees(dead[1]):.3f} deg off")
    assert sum(acc) >= 0.9 * len(out)
    assert all(e[0] < ACCURACY_BOUND[0] and e[1] < ACCURACY_BOUND[1] for e, a in zip(errs, acc) if a)
    assert dead[0] > 10 * ACCURACY_BOUND[0]


CHAINED_BOUND = (0.1, math.radians(0.2))


@pytest.mark.gpu
def test_gpu_chained_loop_localizes_and_moves_nothing_else():
    """process_raw_scan_packed -> (submap_init_frame | scan_match_predicted_async -> submap_update_frame_chained ->
    global_map_append_frame) [-> localize_frame(NULL)]: against the merged map of a first session over the same scans,
    every guess is the restatement's prediction from the downloaded poses and T_map_odom its product, bit for bit, and every
    accepted frame is within CHAINED_BOUND of the first session's odometry pose (not a ground truth: the synthetic HDL-64E
    frames of test_deskew.loop_scans, whose first-session odometry is itself a few centimetres off).  The odometry, the sources, the submap, the global
    map, the registered scan and the launch counts of those calls are those of a handle that never enabled localization,
    with localization enabled and loaded but unused, and with it running."""
    import tloam_b200
    from test_deskew import loop_scans
    from test_loop_closure import assert_same_odometry, process_packed
    scans = loop_scans()
    runs = {}
    prior = None
    for mode in ("off", "enabled", "running"):
        r = tloam_b200.LocalRegistration(fitness_thres=0.3)
        r.enable_global_map(voxel=0.5)
        if mode != "off":
            r.localize_enable()
            r.localize_set_map(prior)
        poses, sources, launches, results = [], [], [], []
        for k, a in enumerate(scans):
            n0 = r.launch_count()
            process_packed(r, a)
            if k == 0:
                r.submap_init_frame()
            else:
                r.scan_matching_predicted_async()
                r.submap_update_frame_chained()
                r.global_map_append_frame()
            launches.append(r.launch_count() - n0)
            if mode == "running":
                results.append(r.localize_frame(np.eye(4) if k == 0 else None))
            if k:
                poses.append(r.get_result())
            sources.append([r.source_cloud(c) for c in range(4)])
        runs[mode] = dict(poses=poses, sources=sources, submap=[r.submap_cloud(c) for c in range(4)], map=r.global_map(),
                          frames=r.global_map_frames(), reg=r.registered_scan(), launches=launches, loc=results)
        if mode == "off":
            prior, _ = r.global_map_merged(0.5)                    # the first session's map, saved by the caller
        r.close()
    off = runs["off"]
    for mode in ("enabled", "running"):
        assert_same_odometry(off, runs[mode])
        assert runs[mode]["launches"] == off["launches"], mode
    O = [np.eye(4)] + runs["running"]["poses"]
    res = runs["running"]["loc"]
    assert same_bits(res[0].guess, np.eye(4))
    for k, x in enumerate(res):
        if k:
            prev = res[k - 1]
            want = lo.predict(prev.T if prev.accepted else prev.guess, O[k - 1], O[k])
            assert same_bits(x.guess, want), k
        assert same_bits(x.T_map_odom, lo.map_odom(x.T, O[k])), k
    accepted = [k for k, x in enumerate(res) if x.accepted]
    errs = [lvo.relative_error(res[k].T, O[k]) for k in accepted]
    print("chained: " + ", ".join(f"{k}: {x.termination}/{x.fitness:.4f}" for k, x in enumerate(res)) +
          f"; max error {max(e[0] for e in errs):.4f} m {math.degrees(max(e[1] for e in errs)):.4f} deg")
    assert len(accepted) >= len(res) - 2
    assert all(e[0] < CHAINED_BOUND[0] and e[1] < CHAINED_BOUND[1] for e in errs)
    assert any(not np.array_equal(x.guess, res[k - 1].T) for k, x in enumerate(res) if k)   # the odometry enters G


@pytest.mark.gpu
def test_gpu_localize_frame_needs_a_processed_scan():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    r.localize_enable()
    r.localize_set_map(structured_cloud(3))
    res = _lib.LocalizeResult()
    assert r._L.tloam_b200_localize_frame(r._h, None, C.byref(res)) == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_localize_shim_matches_the_python_mirror():
    import os
    import struct
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("localize_driver", "front_end_b200.hpp")
    M = structured_cloud(3)
    T_true = se3([1.5, -0.8, 0.1, 0.0, 0.0, 0.35])
    scans = [apply4(np.linalg.inv(T_true @ se3([0.3 * k, 0.0, 0.0, 0.0, 0.0, 0.0])), M[k::3]) for k in range(4)]
    d = os.path.dirname(exe)
    with open(os.path.join(d, "localize_map.bin"), "wb") as fh:
        fh.write(struct.pack("Q", len(M)) + np.ascontiguousarray(M).tobytes())
    with open(os.path.join(d, "localize_scans.bin"), "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p).tobytes())
    guess = (1.7, -0.6, 0.37)
    res = subprocess.run([exe, os.path.join(d, "localize_map.bin"), os.path.join(d, "localize_scans.bin")] +
                         [repr(v) for v in guess], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [l.split() for l in res.stdout.strip().split("\n")]
    r = tloam_b200.LocalRegistration()
    r.localize_enable()
    r.localize_set_map(M)
    G = np.eye(4)
    G[:2, :2] = [[math.cos(guess[2]), -math.sin(guess[2])], [math.sin(guess[2]), math.cos(guess[2])]]
    G[:2, 3] = guess[:2]
    assert len(got) == len(scans)
    for k, p in enumerate(scans):
        x = r.localize(p, G if k == 0 else None)
        g = got[k]
        assert (int(g[0]), int(g[1]), bool(int(g[2])), int(g[3])) == (x.iterations, x.termination, x.accepted, x.inliers)
        assert float(g[4]) == x.fitness and float(g[5]) == x.rmse
        assert np.array_equal(np.array([float(s) for s in g[6:22]]), x.T.ravel(order="F"))
        assert np.array_equal(np.array([float(s) for s in g[22:38]]), x.T_map_odom.ravel(order="F"))
    assert sum(int(g[2]) for g in got) >= 3
    r.close()


def test_localize_driver_compiles_warning_free():
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "mock", "localize_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(root, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr
