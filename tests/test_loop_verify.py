"""Loop verification (include/tloam_b200.h "Loop verification"; k_lv_match / k_lv_reduce / k_lv_step / k_lv_final /
k_lv_commit in libtloam_b200_loopv.so): a down-sampled keyframe per loop frame, kept by the global map's ordered path,
and a scan-to-scan ICP that returns T_cand_query.  tests/loop_verify_oracle.py is the CPU restatement.

CPU: the oracle's nearest neighbour, Gauss-Newton and recovery of a known transform; the symbols, the new library's
kernels, the driver.  GPU: keyframes and verification against the oracle, a revisit in the ray-cast world of
test_loop_closure.py, the existing calls' bits with verification on, determinism and growth, status codes, the shim."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import loop_verify_oracle as lvo
import sass_digest
from tloam_b200 import synth
from test_global_map import with_nonfinite
from test_global_map_intensity import same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_loop_verify_default_config", "tloam_b200_loop_verify_enable", "tloam_b200_loop_keyframe_download",
               "tloam_b200_loop_verify", "tloam_b200_loop_verify_matches"]
# the revisit of the ray-cast world: the bound on T against the route's ground truth.  The restatement on the CPU reaches
# 0.256 m / 0.040 deg there (the yaw alone is 0.50 m / 1.0 deg off); the translation's floor is the 16-beam rings, which a
# point-to-point ICP matches between two sensor positions 0.5 m apart (DESIGN.md section 4c)
REVISIT_BOUND = (0.35, math.radians(0.2))


def rz4(a):
    T = np.eye(4)
    T[:2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
    return T


def se3(xi):
    R, t = lvo.se3_exp(np.asarray(xi, dtype=np.float64))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def apply4(T, p):
    return p @ T[:3, :3].T + T[:3, 3]


def structured_cloud(seed, n=3000):
    """walls, a ground plane and poles: a cloud whose alignment is well conditioned in all six directions"""
    rng = np.random.default_rng(seed)
    g = np.column_stack([rng.uniform(-30, 30, n), rng.uniform(-30, 30, n), rng.normal(-1.7, 0.02, n)])
    w1 = np.column_stack([rng.uniform(-30, 30, n // 2), np.full(n // 2, 12.0), rng.uniform(-1.7, 4.0, n // 2)])
    w2 = np.column_stack([np.full(n // 2, -9.0), rng.uniform(-30, 30, n // 2), rng.uniform(-1.7, 4.0, n // 2)])
    k = n // 6
    c = rng.uniform(-25, 25, (12, 2))
    a = rng.uniform(0, 2 * np.pi, k)
    j = rng.integers(0, 12, k)
    poles = np.column_stack([c[j, 0] + 0.3 * np.cos(a), c[j, 1] + 0.3 * np.sin(a), rng.uniform(-1.7, 6.0, k)])
    roof = np.column_stack([rng.uniform(0, 10, k), rng.uniform(0, 10, k), 0.5 * rng.uniform(0, 10, k) + 4.0])
    return np.vstack([g, w1, w2, poles, roof])


# ---------------------------------------------------------------------------------------------------------------------
def test_oracle_nearest_is_the_kdtree_nearest_and_ties_go_to_the_lower_index():
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(1)
    M = rng.uniform(-20, 20, (3000, 3))
    P = rng.uniform(-25, 25, (2000, 3))
    idx, d2 = lvo.nearest(P, M, chunk=300)
    dist, want = cKDTree(M).query(P)
    assert np.array_equal(idx, want)
    assert np.allclose(d2, dist ** 2, rtol=1e-12)
    M2 = np.vstack([M[:10], M[:10], M[5:6]])                       # rows 10..20 repeat rows 0..9 and row 5
    idx2, _ = lvo.nearest(M2 + 1e-3, M2)
    assert np.array_equal(idx2, np.r_[np.arange(10), np.arange(10), 5])


def test_oracle_gauss_newton_converges_to_the_least_squares_solution():
    """correspondences held fixed: the iterate of gauss_newton_step / apply reaches scipy's least_squares minimum of
    sum |R q + t - m|^2 within 1e-9"""
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(2)
    Q = rng.uniform(-15, 15, (400, 3))
    T0 = se3([0.8, -0.4, 0.2, 0.03, -0.02, 0.4])
    Mm = apply4(T0, Q) + rng.normal(0, 0.05, Q.shape)
    R, t = np.eye(3), np.zeros(3)
    for _ in range(30):
        R, t = lvo.apply(lvo.gauss_newton_step(lvo.transform(Q, R, t), Mm), R, t)

    def res(x):
        return (Q @ Rotation.from_rotvec(x[:3]).as_matrix().T + x[3:] - Mm).ravel()

    sol = least_squares(res, np.zeros(6), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Rl, tl = Rotation.from_rotvec(sol.x[:3]).as_matrix(), sol.x[3:]
    assert np.abs(R - Rl).max() < 1e-9 and np.abs(t - tl).max() < 1e-9


def test_oracle_exp_is_the_deskew_oracles():
    import deskew_oracle
    assert lvo.se3_exp is deskew_oracle.se3_exp


def test_oracle_recovers_a_noise_free_transform_from_a_guess_3_deg_and_2_m_off():
    M = structured_cloud(3)
    T_true = se3([1.5, -0.8, 0.1, 0.01, -0.02, 0.35])
    Q = apply4(np.linalg.inv(T_true), M)                           # p_cand = T_true . p_query exactly
    guess = T_true @ se3([2.0 / math.sqrt(2), 2.0 / math.sqrt(2), 0.0, 0.0, 0.0, math.radians(3.0)])
    r = lvo.run(Q, M, guess, lvo.config())
    dt, dr = lvo.relative_error(r["T"], T_true)
    assert r["termination"] == lvo.CONVERGED and r["accepted"] and dt < 1e-9 and dr < 1e-9, (r["termination"], dt, dr)
    assert r["inliers"] == len(Q) and r["fitness"] < 1e-18
    assert np.array_equal(r["passes"][-1][0], np.arange(len(Q)))


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_loopv_library_holds_only_the_new_kernels_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.LOOPV_LIB))
    kernels = ("k_lv_match", "k_lv_reduce", "k_lv_step", "k_lv_final", "k_lv_commit")
    assert len(names) == 5 and [sum(f"{len(k)}{k}E" in m for m in names) for k in kernels] == [1] * 5
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.LOOPV_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


def test_loop_verify_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "loop_verify_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def refused_cloud():
    """an extent of more than 2^21 voxels of 1.0 m on x: the global map's key-range guard refuses it"""
    p = np.zeros((50, 3))
    p[:, 0] = np.linspace(0.0, 3.0e6, 50)
    return p


def keyframe_clouds():
    rng = np.random.default_rng(4)
    return [with_nonfinite(synth.raw_scan(), 7), with_nonfinite(synth.vlp16_raw_scan(), 9), rng.uniform(-30, 30, (5000, 3)),
            np.zeros((0, 3)), refused_cloud(), np.full((20, 3), np.nan), structured_cloud(5)]


def new_db(**vcfg):
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=0)
    r.loop_verify_enable(**vcfg)
    return r


@pytest.mark.gpu
def test_gpu_keyframes_are_the_global_maps_blocks_and_every_add_owns_one_slot(oracle):
    """HDL-64E and VLP-16 scans with NaN / Inf rows, a host cloud, an empty cloud, a refused cloud, an all-NaN cloud and
    one more cloud after them, at two voxel sizes, and the scan process_raw_scan left on the device: each keyframe is bit
    for bit the global map's block of the same cloud at pose I, and matches the restatement as the global map's blocks do
    (test_global_map.check_block: the same voxel key sequence, coordinates within 1e-10 m)"""
    import global_map_oracle as gmo
    from test_global_map import check_block
    from test_process_cloud import FE
    clouds = keyframe_clouds()
    for voxel in (0.5, 1.0):
        r = new_db(voxel=voxel)
        r.enable_global_map(voxel=voxel)
        for i, p in enumerate(clouds):
            r.loop_add(p)
            got = r.loop_keyframe(i)
            if i in (3, 4, 5):                                         # empty, refused, all non-finite: an empty slot
                assert len(got) == 0, i
                continue
            r.global_map_append(p, pose=np.eye(4))
            off = r.global_map_frames()
            assert same_bits(got, r.global_map(int(off[-2]), int(off[-1] - off[-2]))), (voxel, i)
            check_block(oracle, got, gmo.transform(p, np.eye(4)), voxel)
        raw = synth.raw_scan(seed=3, n_az=900)
        r.process_raw_scan(raw, feature=FE)
        r.loop_add_frame()
        r.global_map_append_frame(np.eye(4))
        off = r.global_map_frames()
        got = r.loop_keyframe(len(clouds))
        assert same_bits(got, r.global_map(int(off[-2]), int(off[-1] - off[-2])))
        check_block(oracle, got, gmo.transform(raw, np.eye(4)), voxel)
        assert r.loop_size() == len(clouds) + 1 and len(r.loop_keyframe(len(clouds) - 1)) > 0
        r.close()


def verify_cases(oracle):
    """(name, Q, M, guess): keyframes as the device builds them"""
    kf = lambda p: lvo.keyframe(oracle, p, 0.5)                   # noqa: E731
    M = kf(structured_cloud(6))
    T = se3([1.2, 0.7, -0.05, 0.01, 0.015, -0.3])
    exact = apply4(np.linalg.inv(T), M)
    rng = np.random.default_rng(7)
    noisy = kf(apply4(np.linalg.inv(T), structured_cloud(6)) + rng.normal(0, 0.03, (len(structured_cloud(6)), 3)))
    from test_loop_closure import route_scans
    poses, scans = route_scans()
    cases = [("exact", exact, M, T @ se3([1.0, -1.0, 0.2, 0.0, 0.0, 0.05])),
             ("noisy", noisy, M, T @ se3([0.5, 0.5, 0.0, 0.0, 0.0, -0.03])),
             ("raycast", kf(scans[-1]), kf(scans[10]), rz4(math.radians(-96.0))),
             ("unrelated", kf(synth.raw_scan(seed=11)), kf(structured_cloud(8)), np.eye(4)),
             ("empty", kf(np.zeros((0, 3))), M, np.eye(4)),
             ("few", M[:5], M + 100.0, np.eye(4))]
    return cases


@pytest.mark.gpu
def test_gpu_verify_is_the_oracles(oracle):
    """first pass bit-identical; no correspondence flips at later passes; iterations, termination, inliers, accepted equal;
    T within 1e-9 m / rad; fitness and rmse within 1e-9 relative"""
    cfg = lvo.config()
    for name, Q, M, guess in verify_cases(oracle):
        r = new_db()
        r.loop_add(Q)                       # a keyframe of a keyframe is itself: voxel centres stay in their voxels
        r.loop_add(M)
        got = r.loop_verify(0, 1, guess)
        kq, km = r.loop_keyframe(0), r.loop_keyframe(1)
        want = lvo.run(kq, km, guess, cfg)
        assert (got.iterations, got.termination, got.inliers, got.accepted) == \
            (want["iterations"], want["termination"], want["inliers"], want["accepted"]), (name, got, want)
        assert (got.n_query_points, got.n_candidate_points) == (len(kq), len(km))
        dt, dr = lvo.relative_error(got.T, want["T"])
        assert dt < 1e-9 and dr < 1e-9, (name, dt, dr)
        for a, b in ((got.fitness, want["fitness"]), (got.rmse, want["rmse"])):
            assert a == b or abs(a - b) <= 1e-9 * abs(b), (name, a, b)
        flips = 0
        for k, (idx, d2) in enumerate(want["passes"]):
            gi, gd = r.loop_verify_matches(k)
            if k == 0:
                assert np.array_equal(gi, idx) and same_bits(gd, d2), name
            flips += int((gi != idx).sum())
        print(f"verify {name}: {len(kq)} x {len(km)} points, {got.iterations} iterations, termination {got.termination}, "
              f"fitness {got.fitness:.4g}, flips {flips}")
        assert flips == 0, name
        if name == "empty":
            assert got.termination == lvo.EMPTY and not want["passes"]
        r.close()


def route_db():
    import tloam_b200
    from test_loop_closure import route_scans
    poses, scans = route_scans()
    r = tloam_b200.LocalRegistration()
    r.loop_enable()
    r.loop_verify_enable()
    res = []
    for p in scans:
        r.loop_add(p)
        res.append(r.loop_result())
    return r, poses, res


def pose4(p):
    T = rz4(p[2])
    T[:2, 3] = p[:2]
    return T


@pytest.mark.gpu
def test_gpu_revisit_is_accepted_and_a_far_frame_is_not():
    r, poses, res = route_db()
    last = res[-1]
    assert last.is_loop
    v = r.loop_verify(last.query, last.candidate, yaw=last.yaw)
    gt = np.linalg.inv(pose4(poses[last.candidate])) @ pose4(poses[last.query])
    dt, dr = lvo.relative_error(v.T, gt)
    dt0, dr0 = lvo.relative_error(rz4(last.yaw), gt)
    print(f"revisit {last.query} -> {last.candidate}: {v.iterations} iterations, fitness {v.fitness:.4f}, rmse {v.rmse:.4f}, "
          f"error {dt:.4f} m {math.degrees(dr):.4f} deg (yaw alone {dt0:.3f} m {math.degrees(dr0):.3f} deg)")
    assert v.accepted and v.termination == v.CONVERGED
    assert dt < REVISIT_BOUND[0] and dr < REVISIT_BOUND[1]
    assert dt < 0.6 * dt0 and dr < dr0 / 10
    far = int(np.argmax([np.hypot(p[0] - poses[-1][0], p[1] - poses[-1][1]) for p in poses[:60]]))
    w = r.loop_verify(last.query, far, yaw=last.yaw)
    print(f"far frame {far}: termination {w.termination}, fitness {w.fitness:.3f}")
    assert not w.accepted
    r.close()


@pytest.mark.gpu
def test_gpu_loop_results_are_bit_identical_with_verification_on():
    from test_loop_closure import database_clouds
    import tloam_b200
    clouds = database_clouds(60, 3)
    runs = []
    for on in (False, True):
        r = tloam_b200.LocalRegistration()
        r.loop_enable(exclude_recent=5)
        if on:
            r.loop_verify_enable()
        res = []
        for p in clouds:
            r.loop_add(p)
            res.append(r.loop_result())
        runs.append((res, [np.concatenate([np.ravel(x) for x in r.loop_descriptor(k)]) for k in range(60)]))
        r.close()
    assert runs[0][0] == runs[1][0] and all(same_bits(a, b) for a, b in zip(runs[0][1], runs[1][1]))


def mapping_loop(scans, verify):
    """the four-call mapping loop with loop_add_frame, as test_loop_closure.odometry_loop, with or without keyframes"""
    import tloam_b200
    from test_loop_closure import process_packed
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()
    r.loop_enable(exclude_recent=2)
    if verify:
        r.loop_verify_enable()
    poses, results = [], []
    for k, a in enumerate(scans):
        process_packed(r, a)
        if k == 0:
            r.submap_init_frame()
        else:
            r.scan_matching_predicted_async()
            r.submap_update_frame_chained()
            r.global_map_append_frame()
        r.loop_add_frame()
        if k:
            poses.append(r.get_result())
        results.append(r.loop_result())
    out = dict(poses=poses, map=r.global_map(), frames=r.global_map_frames(), loop=results)
    if verify:
        out["kf"] = [r.loop_keyframe(k) for k in range(len(scans))]
        out["v"] = r.loop_verify(len(scans) - 1, 0)
    r.close()
    return out


@pytest.mark.gpu
def test_gpu_mapping_loop_is_bit_identical_with_verification_on_and_deterministic():
    from test_deskew import loop_scans
    scans = loop_scans()
    off, on, again = mapping_loop(scans, False), mapping_loop(scans, True), mapping_loop(scans, True)
    for x in (on, again):
        assert all(np.array_equal(a, b) for a, b in zip(off["poses"], x["poses"])) and len(off["poses"]) == len(x["poses"])
        assert same_bits(off["map"], x["map"]) and np.array_equal(off["frames"], x["frames"]) and off["loop"] == x["loop"]
    assert all(same_bits(a, b) for a, b in zip(on["kf"], again["kf"]))
    a, b = on["v"], again["v"]
    assert same_bits(a.T, b.T) and (a.fitness, a.rmse, a.inliers, a.iterations) == (b.fitness, b.rmse, b.inliers, b.iterations)


@pytest.mark.gpu
def test_gpu_grown_keyframe_store_gives_the_preallocated_bits():
    """capacity 1 point (grows on every early add) against the default, on the same clouds: keyframes and a verification"""
    clouds = keyframe_clouds() + [structured_cloud(9)]
    runs = []
    for cap in (1, 1 << 21):
        r = new_db(initial_capacity_points=cap)
        for p in clouds:
            r.loop_add(p)
        v = r.loop_verify(len(clouds) - 1, 6)
        runs.append(([r.loop_keyframe(k) for k in range(len(clouds))], v))
        r.close()
    assert all(same_bits(a, b) for a, b in zip(runs[0][0], runs[1][0]))
    a, b = runs[0][1], runs[1][1]
    assert same_bits(a.T, b.T) and (a.fitness, a.rmse, a.inliers, a.iterations, a.termination) == \
        (b.fitness, b.rmse, b.inliers, b.iterations, b.termination)


@pytest.mark.gpu
def test_gpu_loop_verify_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    res = _lib.LoopVerifyResult()
    n = C.c_size_t(0)
    buf = np.zeros(3 * 200000)
    dp = buf.ctypes.data_as(C.POINTER(C.c_double))
    ibuf = np.zeros(200000, dtype=np.int32)
    ip = ibuf.ctypes.data_as(C.POINTER(C.c_int))

    def cfg(**kw):
        c = _lib.LoopVerifyConfig()
        L.tloam_b200_loop_verify_default_config(C.byref(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    # no loop database: NOT_READY everywhere
    assert L.tloam_b200_loop_verify_enable(h, C.byref(cfg())) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_keyframe_download(h, 0, dp, 10, C.byref(n)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_verify(h, 0, 0, None, C.byref(res)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_verify_matches(h, 0, ip, dp, 10, C.byref(n)) == _lib.ERR_NOT_READY
    r.loop_enable(exclude_recent=0)
    bad = [dict(voxel=0.0), dict(voxel=-1.0), dict(voxel=float("nan")), dict(corr_dist_coarse=float("inf")),
           dict(corr_dist_fine=0.0), dict(corr_dist_fine=5.0), dict(eps_translation=0.0), dict(eps_rotation=float("nan")),
           dict(max_fitness=-0.1), dict(max_iterations=0), dict(max_iterations=201)]
    for kw in bad:
        assert L.tloam_b200_loop_verify_enable(h, C.byref(cfg(**kw))) == _lib.ERR_INVALID_ARG, kw
    assert L.tloam_b200_loop_verify_enable(h, None) == _lib.ERR_INVALID_ARG
    # enabled but off: NOT_READY
    assert L.tloam_b200_loop_verify(h, 0, 0, None, C.byref(res)) == _lib.ERR_NOT_READY
    r.loop_add(structured_cloud(1))
    assert L.tloam_b200_loop_verify_enable(h, C.byref(cfg())) == _lib.ERR_NOT_READY   # the database is not empty
    assert L.tloam_b200_loop_keyframe_download(h, 0, dp, 10, C.byref(n)) == _lib.ERR_NOT_READY
    r.loop_reset()
    assert L.tloam_b200_loop_verify_enable(h, C.byref(cfg(max_iterations=200, corr_dist_fine=4.0))) == _lib.OK
    assert L.tloam_b200_loop_verify_matches(h, 0, ip, dp, 10, C.byref(n)) == _lib.ERR_NOT_READY      # no verification yet
    r.loop_add(structured_cloud(1))
    r.loop_add(structured_cloud(1))
    assert L.tloam_b200_loop_keyframe_download(h, 2, dp, 200000, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_keyframe_download(h, 0, dp, 1, C.byref(n)) == _lib.ERR_INVALID_ARG and n.value > 1
    assert L.tloam_b200_loop_keyframe_download(h, 0, None, 200000, None) == _lib.ERR_INVALID_ARG
    for q, c in ((2, 0), (0, 2), (-1, 0), (0, -1)):
        assert L.tloam_b200_loop_verify(h, q, c, None, C.byref(res)) == _lib.ERR_INVALID_ARG, (q, c)
    assert L.tloam_b200_loop_verify(h, 0, 1, None, None) == _lib.ERR_INVALID_ARG
    for T in (np.diag([1.0, 1.0, 2.0, 1.0]), np.diag([1.0, 1.0, -1.0, 1.0]), np.full((4, 4), np.nan),
              rz4(0.3) + np.array([[0, 0, 0, 0]] * 3 + [[0, 0, 0.5, 0]])):
        g = np.asfortranarray(T).ravel(order="F").copy()
        assert L.tloam_b200_loop_verify(h, 0, 1, g.ctypes.data_as(C.POINTER(C.c_double)), C.byref(res)) == _lib.ERR_BAD_POSE
    v = r.loop_verify(0, 1)                                        # a cloud against itself: converged at once
    assert v.accepted and v.iterations >= 1 and v.fitness == 0.0
    assert L.tloam_b200_loop_verify_matches(h, v.iterations + 1, ip, dp, 200000, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_verify_matches(h, -1, ip, dp, 200000, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_verify_matches(h, 0, ip, dp, 1, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert np.array_equal(r.loop_verify_matches(v.iterations)[0], np.arange(n.value))
    r.loop_reset()                                                 # empties the keyframes, verification stays on
    assert r.loop_size() == 0 and L.tloam_b200_loop_keyframe_download(h, 0, dp, 10, C.byref(n)) == _lib.ERR_INVALID_ARG
    r.loop_add(np.zeros((0, 3)))
    r.loop_add(structured_cloud(2))
    e = r.loop_verify(0, 1)
    assert e.termination == e.EMPTY and not e.accepted and e.fitness == math.inf and e.iterations == 0
    assert L.tloam_b200_loop_verify_matches(h, 0, ip, dp, 10, C.byref(n)) == _lib.ERR_INVALID_ARG    # no pass
    r.loop_enable()                                                # turns verification off
    assert L.tloam_b200_loop_keyframe_download(h, 0, dp, 10, C.byref(n)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_verify(h, 0, 0, None, C.byref(res)) == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_loop_verify_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    from test_process_cloud import FE
    exe = build_driver("loop_verify_driver", "front_end_b200.hpp")
    scans = [synth.raw_scan(seed=s, n_az=900) for s in range(6)]
    scans += [scans[1] @ rz4(0.4)[:3, :3].T + [0.3, -0.2, 0.0], scans[3]]
    path = os.path.join(os.path.dirname(exe), "loop_verify_raw.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path, "3"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [l.split() for l in res.stdout.strip().split("\n")]
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=3)
    r.loop_verify_enable()
    verified = 0
    for k, p in enumerate(scans):
        if k % 2 == 0:
            r.process_raw_scan(p, feature=FE)
            r.loop_add_frame()
        else:
            r.loop_add(p)
        x = r.loop_result()
        g = got[k]
        assert (int(g[0]), int(g[1])) == (x.query, x.candidate)
        if x.candidate >= 0:
            v = r.loop_verify(x.query, x.candidate, yaw=x.yaw)
            assert (int(g[2]), int(g[3]), int(g[4]), bool(int(g[5]))) == (v.iterations, v.termination, v.inliers, v.accepted)
            assert float(g[6]) == v.fitness and float(g[7]) == v.rmse
            assert np.array_equal(np.array([float(s) for s in g[8:24]]), v.T.ravel(order="F"))
            verified += 1
    assert verified >= 4 and int(got[-1][1]) == 3 and int(got[-1][5]) == 1      # an exact repeat of frame 3: accepted
    r.close()
