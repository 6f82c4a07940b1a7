"""Loop verification against a submap (include/tloam_b200.h "Loop verification against a submap"; k_lvs_* in
libtloam_b200_loopvs.so): the query keyframe aligned, point to plane, to the keyframes of the frames around the candidate.
tests/loop_verify_submap_oracle.py is the CPU restatement.

CPU: the oracle's normals, eigen-solve and Gauss-Newton, recovery of a known transform, the ray-cast revisit against the
point-to-point verification, the symbols, the new library's kernels, the driver.  GPU: target, normals, matches and the
whole run against the oracle, the revisit, the existing calls' bits with the feature on, determinism and growth, status
codes, the shim."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import loop_verify_oracle as lvo
import loop_verify_submap_oracle as lso
import sass_digest
from test_global_map_intensity import same_bits
from test_loop_verify import apply4, pose4, rz4, se3, structured_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_loop_verify_submap_default_config", "tloam_b200_loop_verify_submap_enable",
               "tloam_b200_loop_verify_submap", "tloam_b200_loop_verify_submap_target", "tloam_b200_loop_verify_submap_matches"]
KERNELS = ("k_lvs_poses", "k_lvs_assemble", "k_lvs_normals", "k_lvs_match", "k_lvs_reduce", "k_lvs_step", "k_lvs_final")
# the revisit of the ray-cast world with the route's poses: the restatement reaches 0.0020 m / 0.0065 deg where the
# point-to-point verification stops at 0.256 m / 0.040 deg (DESIGN.md section 4c)
REVISIT_BOUND = (0.03, math.radians(0.03))
REVISIT = (117, 10)                                                # the route's last frame and the frame it revisits


# ---- CPU: the restatement ------------------------------------------------------------------------------------------------
def test_oracle_normals_on_planes_a_corner_and_a_pole():
    rng = np.random.default_rng(1)
    n_true = np.array([0.3, -0.5, 0.81])
    n_true /= np.linalg.norm(n_true)
    u = np.cross(n_true, [1.0, 0, 0])
    u /= np.linalg.norm(u)
    w = np.cross(n_true, u)
    ab = rng.uniform(-4, 4, (1500, 2))
    plane = ab[:, :1] * u + ab[:, 1:] * w + 0.01 * rng.normal(size=(1500, 1)) * n_true
    cfg = lso.config()
    nrm, valid, cnt, eig, cov = lso.normals(plane, cfg)
    idx, cnt2 = lso.neighbours(plane, 1.0)
    assert np.array_equal(cnt, cnt2) and valid.mean() > 0.95
    for i in np.flatnonzero(valid)[::50]:                          # the SVD normal of the same neighbourhood
        nb = plane[idx[i][idx[i] >= 0]]
        sv = np.linalg.svd(nb - nb.mean(0))[2][2]
        assert min(np.abs(nrm[i] - sv).max(), np.abs(nrm[i] + sv).max()) < 1e-9
    assert np.abs(np.abs(nrm[valid] @ n_true) - 1.0).max() < 1e-2
    # a wall - ground corner: the rows on the edge see both planes; a pole: a line.  Neither has a plane
    g = np.column_stack([rng.uniform(-3, 3, 3000), rng.uniform(0, 3, 3000), np.zeros(3000)])
    wall = np.column_stack([rng.uniform(-3, 3, 3000), np.zeros(3000), rng.uniform(0, 3, 3000)])
    edge = np.column_stack([np.linspace(-2, 2, 40), np.zeros(40), np.zeros(40)])
    corner = np.vstack([edge, g, wall])
    _, valid_c, _, eig_c, _ = lso.normals(corner, cfg)
    assert not valid_c[:40].any() and (eig_c[:40, 0] > 0.1 * eig_c[:40, 1]).all()
    pole = np.column_stack([0.02 * rng.normal(size=(200, 2)), np.linspace(0, 6, 200)])
    _, valid_p, cnt_p, _, _ = lso.normals(pole, cfg)
    assert not valid_p.any() and cnt_p.min() >= 5
    lone = np.vstack([plane[:3] + 100.0, plane])                   # fewer than min_normal_neighbours
    assert not lso.normals(lone, cfg)[1][:3].any()


def test_oracle_eigen_solve_is_numpys_eigh():
    rng = np.random.default_rng(2)
    A = rng.normal(size=(1000, 3, 3))
    S = A @ A.transpose(0, 2, 1)
    v = rng.normal(size=(300, 3))
    S[:300] = v[:, :, None] * v[:, None, :]                        # rank one
    S[300:500] -= (S[300:500] @ v[:200, :, None]) @ (v[:200, None, :] / np.sum(v[:200] ** 2, axis=1)[:, None, None])
    S[300:500] = S[300:500] @ S[300:500].transpose(0, 2, 1)        # rank two
    S = 0.5 * (S + S.transpose(0, 2, 1))
    c = np.column_stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]])
    eig, nrm = lso.jacobi3(c)
    w, V = np.linalg.eigh(S)
    scale = w[:, 2:3]
    assert np.abs(eig - w).max() <= 1e-12 * scale.max() and (np.abs(eig - w) <= 1e-12 * scale).all()
    assert np.abs(np.linalg.norm(nrm, axis=1) - 1.0).max() < 1e-14
    res = np.einsum("nij,nj->ni", S, nrm) - eig[:, :1] * nrm       # an eigenvector of the least eigenvalue
    assert (np.abs(res) <= 1e-12 * scale).all()
    gap = (w[:, 1] - w[:, 0]) > 1e-3 * w[:, 2]
    assert gap.sum() > 400 and (np.abs(np.abs(np.sum(nrm[gap] * V[gap, :, 0], axis=1)) - 1.0) < 1e-9).all()


def test_oracle_gauss_newton_converges_to_the_point_to_plane_least_squares_solution():
    from scipy.optimize import least_squares
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(3)
    Q = rng.uniform(-15, 15, (500, 3))
    N = rng.normal(size=(500, 3))
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    T0 = se3([0.6, -0.4, 0.2, 0.03, -0.02, 0.2])
    Mm = apply4(T0, Q) + rng.normal(0, 0.05, Q.shape)
    R, t = np.eye(3), np.zeros(3)
    for _ in range(30):
        R, t = lvo.apply(lso.gauss_newton_step(lvo.transform(Q, R, t), Mm, N), R, t)

    def res(x):
        return np.sum(N * (Q @ Rotation.from_rotvec(x[:3]).as_matrix().T + x[3:] - Mm), axis=1)

    sol = least_squares(res, np.zeros(6), xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Rl, tl = Rotation.from_rotvec(sol.x[:3]).as_matrix(), sol.x[3:]
    assert np.abs(R - Rl).max() < 1e-9 and np.abs(t - tl).max() < 1e-9


def test_oracle_recovers_a_noise_free_transform_and_k0_is_the_keyframe():
    M = structured_cloud(3)
    T_true = se3([1.5, -0.8, 0.1, 0.01, -0.02, 0.35])
    Q = apply4(np.linalg.inv(T_true), M)
    guess = T_true @ se3([2.0 / math.sqrt(2), 2.0 / math.sqrt(2), 0.0, 0.0, 0.0, math.radians(3.0)])
    cfg = lso.config(half_window=0)
    kfs = [structured_cloud(4), M, Q]
    poses = [se3([1.0, 2.0, 0.1, 0.0, 0.0, 0.3])] * 3
    r, tgt, nrm, valid, _ = lso.verify(kfs, poses, 2, 1, guess, cfg)
    assert same_bits(tgt, M) and valid.mean() > 0.3
    err = np.abs(r["T"] - T_true).max()                            # entrywise: arccos resolves no angle below 1e-8
    assert r["termination"] == lso.CONVERGED and r["accepted"] and err < 1e-9, (r["termination"], err)
    assert r["fitness"] < 1e-18 and r["rmse"] < 1e-9 and r["inliers"] == int(valid.sum())
    assert np.array_equal(r["passes"][-1][0], np.arange(len(Q)))
    # a window: the neighbours arrive in the candidate's frame, the query is left out, an empty keyframe adds nothing
    kfs = [M[:100], np.zeros((0, 3)), M[100:300], Q, M[300:500]]
    poses = [se3([0.5 * j, 0.1 * j, 0, 0, 0, 0.05 * j]) for j in range(5)]
    tgt = lso.target(kfs, poses, 2, 3, 2)
    assert len(tgt) == 500 and same_bits(tgt[100:300], M[100:300])
    want = apply4(np.linalg.inv(poses[2]) @ poses[4], M[300:500])
    assert np.abs(tgt[300:] - want).max() < 1e-12
    assert lso.window(2, 3, 2, 5) == (0, 4, [0, 1, 2, 4]) and lso.window(0, 9, 3, 6) == (0, 3, [0, 1, 2, 3])


@pytest.fixture(scope="module")
def route():
    """the ray-cast route of test_loop_closure.py: its poses (4 x 4), scans and the restatement's keyframes"""
    from oracle import pyoracle
    from test_loop_closure import route_scans
    pyoracle.build()
    poses, scans = route_scans()
    return [pose4(p) for p in poses], scans, [lvo.keyframe(pyoracle, s, 0.5) for s in scans]


def test_oracle_submap_verification_beats_scan_to_scan_on_the_ray_cast_revisit(route):
    """the point of the feature: the 16-beam revisit, from Scan Context's yaw"""
    P, scans, kf = route
    q, c = REVISIT
    gt = np.linalg.inv(P[c]) @ P[q]
    guess = rz4(math.radians(-96.0))
    p2p = lvo.run(kf[q], kf[c], guess, lvo.config())
    dt0, dr0 = lvo.relative_error(p2p["T"], gt)
    cfg = lso.config()
    r, tgt, _, valid, _ = lso.verify(kf, P, q, c, guess, cfg)
    dt, dr = lvo.relative_error(r["T"], gt)
    print(f"revisit: point to point {dt0:.4f} m {math.degrees(dr0):.4f} deg fitness {p2p['fitness']:.4f}; submap ({len(tgt)} rows, "
          f"{valid.mean():.2f} valid) {dt:.4f} m {math.degrees(dr):.4f} deg fitness {r['fitness']:.4f} rmse {r['rmse']:.4f}")
    assert r["accepted"] and r["termination"] == lso.CONVERGED
    assert dt < REVISIT_BOUND[0] and dr < REVISIT_BOUND[1] and dt < dt0 / 8
    far = int(np.argmax([np.hypot(*(p[:2, 3] - P[q][:2, 3])) for p in P[:60]]))
    false = [lso.verify(kf, P, q, f, guess, cfg)[0] for f in (far, 30, 100)]
    print("false pairs: fitness " + ", ".join(f"{w['fitness']:.2f}" for w in false) + f"; true {r['fitness']:.4f}")
    assert not any(w["accepted"] for w in false) and min(w["fitness"] for w in false) > 20 * r["fitness"]
    from oracle import pyoracle
    from tloam_b200 import synth
    u = lvo.keyframe(pyoracle, synth.raw_scan(seed=11), 0.5)
    s = lvo.keyframe(pyoracle, structured_cloud(8), 0.5)
    nrm, val, _, _, _ = lso.normals(s, cfg)
    assert not lso.run(u, s, nrm, val, np.eye(4), cfg)["accepted"]


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)
    c = _lib.LoopVerifySubmapConfig()
    _lib.load().tloam_b200_loop_verify_submap_default_config(C.byref(c))
    got = {k: getattr(c, k) for k, _ in c._fields_}
    assert got == lso.config()


def test_loopvs_library_holds_only_the_new_kernels_for_sm90a_and_the_normals_do_not_spill():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.LOOPVS_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.LOOPVS_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.LOOPVS_LIB], capture_output=True, text=True, check=True).stdout
    lines = res.splitlines()
    usage = [lines[i + 1] for i, l in enumerate(lines) if "k_lvs_normals" in l]
    assert len(usage) == 1 and " LOCAL:0 " in usage[0] and " STACK:0 " in usage[0], usage
    assert sorted(sass_digest.digests(build.LOOPV_LIB)) == sorted(m for m in sass_digest.digests(build.LOOPV_LIB) if "k_lv_" in m)


def test_loop_verify_submap_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "loop_verify_submap_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def new_db(clouds, poses=None, **cfg):
    """a loop database with a keyframe per cloud, submap verification on, and (with poses) a pose-graph node per frame"""
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=0)
    r.loop_verify_enable()
    r.loop_verify_submap_enable(**cfg)
    if poses is not None:
        r.pose_graph_enable()
    for k, p in enumerate(clouds):
        r.loop_add(p)
        if poses is not None:
            r.pose_graph_add_node(poses[k])
    return r


def check_against_the_oracle(r, n_frames, poses, q, c, guess, cfg, name):
    """one verification with the pose graph's nodes and one with the same poses from the host, both against the
    restatement on the device's keyframes"""
    kfs = [r.loop_keyframe(j) for j in range(n_frames)]
    want, M, nrm, valid, cnt = lso.verify(kfs, poses, q, c, guess, cfg)
    lo, hi, _ = lso.window(c, q, cfg["half_window"], n_frames)
    results = []
    for host in (False, True):
        got = r.loop_verify_submap(q, c, guess, poses=np.array(poses[lo:hi + 1]) if host else None)
        xyz, gn, gv, gc = r.loop_verify_submap_target()
        assert same_bits(xyz, M), name                             # the target, bit for bit
        assert np.array_equal(gc, cnt) and np.array_equal(gv, valid), name
        assert same_bits(gn, nrm), name                            # the same sums and the same eigen-solve
        assert (got.iterations, got.termination, got.inliers, got.accepted) == \
            (want["iterations"], want["termination"], want["inliers"], want["accepted"]), (name, got, want)
        assert (got.n_query_points, got.n_candidate_points) == (len(kfs[q]), len(M))
        if want["termination"] == lso.EMPTY:
            assert got.fitness == math.inf and np.array_equal(got.T, guess)
            continue
        assert np.abs(got.T - want["T"]).max() < 1e-9, (name, np.abs(got.T - want["T"]).max())
        for a, b in ((got.fitness, want["fitness"]), (got.rmse, want["rmse"])):
            assert a == b or abs(a - b) <= 1e-9 * abs(b) + 1e-15, (name, a, b)
        assert len(want["passes"]) == got.iterations + 1
        for k, (idx, d2) in enumerate(want["passes"]):
            gi, gd = r.loop_verify_submap_matches(k)
            if k == 0:
                assert same_bits(gd, d2), name
            assert np.array_equal(gi, idx), (name, k)
        results.append(got)
    a, b = results if results else (None, None)
    if a is not None:
        assert same_bits(a.T, b.T) and (a.fitness, a.rmse) == (b.fitness, b.rmse), name
    print(f"submap verify {name}: {len(kfs[q])} x {len(M)} rows, {int(valid.sum())} valid, {want['iterations']} iterations, "
          f"termination {want['termination']}, fitness {want['fitness']:.4g}")
    return results[0] if results else None


@pytest.fixture(scope="module")
def route_db(route):
    P, scans, _ = route
    r = new_db(scans, P)
    yield r
    r.close()


@pytest.mark.gpu
def test_gpu_route_windows_are_the_oracles(route, route_db):
    """the revisit (device and host poses), a window clipped at frame 0 and one clipped at F - 1, both with the query inside"""
    P, scans, _ = route
    F = len(scans)
    cfg = lso.config()
    q, c = REVISIT
    v = check_against_the_oracle(route_db, F, P, q, c, rz4(math.radians(-96.0)), cfg, "revisit")
    gt = np.linalg.inv(P[c]) @ P[q]
    dt, dr = lvo.relative_error(v.T, gt)
    print(f"revisit on the device: error {dt:.4f} m {math.degrees(dr):.4f} deg, fitness {v.fitness:.4f}, rmse {v.rmse:.4f}")
    assert v.accepted and dt < REVISIT_BOUND[0] and dr < REVISIT_BOUND[1]
    for q, c, name in ((5, 2, "clipped at 0"), (F - 4, F - 2, "clipped at F - 1")):
        guess = np.linalg.inv(P[c]) @ P[q] @ se3([0.3, -0.2, 0.0, 0.0, 0.0, 0.02])
        w = check_against_the_oracle(route_db, F, P, q, c, guess, cfg, name)
        assert w.termination == w.CONVERGED


@pytest.mark.gpu
def test_gpu_revisit_result_is_a_pose_graph_edge(route, route_db):
    P, scans, _ = route
    q, c = REVISIT
    v = route_db.loop_verify_submap(q, c, yaw=math.radians(-96.0))
    old = route_db.loop_verify(q, c, yaw=math.radians(-96.0))
    gt = np.linalg.inv(P[c]) @ P[q]
    e_new, e_old = lvo.relative_error(v.T, gt)[0], lvo.relative_error(old.T, gt)[0]
    print(f"revisit: scan to scan {e_old:.4f} m fitness {old.fitness:.4f}; submap {e_new:.4f} m fitness {v.fitness:.4f}")
    assert v.accepted and e_new < REVISIT_BOUND[0] and e_new < e_old / 8
    far = int(np.argmax([np.hypot(*(p[:2, 3] - P[q][:2, 3])) for p in P[:60]]))
    assert not route_db.loop_verify_submap(q, far, yaw=math.radians(-96.0)).accepted
    route_db.pose_graph_add_loop(v)
    assert route_db.pose_graph_size() == (len(scans), 1)
    res = route_db.pose_graph_optimize()
    assert res.loop_edges == 1 and res.final_cost <= res.initial_cost
    # the nodes a verification reads are the odometry poses, whatever was optimised since
    again = route_db.loop_verify_submap(q, c, yaw=math.radians(-96.0))
    assert same_bits(again.T, v.T) and again.fitness == v.fitness
    route_db.pose_graph_reset()
    for p in P:
        route_db.pose_graph_add_node(p)


def world_db_clouds():
    """seven views of one structured world along a gentle curve, frame 3 empty; the last one revisits frame 2's place"""
    world = structured_cloud(6)
    rng = np.random.default_rng(8)
    poses = [se3([0.8 * j, 0.1 * j, 0.0, 0.0, 0.0, 0.03 * j]) for j in range(6)]
    poses.append(poses[2] @ se3([0.3, -0.2, 0.02, 0.004, -0.003, 0.05]))
    clouds = [apply4(np.linalg.inv(T), world) + rng.normal(0, 0.01, world.shape) for T in poses]
    clouds[3] = np.zeros((0, 3))
    return poses, clouds


@pytest.mark.gpu
def test_gpu_window_with_an_empty_keyframe_k0_and_an_empty_target_are_the_oracles():
    poses, clouds = world_db_clouds()
    r = new_db(clouds, poses, half_window=2)
    cfg = lso.config(half_window=2)
    guess = np.linalg.inv(poses[2]) @ poses[6] @ se3([0.5, 0.4, 0.0, 0.0, 0.0, -0.04])
    v = check_against_the_oracle(r, 7, poses, 6, 2, guess, cfg, "empty keyframe in the window")
    dt, dr = lvo.relative_error(v.T, np.linalg.inv(poses[2]) @ poses[6])
    assert v.accepted and dt < 0.02 and dr < 1e-3, (dt, dr)
    r.loop_verify_submap_enable(half_window=0)                     # allowed on a filled database
    check_against_the_oracle(r, 7, poses, 6, 2, guess, lso.config(half_window=0), "k = 0")
    assert same_bits(r.loop_verify_submap_target()[0], r.loop_keyframe(2))
    e = check_against_the_oracle(r, 7, poses, 6, 3, guess, lso.config(half_window=0), "empty target")
    assert e is None and len(r.loop_verify_submap_target()[0]) == 0
    w = r.loop_verify_submap(3, 2, guess)                          # an empty query
    assert w.termination == w.EMPTY and not w.accepted and w.n_candidate_points == len(r.loop_keyframe(2))
    r.close()


@pytest.mark.gpu
def test_gpu_existing_calls_keep_their_bits_and_runs_are_reproducible():
    """with submap verification on and used: loop results, keyframes and loop_verify as without it; two runs the same
    bits; a scratch grown from a small first run gives the bits of one sized by the large run at once"""
    import tloam_b200
    poses, clouds = world_db_clouds()
    guess = np.linalg.inv(poses[2]) @ poses[6] @ se3([0.5, 0.4, 0.0, 0.0, 0.0, -0.04])
    runs = []
    for mode in ("off", "on", "on", "grown"):
        r = tloam_b200.LocalRegistration()
        r.loop_enable(exclude_recent=2)
        r.loop_verify_enable()
        if mode != "off":
            r.loop_verify_submap_enable(half_window=2)
            r.pose_graph_enable()
        res, launches = [], []
        for k, p in enumerate(clouds):
            n0 = r.launch_count()
            r.loop_add(p)
            launches.append(r.launch_count() - n0)
            res.append(r.loop_result())
            if mode != "off":
                r.pose_graph_add_node(poses[k])
        out = dict(res=res, launches=launches)
        if mode == "grown":
            r.loop_verify_submap_enable(half_window=0)
            r.loop_verify_submap(6, 0, guess)
            r.loop_verify_submap_enable(half_window=2)
        if mode != "off":
            s = r.loop_verify_submap(6, 2, guess)
            out["s"] = (s, r.loop_verify_submap_target(), [r.loop_verify_submap_matches(k) for k in range(s.iterations + 1)])
        out["v"] = r.loop_verify(6, 2, guess)
        out["m"] = [r.loop_verify_matches(k) for k in range(out["v"].iterations + 1)]
        out["kf"] = [r.loop_keyframe(k) for k in range(7)]
        runs.append(out)
        r.close()
    off = runs[0]
    for x in runs[1:]:
        assert x["res"] == off["res"] and x["launches"] == off["launches"]
        assert all(same_bits(a, b) for a, b in zip(x["kf"], off["kf"]))
        a, b = x["v"], off["v"]
        assert same_bits(a.T, b.T) and (a.fitness, a.rmse, a.inliers, a.iterations, a.termination) == \
            (b.fitness, b.rmse, b.inliers, b.iterations, b.termination)
        assert all(np.array_equal(i, j) and same_bits(d, e) for (i, d), (j, e) in zip(x["m"], off["m"]))
    first = runs[1]["s"]
    for x in runs[2:]:
        (a, ta, ma), (b, tb, mb) = first, x["s"]
        assert same_bits(a.T, b.T) and (a.fitness, a.rmse, a.inliers, a.iterations, a.termination) == \
            (b.fitness, b.rmse, b.inliers, b.iterations, b.termination)
        assert all(same_bits(np.asarray(u, dtype=np.float64), np.asarray(w, dtype=np.float64)) for u, w in zip(ta, tb))
        assert all(np.array_equal(i, j) and same_bits(d, e) for (i, d), (j, e) in zip(ma, mb))


@pytest.mark.gpu
def test_gpu_mapping_loop_is_bit_identical_with_submap_verification_on():
    """test_loop_verify.mapping_loop's chained loop with a chained pose-graph node per frame and a submap verification
    in the middle of it: the odometry, the map, the loop results and the keyframes keep their bits"""
    import tloam_b200
    from test_deskew import loop_scans
    from test_loop_closure import process_packed
    scans = loop_scans()
    outs = []
    for on in (False, True):
        r = tloam_b200.LocalRegistration(fitness_thres=0.3)
        r.enable_global_map()
        r.loop_enable(exclude_recent=2)
        r.loop_verify_enable()
        r.pose_graph_enable()
        if on:
            r.loop_verify_submap_enable(half_window=1)
        poses, results, sub = [], [], None
        for k, a in enumerate(scans):
            process_packed(r, a)
            if k == 0:
                r.submap_init_frame()
            else:
                r.scan_matching_predicted_async()
                r.submap_update_frame_chained()
                r.global_map_append_frame()
            r.loop_add_frame()
            r.pose_graph_add_node()
            if k:
                poses.append(r.get_result())
            results.append(r.loop_result())
            if on and k == len(scans) // 2:
                sub = r.loop_verify_submap(k, 1)
        outs.append(dict(poses=poses, map=r.global_map(), frames=r.global_map_frames(), loop=results,
                         kf=[r.loop_keyframe(k) for k in range(len(scans))], v=r.loop_verify(len(scans) - 1, 0),
                         nodes=r.pose_graph_size()))
        if on:
            last = r.loop_verify_submap(len(scans) - 1, 0)
            print(f"mapping loop: submap verification {last.n_query_points} x {last.n_candidate_points} rows, termination "
                  f"{last.termination}, fitness {last.fitness:.4f}; mid-loop termination {sub.termination}")
            assert last.n_candidate_points == len(outs[-1]["kf"][0]) + len(outs[-1]["kf"][1])
        r.close()
    off, on = outs
    assert len(off["poses"]) == len(on["poses"]) and all(np.array_equal(a, b) for a, b in zip(off["poses"], on["poses"]))
    assert same_bits(off["map"], on["map"]) and np.array_equal(off["frames"], on["frames"]) and off["loop"] == on["loop"]
    assert all(same_bits(a, b) for a, b in zip(off["kf"], on["kf"])) and off["nodes"] == on["nodes"]
    a, b = off["v"], on["v"]
    assert same_bits(a.T, b.T) and (a.fitness, a.rmse, a.inliers, a.iterations) == (b.fitness, b.rmse, b.inliers, b.iterations)


@pytest.mark.gpu
def test_gpu_loop_verify_submap_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    res = _lib.LoopVerifyResult()
    n = C.c_size_t(0)
    dbuf = np.zeros(3 * 200000)
    dp = dbuf.ctypes.data_as(C.POINTER(C.c_double))
    ibuf = np.zeros(200000, dtype=np.int32)
    ip = ibuf.ctypes.data_as(C.POINTER(C.c_int))
    cp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))         # noqa: E731

    def cfg(**kw):
        c = _lib.LoopVerifySubmapConfig()
        L.tloam_b200_loop_verify_submap_default_config(C.byref(c))
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    # without loop verification: NOT_READY everywhere
    assert L.tloam_b200_loop_verify_submap_enable(h, C.byref(cfg())) == _lib.ERR_NOT_READY
    r.loop_enable(exclude_recent=0)
    assert L.tloam_b200_loop_verify_submap_enable(h, C.byref(cfg())) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_verify_submap(h, 0, 0, None, None, C.byref(res)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_verify_submap_target(h, None, None, None, None, 0, C.byref(n)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_loop_verify_submap_matches(h, 0, ip, dp, 10, C.byref(n)) == _lib.ERR_NOT_READY
    r.loop_verify_enable()
    assert L.tloam_b200_loop_verify_submap(h, 0, 0, None, None, C.byref(res)) == _lib.ERR_NOT_READY   # on, but not this
    bad = [dict(half_window=-1), dict(half_window=51), dict(normal_radius=0.0), dict(normal_radius=float("nan")),
           dict(min_normal_neighbours=2), dict(max_planarity=0.0), dict(max_planarity=float("inf")),
           dict(corr_dist_coarse=float("inf")), dict(corr_dist_fine=0.0), dict(corr_dist_fine=5.0), dict(eps_translation=0.0),
           dict(eps_rotation=float("nan")), dict(max_fitness=-0.1), dict(max_iterations=0), dict(max_iterations=201)]
    for kw in bad:
        assert L.tloam_b200_loop_verify_submap_enable(h, C.byref(cfg(**kw))) == _lib.ERR_INVALID_ARG, kw
    assert L.tloam_b200_loop_verify_submap_enable(h, None) == _lib.ERR_INVALID_ARG
    poses, clouds = world_db_clouds()
    for p in clouds[:3]:
        r.loop_add(p)
    assert L.tloam_b200_loop_verify_submap_enable(h, C.byref(cfg(half_window=1))) == _lib.OK   # on a filled database
    assert L.tloam_b200_loop_verify_submap_target(h, None, None, None, None, 0, C.byref(n)) == _lib.ERR_NOT_READY   # no run yet
    for q, c in ((3, 0), (0, 3), (-1, 0), (0, -1)):
        assert L.tloam_b200_loop_verify_submap(h, q, c, None, None, C.byref(res)) == _lib.ERR_INVALID_ARG, (q, c)
    assert L.tloam_b200_loop_verify_submap(h, 2, 0, None, None, None) == _lib.ERR_INVALID_ARG
    # device poses: the pose graph is off, then too short
    assert L.tloam_b200_loop_verify_submap(h, 2, 0, None, None, C.byref(res)) == _lib.ERR_NOT_READY
    r.pose_graph_enable()
    r.pose_graph_add_node(poses[0])
    assert L.tloam_b200_loop_verify_submap(h, 2, 0, None, None, C.byref(res)) == _lib.ERR_NOT_READY   # window 0 .. 1, one node
    r.pose_graph_add_node(poses[1])
    assert L.tloam_b200_loop_verify_submap(h, 2, 0, None, None, C.byref(res)) == _lib.OK
    assert L.tloam_b200_loop_verify_submap(h, 0, 2, None, None, C.byref(res)) == _lib.ERR_NOT_READY   # window 1 .. 2
    # host poses need no pose graph; a pose that is not rigid, or such a guess
    hp = np.ascontiguousarray(np.array(poses[1:3]).transpose(0, 2, 1))
    assert L.tloam_b200_loop_verify_submap(h, 0, 2, None, cp(hp), C.byref(res)) == _lib.OK
    assert res.n_candidate_points > 0 and res.query == 0 and res.candidate == 2
    hb = hp.copy()
    hb[1, 2, 2] = 2.0
    assert L.tloam_b200_loop_verify_submap(h, 0, 2, None, cp(hb), C.byref(res)) == _lib.ERR_BAD_POSE
    for T in (np.diag([1.0, 1.0, 2.0, 1.0]), np.diag([1.0, 1.0, -1.0, 1.0]), np.full((4, 4), np.nan)):
        g = np.asfortranarray(T).ravel(order="F").copy()
        assert L.tloam_b200_loop_verify_submap(h, 0, 2, cp(g), cp(hp), C.byref(res)) == _lib.ERR_BAD_POSE
    v = r.loop_verify_submap(0, 2, poses=poses[1:3])
    assert v.iterations >= 1
    assert L.tloam_b200_loop_verify_submap_matches(h, v.iterations + 1, ip, dp, 200000, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_verify_submap_matches(h, -1, ip, dp, 200000, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_loop_verify_submap_matches(h, 0, ip, dp, 1, C.byref(n)) == _lib.ERR_INVALID_ARG and n.value > 1
    assert L.tloam_b200_loop_verify_submap_target(h, dp, None, None, None, 1, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert n.value == v.n_candidate_points
    assert L.tloam_b200_loop_verify_submap_target(h, dp, None, None, ip, 200000, None) == _lib.ERR_INVALID_ARG
    r.loop_reset()                                                 # empties the keyframes, both verifications stay on
    assert L.tloam_b200_loop_verify_submap_target(h, None, None, None, None, 0, C.byref(n)) == _lib.ERR_NOT_READY
    r.loop_add(np.zeros((0, 3)))
    r.loop_add(clouds[0])
    e = r.loop_verify_submap(0, 1, poses=poses[0:2])
    assert e.termination == e.EMPTY and not e.accepted and e.fitness == math.inf and e.iterations == 0
    assert L.tloam_b200_loop_verify_submap_matches(h, 0, ip, dp, 10, C.byref(n)) == _lib.ERR_INVALID_ARG   # no pass
    r.loop_enable()                                                # turns both verifications off
    assert L.tloam_b200_loop_verify_submap(h, 0, 0, None, None, C.byref(res)) == _lib.ERR_NOT_READY
    r.loop_verify_enable()
    assert L.tloam_b200_loop_verify_submap(h, 0, 0, None, None, C.byref(res)) == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_loop_verify_submap_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("loop_verify_submap_driver", "front_end_b200.hpp")
    world = structured_cloud(5)
    rng = np.random.default_rng(12)
    step = 0.75
    places = [np.array([step * k, 0.0, 0.0]) for k in range(9)] + [np.array([step * 2 + 0.2, 0.1, 0.0])]
    scans = [world - p + rng.normal(0, 0.01, world.shape) for p in places]
    path = os.path.join(os.path.dirname(exe), "loop_verify_submap_raw.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path, "4", "2", repr(step)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [l.split() for l in res.stdout.strip().split("\n")]
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=4)
    r.loop_verify_enable()
    r.loop_verify_submap_enable(half_window=2)
    r.pose_graph_enable()
    verified = accepted = 0
    for k, p in enumerate(scans):
        r.loop_add(p)
        T = np.eye(4)
        T[0, 3] = step * k
        r.pose_graph_add_node(T)
        x = r.loop_result()
        g = got[k]
        assert (int(g[0]), int(g[1])) == (x.query, x.candidate)
        if x.candidate >= 0:
            v = r.loop_verify_submap(x.query, x.candidate, yaw=x.yaw)
            assert (int(g[2]), int(g[3]), int(g[4]), bool(int(g[5])), int(g[6])) == \
                (v.iterations, v.termination, v.inliers, v.accepted, v.n_candidate_points)
            assert float(g[7]) == v.fitness and float(g[8]) == v.rmse
            assert np.array_equal(np.array([float(s) for s in g[9:25]]), v.T.ravel(order="F"))
            verified += 1
            if v.accepted:
                r.pose_graph_add_loop(v)
                accepted += 1
    assert verified >= 4 and accepted >= 1 and got[-1] == ["edges", str(accepted)]
    assert r.pose_graph_size() == (len(scans), accepted)
    r.close()
