"""Global registration (include/tloam_b200.h "Global registration"; k_gr_* in libtloam_b200_greg.so): FPFH features, mutual
matches, a RANSAC search and a truncated-least-squares refinement, with no initial guess.
tests/global_registration_oracle.py is the bit-for-bit numpy restatement.

CPU: the restatement's neighbourhoods against scipy's cKDTree, its theta bins against atan2, its mutual matches against a
cKDTree of the features, its Horn fit against an SVD Kabsch and scipy's align_vectors, the sampler, the refinement's
monotone cost, rigid invariance of the features, recovery of large transforms and rejection of an unrelated pair, the
ray-cast revisit with no guess; the symbols, the new library's kernels, every other library's SASS.  GPU: every stage bit
for bit against the restatement through both entry points, the revisit chained into loop_verify, determinism, nothing
else changes, the status codes."""
import ctypes as C
import math
import os
import struct
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree
from scipy.spatial.transform import Rotation

import global_registration_oracle as gro
import loop_verify_oracle as lvo
import sass_digest
from tloam_b200 import synth
from test_global_map_intensity import same_bits

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_global_registration_default_config", "tloam_b200_global_registration_enable",
               "tloam_b200_global_register", "tloam_b200_global_register_loop", "tloam_b200_global_registration_side",
               "tloam_b200_global_registration_correspondences", "tloam_b200_global_registration_hypotheses"]
KERNELS = ("k_gr_orient", "k_gr_spfh", "k_gr_fpfh", "k_gr_match", "k_gr_mutual", "k_gr_hyp", "k_gr_best", "k_gr_refine",
           "k_gr_fitness")
HOT = ("k_gr_match", "k_gr_hyp")
CPU_HYPOTHESES = 4096          # the restatement's hypotheses in the CPU scene tests (the device runs the default 65 536)
# the ray-cast revisit scans[-1] -> scans[10] with no guess: the restatement lands 0.38 m / 1.2 deg from the route's ground
# truth at 8 192 hypotheses (the 16-beam rings and the 0.75 m inlier radius bound it); within loop_verify's 4 m first radius
REVISIT_GLOBAL_BOUND = (0.75, math.radians(3.0))


def rz4(a, t=(0.0, 0.0, 0.0)):
    T = np.eye(4)
    T[:2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
    T[:3, 3] = t
    return T


def apply4(T, p):
    return p @ T[:3, :3].T + T[:3, 3]


def voxel_mean(p, v):
    """a plain voxel-mean down-sample (keypoints for the CPU scene tests; the device's are checked on the GPU)"""
    p = p[np.isfinite(p).all(1)]
    _, inv = np.unique(np.floor(p / v).astype(np.int64), axis=0, return_inverse=True)
    inv = inv.ravel()
    s = np.zeros((inv.max() + 1, 3))
    np.add.at(s, inv, p)
    return s / np.bincount(inv)[:, None]


def pose4(p):
    return rz4(p[2], (p[0], p[1], 0.0))


# ---- the restatement --------------------------------------------------------------------------------------------------
def test_oracle_neighbourhoods_are_the_kdtree_balls():
    rng = np.random.default_rng(1)
    P = np.vstack([rng.uniform(-8, 8, (1500, 3)), np.round(rng.uniform(-4, 4, (300, 3)), 1)])   # grid-aligned rows: ties
    g = gro.lo.grid(P, 1.0)
    valid = rng.random(len(P)) < 0.9
    for r in (0.5, 1.0, 2.5):
        i, v, d2 = gro.neighbour_pairs(g, P, valid, r)
        got = set(zip(i.tolist(), v.tolist()))
        want = set()
        for a, nb in enumerate(cKDTree(P).query_ball_point(P, r * (1 + 1e-9))):
            for b in nb:
                if a != b and valid[a] and valid[b] and 0 < gro._d2(P[a], P[b]) <= r * r:
                    want.add((a, b))
        assert got == want, r
        pos = np.argsort(g["srow"])                             # each row's neighbours in ascending sorted position
        assert all(np.all(np.diff(pos[v[i == a]]) > 0) for a in range(0, len(P), 97))


def test_oracle_theta_bins_are_atan2_bins_away_from_edges():
    rng = np.random.default_rng(2)
    x, y = rng.normal(size=200000), rng.normal(size=200000)
    x[:4], y[:4] = [1.0, -1.0, 0.0, -1.0], [0.0, 0.0, 1.0, -1e-300]
    th = np.arctan2(y, x)
    want = np.clip(np.floor(11 * (th + np.pi) / (2 * np.pi)), 0, 10).astype(np.int64)
    edges = (2.0 * np.arange(12) / 11.0 - 1.0) * np.pi
    far = np.min(np.abs(th[:, None] - edges[None, :]), axis=1) > 1e-12
    got = gro.theta_bin(x, y)
    assert far.sum() > 199000 and np.array_equal(got[far], want[far])


def test_oracle_mutual_matches_are_the_kdtree_mutual_nearest():
    rng = np.random.default_rng(3)
    A, B = rng.random((700, 33)) * 20, rng.random((650, 33)) * 20
    B[:300] = A[:300] + rng.normal(0, 0.3, (300, 33))
    ha, hb = rng.random(700) < 0.95, rng.random(650) < 0.95
    got = gro.mutual(dict(feature=A, has_feature=ha), dict(feature=B, has_feature=hb))
    ia, ib = np.flatnonzero(ha), np.flatnonzero(hb)
    a2b = ib[cKDTree(B[ib]).query(A[ia])[1]]
    b2a = ia[cKDTree(A[ia]).query(B[ib])[1]]
    back = dict(zip(ib.tolist(), b2a.tolist()))
    want = [(a, b) for a, b in zip(ia.tolist(), a2b.tolist()) if back[b] == a]
    assert [tuple(r) for r in got.tolist()] == want and len(want) > 250


def test_oracle_horn_fit_is_the_svd_kabsch_and_align_vectors():
    rng = np.random.default_rng(4)
    for k in range(20):
        R = Rotation.random(random_state=k).as_matrix()
        t = rng.uniform(-10, 10, 3)
        p = rng.uniform(-20, 20, (int(rng.integers(3, 400)), 3))
        q = p @ R.T + t + rng.normal(0, 0.05 * (k % 2), p.shape)
        Rf, tf = gro.fit(p, q)
        cp, cq = p.mean(0), q.mean(0)
        U, _, Vt = np.linalg.svd((p - cp).T @ (q - cq))
        D = np.diag([1, 1, np.sign(np.linalg.det(Vt.T @ U.T))])
        Rk = Vt.T @ D @ U.T
        Ra = Rotation.align_vectors(q - cq, p - cp)[0].as_matrix()
        assert np.abs(Rf - Rk).max() < 1e-12 and np.abs(Rf - Ra).max() < 1e-12, k
        assert np.abs(tf - (cq - Rk @ cp)).max() < 1e-11, k


def test_oracle_sampler_draws_distinct_pairs_and_a_fixed_seed_fixes_them():
    h = np.arange(100000)
    for nc in (3, 4, 7, 1000):
        d = gro.draws(42, h, nc)
        assert d.min() >= 0 and d.max() < nc
        assert np.all((d[:, 0] != d[:, 1]) & (d[:, 0] != d[:, 2]) & (d[:, 1] != d[:, 2])), nc
        assert np.array_equal(d, gro.draws(42, h, nc))
        if nc == 1000:
            assert not np.array_equal(d, gro.draws(43, h, nc))
            assert np.abs(np.bincount(d.ravel(), minlength=nc) / 300.0 - 1).max() < 0.25   # all indices, about evenly


def test_oracle_refinement_never_increases_the_truncated_cost():
    rng = np.random.default_rng(5)
    for k in range(10):
        p = rng.uniform(-15, 15, (400, 3))
        T = rz4(rng.uniform(-np.pi, np.pi), rng.uniform(-5, 5, 3))
        q = apply4(T, p) + rng.normal(0, 0.1, p.shape)
        q[: 150 + 10 * k] = rng.uniform(-15, 15, (150 + 10 * k, 3))          # outliers
        E = T @ rz4(0.05, (0.3, -0.2, 0.0))                                    # a start off by 3 deg and 0.36 m
        *_, costs = gro.refine(p, q, E[:3, :3], E[:3, 3], gro.config(max_refine_iterations=50))
        assert all(b <= a * (1 + 1e-12) for a, b in zip(costs, costs[1:])), (k, costs)
        assert costs[-1] < costs[0]


def test_oracle_features_are_invariant_to_a_rigid_motion():
    """the keypoints of an HDL-64E scan, and the same keypoints rotated about the sensor (the viewpoint stays the origin):
    the integer SPFH counts agree except for the pairs that sit within rounding of a bin edge"""
    P = voxel_mean(synth.raw_scan(), 0.5)
    T = np.eye(4)
    T[:3, :3] = Rotation.from_euler("zyx", [2.4, 0.05, -0.03]).as_matrix()
    cfg = gro.config()
    a, b = gro.side(P, cfg), gro.side(apply4(T, P), cfg)
    ok = a["has_feature"]
    assert np.array_equal(a["valid"], b["valid"]) and np.array_equal(a["pairs"], b["pairs"])
    same = np.all(a["spfh"] == b["spfh"], axis=1)
    print(f"{ok.sum()} features, {(~same[ok]).sum()} with a count moved across an edge")
    assert ok.sum() > 1000 and (~same[ok]).sum() <= 0.002 * ok.sum()
    assert np.abs(a["feature"][same] - b["feature"][same]).max() < 1e-6


def recover(P_src, P_tgt, n_hypotheses=CPU_HYPOTHESES, **cfg):
    return gro.run(voxel_mean(P_src, 0.5), voxel_mean(P_tgt, 0.5), gro.config(n_hypotheses=n_hypotheses, **cfg))


@pytest.mark.parametrize("yaw,t", [(math.radians(90), (5.0, 0.0, 0.0)), (math.radians(135), (6.0, -4.0, 0.2)),
                                   (math.radians(180), (-7.0, 7.0, 0.0))])
def test_oracle_recovers_a_large_transform_of_a_noisy_partial_scan(yaw, t):
    """the scan seen from a sensor moved by T (5 - 10 m, 90 - 180 deg), with noise and a 60-degree sector cut away"""
    rng = np.random.default_rng(6)
    P = synth.raw_scan()
    P = P[np.isfinite(P).all(1)]
    T = rz4(yaw, t)
    az = np.arctan2(P[:, 1], P[:, 0])
    Q = P[(az < 0.3) | (az > 0.3 + np.pi / 3)]                                  # partial overlap
    src = apply4(np.linalg.inv(T), Q) + rng.normal(0, 0.02, Q.shape)          # target <- source = T
    r = recover(src, P)
    dt, dr = lvo.relative_error(r["T"], T)
    print(f"yaw {math.degrees(yaw):.0f}: {r['n_correspondences']} pairs, best {r['best_inliers']}, inliers {r['inliers']}, "
          f"fitness {r['fitness']:.3f}, error {dt:.3f} m {math.degrees(dr):.3f} deg")
    assert r["accepted"] and dt < 0.2 and dr < math.radians(1.0)


def test_oracle_recovers_a_map_scene_and_rejects_an_unrelated_pair():
    T = rz4(math.radians(-120), (-6.0, 3.0, 0.0))
    M = np.vstack(synth.make_map(synth.config1()["cfg"], np.eye(4)))
    M = M[np.linalg.norm(M[:, :2], axis=1) < 20]
    src = apply4(np.linalg.inv(T), M[M[:, 0] > -8]) + np.random.default_rng(7).normal(0, 0.02, (int((M[:, 0] > -8).sum()), 3))
    r = recover(src, M)
    dt, dr = lvo.relative_error(r["T"], T)
    print(f"map scene: {r['n_correspondences']} pairs, inliers {r['inliers']}, fitness {r['fitness']:.3f}, "
          f"error {dt:.3f} m {math.degrees(dr):.3f} deg")
    assert r["accepted"] and dt < 0.2 and dr < math.radians(1.0)
    from test_loop_verify import structured_cloud
    u = recover(synth.raw_scan(seed=11), structured_cloud(8))
    print(f"unrelated: inliers {u['inliers']}, fitness {u['fitness']:.3f}")
    assert not u["accepted"]


def route_keypoints():
    from test_loop_closure import route_scans
    poses, scans = route_scans()
    return poses, scans


def test_oracle_aligns_the_ray_cast_revisit_with_no_guess():
    poses, scans = route_keypoints()
    gt = np.linalg.inv(pose4(poses[10])) @ pose4(poses[-1])
    r = recover(scans[-1], scans[10], n_hypotheses=8192)
    dt, dr = lvo.relative_error(r["T"], gt)
    print(f"revisit: {r['n_correspondences']} pairs, inliers {r['inliers']}, error {dt:.3f} m {math.degrees(dr):.3f} deg")
    assert r["accepted"] and dt < REVISIT_GLOBAL_BOUND[0] and dr < REVISIT_GLOBAL_BOUND[1]


# ---- the library ------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_greg_library_holds_only_its_kernels_for_sm90a_and_the_hot_ones_do_not_spill():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.GREG_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.GREG_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.GREG_LIB], capture_output=True, text=True,
                         check=True).stdout.splitlines()
    usage = {k: res[i + 1] for i, l in enumerate(res) for k in HOT if f"{len(k)}{k}E" in l}
    assert len(usage) == len(HOT) and all("STACK:0 " in u for u in usage.values()), usage


def test_every_other_library_keeps_its_sass():
    import json
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_greg.json")))
    assert len(want) == 18 and "libtloam_b200_greg.so" not in want and "libtloam_b200_plan.so" in want
    for lib in want:
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


def test_global_registration_driver_compiles_warning_free():
    """the drop-in (global_registration_b200.hpp) and FrontEndB200's calls, through the mock driver, as C++14"""
    src = os.path.join(ROOT, "tests", "mock", "global_registration_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def gpu_handle(**cfg):
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.global_registration_enable(**cfg)
    return r


def check_run(r, got, cfg, name):
    """every stage of the device's last run against the restatement from the device's own keypoints"""
    S, T = r.global_registration_side(0), r.global_registration_side(1)
    want = gro.run(S["xyz"], T["xyz"], cfg)
    assert got.termination == want["termination"], (name, got, want["termination"])
    if got.termination == gro.EMPTY:
        return want
    for dev, ref in ((S, want["src"]), (T, want["tgt"])):
        assert same_bits(dev["normal"], ref["normal"]) and np.array_equal(dev["valid"], ref["valid"]), name
        assert np.array_equal(dev["spfh"], ref["spfh"]) and np.array_equal(dev["has_feature"], ref["has_feature"]), name
        assert same_bits(dev["feature"], ref["feature"]), name
    assert np.array_equal(r.global_registration_correspondences(), want["corr"]), name
    assert np.array_equal(r.global_registration_hypotheses(), want["hyp"]), name
    assert (got.n_correspondences, got.n_valid_hypotheses, got.best_hypothesis, got.best_inliers, got.inliers,
            got.refine_iterations) == (want["n_correspondences"], want["n_valid_hypotheses"], want["best_hypothesis"],
                                       want["best_inliers"], want["inliers"], want["refine_iterations"]), name
    assert same_bits(got.T, want["T"]) and got.fitness == want["fitness"] and got.inlier_rmse == want["inlier_rmse"], name
    assert got.accepted == want["accepted"]
    assert (got.n_source_features, got.n_target_features) == (want["src"]["has_feature"].sum(), want["tgt"]["has_feature"].sum())
    return want


def host_cases():
    from test_loop_verify import structured_cloud
    P = synth.raw_scan()
    T = rz4(math.radians(135), (6.0, -4.0, 0.2))
    rng = np.random.default_rng(8)
    return [("scan", apply4(np.linalg.inv(T), P[np.isfinite(P).all(1)]) + rng.normal(0, 0.02, (int(np.isfinite(P).all(1).sum()), 3)), P, T),
            ("unrelated", synth.raw_scan(seed=11), structured_cloud(8), None),
            ("few", np.array([[0.0, 0.0, 0.0], [5.0, 0.0, 0.0]]), P, None),
            ("empty", np.zeros((0, 3)), P, None)]


@pytest.mark.gpu
def test_gpu_host_clouds_are_the_restatement_bit_for_bit():
    cfg = gro.config()
    r = gpu_handle()
    for name, src, tgt, T in host_cases():
        got = r.global_register(src, tgt)
        check_run(r, got, cfg, name)
        print(f"{name}: {got.n_source_points} x {got.n_target_points} keypoints, {got.n_correspondences} pairs, "
              f"{got.n_valid_hypotheses} valid, best {got.best_inliers}, inliers {got.inliers}, fitness {got.fitness:.3f}, "
              f"termination {got.termination}")
        if T is not None:
            dt, dr = lvo.relative_error(got.T, T)
            assert got.accepted and dt < 0.2 and dr < math.radians(1.0), (dt, dr)
        if name == "unrelated":
            assert not got.accepted
        if name == "empty":
            assert got.termination == got.EMPTY and np.array_equal(got.T, np.eye(4)) and got.n_source_points == 0
    r.close()


@pytest.mark.gpu
def test_gpu_keypoints_are_the_keyframes_and_the_loop_entry_is_the_restatement():
    """a host cloud's keypoints are bit for bit the loop keyframe of the same cloud; global_register_loop on those
    keyframes gives the host call's bits"""
    import tloam_b200
    from test_loop_verify import structured_cloud
    P, Q = synth.raw_scan(), structured_cloud(6)
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=0)
    r.loop_verify_enable(voxel=0.5)
    r.global_registration_enable()
    r.loop_add(P)
    r.loop_add(Q)
    a = r.global_register(Q, P)
    S, T = r.global_registration_side(0), r.global_registration_side(1)
    assert same_bits(S["xyz"], r.loop_keyframe(1)) and same_bits(T["xyz"], r.loop_keyframe(0))
    b = r.global_register_loop(1, 0)
    assert same_bits(a.T, b.T)
    assert (a.n_correspondences, a.inliers, a.fitness, a.best_hypothesis) == (b.n_correspondences, b.inliers, b.fitness, b.best_hypothesis)
    check_run(r, b, gro.config(), "loop")
    r.close()


@pytest.mark.gpu
def test_gpu_revisit_with_no_guess_then_loop_verify_meets_the_revisit_bound():
    import tloam_b200
    from test_loop_verify import REVISIT_BOUND
    poses, scans = route_keypoints()
    r = tloam_b200.LocalRegistration()
    r.loop_enable()
    r.loop_verify_enable()
    r.global_registration_enable()
    for p in scans:
        r.loop_add(p)
    q, c = len(scans) - 1, 10
    g = r.global_register_loop(q, c)
    gt = np.linalg.inv(pose4(poses[c])) @ pose4(poses[q])
    dt0, dr0 = lvo.relative_error(g.T, gt)
    v = r.loop_verify(q, c, g.T)
    dt, dr = lvo.relative_error(v.T, gt)
    print(f"revisit {q} -> {c}: global {dt0:.3f} m {math.degrees(dr0):.3f} deg ({g.inliers} inliers, fitness {g.fitness:.3f}); "
          f"verified {dt:.3f} m {math.degrees(dr):.4f} deg, fitness {v.fitness:.4f}")
    assert g.accepted and dt0 < REVISIT_GLOBAL_BOUND[0] and dr0 < REVISIT_GLOBAL_BOUND[1]
    assert v.accepted and dt < REVISIT_BOUND[0] and dr < REVISIT_BOUND[1]
    check_run(r, g, gro.config(), "revisit")
    r.close()


@pytest.mark.gpu
def test_gpu_repeated_calls_give_the_same_bits():
    name, src, tgt, _ = host_cases()[0]
    r = gpu_handle(seed=7)
    outs = [r.global_register(src, tgt) for _ in range(3)]
    sides = r.global_registration_side(0)
    hyp = r.global_registration_hypotheses()
    for o in outs[1:]:
        assert same_bits(o.T, outs[0].T) and o.fitness == outs[0].fitness and o.inliers == outs[0].inliers
    r2 = gpu_handle(seed=7)
    o2 = r2.global_register(src, tgt)
    assert same_bits(o2.T, outs[0].T) and np.array_equal(r2.global_registration_hypotheses(), hyp)
    assert same_bits(r2.global_registration_side(0)["feature"], sides["feature"])
    r.close()
    r2.close()


def loop_flow(scans, greg):
    """loop adds, a verification of the last frame against frame 10, and the launch count of each call"""
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(voxel=1.0)
    r.loop_enable()
    r.loop_verify_enable()
    if greg:
        r.global_registration_enable()
    res, launches = [], []
    for k, p in enumerate(scans):
        n0 = r._L.tloam_b200_launch_count(r._h)
        r.loop_add(p)
        r.global_map_append(p, pose=np.eye(4))
        launches.append(r._L.tloam_b200_launch_count(r._h) - n0)
        res.append(r.loop_result())
        if greg and k >= 12 and k % 10 == 0:
            r.global_register_loop(k, 10)
            r.global_register(p, scans[10])
    n0 = r._L.tloam_b200_launch_count(r._h)
    v = r.loop_verify(len(scans) - 1, 10, rz4(math.radians(-96.0)))
    launches.append(r._L.tloam_b200_launch_count(r._h) - n0)
    out = dict(res=res, launches=launches, v=v, map=r.global_map(), kf=r.loop_keyframe(len(scans) - 1))
    r.close()
    return out


@pytest.mark.gpu
def test_gpu_global_registration_changes_nothing_else():
    _, scans = route_keypoints()
    scans = scans[:40] + scans[-1:]
    off, on = loop_flow(scans, False), loop_flow(scans, True)
    assert off["res"] == on["res"] and off["launches"] == on["launches"]
    assert same_bits(off["map"], on["map"]) and same_bits(off["kf"], on["kf"])
    assert same_bits(off["v"].T, on["v"].T) and off["v"].fitness == on["v"].fitness


@pytest.mark.gpu
def test_gpu_global_registration_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    from tloam_b200.registration import RegistrationError
    r = tloam_b200.LocalRegistration()
    P = synth.raw_scan()
    with pytest.raises(RegistrationError) as e:
        r.global_register(P, P)                                     # off
    assert e.value.status == _lib.ERR_NOT_READY
    for bad in (dict(voxel=0.0), dict(feature_radius=3.5), dict(normal_radius=-1.0), dict(n_hypotheses=0),
                dict(n_hypotheses=(1 << 20) + 1), dict(edge_similarity=1.5), dict(min_triangle_area=0.0),
                dict(max_refine_iterations=0), dict(min_fitness=1.5), dict(min_normal_neighbours=2),
                dict(max_correspondence_distance=float("nan"))):
        with pytest.raises(RegistrationError) as e:
            r.global_registration_enable(**bad)
        assert e.value.status == _lib.ERR_INVALID_ARG, bad
    r.global_registration_enable()
    with pytest.raises(RegistrationError) as e:
        r.global_registration_side(0)                               # no run yet
    assert e.value.status == _lib.ERR_NOT_READY
    with pytest.raises(RegistrationError) as e:
        r.global_register_loop(0, 1)                                # loop verification off
    assert e.value.status == _lib.ERR_NOT_READY
    far = np.zeros((50, 3))
    far[:, 0] = np.linspace(0.0, 3.0e6, 50)
    with pytest.raises(RegistrationError) as e:
        r.global_register(far, P)
    assert e.value.status == _lib.ERR_VOXEL_RANGE
    res = _lib.GlobalRegistrationResult()
    assert r._L.tloam_b200_global_register(r._h, None, 5, None, 0, C.byref(res)) == _lib.ERR_INVALID_ARG
    nan = P.copy()
    nan[::3] = np.nan
    got = r.global_register(nan, P)                                 # non-finite rows are dropped
    assert got.n_source_points > 0 and got.termination != got.EMPTY
    assert r.global_register(np.zeros((0, 3)), P).termination == got.EMPTY
    with pytest.raises(RegistrationError) as e:
        r.global_registration_side(2)
    assert e.value.status == _lib.ERR_INVALID_ARG
    r.loop_enable(exclude_recent=0)
    r.loop_verify_enable()
    r.loop_add(P)
    with pytest.raises(RegistrationError) as e:
        r.global_register_loop(0, 1)                                # out of range
    assert e.value.status == _lib.ERR_INVALID_ARG
    r.close()


@pytest.mark.gpu
def test_gpu_global_registration_shim_matches_the_python_mirror():
    """GlobalRegistrationB200::scanMatching / getFitnessScore and FrontEndB200::globalRegister give the Python call's bits"""
    from test_cpp_shim import build_driver
    exe = build_driver("global_registration_driver", "global_registration_b200.hpp")
    d = os.path.dirname(exe)
    in_path, out_path = os.path.join(d, "greg_in.bin"), os.path.join(d, "greg_out.bin")
    _, src, tgt, _ = host_cases()[0]
    src = src[np.isfinite(src).all(1)]
    tgt = tgt[np.isfinite(tgt).all(1)]
    with open(in_path, "wb") as fh:
        for p in (src, tgt):
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p, dtype=np.float64).tobytes())
    run = subprocess.run([exe, in_path, out_path], capture_output=True, text=True)
    assert run.returncode == 0, run.stderr
    r = gpu_handle()
    want = r.global_register(src, tgt)
    r.close()
    assert [int(v) for v in run.stdout.split()] == [want.termination, int(want.accepted), want.inliers]
    blob = open(out_path, "rb").read()
    for k in range(2):
        o = k * (18 * 8 + 3 * 8)
        T = np.frombuffer(blob, dtype=np.float64, count=16, offset=o).reshape(4, 4, order="F")
        fit, rmse = np.frombuffer(blob, dtype=np.float64, count=2, offset=o + 128)
        inl, nc, best = np.frombuffer(blob, dtype=np.int64, count=3, offset=o + 144)
        assert same_bits(T, want.T) and fit == want.fitness and rmse == want.inlier_rmse, k
        assert (inl, nc, best) == (want.inliers, want.n_correspondences, want.best_hypothesis), k
