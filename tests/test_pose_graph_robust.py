"""Robust pose graph (include/tloam_b200.h "Robust pose graph"; k_pgr_* in libtloam_b200_pgr.so, the weighted stages in
libtloam_b200_pg.so): graduated non-convexity with a truncated-least-squares cost over the loop edges.
tests/pose_graph_robust_oracle.py is the CPU restatement.

Outliers are injected into test_pose_graph.seq_graph graphs with a seeded generator: (a) node pairs >= 50 m apart with
Z = I; (b) a true loop's measurement composed with a 2-10 m / 5-30 degree error (aliasing); (c) three (b)-type edges on
adjacent node pairs that agree with each other.  The restatement costs about 1 s per Gauss-Newton step on the 1 700-node
seq-00 sub-graph (71 loops), and a GNC run takes 60-90 steps, so the tests against it use sub-graphs.

CPU: the TLS rule against T-LOAM's updateWeight, the all-inlier stop, the rejection of families (a) and (b), the symbols,
the new library's kernels, the shim's driver.  GPU: the outlier-free seq graphs bit for bit against the plain optimise, the
outlier graphs against the restatement, the full seq-00 graph against ground truth, determinism and growth, the calls that
read the result, status codes, the shim."""
import ctypes as C
import functools
import os
import subprocess

import numpy as np
import pytest

import pose_graph_oracle as pgo
import pose_graph_robust_oracle as pgr
import sass_digest
from test_global_map_intensity import same_bits
from test_pose_graph import POSE_TOL, assert_poses_close, device_graph, loop_pair_error, loop_result, seq_graph

NEW_SYMBOLS = ["tloam_b200_pose_graph_robust_default_config", "tloam_b200_pose_graph_optimize_robust",
               "tloam_b200_pose_graph_loop_weights"]
KERNELS = ("k_pgr_residual", "k_pgr_weights")
# the sub-graphs: the first n nodes of a seq graph and the loops among them
SUB = {"00": 1700, "08": 1500}
FRACTIONS = (0.05, 0.1, 0.2)


def sub_graph(seq, n=None):
    G, O, loops = seq_graph(seq)
    if n is None:
        return G, O, loops
    return G[:n], O[:n], [x for x in loops if x[1] < n]


def outliers(G, loops, fraction, family, seed=7):
    """round(fraction * len(loops)) (at least 1) seeded outlier edges of one family"""
    rng = np.random.default_rng(seed)
    n = max(1, int(round(fraction * len(loops))))
    p = np.array([g[:3, 3] for g in G])

    def error():
        a = rng.normal(size=3)
        u = rng.normal(size=3)
        E = pgo.exp4(np.concatenate([[0.0, 0.0, 0.0], a / np.linalg.norm(a) * np.deg2rad(rng.uniform(5.0, 30.0))]))
        E[:3, 3] = u / np.linalg.norm(u) * rng.uniform(2.0, 10.0)
        return E

    out = []
    while len(out) < n:
        if family == "a":
            i, j = sorted(int(x) for x in rng.choice(len(G), 2, replace=False))
            if np.linalg.norm(p[i] - p[j]) >= 50.0:
                out.append((i, j, np.eye(4)))
        elif family == "b":
            i, j, Z = loops[int(rng.integers(len(loops)))]
            out.append((i, j, Z @ error()))
        else:                                        # (c): three agreeing edges on adjacent node pairs
            i, j, _ = loops[int(rng.integers(len(loops)))]
            E = error()
            for k in range(3):
                if j + k < len(G) and len(out) < n:
                    out.append((i + k, j + k, pgo.inv_mul(G[i + k], G[j + k]) @ E))
    return out


@functools.lru_cache(maxsize=None)
def case(seq, family, fraction):
    """(G, O, true loops, outliers, the restatement's robust run, its plain run, the plain run without outliers)"""
    G, O, loops = sub_graph(seq, SUB.get(seq))
    bad = outliers(G, loops, fraction, family)
    cfg = pgo.config()
    return (G, O, loops, bad, pgr.optimize_robust(O, loops + bad, cfg, pgr.config()), pgo.optimize(O, loops + bad, cfg),
            pgo.optimize(O, loops, cfg))


# ---------------------------------------------------------------------------------------------------------------------
def update_weight(weights, residuals, noise_bound_sq, th1, th2, mu):
    """T-LOAM's LocalRegistration::updateWeight (ref: src/models/registration/registration.cpp:858-876) transcribed
    literally; a zero residual keeps the weight it had, which is 1 at the first update"""
    for i in range(len(residuals)):
        if residuals[i] == 0:
            continue
        if residuals[i] >= th1:
            weights[i] = 0.0
        elif residuals[i] <= th2:
            weights[i] = 1.0
        else:
            weights[i] = np.sqrt(noise_bound_sq * mu * (mu + 1) / residuals[i]) - mu
            assert 0.0 <= weights[i] <= 1.0
    return weights


@pytest.mark.parametrize("mu", [1e-10, 3.7e-6, 0.01, 0.5, 1.0, 1.4 ** 20, 1e6])
def test_tls_rule_is_tloams_update_weight(mu):
    c2 = 16.81
    th1, th2 = (mu + 1) / mu * c2, mu / (mu + 1) * c2
    rho = [0.0, th1, th2, np.nextafter(th1, 0), np.nextafter(th1, np.inf), np.nextafter(th2, 0), np.nextafter(th2, np.inf),
           0.5 * (th1 + th2), c2, 1e-300, 1e300]
    rho += list(np.geomspace(th2 / 4, th1 * 4, 64))
    got = pgr.tls(np.array(rho), mu, c2)
    want = update_weight(np.ones(len(rho)), rho, c2, th1, th2, mu)
    assert same_bits(got, want)
    assert got[0] == 1.0 and got[1] == 0.0 and got[2] == 1.0 and got[4] == 0.0 and got[5] == 1.0


def test_oracle_stops_at_all_inliers_with_the_plain_result():
    """without outliers every true loop's rho is below chi2_threshold after stage 0 (max 9.33 on the seq-00 sub-graph),
    so the run is pose_graph_oracle.optimize bit for bit"""
    G, O, loops = sub_graph("00", SUB["00"])
    cfg = pgo.config()
    want = pgo.optimize(O, loops, cfg)
    got = pgr.optimize_robust(O, loops, cfg, pgr.config())
    rho = pgr.residuals(got["T"], loops, cfg)
    print(f"seq 00[:{SUB['00']}]: {len(loops)} loops, max rho {rho.max():.3f}")
    assert got["gnc_termination"] == pgr.ALL_INLIERS and got["outer_iterations"] == 0 and got["inliers"] == len(loops)
    assert same_bits(got["T"], want["T"]) and np.all(got["weights"] == 1.0)
    for k in ("iterations", "termination", "initial_cost", "final_cost", "step_translation", "step_rotation"):
        assert got[k] == want[k], k


@pytest.mark.parametrize("family", ["a", "b"])
@pytest.mark.parametrize("fraction", FRACTIONS)
def test_oracle_rejects_every_injected_edge(family, fraction):
    """on the seq-00 sub-graph (1 700 nodes, 71 loops; 4 / 7 / 14 outliers) every injected edge ends at w = 0 and every
    true loop at w = 1, and the loop-pair error is the outlier-free optimum's (0.083649 m) within 1e-6 m (measured: equal
    to the printed 6 digits); GNC converges after 41-43 outer steps and 79-84 Gauss-Newton steps for (a), 28 and 59-61
    for (b).  The plain optimise with the same outliers ends at 10.63 m for (a) and 0.398 / 0.520 / 0.583 m for (b)"""
    G, O, loops, bad, r, plain, clean = case("00", family, fraction)
    L = len(loops)
    w = r["weights"]
    e_clean, e_robust, e_plain = (loop_pair_error(T, G, loops) for T in (clean["T"], r["T"], plain["T"]))
    print(f"({family}) {len(bad)} outliers: GNC {r['gnc_termination']} after {r['outer_iterations']} outer steps, "
          f"{r['iterations']} steps; loop-pair error clean {e_clean:.6f}, robust {e_robust:.6f}, plain {e_plain:.4f} m")
    assert r["gnc_termination"] == pgr.CONVERGED
    assert np.all(w[:L] == 1.0) and np.all(w[L:] == 0.0) and (r["inliers"], r["rejected"]) == (L, len(bad))
    assert abs(e_robust - e_clean) <= 1e-6
    assert e_plain > 4 * e_clean


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_pgr_library_holds_only_the_new_kernels_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.PGR_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.PGR_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


def test_pose_graph_robust_driver_compiles_warning_free():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "mock", "pose_graph_robust_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(root, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("seq", ["00", "05", "08"])
def test_gpu_outlier_free_graphs_are_the_plain_optimise_bit_for_bit(seq):
    """stage 0 runs with every weight 1 (sqrt(1) scales by exactly 1.0): poses, costs and iterations are the plain
    optimise's bits; at the default chi2_threshold every true loop is an inlier, so the run stops at ALL_INLIERS"""
    G, O, loops = seq_graph(seq)
    r = device_graph(O, loops)
    plain = r.pose_graph_optimize()
    T_plain, C_plain = r.pose_graph_poses(), r.pose_graph_correction()
    assert np.all(r.pose_graph_loop_weights() == 1.0)
    n0 = r.launch_count()
    got = r.pose_graph_optimize_robust()
    print(f"seq {seq}: {got}, {r.launch_count() - n0} launches")
    assert got.pg == plain and got.gnc_termination == got.ALL_INLIERS and got.outer_iterations == 0
    assert (got.inliers, got.rejected, got.mu_final) == (len(loops), 0, 0.0)
    assert same_bits(r.pose_graph_poses(), T_plain) and same_bits(r.pose_graph_correction(), C_plain)
    w = r.pose_graph_loop_weights()
    assert w.shape == (len(loops),) and np.all(w == 1.0)
    # the plain optimise's launches plus the residual and weight kernels
    assert r.launch_count() - n0 == 2 + 8 * pgo.config()["max_iterations"] + 2
    r.close()


GPU_CASES = [("00", "a", 0.1), ("00", "b", 0.1), ("00", "c", 0.1), ("08", "b", 0.2)]


@pytest.mark.gpu
@pytest.mark.parametrize("seq,family,fraction", GPU_CASES)
def test_gpu_outlier_graphs_are_the_restatement(seq, family, fraction):
    """the weights, outer_iterations and GNC termination equal the restatement's exactly (every final weight is 0 or 1,
    and no injected rho lies within 1e-6 relative of a threshold); the final poses within test_pose_graph's 1e-6 m /
    1e-8 rad and the final weighted cost within 1e-9 relative"""
    G, O, loops, bad, want, _, _ = case(seq, family, fraction)
    r = device_graph(O, loops + bad)
    got = r.pose_graph_optimize_robust()
    w = r.pose_graph_loop_weights()
    print(f"seq {seq} ({family}) {len(bad)} outliers: {got}; restatement {want['outer_iterations']} outer, "
          f"{want['iterations']} steps, final cost {want['final_cost']!r}")
    assert (got.gnc_termination, got.outer_iterations) == (want["gnc_termination"], want["outer_iterations"])
    assert np.array_equal(w, want["weights"]) and set(np.unique(w)) <= {0.0, 1.0}
    assert (got.inliers, got.rejected) == (want["inliers"], want["rejected"])
    assert got.pg.iterations == want["iterations"] and got.pg.termination == want["termination"]
    assert abs(got.pg.final_cost - want["final_cost"]) <= 1e-9 * want["final_cost"], (got.pg.final_cost, want["final_cost"])
    worst = assert_poses_close(r.pose_graph_poses(), want["T"], POSE_TOL)
    print(f"worst pose difference {worst[0]:.2e} m {worst[1]:.2e} rad")
    r.close()


@pytest.mark.gpu
def test_gpu_full_seq00_with_outliers_rejects_them():
    """4 541 nodes, 183 loops and 18 family-(b) outliers: every outlier ends at w = 0, every true loop at w = 1, and the
    loop-pair error is below 0.1 m, as the plain optimise reaches without outliers; the plain optimise with them is not"""
    import time
    G, O, loops = seq_graph("00")
    bad = outliers(G, loops, 0.1, "b")
    r = device_graph(O, loops + bad)
    plain = r.pose_graph_optimize()
    e_plain = loop_pair_error(r.pose_graph_poses(), G, loops)
    t0 = time.perf_counter()
    got = r.pose_graph_optimize_robust()
    dt = time.perf_counter() - t0
    w = r.pose_graph_loop_weights()
    e = loop_pair_error(r.pose_graph_poses(), G, loops)
    print(f"seq 00 + {len(bad)} outliers: {got}; {dt:.2f} s; loop-pair error plain {e_plain:.4f} m ({plain.iterations} "
          f"iterations), robust {e:.4f} m")
    assert got.gnc_termination == got.CONVERGED
    assert np.all(w[:len(loops)] == 1.0) and np.all(w[len(loops):] == 0.0)
    assert e < 0.1 < e_plain
    r.close()


@pytest.mark.gpu
def test_gpu_runs_are_bit_reproducible_and_a_grown_store_gives_the_preallocated_bits():
    G, O, loops = sub_graph("08", SUB["08"])
    E = loops + outliers(G, loops, 0.1, "b")
    runs = []
    for cap in (4096, 4096, 1):
        r = device_graph(O, E, initial_capacity_nodes=cap)
        a = r.pose_graph_optimize_robust()
        T, w = r.pose_graph_poses(), r.pose_graph_loop_weights()
        b = r.pose_graph_optimize_robust()                           # restarts from the odometry poses
        runs.append((a, T, w))
        assert a == b and same_bits(r.pose_graph_poses(), T) and same_bits(r.pose_graph_loop_weights(), w)
        r.close()
    assert runs[0][0].rejected > 0
    for a, T, w in runs[1:]:
        assert a == runs[0][0] and same_bits(T, runs[0][1]) and same_bits(w, runs[0][2])


@pytest.mark.gpu
def test_gpu_download_correction_and_map_correct_read_the_robust_run():
    """after a robust run: pose_graph_correction and global_map_correct equal map_correct_oracle fed with the downloaded
    robust poses, bit for bit, and those poses are the robust run's (not the plain run's)"""
    import map_correct_oracle as mco
    import tloam_b200
    from test_map_correct import map_state, synthetic_frame
    G, O, loops = sub_graph("08", SUB["08"])
    E = loops + outliers(G, loops, 0.1, "b")
    rng = np.random.default_rng(5)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=len(O) * 300)
    r.global_map_correction_enable()
    r.pose_graph_enable()
    for T in O:
        r.pose_graph_add_node(T)
        r.global_map_append(synthetic_frame(rng, 300), T)
    for i, j, Z in E:
        r.pose_graph_add_loop(loop_result(i, j, Z))
    r.pose_graph_optimize()
    T_plain = r.pose_graph_poses()
    res = r.pose_graph_optimize_robust()
    assert res.rejected > 0
    T_opt = r.pose_graph_poses()
    assert not same_bits(T_opt, T_plain)
    C_ = r.pose_graph_correction()
    assert same_bits(C_, mco.correction(T_opt, np.array(O)))
    before = map_state(r)
    nodes = np.arange(len(O))
    r.global_map_correct(nodes)
    after = map_state(r)
    want, want_P, want_M = mco.correct(before["map"], before["frames"], before["O"], before["P"], nodes, T_opt, np.array(O))
    assert same_bits(after["map"], want) and same_bits(after["P"], want_P) and same_bits(want_M, C_)
    r.close()


@pytest.mark.gpu
def test_gpu_pose_graph_robust_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.PoseGraphRobustConfig()
    L.tloam_b200_pose_graph_robust_default_config(C.byref(cfg))
    assert (cfg.chi2_threshold, cfg.gnc_factor, cfg.inner_iterations, cfg.max_outer_iterations) == (16.81, 1.4, 2, 100)
    res = _lib.PoseGraphRobustResult()
    w = np.zeros(4)
    wp = w.ctypes.data_as(C.POINTER(C.c_double))
    assert L.tloam_b200_pose_graph_optimize_robust(h, C.byref(cfg), C.byref(res)) == _lib.ERR_NOT_READY
    assert L.tloam_b200_pose_graph_loop_weights(h, 0, 0, wp) == _lib.ERR_NOT_READY
    r.pose_graph_enable()
    assert L.tloam_b200_pose_graph_optimize_robust(h, None, C.byref(res)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_pose_graph_optimize_robust(h, C.byref(cfg), None) == _lib.ERR_INVALID_ARG
    for kw in (dict(chi2_threshold=0.0), dict(chi2_threshold=-1.0), dict(chi2_threshold=float("nan")),
               dict(chi2_threshold=float("inf")), dict(gnc_factor=1.0), dict(gnc_factor=float("nan")),
               dict(inner_iterations=0), dict(inner_iterations=101), dict(max_outer_iterations=0),
               dict(max_outer_iterations=1001)):
        with pytest.raises(tloam_b200.RegistrationError) as e:
            r.pose_graph_optimize_robust(**kw)
        assert e.value.status == _lib.ERR_INVALID_ARG, kw
    for k in range(6):
        r.pose_graph_add_node(pgo.exp4([k, 0, 0, 0, 0, 0.1 * k]))
    n0 = r.launch_count()
    got = r.pose_graph_optimize_robust()                            # no loop edge
    assert got.gnc_termination == got.NO_LOOPS and got.pg.termination == got.pg.NO_LOOPS and r.launch_count() == n0
    assert r.pose_graph_loop_weights().shape == (0,)
    Z = pgo.exp4([1.0, 0, 0, 0, 0, 0.1])
    r.pose_graph_add_loop(loop_result(0, 1, Z))
    r.pose_graph_add_loop(loop_result(2, 5, pgo.exp4([30.0, 0, 0, 0, 0, 1.0])))
    r.pose_graph_add_loop(loop_result(1, 3, pgo.inv_mul(pgo.exp4([1, 0, 0, 0, 0, 0.1]), pgo.exp4([3, 0, 0, 0, 0, 0.3]))))
    assert np.all(r.pose_graph_loop_weights() == 1.0)               # before any optimisation
    r.pose_graph_optimize()
    assert np.all(r.pose_graph_loop_weights() == 1.0)               # after a plain one
    got = r.pose_graph_optimize_robust(max_outer_iterations=1)
    w3 = r.pose_graph_loop_weights()
    assert got.outer_iterations == 1 and got.gnc_termination in (got.CONVERGED, got.OUTER_LIMIT)
    for first, count in ((4, None), (-1, None), (2, 2), (0, -1)):
        with pytest.raises(tloam_b200.RegistrationError) as e:
            r.pose_graph_loop_weights(first, count)
        assert e.value.status == _lib.ERR_INVALID_ARG, (first, count)
    assert L.tloam_b200_pose_graph_loop_weights(h, 2, 2, wp) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_pose_graph_loop_weights(h, 4, 0, wp) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_pose_graph_loop_weights(h, 0, 1, None) == _lib.ERR_INVALID_ARG
    assert same_bits(r.pose_graph_loop_weights(1, 2), w3[1:])
    r.pose_graph_add_loop(loop_result(0, 2, Z))                     # added after the robust run: weight 1
    w4 = r.pose_graph_loop_weights()
    assert same_bits(w4[:3], w3) and w4[3] == 1.0
    r.pose_graph_reset()
    assert r.pose_graph_loop_weights().shape == (0,)
    r.close()


@pytest.mark.gpu
def test_gpu_pose_graph_robust_shim_matches_the_python_mirror():
    import dataclasses
    import struct
    import tloam_b200
    from tloam_b200 import synth
    from test_cpp_shim import build_driver
    from test_loop_verify import rz4
    exe = build_driver("pose_graph_robust_driver", "front_end_b200.hpp")
    scans = [synth.raw_scan(seed=s, n_az=900) for s in range(6)]
    scans += [scans[1] @ rz4(0.4)[:3, :3].T + [0.3, -0.2, 0.0], scans[3]]
    path = os.path.join(os.path.dirname(exe), "pose_graph_robust_raw.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p, dtype=np.float64).tobytes())
    shift = 5.0
    res = subprocess.run([exe, path, "3", str(shift)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [l.split() for l in res.stdout.strip().split("\n")]
    r = tloam_b200.LocalRegistration()
    r.loop_enable(exclude_recent=3)
    r.loop_verify_enable()
    r.pose_graph_enable()
    edges = 0
    for k, p in enumerate(scans):
        r.loop_add(p)
        r.pose_graph_add_node()
        x = r.loop_result()
        acc = 0
        if x.candidate >= 0:
            v = r.loop_verify(x.query, x.candidate, yaw=x.yaw)
            acc = int(v.accepted)
            if v.accepted:
                r.pose_graph_add_loop(v)
                T = v.T.copy()
                T[0, 3] += shift
                r.pose_graph_add_loop(dataclasses.replace(v, T=T))
                edges += 2
        assert [int(s) for s in got[k]] == [x.query, x.candidate, acc]
    out = r.pose_graph_optimize_robust()
    g = got[len(scans)]
    p = out.pg
    assert [int(s) for s in g[:4]] == [p.nodes, p.loop_edges, p.iterations, p.termination] and edges >= 2
    assert (float(g[4]), float(g[5])) == (p.initial_cost, p.final_cost)
    assert [int(g[6]), int(g[7]), float(g[8]), int(g[9]), int(g[10])] == [out.outer_iterations, out.gnc_termination,
                                                                        out.mu_final, out.inliers, out.rejected]
    assert np.array_equal(np.array([float(s) for s in got[len(scans) + 1]]), r.pose_graph_loop_weights())
    print(out, r.pose_graph_loop_weights())
    T = r.pose_graph_poses()
    for k in range(len(scans)):
        assert np.array_equal(np.array([float(s) for s in got[len(scans) + 2 + k]]), T[k].ravel(order="F"))
    assert np.array_equal(np.array([float(s) for s in got[-1]]), r.pose_graph_correction().ravel(order="F"))
    r.close()
