"""Loop-corrected global map (include/tloam_b200.h "Loop-corrected global map"; k_gmc_* in libtloam_b200_gmc.so): every
map frame's block moved to its pose-graph pose, later appends through the map -> odom correction.
tests/map_correct_oracle.py is the bit-for-bit numpy restatement.

CPU: the restatement's self-checks, the symbols, the new library's kernels, the shim's driver.  GPU: tracking changes no
bit of the map, the correction of the seq 00 / 05 / 08 graphs equals the restatement bit for bit, repeated and chained
corrections, the mapping loop end to end, status codes, the shim."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import map_correct_oracle as mco
import pose_graph_oracle as pgo
import sass_digest
from test_global_map_intensity import same_bits

NEW_SYMBOLS = ["tloam_b200_global_map_correction_enable", "tloam_b200_global_map_correct", "tloam_b200_global_map_frame_poses"]
KERNELS = ("k_gmc_pose", "k_gmc_frames", "k_gmc_points")


def random_pose(rng, t=20.0, a=0.5):
    return pgo.exp4(np.concatenate([rng.normal(0, t, 3), rng.normal(0, a, 3)]))


def synthetic_frame(rng, n, extent=40.0):
    """n points spread over a cube (about one per 1 m voxel), a few non-finite rows"""
    p = rng.uniform(-extent, extent, (n, 3))
    p[rng.choice(n, max(n // 200, 1), replace=False)] = np.nan
    return p


def synthetic_map(rng, n_frames, pts=500):
    """blocks of distinct points at random poses: (points, offsets, O, P = O)"""
    blocks = [rng.uniform(-30, 30, (pts + int(rng.integers(0, 50)), 3)) for _ in range(n_frames)]
    offsets = np.concatenate([[0], np.cumsum([len(b) for b in blocks])])
    O = np.array([random_pose(rng) for _ in range(n_frames)])
    return np.concatenate(blocks), offsets, O, O.copy()


# ---------------------------------------------------------------------------------------------------------------------
def test_oracle_identity_moves_nothing():
    rng = np.random.default_rng(1)
    pts, off, O, P = synthetic_map(rng, 30)
    nodes = rng.integers(-1, 30, 30)
    got, gP, M = mco.correct(pts, off, O, P, nodes, [], O)                 # no optimisation: Delta = I everywhere
    assert same_bits(got, pts) and same_bits(gP, P) and same_bits(M, np.eye(4))
    assert same_bits(mco.append_pose(np.eye(4), O[3]), O[3])


def test_oracle_keeps_distances_within_a_frame():
    rng = np.random.default_rng(2)
    pts, off, O, P = synthetic_map(rng, 20)
    T_opt = np.array([random_pose(rng, 1.0, 0.05) @ x for x in O[:15]])
    nodes = np.arange(20)
    nodes[3] = -1
    got, gP, _ = mco.correct(pts, off, O, P, nodes, T_opt, O)
    moved = 0
    for f in range(20):
        a, b = off[f], off[f + 1]
        d0 = np.linalg.norm(pts[a:b] - pts[a], axis=1)
        d1 = np.linalg.norm(got[a:b] - got[a], axis=1)
        assert np.abs(d1 - d0).max() <= 1e-12 * d0.max(), f
        moved += not same_bits(got[a:b], pts[a:b])
    assert moved == 19 and same_bits(gP[3], P[3])
    # every frame bound to a node lands at Delta O_f
    assert np.allclose(gP[0], T_opt[0], atol=1e-9) and np.allclose(gP[16], mco.correction(T_opt, O) @ O[16], atol=1e-9)


def test_oracle_two_corrections_equal_the_second():
    rng = np.random.default_rng(3)
    pts, off, O, P = synthetic_map(rng, 25)
    nodes = np.arange(25)
    T1 = np.array([random_pose(rng, 1.0, 0.05) @ x for x in O[:20]])
    T2 = np.array([random_pose(rng, 1.0, 0.05) @ x for x in O[:22]])
    p1, P1, _ = mco.correct(pts, off, O, P, nodes, T1, O)
    p12, P12, M12 = mco.correct(p1, off, O, P1, nodes, T2, O)
    p2, P2, M2 = mco.correct(pts, off, O, P, nodes, T2, O)
    assert same_bits(P12, P2) and same_bits(M12, M2)
    assert np.abs(p12 - p2).max() <= 1e-12 * np.abs(p2).max()
    again, Pa, _ = mco.correct(p2, off, O, P2, nodes, T2, O)                # the same optimisation twice: no bit moves
    assert same_bits(again, p2) and same_bits(Pa, P2)


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_gmc_library_holds_only_the_new_kernels_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.GMC_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.GMC_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


def test_map_correct_driver_compiles_warning_free():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "mock", "map_correct_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(root, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
def tracked_mapping_loop(scans, track, keep=False):
    """test_pose_graph.graph_mapping_loop with, when track, the map's pose tracking on: every frame after the first is
    appended chained (map frame f is node f + 1), every frame gets a chained node; the launches of every append are
    counted.  keep: the handle stays open and is returned under "r"."""
    import tloam_b200
    from test_loop_closure import process_packed
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()
    if track:
        r.global_map_correction_enable()
    r.loop_enable(exclude_recent=2)
    r.loop_verify_enable()
    r.pose_graph_enable()
    poses, sources, results, launches = [], [], [], []
    for k, a in enumerate(scans):
        process_packed(r, a)
        if k == 0:
            r.submap_init_frame()
        else:
            r.scan_matching_predicted_async()
            r.submap_update_frame_chained()
            n0 = r.launch_count()
            r.global_map_append_frame()
            launches.append(r.launch_count() - n0)
        r.loop_add_frame()
        r.pose_graph_add_node()
        if k:
            poses.append(r.get_result())
        sources.append([r.source_cloud(c) for c in range(4)])
        results.append(r.loop_result())
    out = dict(poses=poses, sources=sources, submap=[r.submap_cloud(c) for c in range(4)], map=r.global_map(),
               frames=r.global_map_frames(), reg=r.registered_scan(), loop=results, launches=launches)
    if track:
        out["O"], out["P"] = r.global_map_frame_poses()
    if keep:
        out["r"] = r
    else:
        r.close()
    return out


@pytest.mark.gpu
def test_gpu_tracking_changes_nothing_in_the_mapping_loop():
    """chained appends: the odometry, the map, the frame table and the registered scan are the untracked bits; one more
    launch per append; O_f is get_result's pose of the frame and P_f its copy"""
    from test_deskew import loop_scans
    from test_loop_closure import assert_same_odometry
    scans = loop_scans()
    on, off = tracked_mapping_loop(scans, True), tracked_mapping_loop(scans, False)
    assert_same_odometry(on, off)
    assert [a - b for a, b in zip(on["launches"], off["launches"])] == [1] * (len(scans) - 1)
    assert len(on["O"]) == len(scans) - 1
    for f in range(len(scans) - 1):
        assert same_bits(on["O"][f], on["poses"][f]) and same_bits(on["P"][f], on["O"][f]), f


def host_appends(frames, track, capacity=1 << 20):
    """host appends (scan, pose, intensity or None); returns the map, its frame table, intensity, every registered scan,
    the VOXEL_RANGE refusals reported, and with track the frame poses"""
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=capacity)
    if track:
        r.global_map_correction_enable()
    regs, refused = [], 0
    for scan, pose, inten in frames:
        r.global_map_append(scan, pose, intensity=inten)
        regs.append(r.registered_scan())
    try:
        r.global_map_size()
    except tloam_b200.RegistrationError as e:
        assert e.status == _lib.ERR_VOXEL_RANGE
        refused += 1
    out = dict(map=r.global_map(), frames=r.global_map_frames(), regs=regs, refused=refused, growths=r.global_map_capacity()[1])
    out["intensity"] = r.global_map_intensity() if r.global_map_has_intensity() else None
    if track:
        out["O"], out["P"] = r.global_map_frame_poses()
    r.close()
    return out


def assert_same_map(a, b):
    assert same_bits(a["map"], b["map"]) and np.array_equal(a["frames"], b["frames"])
    assert len(a["regs"]) == len(b["regs"]) and all(same_bits(x, y) for x, y in zip(a["regs"], b["regs"]))
    assert (a["intensity"] is None) == (b["intensity"] is None)
    if a["intensity"] is not None:
        assert same_bits(a["intensity"], b["intensity"])


@pytest.mark.gpu
def test_gpu_tracking_changes_nothing_for_host_appends_with_intensity():
    """host appends with an intensity array and a refused frame (an extent past 2^21 voxels): map, frame table, intensity
    and registered scans are the untracked bits; O_f are the appended poses bit for bit and the refused frame took no slot"""
    rng = np.random.default_rng(11)
    frames = []
    for k in range(12):
        p = synthetic_frame(rng, 3000)
        if k == 5:
            p[7] = [4.0e6, 0.0, 0.0]                                   # refused on the device: its slot is taken by frame 6
        frames.append((p, random_pose(rng), rng.uniform(0, 100, len(p))))
    on, off = host_appends(frames, True), host_appends(frames, False)
    assert_same_map(on, off)
    assert on["refused"] == off["refused"] == 1 and len(on["frames"]) == len(frames)       # 11 frames + the end
    kept = [pose for k, (_, pose, _) in enumerate(frames) if k != 5]
    assert same_bits(on["O"], np.array(kept)) and same_bits(on["P"], on["O"])


@pytest.mark.gpu
def test_gpu_pose_tables_grow_with_the_frame_table():
    """a map that starts at one point and passes the frame table's first 1 024 entries gives the preallocated bits and the
    untracked bits"""
    rng = np.random.default_rng(12)
    frames = [(synthetic_frame(rng, 40, 10.0), random_pose(rng), None) for _ in range(1100)]
    grown, pre, off = host_appends(frames, True, capacity=1), host_appends(frames, True), host_appends(frames, False, capacity=1)
    assert grown["growths"] > 0 and len(grown["frames"]) == 1101
    assert_same_map(grown, pre)
    assert_same_map(grown, off)
    assert same_bits(grown["O"], pre["O"]) and same_bits(grown["P"], pre["P"])
    assert same_bits(grown["O"], np.array([p for _, p, _ in frames]))


def correction_setup(seq, pts=1500, late=20, seed=5):
    """the seq graph of test_pose_graph.seq_graph: a map frame per node appended at O_k (a seeded synthetic scan), plus a
    frame bound to -1 every 500 nodes; the graph is optimised over all but the last `late` nodes, which are added after"""
    import tloam_b200
    from test_pose_graph import loop_result, seq_graph
    G, O, loops = seq_graph(seq)
    rng = np.random.default_rng(seed)
    N = len(O)
    n_opt = N - late
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=N * pts)
    r.global_map_correction_enable()
    r.pose_graph_enable()
    for T in O[:n_opt]:
        r.pose_graph_add_node(T)
    opt_loops = [l for l in loops if l[1] < n_opt]
    for i, j, Z in opt_loops:
        r.pose_graph_add_loop(loop_result(i, j, Z))
    nodes = []
    for k in range(N):
        if k % 500 == 250:
            r.global_map_append(synthetic_frame(rng, pts), random_pose(rng))
            nodes.append(-1)
        r.global_map_append(synthetic_frame(rng, pts), O[k])
        nodes.append(k)
    res = r.pose_graph_optimize()
    for T in O[n_opt:]:
        r.pose_graph_add_node(T)
    return r, np.array(O), loops, np.array(nodes), n_opt, res


def map_state(r):
    O, P = r.global_map_frame_poses()
    return dict(map=r.global_map(), frames=r.global_map_frames(), O=O, P=P)


@pytest.mark.gpu
@pytest.mark.parametrize("seq", ["00", "05", "08"])
def test_gpu_correction_is_the_restatement(seq):
    """the map, P_f and M after global_map_correct equal map_correct_oracle fed with the downloaded T_opt and O, bit for
    bit; frames bound to -1 keep their bits; the offsets and O_f do not change; M is pose_graph_correction's T"""
    import time
    r, O, loops, nodes, n_opt, res = correction_setup(seq)
    assert res.termination != pgo.NO_LOOPS
    before = map_state(r)
    T_opt = r.pose_graph_poses(0, n_opt)
    t0 = time.perf_counter()
    r.global_map_correct(nodes)
    t_dev = time.perf_counter() - t0
    after = map_state(r)
    t0 = time.perf_counter()
    want, want_P, want_M = mco.correct(before["map"], before["frames"], before["O"], before["P"], nodes, T_opt, O)
    t_np = time.perf_counter() - t0
    print(f"seq {seq}: {len(nodes)} frames, {len(want)} points, {res}; correct {t_dev * 1e3:.2f} ms (host clock), "
          f"restatement {t_np:.2f} s")
    assert same_bits(after["O"], before["O"]) and np.array_equal(after["frames"], before["frames"])
    assert same_bits(after["P"], want_P)
    bad = np.nonzero(~np.all(after["map"].view(np.uint64) == want.view(np.uint64), axis=1))[0]
    assert bad.size == 0, (bad.size, bad[:5])
    off = before["frames"]
    for f in np.nonzero(nodes < 0)[0]:
        assert same_bits(after["map"][off[f]:off[f + 1]], before["map"][off[f]:off[f + 1]]) and same_bits(after["P"][f],
                                                                                                            before["P"][f])
    assert not same_bits(after["map"], before["map"])
    # M: the correction pose_graph_correction returns, bit for bit, and the pose of the next append is M X
    C_ = r.pose_graph_correction()
    assert same_bits(want_M, C_)
    X = pgo.exp4([1.0, 2.0, 0.5, 0.01, -0.02, 0.3])
    r.global_map_append(synthetic_frame(np.random.default_rng(9), 200), X)
    Ox, Px = r.global_map_frame_poses(len(nodes), 1)
    assert same_bits(Ox[0], X) and same_bits(Px[0], mco.append_pose(C_, X))
    r.close()


@pytest.mark.gpu
def test_gpu_repeated_and_chained_corrections():
    """correcting twice from one optimisation moves no bit; after another loop and optimisation the correction equals the
    restatement applied from the current P_f; a host append after it lands at M O_f, its registered scan and its block
    are those of an untracked map appended at M O_f"""
    import tloam_b200
    from test_pose_graph import loop_result, seq_graph
    G, O, loops = seq_graph("05")
    O, loops = np.array(O[:1500]), [x for x in loops if x[1] < 1500]
    rng = np.random.default_rng(21)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_correction_enable()
    r.pose_graph_enable()
    for k, T in enumerate(O):
        r.pose_graph_add_node(T)
        r.global_map_append(synthetic_frame(rng, 800), T)
    half = len(loops) // 2
    assert half >= 1
    for i, j, Z in loops[:half]:
        r.pose_graph_add_loop(loop_result(i, j, Z))
    nodes = np.arange(len(O))
    r.pose_graph_optimize()
    r.global_map_correct(nodes)
    once = map_state(r)
    n0 = r.launch_count()
    r.global_map_correct(nodes)
    twice = map_state(r)
    assert r.launch_count() - n0 == 2
    assert same_bits(twice["map"], once["map"]) and same_bits(twice["P"], once["P"])
    for i, j, Z in loops[half:]:
        r.pose_graph_add_loop(loop_result(i, j, Z))
    r.pose_graph_optimize()
    T_opt = r.pose_graph_poses()
    r.global_map_correct(nodes)
    third = map_state(r)
    want, want_P, want_M = mco.correct(once["map"], once["frames"], once["O"], once["P"], nodes, T_opt, O)
    assert same_bits(third["P"], want_P) and same_bits(third["map"], want)
    assert not same_bits(third["map"], once["map"])
    # a later host append: P = M X, registered scan and block as an untracked map's append at M X
    X = O[-1] @ pgo.exp4([0.8, 0.0, 0.0, 0.0, 0.0, 0.01])
    scan = synthetic_frame(rng, 1000)
    r.global_map_append(scan, X)
    Ox, Px = r.global_map_frame_poses(len(O), 1)
    P_want = mco.append_pose(want_M, X)
    assert same_bits(Ox[0], X) and same_bits(Px[0], P_want) and not same_bits(P_want, X)
    ref = tloam_b200.LocalRegistration()
    ref.enable_global_map()
    ref.global_map_append(scan, P_want)
    assert same_bits(r.registered_scan(), ref.registered_scan())
    off = r.global_map_frames()
    assert same_bits(r.global_map(off[-2], off[-1] - off[-2]), ref.global_map())
    ref.close()
    r.close()


def mean_nn(a, b):
    from scipy.spatial import cKDTree
    return float(np.mean(cKDTree(b).query(a)[0]))


@pytest.mark.gpu
def test_gpu_mapping_loop_end_to_end():
    """the seven packed frames of test_deskew.loop_scans through the four-call mapping loop with detection, verification
    and the graph, node[f] = f + 1: after global_map_correct the query frame's block lies closer to the candidate's, and
    P_cand^-1 P_query is within the verification bound of the ground truth; a chained append after it lands at M O_f"""
    import tloam_b200
    from test_deskew import loop_scans
    from test_loop_closure import process_packed
    from test_loop_verify import REVISIT_BOUND
    from tloam_b200 import synth
    scans = loop_scans()
    out = tracked_mapping_loop(scans, True, keep=True)
    r = out["r"]
    last = out["loop"][-1]
    v = r.loop_verify(last.query, last.candidate, yaw=last.yaw)
    assert v.accepted and v.query == len(scans) - 1 and 1 <= v.candidate <= v.query - 2
    r.pose_graph_add_loop(v)
    res = r.pose_graph_optimize()
    assert res.termination == res.CONVERGED
    nodes = np.arange(1, len(scans))
    fq, fc = v.query - 1, v.candidate - 1
    off = r.global_map_frames()
    block = lambda m, f: m[off[f]:off[f + 1]]
    m0 = r.global_map()
    r.global_map_correct(nodes)
    m1 = r.global_map()
    O, P = r.global_map_frame_poses()
    before, after = mean_nn(block(m0, fq), block(m0, fc)), mean_nn(block(m1, fq), block(m1, fc))
    truth = [synth.se3_exp(np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k + 0.001 * (k % 2)])) if k else np.eye(4)
             for k in range(len(scans))]
    gt = np.linalg.inv(truth[v.candidate]) @ truth[v.query]
    err = pgo.relative_error(pgo.inv_mul(P[fc], P[fq]), gt)
    print(f"loop {v.query} -> {v.candidate}: {res}; mean nearest-neighbour distance query -> candidate block "
          f"{before:.4f} m -> {after:.4f} m; corrected relative pose {err[0]:.4f} m {err[1]:.2e} rad")
    assert after < before
    assert err[0] < REVISIT_BOUND[0] and err[1] < REVISIT_BOUND[1]
    T_opt = r.pose_graph_poses()
    node_O = np.array([np.eye(4)] + out["poses"])                 # node 0: identity, before the first match
    want, want_P, want_M = mco.correct(m0, off, O, out["P"], nodes, T_opt, node_O)
    assert same_bits(m1, want) and same_bits(P, want_P)
    # a chained append after the correction: O_f = get_result's pose, P_f = M O_f, registered scan = P_f p
    process_packed(r, scans[-1])
    r.scan_matching_predicted_async()
    r.submap_update_frame_chained()
    r.global_map_append_frame()
    pose = r.get_result()
    Ox, Px = r.global_map_frame_poses(len(nodes), 1)
    assert same_bits(Ox[0], pose) and same_bits(Px[0], mco.append_pose(want_M, pose))
    ref = tloam_b200.LocalRegistration()
    ref.enable_global_map()
    process_packed(ref, scans[-1])
    ref.global_map_append_frame(Px[0])
    assert same_bits(r.registered_scan(), ref.registered_scan())
    off = r.global_map_frames()
    assert same_bits(r.global_map(off[-2], off[-1] - off[-2]), ref.global_map())
    ref.close()
    r.close()


@pytest.mark.gpu
def test_gpu_map_correct_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    buf = np.zeros(64)
    bp = buf.ctypes.data_as(C.POINTER(C.c_double))
    nodes = (C.c_longlong * 4)(0, 1, -1, 0)
    assert L.tloam_b200_global_map_correction_enable(None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_correction_enable(h) == _lib.ERR_NOT_READY                # mapping off
    assert L.tloam_b200_global_map_correct(h, nodes, 0) == _lib.ERR_NOT_READY
    assert L.tloam_b200_global_map_frame_poses(h, 0, 0, bp, bp) == _lib.ERR_NOT_READY
    r.enable_global_map()
    assert L.tloam_b200_global_map_correct(h, nodes, 0) == _lib.ERR_NOT_READY                # tracking off
    assert L.tloam_b200_global_map_frame_poses(h, 0, 0, bp, bp) == _lib.ERR_NOT_READY
    rng = np.random.default_rng(4)
    r.global_map_append(synthetic_frame(rng, 100), np.eye(4))
    assert L.tloam_b200_global_map_correction_enable(h) == _lib.ERR_NOT_READY                # not empty
    r.reset_global_map()
    r.global_map_correction_enable()
    assert L.tloam_b200_global_map_correct(h, nodes, 0) == _lib.ERR_NOT_READY                # pose graph off
    r.pose_graph_enable()
    n0 = r.launch_count()
    assert L.tloam_b200_global_map_correct(h, None, 0) == _lib.OK                            # empty map: nothing launched
    assert r.launch_count() == n0
    poses = [random_pose(rng) for _ in range(3)]
    for T in poses:
        r.global_map_append(synthetic_frame(rng, 100), T)
    r.pose_graph_add_node(poses[0])
    r.pose_graph_add_node(poses[1])
    assert L.tloam_b200_global_map_correct(h, None, 3) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_correct(h, nodes, 2) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_correct(h, nodes, 4) == _lib.ERR_INVALID_ARG
    for bad in ((0, 2, -1), (0, 1, -2)):
        assert L.tloam_b200_global_map_correct(h, (C.c_longlong * 3)(*bad), 3) == _lib.ERR_INVALID_ARG, bad
    assert L.tloam_b200_global_map_frame_poses(h, 2, 2, bp, bp) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_frame_poses(h, 4, 0, bp, bp) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_frame_poses(h, 3, 0, bp, bp) == _lib.OK
    assert L.tloam_b200_global_map_frame_poses(h, 1, 2, None, None) == _lib.OK
    m = r.global_map()
    r.global_map_correct([0, 1, -1])                               # before any optimisation: Delta = I, no bit moves
    assert same_bits(r.global_map(), m) and same_bits(r.global_map_frame_poses()[1], np.array(poses))
    r.pose_graph_add_loop(tloam_b200.LoopVerifyResult(query=1, candidate=0, T=pgo.inv_mul(poses[0], poses[1]) @ pgo.exp4(
        [0.5, 0, 0, 0, 0, 0.01]), fitness=0.1, rmse=0.1, inliers=100, n_query_points=100, n_candidate_points=100,
        iterations=3, termination=0, accepted=True))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct([0, 1, -1])
    assert not same_bits(r.global_map(), m)
    r.pose_graph_reset()                                           # no optimisation: Delta = I puts every frame back at O_f
    r.pose_graph_add_node(poses[0])
    r.global_map_correct([0, -1, -1])
    assert same_bits(r.global_map_frame_poses()[1], np.array(poses))
    r.reset_global_map()                                           # keeps tracking on
    assert r.global_map_frame_poses()[0].shape == (0, 4, 4)
    r.enable_global_map()                                          # turns it off
    assert L.tloam_b200_global_map_frame_poses(h, 0, 0, bp, bp) == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_map_correct_shim_matches_the_python_mirror():
    import struct
    import tloam_b200
    from tloam_b200 import synth
    from test_cpp_shim import build_driver
    from test_loop_verify import rz4
    exe = build_driver("map_correct_driver", "front_end_b200.hpp")
    scans = [synth.raw_scan(seed=s, n_az=900) for s in range(6)]
    scans += [scans[1] @ rz4(0.4)[:3, :3].T + [0.3, -0.2, 0.0], scans[3]]
    path = os.path.join(os.path.dirname(exe), "map_correct_raw.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path, "3"], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.strip().split("\n")
    n_pts, n_frames, term = (int(s) for s in lines[0].split())
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_correction_enable()
    r.loop_enable(exclude_recent=3)
    r.loop_verify_enable()
    r.pose_graph_enable()
    edges = 0
    for k, p in enumerate(scans):
        if k:
            r.global_map_append(p)
        r.loop_add(p)
        r.pose_graph_add_node()
        x = r.loop_result()
        if x.candidate >= 0:
            v = r.loop_verify(x.query, x.candidate, yaw=x.yaw)
            if v.accepted:
                r.pose_graph_add_loop(v)
                edges += 1
    res = r.pose_graph_optimize()
    r.global_map_correct(np.arange(1, len(scans)))
    O, P = r.global_map_frame_poses()
    m = r.global_map()
    assert edges >= 1 and (n_pts, n_frames, term) == (len(m), len(scans) - 1, res.termination)
    for f in range(n_frames):
        got = np.array([float(s) for s in lines[1 + f].split()])
        assert np.array_equal(got[:16], O[f].ravel(order="F")) and np.array_equal(got[16:], P[f].ravel(order="F")), f
    got = np.array([[float(s) for s in l.split()] for l in lines[1 + n_frames:]])
    assert same_bits(got, m)
    r.close()
