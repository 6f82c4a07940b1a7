"""The merged global map (include/tloam_b200.h "Merged global map"; k_gmm_* in libtloam_b200_gmm.so): the map, or its
static rows, merged into one voxel grid -- VoxelDownSample of the whole map.  tests/global_map_merge_oracle.py is the
bit-for-bit numpy restatement.

CPU: the restatement against a literal transcription of the reference's loop (rows on voxel faces, negative coordinates,
one row, one voxel, signed zero / NaN / Inf intensities, a 2 000-row voxel, the key-range limit), the symbols, the new
library's kernels and its DFMA, the shim's driver.  GPU: merges equal the restatement bit for bit (host appends with and
without intensity at three voxel sizes, a map of more than a million rows, static_only, after a correction, the chained
mapping loop, 2 000-row voxels, a grown map), nothing else changes, status codes, the shim."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

import global_map_merge_oracle as gmo
import map_dynamic_oracle as mdo
import sass_digest
from test_global_map_intensity import same_bits

NEW_SYMBOLS = ["tloam_b200_global_map_merge", "tloam_b200_global_map_merged_download"]
KERNELS = ("k_gmm_bounds", "k_gmm_keys", "k_gmm_hist", "k_gmm_offsets", "k_gmm_scatter", "k_gmm_head_count",
           "k_gmm_head_scatter", "k_gmm_average")


def faces_cloud(rng):
    """rows exactly on voxel faces (voxel 0.5, min -3.25: mb = -3.5, faces at -3.5 + k / 2) and negative coordinates"""
    k = rng.integers(0, 20, (400, 3))
    p = -3.5 + 0.5 * k.astype(np.float64)
    p = np.concatenate([p, rng.uniform(-3.25, 6.0, (400, 3)), [[-3.25, -3.25, -3.25]]])
    return p


def small_clouds():
    rng = np.random.default_rng(5)
    out = []
    p = faces_cloud(rng)
    out.append(("faces", p, 0.5, rng.uniform(0, 100, len(p))))
    out.append(("one row", np.array([[-1.5, 2.25, -7.0]]), 1.0, np.array([42.0])))
    p = rng.uniform(0.1, 0.9, (300, 3)) - 5.0
    out.append(("one voxel", p, 2.0, rng.uniform(-1, 1, len(p))))
    p = rng.uniform(-4, 4, (200, 3))
    inten = rng.uniform(0, 1, len(p))
    inten[::7] = -0.0
    inten[1::7] = 0.0
    inten[3] = np.nan
    inten[50] = np.inf
    inten[51] = -np.inf
    out.append(("signed zero nan inf", p, 1.0, inten))
    # min -20: mb = -20.25, so [9.75, 10.25) is one voxel on every axis
    p = np.concatenate([rng.uniform(9.9, 10.1, (2000, 3)), rng.uniform(-19.9, 20, (500, 3)), [[-20.0, -20.0, -20.0]]])
    p = p[rng.permutation(len(p))]
    out.append(("2000-row voxel", p, 0.5, rng.normal(0, 30, len(p))))
    p = rng.normal(0, 30, (3000, 3))
    out.append(("gaussian 0.3", p, 0.3, None))
    return out


@pytest.mark.parametrize("k", range(6))
def test_oracle_matches_the_literal_transcription(k):
    name, p, voxel, inten = small_clouds()[k]
    xyz, vi = gmo.merge(p, voxel, inten)
    lx, li = gmo.merge_literal(p, voxel, inten)
    assert same_bits(xyz, lx), name
    assert (vi is None) == (inten is None) and (vi is None or same_bits(vi, li)), name
    key, idx = gmo.keys(p, voxel)
    assert idx.min() >= 0 and len(xyz) == len(np.unique(key))
    if name == "one voxel":
        assert len(xyz) == 1
    if name == "2000-row voxel":
        assert np.bincount(np.unique(key, return_inverse=True)[1].reshape(-1)).max() == 2000


def test_empty_cloud_gives_no_voxels():
    xyz, inten = gmo.merge(np.zeros((0, 3)), 1.0, np.zeros(0))
    assert xyz.shape == (0, 3) and inten.shape == (0,)


def test_key_range_limit():
    """the largest index 2^21 - 1 is kept, 2^21 refused (voxel 1: mb = -0.5, index of x = floor(x + 0.5))"""
    top = float((1 << 21) - 1)
    kept = np.array([[0.0, 0.0, 0.0], [top, 1.0, 2.0], [3.0, top, 0.0], [1.0, 2.0, top]])
    xyz, _ = gmo.merge(kept, 1.0)
    assert same_bits(xyz, gmo.merge_literal(kept, 1.0)[0]) and len(xyz) == 4
    key, idx = gmo.keys(kept, 1.0)
    assert idx.max() == (1 << 21) - 1 and key.max() < (1 << 63)
    for d in range(3):
        bad = kept.copy()
        bad[1 + d, d] = top + 1.0
        for f in (gmo.merge, gmo.merge_literal):
            with pytest.raises(gmo.VoxelRangeError):
                f(bad, 1.0)
    with pytest.raises(gmo.VoxelRangeError):
        gmo.merge(np.array([[0.0, 0.0, 0.0], [np.nan, 0.0, 0.0]]), 1.0)


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_gmm_library_holds_only_the_new_kernels_for_sm90a():
    """the eight kernels, sm_90a only.  The only DFMA are those of the correctly rounded division (k_gmm_keys: the index,
    k_gmm_average: the averages); the subtractions and sums stay separate DADD"""
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.GMM_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.GMM_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    sass = subprocess.run([sass_digest.cuobjdump(), "-sass", build.GMM_LIB], capture_output=True, text=True, check=True).stdout
    dfma, dadd, fn = {}, {}, None
    for line in sass.splitlines():
        if "Function :" in line:
            fn = next(k for k in KERNELS if f"{len(k)}{k}E" in line)
            dfma[fn] = dadd[fn] = 0
        elif fn and "DFMA" in line:
            dfma[fn] += 1
        elif fn and "DADD" in line:
            dadd[fn] += 1
    assert all(dfma[k] == 0 for k in KERNELS if k not in ("k_gmm_keys", "k_gmm_average")), dfma
    assert dfma["k_gmm_keys"] > 0 and dfma["k_gmm_average"] > 0, dfma
    assert dadd["k_gmm_keys"] >= 3 and dadd["k_gmm_average"] >= 4, dadd


def test_map_merge_driver_compiles_warning_free():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "mock", "map_merge_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(root, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


# ---- GPU ------------------------------------------------------------------------------------------------------------
VOXELS = (0.3, 1.0, 2.5)


def merged_restatement(r, voxel):
    """the restatement applied to what the existing download calls return"""
    inten = r.global_map_intensity() if r.global_map_has_intensity() else None
    return gmo.merge(r.global_map(), voxel, inten)


def assert_merged(got, want):
    assert same_bits(got[0], want[0]), (got[0].shape, want[0].shape)
    assert (got[1] is None) == (want[1] is None)
    if want[1] is not None:
        assert same_bits(got[1], want[1])


def state_of(r):
    """every observable bit that a merge must leave alone"""
    out = dict(map=r.global_map(), frames=r.global_map_frames(), size=r.global_map_size())
    out["intensity"] = r.global_map_intensity() if r.global_map_has_intensity() else None
    return out


def assert_same_state(a, b):
    assert same_bits(a["map"], b["map"]) and np.array_equal(a["frames"], b["frames"]) and a["size"] == b["size"]
    assert (a["intensity"] is None) == (b["intensity"] is None)
    if a["intensity"] is not None:
        assert same_bits(a["intensity"], b["intensity"])


@pytest.mark.gpu
@pytest.mark.parametrize("intensity", [True, False])
def test_gpu_host_appends_are_the_restatement(intensity):
    """host appends of the ray-cast drive merged at 0.3, 1.0 and 2.5 m; the map's own voxel by default; two merges give
    the same bits; the map is untouched"""
    import tloam_b200
    from test_map_dynamic import ray_cast_frames
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    for scan, pose, inten in ray_cast_frames(14):
        r.global_map_append(scan, pose, intensity=inten if intensity else None)
    before = state_of(r)
    for v in VOXELS:
        got = r.global_map_merged(v)
        assert_merged(got, merged_restatement(r, v))
        assert_merged(r.global_map_merged(v), got)
        assert (got[1] is None) == (not intensity)
        print(f"voxel {v}: {len(before['map'])} map points -> {len(got[0])} voxels")
        assert 0 < len(got[0]) < len(before["map"])
    assert_merged(r.global_map_merged(), merged_restatement(r, 1.0))
    assert_same_state(state_of(r), before)
    r.close()


@pytest.mark.gpu
def test_gpu_million_row_map_is_the_restatement():
    """more than a million rows: several radix passes over many tiles"""
    import tloam_b200
    from test_map_dynamic import pose_of
    rng = np.random.default_rng(11)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(voxel=0.3, initial_capacity=1 << 21)
    for k in range(60):
        p = rng.uniform(-40.0, 40.0, (20000, 3))
        r.global_map_append(p, pose_of(2.0 * k, 0.5 * k, 0.01 * k), intensity=rng.uniform(0, 255, len(p)))
    n = r.global_map_size()[0]
    assert n >= 1_000_000
    for v in VOXELS:
        got = r.global_map_merged(v)
        assert_merged(got, merged_restatement(r, v))
        print(f"voxel {v}: {n} map points -> {len(got[0])} voxels")
    r.close()


@pytest.mark.gpu
def test_gpu_static_only_is_the_restatement_of_the_static_rows():
    import tloam_b200
    from test_map_dynamic import VLP, ray_cast_frames
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_dynamic_enable(**VLP)
    for scan, pose, inten in ray_cast_frames(14):
        r.global_map_append(scan, pose, intensity=inten)
    votes = r.global_map_votes()
    before = state_of(r)
    t, h = votes
    dyn = mdo.dynamic(t, h, mdo.config(**VLP))
    assert dyn.any()
    for v in VOXELS:
        xyz, inten = mdo.static_map(before["map"], before["intensity"], t, h, mdo.config(**VLP))
        assert_merged(r.global_map_merged(v, static=True), gmo.merge(xyz, v, inten))
        assert_merged(r.global_map_merged(v), gmo.merge(before["map"], v, before["intensity"]))
    after = r.global_map_votes()
    assert np.array_equal(after[0], t) and np.array_equal(after[1], h)
    assert_same_state(state_of(r), before)
    r.close()


@pytest.mark.gpu
def test_gpu_merge_after_a_correction_is_the_restatement_of_the_corrected_map():
    import tloam_b200
    from test_map_dynamic import ray_cast_frames
    from test_pose_graph import loop_result
    import pose_graph_oracle as pgo
    frames = ray_cast_frames(8)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_correction_enable()
    r.pose_graph_enable()
    O = []
    for scan, pose, inten in frames:
        r.global_map_append(scan, pose, intensity=inten)
        r.pose_graph_add_node(pose)
        O.append(pose)
    drifted = r.global_map()
    r.pose_graph_add_loop(loop_result(1, 6, pgo.inv_mul(O[1], O[6]) @ pgo.exp4([0.4, -0.2, 0.0, 0.0, 0.0, 0.03])))
    assert r.pose_graph_optimize().termination != pgo.NO_LOOPS
    r.global_map_correct(np.arange(len(frames)))
    moved = r.global_map()
    assert not same_bits(moved, drifted)
    for v in (0.3, 1.0):
        assert_merged(r.global_map_merged(v), gmo.merge(moved, v, r.global_map_intensity()))
    assert same_bits(r.global_map(), moved)
    r.close()


def chained_run(merge_at=None):
    """the four-call mapping loop of test_map_dynamic; merge_at: merge (1 m, and static) after that frame's append"""
    import tloam_b200
    from test_global_map import with_nonfinite
    from test_process_cloud import FE, moved
    from tloam_b200 import synth
    scan0 = synth.raw_scan()
    scans = [with_nonfinite(scan0, 90)] + [with_nonfinite(moved(scan0, np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k]),
                                                                100 + k), 200 + k) for k in range(1, 8)]
    cfg = dict(n_rows=64, fov_down=-25.0, fov_up=3.0, n_cols=900, min_range=2.0)
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()
    r.global_map_dynamic_enable(**cfg)
    poses, launches, mid = [], [], None
    for k, scan in enumerate(scans):
        n0 = r.launch_count()
        r.process_raw_scan(scan, feature=FE)
        if k == 0:
            r.submap_init_frame()
            launches.append(r.launch_count() - n0)
            continue
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        r.global_map_append_frame()
        poses.append(r.get_result())
        launches.append(r.launch_count() - n0)
        if k == merge_at:
            mid = (r.global_map_merged(1.0), r.global_map_merged(1.0, static=True), r.global_map())
    out = dict(poses=poses, launches=launches, mid=mid, map=r.global_map(), frames=r.global_map_frames(),
               reg=r.registered_scan(), votes=r.global_map_votes())
    out["merged"] = r.global_map_merged(1.0)
    out["static"] = r.global_map_static()
    out["merged_static"] = r.global_map_merged(1.0, static=True)
    r.close()
    return out


@pytest.mark.gpu
def test_gpu_chained_mapping_loop_merged_at_the_end():
    """process_raw_scan -> scan_matching_predicted_async -> submap_update_frame_chained -> global_map_append_frame, merged
    in the middle and at the end: poses, map, votes and registered scan are the bits of the loop without the mid-run merge,
    its per-frame launch counts are unchanged, and every merge is the restatement"""
    plain, merged = chained_run(), chained_run(merge_at=4)
    assert all(np.array_equal(a, b) for a, b in zip(merged["poses"], plain["poses"]))
    assert same_bits(merged["map"], plain["map"]) and np.array_equal(merged["frames"], plain["frames"])
    assert same_bits(merged["reg"], plain["reg"])
    assert all(np.array_equal(a, b) for a, b in zip(merged["votes"], plain["votes"]))
    assert merged["launches"] == plain["launches"]
    assert_merged(merged["merged"], gmo.merge(merged["map"], 1.0))
    assert_merged(merged["merged_static"], gmo.merge(merged["static"][0], 1.0))
    m_all, m_static, m_map = merged["mid"]
    assert_merged(m_all, gmo.merge(m_map, 1.0))
    assert len(m_static[0]) <= len(m_all[0]) < len(m_map)
    print(f"chained: {len(merged['map'])} map points -> {len(merged['merged'][0])} voxels, "
          f"{len(merged['merged_static'][0])} static")


@pytest.mark.gpu
def test_gpu_stationary_scan_gives_2000_row_voxels():
    """one scan at one pose appended 2 000 times: every voxel of the merge holds 2 000 rows"""
    import tloam_b200
    from test_map_dynamic import pose_of
    rng = np.random.default_rng(3)
    scan = rng.uniform(-20.0, 20.0, (300, 3))
    inten = rng.uniform(0, 100, len(scan))
    T = pose_of(1.0, -2.0, 0.4, 0.3)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 20)
    for _ in range(2000):
        r.global_map_append(scan, T, intensity=inten)
    m = r.global_map()
    block = len(m) // 2000
    assert len(m) == 2000 * block
    got = r.global_map_merged()
    assert len(got[0]) == block
    assert_merged(got, gmo.merge(m, 1.0, r.global_map_intensity()))
    assert_merged(r.global_map_merged(0.5), gmo.merge(m, 0.5, r.global_map_intensity()))
    r.close()


@pytest.mark.gpu
def test_gpu_merge_between_appends_changes_no_later_append():
    import tloam_b200
    from test_map_dynamic import ray_cast_frames
    frames = ray_cast_frames(8)

    def run(merge):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map()
        regs, launches = [], []
        for k, (scan, pose, inten) in enumerate(frames):
            if merge and k % 2:
                r.global_map_merged(0.7)
            n0 = r.launch_count()
            r.global_map_append(scan, pose, intensity=inten)
            launches.append(r.launch_count() - n0)
            regs.append(r.registered_scan())
        out = state_of(r)
        out.update(regs=regs, launches=launches, merged=r.global_map_merged(0.7))
        r.close()
        return out

    a, b = run(True), run(False)
    assert_same_state(a, b)
    assert all(same_bits(x, y) for x, y in zip(a["regs"], b["regs"])) and a["launches"] == b["launches"]
    assert_merged(a["merged"], b["merged"])


@pytest.mark.gpu
def test_gpu_grown_map_gives_the_preallocated_merge():
    import tloam_b200
    from test_map_dynamic import ray_cast_frames
    frames = ray_cast_frames(10)

    def run(cap):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map(initial_capacity=cap)
        for k, (scan, pose, inten) in enumerate(frames):
            r.global_map_append(scan, pose, intensity=inten)
            if k == 3:
                r.global_map_merged(0.5)                           # the merge buffers grow with the map after this
        out = (r.global_map_merged(0.5), r.global_map_merged(2.5), r.global_map_capacity()[1])
        r.close()
        return out

    grown, pre = run(1), run(1 << 20)
    assert grown[2] >= 3 and pre[2] == 0
    assert_merged(grown[0], pre[0])
    assert_merged(grown[1], pre[1])


@pytest.mark.gpu
def test_gpu_map_merge_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    from test_map_dynamic import VLP, ray_cast_frames
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    n = C.c_size_t(7)
    xyz = np.zeros((4, 3))
    dp = C.POINTER(C.c_double)
    xp = xyz.ctypes.data_as(dp)
    assert L.tloam_b200_global_map_merge(None, 1.0, 0, C.byref(n)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_merge(h, 1.0, 0, C.byref(n)) == _lib.ERR_NOT_READY and n.value == 0   # mapping off
    assert L.tloam_b200_global_map_merged_download(h, 0, 0, xp, None) == _lib.ERR_NOT_READY
    r.enable_global_map()
    assert L.tloam_b200_global_map_merge(h, 1.0, 0, None) == _lib.ERR_INVALID_ARG
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        assert L.tloam_b200_global_map_merge(h, bad, 0, C.byref(n)) == _lib.ERR_INVALID_ARG, bad
    assert L.tloam_b200_global_map_merge(h, 1.0, 1, C.byref(n)) == _lib.ERR_NOT_READY                # removal off
    assert L.tloam_b200_global_map_merged_download(h, 0, 0, xp, None) == _lib.ERR_NOT_READY         # no merge yet
    n.value = 7
    assert L.tloam_b200_global_map_merge(h, 1.0, 0, C.byref(n)) == _lib.OK and n.value == 0        # empty map
    assert L.tloam_b200_global_map_merged_download(h, 0, 0, xp, None) == _lib.OK
    assert L.tloam_b200_global_map_merged_download(h, 0, 1, xp, None) == _lib.ERR_INVALID_ARG
    xyz0, inten0 = r.global_map_merged()
    assert xyz0.shape == (0, 3) and inten0 is None
    frames = ray_cast_frames(3)
    for scan, pose, inten in frames:
        r.global_map_append(scan, pose, intensity=inten)
    assert L.tloam_b200_global_map_merge(h, 1.0, 0, C.byref(n)) == _lib.OK and n.value > 4
    nv = n.value
    assert L.tloam_b200_global_map_merged_download(h, nv, 0, xp, None) == _lib.OK
    assert L.tloam_b200_global_map_merged_download(h, nv, 1, xp, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_merged_download(h, nv - 4, 5, xp, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_merged_download(h, 0, 4, None, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_merged_download(h, nv - 4, 4, xp, None) == _lib.OK              # intensity may be null
    assert same_bits(xyz, r.global_map_merged()[0][nv - 4:])
    # a tiny voxel on a wide map: the key range is refused, and no snapshot is left
    assert L.tloam_b200_global_map_merge(h, 1e-5, 0, C.byref(n)) == _lib.ERR_VOXEL_RANGE and n.value == 0
    assert L.tloam_b200_global_map_merged_download(h, 0, 0, xp, None) == _lib.ERR_NOT_READY
    with pytest.raises(tloam_b200.RegistrationError) as e:
        r.global_map_merged(1e-5)
    assert e.value.status == _lib.ERR_VOXEL_RANGE
    assert r.global_map_size()[0] > 0                                # the map and its flags are untouched
    assert L.tloam_b200_global_map_merge(h, 1.0, 0, C.byref(n)) == _lib.OK
    r.reset_global_map()                                             # drops the snapshot
    assert L.tloam_b200_global_map_merged_download(h, 0, 0, xp, None) == _lib.ERR_NOT_READY
    r.global_map_dynamic_enable(**VLP)
    assert L.tloam_b200_global_map_merge(h, 1.0, 1, C.byref(n)) == _lib.OK and n.value == 0
    for scan, pose, inten in frames:
        r.global_map_append(scan, pose)
    assert L.tloam_b200_global_map_merge(h, 1.0, 1, C.byref(n)) == _lib.OK and n.value > 0
    r.enable_global_map()                                            # drops the snapshot and removal
    assert L.tloam_b200_global_map_merged_download(h, 0, 0, xp, None) == _lib.ERR_NOT_READY
    assert L.tloam_b200_global_map_merge(h, 1.0, 1, C.byref(n)) == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_map_merge_shim_matches_the_python_mirror():
    import tloam_b200
    from test_cpp_shim import build_driver
    from test_map_dynamic import VLP, ray_cast_frames
    exe = build_driver("map_merge_driver", "front_end_b200.hpp")
    frames = ray_cast_frames(8)
    path = os.path.join(os.path.dirname(exe), "map_merge_raw.bin")
    out_path = os.path.join(os.path.dirname(exe), "map_merge_out.bin")
    with open(path, "wb") as fh:
        fh.write(struct.pack("Q", len(frames)))
        for p, T, inten in frames:
            fh.write(np.ascontiguousarray(T.ravel(order="F")).tobytes() + struct.pack("Q", len(p)))
            fh.write(np.ascontiguousarray(p, dtype=np.float64).tobytes() + np.ascontiguousarray(inten).tobytes())
    res = subprocess.run([exe, path, out_path, "0.7", str(VLP["n_rows"]), str(VLP["n_cols"]), repr(VLP["fov_down"]),
                          repr(VLP["fov_up"])], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    n_all, n_static = (int(s) for s in res.stdout.split())
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_dynamic_enable(**VLP)
    for scan, pose, inten in frames:
        r.global_map_append(scan, pose, intensity=inten)
    py = [r.global_map_merged(0.7), r.global_map_merged(0.7, static=True)]
    r.close()
    with open(out_path, "rb") as fh:
        blob = fh.read()
    o = 0
    for want, n_want in zip(py, (n_all, n_static)):
        (n,) = struct.unpack_from("Q", blob, o)
        xyz = np.frombuffer(blob, dtype=np.float64, count=3 * n, offset=o + 8).reshape(-1, 3)
        o += 8 + 24 * n
        (ni,) = struct.unpack_from("Q", blob, o)
        inten = np.frombuffer(blob, dtype=np.float64, count=ni, offset=o + 8)
        o += 8 + 8 * ni
        assert n == n_want == len(want[0]) and ni == n
        assert same_bits(xyz, want[0]) and same_bits(inten, want[1])
    assert 0 < n_static <= n_all
