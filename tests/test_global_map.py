"""Global map of FrontEnd on the device (tloam_b200_global_map_*, ref: src/front_end/front_end.cpp:269-274 with mapping_flag):
each appended raw scan is transformed, voxel-down-sampled on its own and concatenated to a map that stays on the GPU.

CPU: the restatement (tests/global_map_oracle.py) is pinned against an independent numpy form, on frame order, on an empty
frame and on the frame-0 rule; the new symbols are in the header and the binding; the shim compiles as C++14; every kernel
that existed before the global map compiles to the same SASS.  GPU: host-pose appends against the restatement (HDL-64E with
NaN / Inf rows, VLP-16 with near and non-finite rows), a 7-frame chained loop (poses unchanged by mapping, the map equal to
host-pose appends and to the restatement, no growth), determinism, growth, the key-range refusal, status codes, the shim."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from tloam_b200 import synth
import global_map_oracle as gmo
import process_cloud_oracle as pco
import sass_digest
from test_process_cloud import FE, moved

NEW_SYMBOLS = ["tloam_b200_global_map_default_config", "tloam_b200_global_map_enable", "tloam_b200_global_map_reset",
               "tloam_b200_global_map_append", "tloam_b200_global_map_append_chained", "tloam_b200_global_map_append_frame",
               "tloam_b200_global_map_append_frame_chained", "tloam_b200_global_map_size", "tloam_b200_global_map_download",
               "tloam_b200_global_map_frame_offsets", "tloam_b200_global_map_capacity", "tloam_b200_registered_scan_download"]


def numpy_block(registered, voxel):
    """independent form of one frame's block: np.unique over the floor indices of the finite rows, then a group mean"""
    fin = registered[np.isfinite(registered).all(axis=1)]
    if len(fin) == 0:
        return np.zeros((0, 3))
    idx = np.floor((fin - (fin.min(0) - 0.5 * voxel)) / voxel).astype(np.int64)
    uniq, inv, cnt = np.unique(idx, axis=0, return_inverse=True, return_counts=True)
    out = np.zeros((cnt.size, 3))
    np.add.at(out, inv.reshape(-1), fin)
    return out / cnt[:, None]


def with_nonfinite(scan, seed):
    """the scan with NaN / Inf rows and a partly-NaN row inserted at random places"""
    rng = np.random.default_rng(seed)
    rows = [np.full((200, 3), np.nan), np.array([[np.inf, 1.0, 0.0], [1.0, np.nan, 2.0], [-np.inf, -np.inf, 5.0]] * 40)]
    out = scan.copy()
    for r in rows:
        out = np.insert(out, np.sort(rng.choice(len(out), len(r), replace=False)), r, axis=0)
    return out


# ---------------------------------------------------------------------------------------------------------------------
def test_restatement_matches_an_independent_numpy_form(oracle):
    rng = np.random.default_rng(4)
    raw = with_nonfinite(synth.raw_scan(n_az=400), 1)
    T = synth.se3_exp([3.0, -1.0, 0.2, 0.01, -0.02, 0.4])
    reg = gmo.transform(raw, T)
    bad = ~np.isfinite(raw).all(axis=1)
    assert bad.sum() == 320 and np.array_equal(~np.isfinite(reg).all(axis=1), bad)
    for voxel in (1.0, 0.37):
        got = gmo.frame_block(oracle, reg, voxel)
        want = numpy_block(reg, voxel)
        assert len(got) > 300 and got.shape == want.shape
        assert np.allclose(got, want, rtol=0, atol=1e-10)
        fin = reg[~bad]
        keys = pco.packed_keys(pco.voxel_indices(got, voxel, fin.min(0)))
        assert np.all(np.diff(keys) > 0)                                    # ascending voxel index
    assert len(gmo.frame_block(oracle, rng.uniform(-5, 5, (10, 3)) * np.nan, 1.0)) == 0


def test_restatement_concatenates_frames_in_call_order_and_keeps_empty_frames(oracle):
    scan = synth.raw_scan(n_az=300)
    regs = [gmo.transform(scan, synth.se3_exp([2.0 * k, 0.1 * k, 0, 0, 0, 0.05 * k])) for k in range(3)]
    regs.insert(1, np.zeros((0, 3)))
    regs.append(np.full((50, 3), np.nan))
    mp, off = gmo.global_map(oracle, regs)
    blocks = [gmo.frame_block(oracle, r) for r in regs]
    assert list(np.diff(off)) == [len(b) for b in blocks] and off[1] == off[2] and off[-1] == off[-2] == len(mp)
    for f, b in enumerate(blocks):
        assert np.array_equal(mp[off[f]:off[f + 1]], b)
    # frames are never merged: two identical frames give the block twice
    twice, _ = gmo.global_map(oracle, [regs[0], regs[0]])
    assert np.array_equal(twice, np.concatenate([blocks[0], blocks[0]]))


def test_restatement_of_the_loop_leaves_frame_zero_out(oracle):
    scan = synth.raw_scan(n_az=300)
    poses = [synth.se3_exp([1.5 * k, 0, 0, 0, 0, 0.02 * k]) for k in range(4)]
    raws = [scan] * 4
    mp, off = gmo.front_end_map(oracle, raws, poses)
    want, _ = gmo.global_map(oracle, [gmo.transform(scan, P) for P in poses[1:]])
    assert len(off) == 4 and np.array_equal(mp, want)


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)
    assert _lib.ERR_VOXEL_RANGE == 9


def test_front_end_shim_with_mapping_compiles_as_cpp14():
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("front_end_map_driver", "front_end_b200.hpp"))


def test_existing_kernels_compile_to_the_same_sass():
    """every kernel of the commit before the global map: same instructions (the new ones are only added)"""
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "sass_digests.json")))
    got = sass_digest.digests()
    assert len(want) == 89
    changed = [k for k in want if got.get(k) != want[k]]
    assert changed == []
    assert sorted(k for k in got if k not in want) == sorted(k for k in got if "k_gmap_" in k) and len(got) == len(want) + 4


# ---------------------------------------------------------------------------------------------------------------------
def check_block(oracle, got, registered, voxel=1.0):
    """one frame's block against the restatement applied to the device's own registered scan (so that the transform's FMA
    rounding cannot flip a voxel): same voxel key sequence, strictly ascending, coordinates within 1e-10 m"""
    fin = registered[np.isfinite(registered).all(axis=1)]
    want = gmo.frame_block(oracle, registered, voxel)
    assert got.shape == want.shape, (got.shape, want.shape)
    if len(fin) == 0:
        return
    kg = pco.packed_keys(pco.voxel_indices(got, voxel, fin.min(0)))
    kw = pco.packed_keys(pco.voxel_indices(want, voxel, fin.min(0)))
    assert np.array_equal(kg, kw) and np.all(np.diff(kg) > 0)
    assert np.allclose(got, want, rtol=0, atol=1e-10)


def hdl_scan():
    return with_nonfinite(synth.raw_scan(), 7)


@pytest.mark.gpu
def test_gpu_host_pose_append_matches_the_restatement(oracle):
    import tloam_b200
    reg = tloam_b200.LocalRegistration()
    reg.enable_global_map()
    hdl = hdl_scan()
    vlp = synth.vlp16_raw_scan(seed=31, nonfinite=0.01, near=0.01)
    poses = [synth.se3_exp([5.0, -2.0, 0.3, 0.01, 0.02, 0.7]), synth.se3_exp([-3.0, 4.0, 0.0, 0.0, 0.0, -1.2])]
    blocks = []
    for raw, T in zip((hdl, vlp), poses):
        reg.global_map_append(raw, T)
        R = reg.registered_scan()
        want = gmo.transform(raw, T)
        bad = ~np.isfinite(raw).all(axis=1)
        assert R.shape == raw.shape and bad.any()
        assert np.array_equal(~np.isfinite(R).all(axis=1), bad)                       # non-finite in the same rows
        assert np.allclose(R[~bad], want[~bad], rtol=0, atol=1e-12)
        blocks.append(R)
    off = reg.global_map_frames()
    mp = reg.global_map()
    assert len(off) == 3 and off[0] == 0 and off[-1] == len(mp) == reg.global_map_size()[0]
    for f, R in enumerate(blocks):
        check_block(oracle, mp[off[f]:off[f + 1]], R)
    assert np.array_equal(reg.global_map(off[1], off[2] - off[1]), mp[off[1]:])          # a range: only the new frame
    assert off[1] > 1000 and off[2] - off[1] > 200
    # determinism: the same appends after a reset, and on a second handle, give the same bits
    reg.reset_global_map()
    assert reg.global_map_size() == (0, 0)
    for raw, T in zip((hdl, vlp), poses):
        reg.global_map_append(raw, T)
    other = tloam_b200.LocalRegistration()
    other.enable_global_map()
    for raw, T in zip((hdl, vlp), poses):
        other.global_map_append(raw, T)
    assert np.array_equal(reg.global_map(), mp) and np.array_equal(other.global_map(), mp)
    assert np.array_equal(other.global_map_frames(), off)
    reg.close()
    other.close()


def run_loop(scans, mapping=None, host_poses=None, capacity=1 << 20):
    """frame 0: process_raw_scan -> submap_init_frame; frames 1..: process_raw_scan -> scan_match_predicted_async ->
    submap_update_frame_chained [-> global_map_append_frame(_chained)] -> get_result.  Returns (poses, handle)."""
    import tloam_b200
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    if mapping:
        r.enable_global_map(initial_capacity=capacity)
    r.process_raw_scan(scans[0], feature=FE)
    r.submap_init_frame()                                              # frame 0: no append (front_end.cpp:285-305)
    r.set_pose_history(synth.se3_exp(-np.array([0.3, 0.02, 0, 0, 0, 0.005])), np.eye(4))
    poses, regs = [], []
    for k, s in enumerate(scans[1:]):
        r.process_raw_scan(s, feature=FE)
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        if mapping == "chained":
            r.global_map_append_frame()
        elif mapping == "host":
            r.global_map_append_frame(host_poses[k])
            regs.append(r.registered_scan())
        poses.append(r.get_result())
    return poses, r, regs


@pytest.mark.gpu
def test_gpu_chained_loop_maps_without_changing_the_poses(oracle):
    xis = [np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k + 0.001 * (k % 2)]) for k in range(7)]
    scan0 = synth.raw_scan()
    scans = [with_nonfinite(scan0, 90)] + [with_nonfinite(moved(scan0, xi, 100 + k), 200 + k) for k, xi in enumerate(xis) if k > 0]
    plain, a, _ = run_loop(scans)
    a.close()
    chained, b, _ = run_loop(scans, "chained")
    for k in range(6):
        assert np.array_equal(chained[k], plain[k]), k                   # mapping does not touch the odometry
    mp, off = b.global_map(), b.global_map_frames()
    cap, growths = b.global_map_capacity()
    assert growths == 0 and cap == 1 << 20                             # no synchronisation: the buffer never grew
    assert len(off) == 7 and off[0] == 0 and off[-1] == len(mp) and np.all(np.diff(off) > 1000)
    b.close()
    hosted, c, regs = run_loop(scans, "host", host_poses=chained)
    assert all(np.array_equal(x, y) for x, y in zip(hosted, plain))
    assert np.array_equal(c.global_map(), mp) and np.array_equal(c.global_map_frames(), off)
    for k in range(6):
        R = regs[k]
        want = gmo.transform(scans[k + 1], chained[k])
        ok = np.isfinite(scans[k + 1]).all(axis=1)
        assert np.allclose(R[ok], want[ok], rtol=0, atol=1e-12) and not np.isfinite(R[~ok]).all(axis=1).any()
        check_block(oracle, mp[off[k]:off[k + 1]], R)
    c.close()


@pytest.mark.gpu
def test_gpu_growth_gives_the_same_map():
    """a sparse cloud (about one voxel per point) so that the map outgrows a small buffer frame after frame, whatever the
    timing of the asynchronous size read-backs"""
    import tloam_b200
    sparse = with_nonfinite(np.random.default_rng(6).uniform(-1000, 1000, (20000, 3)), 8)
    scans = [sparse, hdl_scan()] * 4
    poses = [synth.se3_exp([4.0 * k, 1.0 * k, 0.0, 0.0, 0.0, 0.3 * k]) for k in range(8)]
    maps = []
    for cap in (1 << 22, 5000):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map(initial_capacity=cap)
        for s, T in zip(scans, poses):
            r.global_map_append(s, T)
        maps.append((r.global_map(), r.global_map_frames(), r.global_map_capacity()))
        r.close()
    (m0, o0, (c0, g0)), (m1, o1, (c1, g1)) = maps
    assert g0 == 0 and c0 == 1 << 22
    assert g1 >= 3 and c1 >= len(m1), (c1, g1)
    assert o0[1] > 19000 and len(o0) == 9
    assert np.array_equal(m0, m1) and np.array_equal(o0, o1)


@pytest.mark.gpu
def test_gpu_key_range_refusal_leaves_the_map_unchanged():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(voxel=1e-5)
    small = np.random.default_rng(3).uniform(-0.5, 0.5, (3000, 3))
    r.global_map_append(small, np.eye(4))
    before, off = r.global_map(), r.global_map_frames()
    assert len(before) == 3000 and list(off) == [0, 3000]
    big = synth.raw_scan()
    r.global_map_append(big, np.eye(4))                                  # ~120 m / 1e-5 m: more than 2^21 voxels
    with pytest.raises(tloam_b200.RegistrationError) as e:
        r.global_map_size()
    assert e.value.status == _lib.ERR_VOXEL_RANGE
    assert r.global_map_size() == (3000, 1)                              # reported once; the map is unchanged
    assert np.array_equal(r.global_map(), before) and np.array_equal(r.global_map_frames(), off)
    assert np.array_equal(r.registered_scan(), big)                      # the scan itself was still registered (T = I)
    r.global_map_append(small, np.eye(4))                                # later frames append normally
    assert r.global_map_size() == (6000, 2)
    r.close()


@pytest.mark.gpu
def test_gpu_global_map_status_codes_and_empty_scans():
    import ctypes as C
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    I = np.eye(4)
    pts = np.ascontiguousarray(synth.raw_scan(n_az=200))
    p = pts.ctypes.data_as(C.POINTER(C.c_double))
    pose = np.ascontiguousarray(I).ctypes.data_as(C.POINTER(C.c_double))
    n, f = C.c_size_t(0), C.c_size_t(0)
    # not enabled: every call is NOT_READY and nothing is launched
    launches = r.launch_count()
    for call in (lambda: r.global_map_append(pts, I), lambda: r.global_map_append(pts), lambda: r.global_map_append_frame(I),
                 r.global_map_append_frame, r.global_map_size, r.global_map_frames, r.registered_scan, r.reset_global_map,
                 r.global_map_capacity):
        with pytest.raises(tloam_b200.RegistrationError) as e:
            call()
        assert e.value.status == _lib.ERR_NOT_READY
    assert r.launch_count() == launches
    cfg = _lib.GlobalMapConfig()
    L.tloam_b200_global_map_default_config(C.byref(cfg))
    assert cfg.voxel == 1.0
    bad_cfg = [_lib.GlobalMapConfig(0.0, 100), _lib.GlobalMapConfig(-1.0, 100), _lib.GlobalMapConfig(float("nan"), 100),
               _lib.GlobalMapConfig(float("inf"), 100)]
    assert [L.tloam_b200_global_map_enable(h, C.byref(c)) for c in bad_cfg] == [_lib.ERR_INVALID_ARG] * 4
    assert L.tloam_b200_global_map_enable(h, None) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_enable(None, C.byref(cfg)) == _lib.ERR_INVALID_ARG
    r.enable_global_map()
    with pytest.raises(tloam_b200.RegistrationError) as e:              # before any append
        r.registered_scan()
    assert e.value.status == _lib.ERR_NOT_READY
    with pytest.raises(tloam_b200.RegistrationError) as e:              # no process_raw_scan yet
        r.global_map_append_frame()
    assert e.value.status == _lib.ERR_NOT_READY
    bad = [
        L.tloam_b200_global_map_append(None, pose, p, 10), L.tloam_b200_global_map_append(h, None, p, 10),
        L.tloam_b200_global_map_append(h, pose, None, 10), L.tloam_b200_global_map_append_chained(h, None, 10),
        L.tloam_b200_global_map_append_frame(h, None), L.tloam_b200_global_map_append_frame_chained(None),
        L.tloam_b200_global_map_size(h, None, C.byref(f)), L.tloam_b200_global_map_download(h, 0, 1, p),        # past the end
        L.tloam_b200_global_map_download(h, 0, 1, None), L.tloam_b200_global_map_frame_offsets(h, None, 5),
        L.tloam_b200_global_map_capacity(h, None, C.byref(n)), L.tloam_b200_registered_scan_download(h, p, 10, None),
        L.tloam_b200_global_map_reset(None),
    ]
    assert bad == [_lib.ERR_INVALID_ARG] * len(bad), bad
    # empty and all-non-finite scans append frames of 0 points
    r.global_map_append(np.zeros((0, 3)), I)
    assert len(r.registered_scan()) == 0
    r.global_map_append(np.full((500, 3), np.nan), I)
    r.global_map_append(pts, I)
    off = r.global_map_frames()
    assert off[0] == off[1] == off[2] == 0 and off[3] > 100
    offs = (C.c_size_t * 3)()
    assert L.tloam_b200_global_map_frame_offsets(h, offs, 3) == _lib.ERR_INVALID_ARG                        # needs 4
    assert L.tloam_b200_global_map_download(h, int(off[3]), 1, p) == _lib.ERR_INVALID_ARG
    reg_n = C.c_size_t(0)
    assert L.tloam_b200_registered_scan_download(h, p, 5, C.byref(reg_n)) == _lib.ERR_INVALID_ARG and reg_n.value == len(pts)
    # the raw scan of process_raw_scan: valid until the next segmentation / process call
    scan = synth.raw_scan(n_az=400)
    r.process_raw_scan(scan, feature=FE)
    r.global_map_append_frame(I)
    assert np.array_equal(r.registered_scan(), r.registered_scan()) and len(r.registered_scan()) == len(scan)
    r.segment_raw_scan(scan)
    with pytest.raises(tloam_b200.RegistrationError) as e:
        r.global_map_append_frame(I)
    assert e.value.status == _lib.ERR_NOT_READY
    r.process_raw_scan(np.zeros((0, 3)))                                 # an empty raw scan: an empty frame
    r.global_map_append_frame(I)
    assert r.global_map_size()[1] == 5
    r.reset_global_map()
    assert r.global_map_size() == (0, 0) and list(r.global_map_frames()) == [0]
    r.close()


@pytest.mark.gpu
def test_gpu_front_end_shim_maps_like_the_python_mirror():
    """FrontEndB200 with mapping on over three frames (seed, then two registered, submap-updated and appended): the global
    map and the registered scan of the Python mirror, bit for bit"""
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("front_end_map_driver", "front_end_b200.hpp")
    reg = tloam_b200.LocalRegistration()
    scan0 = synth.raw_scan(n_az=1200)
    xis = [np.zeros(6), np.array([0.3, 0.02, 0, 0, 0, 0.004]), np.array([0.6, 0.05, 0, 0, 0, 0.009])]
    raws = [with_nonfinite(scan0 if k == 0 else moved(scan0, xi, 50 + k), 60 + k) for k, xi in enumerate(xis)]
    frames = []
    for raw in raws:
        s = reg.segment_raw_scan(raw)
        frames.append([np.ascontiguousarray(raw[s[k]]) for k in ("ground", "edge", "general")])
    predicts = [synth.se3_exp(xi) @ synth.se3_exp(synth.CONFIG1_PERTURB) for xi in xis[1:]]
    d = os.path.dirname(exe)
    paths = [os.path.join(d, x) for x in ("front_end_map.bin", "front_end_raw.bin", "front_end_out.bin")]
    with open(paths[0], "wb") as fh:
        for fr in frames:
            for c in fr:
                fh.write(struct.pack("Q", c.shape[0]))
                fh.write(np.ascontiguousarray(c, dtype=np.float64).tobytes())
        for P in predicts:
            fh.write(np.ascontiguousarray(P.T, dtype=np.float64).tobytes())
    with open(paths[1], "wb") as fh:
        for raw in raws:
            fh.write(struct.pack("Q", raw.shape[0]))
            fh.write(np.ascontiguousarray(raw, dtype=np.float64).tobytes())
    res = subprocess.run([exe] + paths, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert len(res.stdout.strip().split("\n")) == 4
    with open(paths[2], "rb") as fh:
        blob = fh.read()
    n_map = struct.unpack_from("Q", blob, 0)[0]
    cpp_map = np.frombuffer(blob, dtype=np.float64, count=3 * n_map, offset=8).reshape(-1, 3)
    o = 8 + 24 * n_map
    n_reg = struct.unpack_from("Q", blob, o)[0]
    cpp_reg = np.frombuffer(blob, dtype=np.float64, count=3 * n_reg, offset=o + 8).reshape(-1, 3)
    reg.enable_global_map()
    reg.process_cloud(*frames[0], **FE)
    reg.submap_init_frame()
    for k in (1, 2):
        reg.process_cloud(*frames[k], **FE)
        T = reg.scan_matching(predicts[k - 1])
        reg.submap_update_frame(T)
        reg.global_map_append(raws[k], T)
    assert n_map > 1000 and np.array_equal(cpp_map, reg.global_map())
    assert np.array_equal(cpp_reg, reg.registered_scan(), equal_nan=True)
    reg.close()
