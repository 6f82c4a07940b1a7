"""FrontEnd::processCloud on the device (tloam_b200_process_cloud / _process_raw_scan, ref: src/front_end/front_end.cpp:181-199)
and the frame-fed submap calls (submap_init_frame :285-305, submap_update_frame[_chained] :201-267).

CPU: the restatement (tests/process_cloud_oracle.py) is pinned -- the oracle's voxels come out in strictly ascending key, which
is numpy's lexicographic order, and the sphere feature is the general cloud's first n_sphere_scan points; the front-end shim
compiles as C++14.  GPU: the street scene against the restatement (planar / sphere bit-identical, ground / edge in the same
order to 1e-10 m, with the ground cap binding), determinism, the raw-scan form against the host-glue path, a multi-frame loop
against the existing submap calls and the oracle, status codes, the C++ shim against the Python mirror."""
import os
import struct
import subprocess

import numpy as np
import pytest

from tloam_b200 import synth
import process_cloud_oracle as pco

FE = dict(cvr_submap=0.005, cvr_scan=0.01)                 # the street scene has few curvature maxima (test_front_end_chain.py)
VLP = dict(sensor_model=16, vertical_res=2.0, init_angle=-15.0)
FE16 = dict(cvr_submap=0.005, cvr_scan=0.01, radius=0.8)   # 16 rings 2 deg apart: a wider PCA neighbourhood (test_vlp16.py)


def numpy_voxel_down_sample(p, voxel):
    """independent restatement: np.unique over the integer voxel indices (lexicographically sorted rows)"""
    mb = p.min(0) - 0.5 * voxel
    idx = np.floor((p - mb) / voxel).astype(np.int64)
    uniq, inv, cnt = np.unique(idx, axis=0, return_inverse=True, return_counts=True)
    out = np.zeros((cnt.size, 3))
    np.add.at(out, inv.reshape(-1), p)
    return uniq, out / cnt[:, None]


def test_restatement_voxels_come_out_in_ascending_key(oracle):
    rng = np.random.default_rng(5)
    clouds = [rng.uniform(-30, 30, (20000, 3)) * [1, 1, 0.05], synth.general_cloud(8000, seed=3)]
    for p in clouds:
        for voxel in (0.1, 0.3):
            out = oracle.voxel_down_sample(p, voxel)
            idx = pco.voxel_indices(out, voxel, p.min(0))
            keys = pco.packed_keys(idx)
            assert len(out) > 500 and np.all(idx >= 0) and np.all(idx < (1 << 21))
            assert np.all(np.diff(keys) > 0)                                      # strictly ascending packed key
            assert np.array_equal(np.lexsort((idx[:, 2], idx[:, 1], idx[:, 0])), np.arange(len(idx)))
            uniq, avg = numpy_voxel_down_sample(p, voxel)
            assert np.array_equal(uniq, idx) and np.allclose(avg, out, rtol=0, atol=1e-12)


def test_restatement_sphere_feature_is_the_general_prefix(oracle):
    general = synth.general_cloud(20000, seed=9)
    p_scan, p_sub, s_scan, s_sub, _ = oracle.extract_planar_sphere(general)
    assert len(s_scan) > 10 and np.array_equal(s_scan, np.arange(len(s_scan)))   # ranks, not point indices (SURVEY Q12)
    ground, edge = general[:3000], general[3000:4000]
    fr = pco.process_cloud(oracle, ground, edge, general)
    assert np.array_equal(fr["sphere"], general[:len(s_scan)]) and np.array_equal(fr["sphere_sub"], general[:len(s_sub)])
    assert np.array_equal(fr["planar"], general[p_scan]) and np.array_equal(fr["planar_sub"], general[p_sub])
    assert np.array_equal(fr["ground"], oracle.voxel_down_sample(ground, 0.3))
    empty = pco.process_cloud(oracle, ground, edge, np.zeros((0, 3)))
    assert all(len(empty[k]) == 0 for k in ("planar", "sphere", "planar_sub", "sphere_sub"))


def test_front_end_shim_compiles_as_cpp14():
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("front_end_driver", "front_end_b200.hpp"))


# ---------------------------------------------------------------------------------------------------------------------
def moved(scan, xi, seed):
    """the scan seen from a sensor moved by exp(xi), with 5 mm of noise (non-finite rows stay non-finite)"""
    Ti = np.linalg.inv(synth.se3_exp(xi))
    with np.errstate(invalid="ignore"):
        return np.ascontiguousarray((scan @ Ti[:3, :3].T + Ti[:3, 3]) + np.random.default_rng(seed).normal(0, 0.005, scan.shape))


def segmented(reg, scan, **kw):
    s = reg.segment_raw_scan(scan, **kw)
    return [np.ascontiguousarray(scan[s[k]]) for k in ("ground", "edge", "general")]


def source_of(reg):
    return [reg.source_cloud(c) for c in range(4)]


def check_against_restatement(got, want, voxels=(0.3, 0.1), raw=None):
    """planar / sphere bit-identical; ground / edge: same count, same voxel key row by row, coordinates within 1e-10 m"""
    assert np.array_equal(got[1], want["sphere"]) and np.array_equal(got[2], want["planar"])
    for c, name, voxel, cloud in ((3, "ground", voxels[0], raw[0]), (0, "edge", voxels[1], raw[1])):
        assert got[c].shape == want[name].shape, name
        kg = pco.packed_keys(pco.voxel_indices(got[c], voxel, cloud.min(0)))
        kw = pco.packed_keys(pco.voxel_indices(want[name], voxel, cloud.min(0)))
        assert np.array_equal(kg, kw) and np.all(np.diff(kg) > 0), name
        assert np.allclose(got[c], want[name], rtol=0, atol=1e-10), name


def pose_close(A, B, dt_max=1e-4, dr_max=1e-5):
    d = np.linalg.inv(A) @ B
    dt, dr = np.linalg.norm(d[:3, 3]), np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))
    return dt < dt_max and dr < dr_max, (dt, dr)


@pytest.mark.gpu
def test_gpu_process_cloud_matches_the_restatement_and_registers_like_set_source(oracle):
    import tloam_b200
    reg = tloam_b200.LocalRegistration()
    xi = [0.4, 0.05, 0.0, 0.0, 0.0, 0.01]
    scan0 = synth.raw_scan()
    scan1 = moved(scan0, xi, 3)
    raw0, raw1 = segmented(reg, scan0), segmented(reg, scan1)
    want0, want1 = (pco.process_cloud(oracle, *r, **FE) for r in (raw0, raw1))
    n = reg.process_cloud(*raw1, **FE)
    got = source_of(reg)
    assert n == [len(c) for c in got]
    check_against_restatement(got, want1, raw=raw1)
    assert n[3] > reg.cfg.ground_maxnum and n[2] > 500 and n[1] > 50 and n[0] > 500     # the ground cap binds
    # frame 0 as the map (the first-frame selections of the restatement), frame 1 registered from the process_cloud source
    target = [raw0[1], want0["sphere_sub"], want0["planar_sub"], oracle.voxel_down_sample(raw0[0], 0.3)]
    predict = synth.se3_exp(xi) @ synth.se3_exp(synth.CONFIG1_PERTURB)
    reg.set_input_target(target)
    T = reg.scan_matching(predict)
    # determinism: the same call again gives the same bits, and so does the registration
    reg.process_cloud(*raw1, **FE)
    assert all(np.array_equal(a, b) for a, b in zip(source_of(reg), got))
    assert np.array_equal(reg.scan_matching(predict), T)
    # == a second handle given the downloaded source through set_input_source
    other = tloam_b200.LocalRegistration()
    other.set_input_target(target)
    other.set_input_source(got)
    assert np.array_equal(other.scan_matching(predict), T)
    orc = oracle.Oracle(threads_mode=1)
    orc.set_input_target(target)
    orc.set_input_source(pco.source(want1))
    rc, To, _ = orc.scan_matching(predict)
    ok, d = pose_close(To, T)
    assert rc == 0 and ok, d
    reg.close()
    other.close()


@pytest.mark.gpu
def test_gpu_ordered_emission_of_long_voxel_lists(oracle):
    """more than 32 768 voxels: the sort falls through to the bitonic network (tiles in shared memory + global-memory
    steps), and the order is still the restatement's"""
    import tloam_b200
    reg = tloam_b200.LocalRegistration()
    rng = np.random.default_rng(12)
    ground = rng.uniform(-60, 60, (90000, 3)) * [1, 1, 0.02]
    edge = rng.uniform(-10, 10, (40000, 3))
    n = reg.process_cloud(ground, edge, np.zeros((0, 3)))
    assert n[3] > 40000 and n[0] > 33000, n
    got = source_of(reg)
    want = dict(ground=oracle.voxel_down_sample(ground, 0.3), edge=oracle.voxel_down_sample(edge, 0.1),
                sphere=np.zeros((0, 3)), planar=np.zeros((0, 3)))
    check_against_restatement(got, want, raw=(ground, edge))
    reg.close()


@pytest.mark.gpu
def test_gpu_process_raw_scan_equals_segment_raw_scan_plus_process_cloud():
    import tloam_b200
    a, b = tloam_b200.LocalRegistration(), tloam_b200.LocalRegistration()
    scan = synth.raw_scan()
    rng = np.random.default_rng(8)
    rows = [np.full((300, 3), np.nan), rng.normal(0, 1.0, (300, 3)), np.array([[np.inf, 1.0, 0.0], [1.0, np.nan, 2.0]] * 50)]
    hdl = scan.copy()
    for r in rows:
        at = np.sort(rng.choice(len(hdl), len(r), replace=False))
        hdl = np.insert(hdl, at, r, axis=0)
    vlp = synth.vlp16_raw_scan(seed=31, nonfinite=0.01, near=0.01)
    for raw, ground, fe in ((hdl, None, FE), (vlp, VLP, FE16)):
        n = a.process_raw_scan(raw, ground=ground, feature=fe)
        assert b.process_cloud(*segmented(b, raw, ground=ground), **fe) == n
        sa, sb = source_of(a), source_of(b)
        for c in range(4):
            assert np.array_equal(sa[c], sb[c]), c
        assert n[0] > 20 and n[2] > 200 and n[3] > 500, n
        # the frames' submap selections are the same too
        a.submap_init_frame()
        b.submap_init_frame()
        for c in range(4):
            assert np.array_equal(a.submap_cloud(c)[np.lexsort(a.submap_cloud(c).T)], b.submap_cloud(c)[np.lexsort(b.submap_cloud(c).T)]), c
    a.close()
    b.close()


@pytest.mark.gpu
def test_gpu_three_call_loop_equals_the_existing_calls_and_the_oracle(oracle):
    """Run A: process_raw_scan -> submap_init_frame on frame 0, then process_raw_scan -> scan_match_predicted_async ->
    submap_update_frame_chained -> get_result.  Run B: the same frames through segment_raw_scan, host gathers, process_cloud
    and the host-input submap calls (submap_init / submap_update_chained with the host-gathered planar selection), with the maps
    downloaded before every frame: bit-identical poses, and the oracle on identical inputs within 1e-4 m / 1e-5 rad per frame."""
    import tloam_b200
    caps = dict(fitness_thres=0.3)
    scan0 = synth.raw_scan()
    xis = [np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k + 0.001 * (k % 2)]) for k in range(7)]
    scans = [scan0] + [moved(scan0, xi, 100 + k) for k, xi in enumerate(xis) if k > 0]
    prev = synth.se3_exp(-xis[1])

    # ---- run A ----
    a = tloam_b200.LocalRegistration(**caps)
    a.process_raw_scan(scans[0], feature=FE)
    a.submap_init_frame()
    a.set_pose_history(prev, np.eye(4))
    got = []
    for s in scans[1:]:
        a.process_raw_scan(s, feature=FE)
        a.scan_matching_predicted_async()
        a.submap_update_frame_chained()
        got.append(a.get_result())
    a.close()

    # ---- run B ----
    b = tloam_b200.LocalRegistration(**caps)
    orc = oracle.Oracle(threads_mode=1, **caps)

    def host_frame(s):
        ground, edge, general = segmented(b, s)
        p_scan, p_sub, s_scan, s_sub, _ = b.extract_planar_sphere(general, **FE)
        return ground, edge, general, general[p_sub], general[:len(s_sub)]

    ground, edge, general, p_sub, s_sub = host_frame(scans[0])
    b.submap_init(edge, ground, p_sub, s_sub)
    b.set_pose_history(prev, np.eye(4))
    last, cur = prev, np.eye(4)
    for k, s in enumerate(scans[1:]):
        maps = [b.submap_cloud(c) for c in range(4)]
        ground, edge, general, p_sub, _ = host_frame(s)
        b.process_cloud(ground, edge, general, **FE)
        src = source_of(b)
        b.scan_matching_predicted_async()
        b.submap_update_chained(p_sub)
        T = b.get_result()
        assert np.array_equal(T, got[k]), k
        orc.set_input_target(maps)
        orc.set_input_source(src)
        rc, To, _ = orc.scan_matching(cur @ (np.linalg.inv(last) @ cur))
        ok, d = pose_close(To, T)
        assert rc == 0 and ok, (k, d)
        last, cur = cur, T
    # and it follows the motion: the street canyon constrains the along-street translation weakly (test_front_end_chain.py),
    # so after 6 frames the chain is ~15 cm off along the street (measured), within 2 mrad in rotation
    ok, d = pose_close(synth.se3_exp(xis[-1]), cur, 0.3, 2e-3)
    assert ok, d
    b.close()


@pytest.mark.gpu
def test_gpu_process_status_codes_and_empty_inputs():
    import ctypes as C
    import tloam_b200
    from tloam_b200 import _lib
    reg = tloam_b200.LocalRegistration()
    L = reg._L
    for call in (reg.submap_init_frame, lambda: reg.submap_update_frame(np.eye(4)), reg.submap_update_frame_chained,
                 lambda: reg.source_cloud(0)):
        with pytest.raises(tloam_b200.RegistrationError) as e:
            call()
        assert e.value.status == _lib.ERR_NOT_READY
    fc, gc, dc = _lib.FeatureConfig(), _lib.GroundConfig(), _lib.DcvcConfig()
    L.tloam_b200_feature_default_config(C.byref(fc))
    L.tloam_b200_ground_default_config(C.byref(gc))
    L.tloam_b200_dcvc_default_config(C.byref(dc))
    pts = np.ascontiguousarray(synth.general_cloud(2000, seed=1))
    p = pts.ctypes.data_as(C.POINTER(C.c_double))
    ns = (C.c_size_t * 4)()
    bad = [
        L.tloam_b200_process_cloud(None, C.byref(fc), 0.3, 0.1, p, 2000, p, 2000, p, 2000, ns),
        L.tloam_b200_process_cloud(reg._h, None, 0.3, 0.1, p, 2000, p, 2000, p, 2000, ns),
        L.tloam_b200_process_cloud(reg._h, C.byref(fc), 0.3, 0.1, None, 2000, p, 2000, p, 2000, ns),
        L.tloam_b200_process_cloud(reg._h, C.byref(fc), 0.3, 0.1, p, 2000, None, 5, p, 2000, ns),
        L.tloam_b200_process_cloud(reg._h, C.byref(fc), 0.3, 0.1, p, 2000, p, 2000, None, 1, ns),
        L.tloam_b200_process_cloud(reg._h, C.byref(fc), 0.0, 0.1, None, 0, None, 0, None, 0, ns),        # checked for empty clouds too
        L.tloam_b200_process_cloud(reg._h, C.byref(fc), 0.3, float("nan"), None, 0, None, 0, None, 0, ns),
        L.tloam_b200_process_cloud(reg._h, C.byref(fc), 0.3, 0.1, p, 2000, p, 2000, p, 2000, None),
        L.tloam_b200_process_raw_scan(None, C.byref(gc), C.byref(dc), 131, 3.0, C.byref(fc), 0.3, 0.1, p, 2000, ns),
        L.tloam_b200_process_raw_scan(reg._h, None, C.byref(dc), 131, 3.0, C.byref(fc), 0.3, 0.1, p, 2000, ns),
        L.tloam_b200_process_raw_scan(reg._h, C.byref(gc), None, 131, 3.0, C.byref(fc), 0.3, 0.1, p, 2000, ns),
        L.tloam_b200_process_raw_scan(reg._h, C.byref(gc), C.byref(dc), 131, 3.0, None, 0.3, 0.1, p, 2000, ns),
        L.tloam_b200_process_raw_scan(reg._h, C.byref(gc), C.byref(dc), 131, 3.0, C.byref(fc), -1.0, 0.1, None, 0, ns),
        L.tloam_b200_process_raw_scan(reg._h, C.byref(gc), C.byref(dc), 131, 3.0, C.byref(fc), 0.3, 0.1, None, 10, ns),
        L.tloam_b200_submap_init_frame(None, None), L.tloam_b200_submap_init_frame(reg._h, None),
        L.tloam_b200_submap_update_frame(reg._h, None), L.tloam_b200_submap_update_frame(None, p),
        L.tloam_b200_submap_update_frame_chained(None), L.tloam_b200_source_download(None, 0, p, 10),
    ]
    assert bad == [_lib.ERR_INVALID_ARG] * len(bad), bad
    # empty inputs behave like the reference: nothing selected from an empty general cloud, empty ground / edge features
    e = np.zeros((0, 3))
    assert reg.process_cloud(e, e, e) == [0, 0, 0, 0]
    assert reg.process_cloud(pts[:500], e, e) == [0, 0, 0, len(reg.source_cloud(3))] and len(reg.source_cloud(3)) > 0
    assert reg.process_cloud(e, pts[:500], e)[1:] == [0, 0, 0]
    n = reg.process_cloud(e, e, pts, **FE)
    assert n[0] == 0 and n[3] == 0 and n[2] > 0
    for raw in (e, np.full((1000, 3), np.nan), np.ones((1000, 3))):                  # empty, all NaN, all within 9 m
        assert reg.process_raw_scan(raw) == [0, 0, 0, 0]
        assert all(len(reg.source_cloud(c)) == 0 for c in range(4))
    reg.submap_init_frame()                                                         # an empty frame seeds an empty map
    assert all(len(reg.submap_cloud(c)) == 0 for c in range(4))
    with pytest.raises(tloam_b200.RegistrationError) as err:                          # a bad configuration of the PCA
        reg.process_cloud(e, e, pts, K=2)
    assert err.value.status == _lib.ERR_INVALID_ARG
    with pytest.raises(tloam_b200.RegistrationError) as err:                          # a failed call leaves no frame behind
        reg.submap_init_frame()
    assert err.value.status == _lib.ERR_NOT_READY
    reg.close()


@pytest.mark.gpu
def test_gpu_front_end_shim_matches_the_python_mirror():
    """tloam::FrontEndB200 over three frames (seed, then two registered and appended): the poses of the Python mirror, bit for bit"""
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("front_end_driver", "front_end_b200.hpp")
    reg = tloam_b200.LocalRegistration()
    scan0 = synth.raw_scan(n_az=1200)
    xis = [np.zeros(6), np.array([0.3, 0.02, 0, 0, 0, 0.004]), np.array([0.6, 0.05, 0, 0, 0, 0.009])]
    frames = [segmented(reg, scan0 if k == 0 else moved(scan0, xi, 50 + k)) for k, xi in enumerate(xis)]
    predicts = [synth.se3_exp(xi) @ synth.se3_exp(synth.CONFIG1_PERTURB) for xi in xis[1:]]
    path = os.path.join(os.path.dirname(exe), "front_end.bin")
    with open(path, "wb") as f:
        for fr in frames:
            for c in fr:
                f.write(struct.pack("Q", c.shape[0]))
                f.write(np.ascontiguousarray(c, dtype=np.float64).tobytes())
        for P in predicts:
            f.write(np.ascontiguousarray(P.T, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.strip().split("\n")
    assert len(lines) == 4
    reg.process_cloud(*frames[0], **FE)
    reg.submap_init_frame()
    for k in (1, 2):
        n = reg.process_cloud(*frames[k], **FE)
        T = reg.scan_matching(predicts[k - 1])
        reg.submap_update_frame(T)
        assert [int(v) for v in lines[2 * k - 2].split()] == n
        T_cpp = np.array([float(v) for v in lines[2 * k - 1].split()]).reshape(4, 4).T
        assert np.array_equal(T_cpp, T), k
    reg.close()
