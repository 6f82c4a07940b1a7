"""VLP-16 segmentation and the raw-scan entry point (ref: src/models/segmentation/segmentation.cpp:47-66 spinOnce, :386-429
estimateRingsAndTimes2 VLP_16, :472-499 RemoveClosedNonFinitePoints, :174-238 initSections / getSection).

CPU: the literal restatement of the VLP-16 branch (tests/vlp16_oracle.py) against an independent vectorised form, the
one-bound section table of the VLP-16 configuration, the restated removal step against numpy.  GPU: ground_remove / segment_raw_scan against the oracle
chain, segment_raw_scan on an HDL-64E scan against segment_scan, bad arguments, VLP-16 from raw scan to a pose."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

from tloam_b200 import synth
import vlp16_oracle as vo

VLP = dict(sensor_model=16, vertical_res=2.0, init_angle=-15.0)          # what a VLP-16 user sets (INTEGRATION.md)
# 16 rings 2 deg apart: a PCA neighbourhood must span several rings to see a plane (0.2 m finds none); the sparse scan has no
# sphere features, so the registration runs with factor_num 3 (planar + ground + edge) and a placeholder sphere cloud
FE = dict(cvr_submap=0.005, cvr_scan=0.01, radius=0.8)


def vlp16_numpy(pts, init_angle=-15.0, vertical_res=2.0):
    """an independent, vectorised form of the VLP_16 lambda (numpy's arctan2, the half pass found from the signs of y and x):
    returns (channel, index of the first half-pass point or None)"""
    p = np.asarray(pts, dtype=np.float64).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    start, end = np.arctan2(y[0], x[0]), np.arctan2(y[-1], x[-1])
    end = end - 2 * np.pi if end - start > 3 * np.pi else (end + 2 * np.pi if end - start < np.pi else end)
    scan_ori = end - start
    beam_id = np.trunc(np.arctan2(z, np.sqrt(x * x + y * y)) * 180.0 / np.pi + (abs(init_angle) + 0.1)) / vertical_res
    ori = np.arctan2(y, x)
    neg = (y < 0) | ((y == 0) & np.signbit(y) & np.signbit(x))
    pos = (y > 0) | ((y == 0) & ~np.signbit(y) & np.signbit(x))
    tr = np.flatnonzero(pos[1:] & neg[:-1]) + 1
    first = int(tr[0]) if len(tr) else None
    t = np.abs(ori - start) / scan_ori
    if first is not None:
        after = (np.pi - ori[first:] + np.abs(ori[first - 1] - start)) / scan_ori
        t[first:] = np.where(after > 1.0, 0.99999, after)
    return beam_id + t, first


def sweep(azimuths, rng, r=20.0):
    """one column of 16 lasers per azimuth (driver order), at range r"""
    el = np.radians(-15.0 + 2.0 * np.arange(16))
    a, e = np.meshgrid(azimuths, el, indexing="ij")
    p = r * np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], axis=-1).reshape(-1, 3)
    return np.ascontiguousarray(p + rng.normal(0, 0.01, p.shape))


def x_axis_points():
    """points on the x axis with y = +-0: atan2(+-0, x < 0) = +-pi, atan2(+-0, x > 0) = +-0 (only -pi -> +pi is a half pass)"""
    rows = [(5.0, 1.0, -1.0), (-5.0, 0.5, -1.0), (-5.0, -0.0, -1.2), (-5.0, 0.0, -1.1), (-4.0, -1.0, -1.0), (5.0, -0.0, -1.0),
            (5.0, 0.0, -1.0), (6.0, -1.0, -0.5), (-0.0, -0.0, 2.0), (4.0, -0.0, 1.0), (-3.0, 0.0, 1.0)]
    return np.array(rows, dtype=np.float64)


def vlp_scans():
    """several VLP-16 scans: both directions, two start azimuths"""
    return [synth.vlp16_raw_scan(seed=s, clockwise=cw, start_azimuth=a)
            for s, (cw, a) in enumerate(((True, np.pi / 2), (True, -2.0), (False, np.pi / 2), (False, -2.0)), start=11)]


def host_filter(raw, near_dis=3.0):
    x, y, z = raw[:, 0], raw[:, 1], raw[:, 2]
    with np.errstate(invalid="ignore"):
        keep = np.isfinite(raw).all(axis=1) & (np.sqrt((x * x + y * y) + z * z) >= near_dis * near_dis)
    return np.flatnonzero(keep)


def close_ulps(got, want, ulps=8):
    """|got - want| <= ulps ulp of max(|want|, 1): the channel's error comes from atan2 of angles of magnitude ~pi"""
    return bool(np.all(np.abs(got - want) <= ulps * np.spacing(np.maximum(np.abs(want), 1.0))))


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_vlp16_restatement_against_an_independent_vectorised_form(oracle):
    """the literal restatement (tests/vlp16_oracle.py, libm) against numpy's arctan2 and a sign-based half pass: within a
    few ulp, identical (int), the same half-pass point; the inputs cover both directions, a partial sweep without a half
    pass, the 0.99999 clamp, points on the x axis with y = +-0 and a single point"""
    rng = np.random.default_rng(5)
    full = 2 * np.pi / 1800 * (np.arange(1800) + 0.5)
    cases = {
        "clockwise": synth.vlp16_raw_scan(clockwise=True),
        "clockwise_start_-2": synth.vlp16_raw_scan(seed=3, clockwise=True, start_azimuth=-2.0),
        "counter_clockwise": synth.vlp16_raw_scan(clockwise=False),
        "counter_clockwise_start_-2": synth.vlp16_raw_scan(seed=4, clockwise=False, start_azimuth=-2.0),
        "partial_no_transition": sweep(0.1 + 0.9 * full / (2 * np.pi), rng),
        "clamped": sweep(np.pi / 2 - full * (2 * np.pi + 0.3) / (2 * np.pi), rng),
        "x_axis": x_axis_points(),
        "one_point": np.array([[10.0, -3.0, -1.0]]),
    }
    for name, pts in cases.items():
        st = {}
        got = vo.vlp16_channel(pts, stats=st)
        want, first = vlp16_numpy(pts)
        assert close_ulps(got, want), name
        assert np.array_equal(got.astype(np.int64), want.astype(np.int64)), name
        assert st["half_pass"] == first, name
        if name.startswith("clockwise") or name.startswith("counter"):
            assert first is not None and 0 < first < len(pts)
        if name == "clamped":
            assert st["clamped"] > 100
        if name == "partial_no_transition":
            assert first is None
        if name == "x_axis":
            assert first == 3                                                   # (-5, -0) -> (-5, +0): -pi -> +pi
    assert vo.vlp16_channel(cases["one_point"])[0] == math.trunc(math.degrees(math.atan2(-1.0, math.hypot(10.0, 3.0))) + 15.1) / 2.0
    # groundRemove carries that channel; HDL-64E: the beam estimate as doubles; other sensors: the `default:` branch
    scan = cases["clockwise"]
    assert np.array_equal(vo.ground_remove(oracle, scan, **VLP)["intensity"], vo.vlp16_channel(scan))
    hdl = synth.raw_scan(seed=4, n_az=300)
    assert np.array_equal(vo.ground_remove(oracle, hdl)["intensity"], oracle.ground_extract(hdl)["beam"].astype(np.float64))
    assert vo.ground_remove(oracle, hdl, sensor_model=32) is None


def test_vlp16_section_table_has_one_bound(oracle):
    """initSections with sensorModel 16 stalls after the first boundary (the -7 -> -5 deg radius jump is 5.7 m): one bound,
    so a missing bound reads as the last section and section 1 stays empty"""
    b = oracle.ground_section_bounds(sensor_model=16, sensor_height=1.73, init_angle=-15.0, vertical_res=2.0)
    assert b == [float(np.float32(1.73 / math.tan(math.fabs(-7.0 / 180 * math.pi))))]
    ge = vo.ground_remove(oracle, synth.vlp16_raw_scan(), **VLP)
    r = ge["region"][ge["region"] < 12]
    assert len(r) > 1000 and not np.any(r % 3 == 1) and np.any(r % 3 == 0) and np.any(r % 3 == 2)


def test_remove_closed_nonfinite_restatement_against_numpy():
    rng = np.random.default_rng(2)
    pts = rng.normal(0, 8, (5000, 3))
    nine = 9.0
    edge = [(nine, 0.0, 0.0), (np.nextafter(nine, 0), 0.0, 0.0), (np.nextafter(nine, 20), 0.0, 0.0), (0.0, -nine, 0.0),
            (0.0, 0.0, np.nextafter(-nine, 0)), (3.0, 3.0, math.sqrt(81 - 18)), (np.nan, 1e3, 0.0), (1e3, np.nan, 0.0),
            (1e3, 0.0, np.nan), (np.inf, 0.0, 0.0), (0.0, -np.inf, 0.0), (0.0, 0.0, np.inf), (0.0, 0.0, 0.0)]
    pts = np.vstack([pts[:2500], np.array(edge), pts[2500:]])
    for dis in (3.0, 1.0, 0.0):
        keep = vo.remove_closed_nonfinite(pts, dis)
        assert np.array_equal(keep, host_filter(pts, dis)), dis
    keep = vo.remove_closed_nonfinite(pts, 3.0)
    assert 2500 in keep and 2501 not in keep and 2502 in keep                 # norm 9, 9 - 1 ulp, 9 + 1 ulp
    assert not np.any((keep >= 2506) & (keep <= 2511))                        # NaN / Inf in one coordinate
    assert len(vo.remove_closed_nonfinite(np.zeros((0, 3)), 3.0)) == 0


def test_vlp16_driver_compiles_as_cpp14():
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("vlp16_driver", "segmentation_b200.hpp"))


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_ground_remove_vlp16_matches_the_oracle(oracle):
    import tloam_b200
    reg = tloam_b200.LocalRegistration()
    for scan in vlp_scans() + [x_axis_points()]:
        got, want = reg.ground_remove(scan, **VLP), vo.ground_remove(oracle, scan, **VLP)
        for k in ("ground", "object", "region"):
            assert np.array_equal(got[k], want[k]), k
        assert got["height_threshold"] == want["height_threshold"]
        assert np.array_equal(got["planes"], want["planes"], equal_nan=True)
        c, w = got["intensity"], want["intensity"]
        assert close_ulps(c, w)
        exact = c == w
        assert not np.any(~exact & (np.abs(w - np.round(w)) < 1e-9))          # the (int) check below is not luck
        assert np.array_equal(c.astype(np.int64), w.astype(np.int64))
        # tloam_b200_ground_extract hands out (int) of the same channel
        assert np.array_equal(reg.ground_extract(scan, **VLP)["beam"], c.astype(np.int32))
    hdl = synth.raw_scan(seed=4, n_az=600)
    assert np.array_equal(reg.ground_remove(hdl)["intensity"], reg.ground_extract(hdl)["beam"].astype(np.float64))
    reg.close()


@pytest.mark.gpu
def test_gpu_segment_raw_scan_vlp16_matches_the_oracle_chain(oracle):
    import tloam_b200
    reg = tloam_b200.LocalRegistration()
    for cw, start in ((True, np.pi / 2), (False, -2.0)):
        raw = synth.vlp16_raw_scan(seed=21 + cw, clockwise=cw, start_azimuth=start, nonfinite=0.02, near=0.02)
        got = reg.segment_raw_scan(raw, ground=VLP)
        want = vo.raw_chain(oracle, raw)
        for k in ("ground", "edge", "general", "sizes", "boxes"):
            assert np.array_equal(got[k], want[k]), k
        keep = want["keep"]
        assert np.all(np.isnan(np.delete(got["intensity"], keep)))
        assert close_ulps(got["intensity"][keep], want["intensity"])
        assert np.array_equal(got["intensity"][keep].astype(np.int64), want["intensity"].astype(np.int64))
        assert len(keep) < len(raw) - 500 and len(got["edge"]) > 20 and len(got["general"]) > 2000 and len(got["ground"]) > 2000
        # the oracle's edge step fed the DEVICE's channel
        dev = vo.raw_chain(oracle, raw, channel=got["intensity"])
        assert np.array_equal(got["edge"], dev["edge"]) and np.array_equal(got["general"], dev["general"])
    reg.close()


@pytest.mark.gpu
def test_gpu_segment_raw_scan_hdl64_equals_segment_scan_on_the_filtered_scan():
    import tloam_b200
    reg = tloam_b200.LocalRegistration()
    scan = synth.raw_scan()
    rng = np.random.default_rng(8)
    rows = [np.full((300, 3), np.nan), rng.normal(0, 1.0, (300, 3)), np.array([[np.inf, 1.0, 0.0], [1.0, np.nan, 2.0]] * 50)]
    raw = scan.copy()
    for r in rows:
        at = np.sort(rng.choice(len(raw), len(r), replace=False))
        raw = np.insert(raw, at, r, axis=0)
    keep = host_filter(raw)
    got = reg.segment_raw_scan(raw)
    ref = reg.segment_scan(np.ascontiguousarray(raw[keep]))
    for k in ("ground", "edge", "general"):
        assert np.array_equal(got[k], keep[ref[k]]), k
    assert np.array_equal(got["sizes"], ref["sizes"]) and np.array_equal(got["boxes"], ref["boxes"])
    assert np.array_equal(got["intensity"][keep], ref["beam"].astype(np.float64))
    assert np.all(np.isnan(np.delete(got["intensity"], keep)))
    reg.close()


@pytest.mark.gpu
def test_gpu_bad_arguments_and_empty_inputs():
    import tloam_b200
    from tloam_b200 import _lib
    reg = tloam_b200.LocalRegistration()
    scan = synth.vlp16_raw_scan(columns=300)
    for call in (lambda: reg.ground_remove(scan, sensor_model=32), lambda: reg.segment_raw_scan(scan, ground=dict(sensor_model=32)),
                 lambda: reg.ground_extract(scan, sensor_model=32), lambda: reg.segment_raw_scan(np.full((50, 3), np.nan), ground=dict(sensor_model=32))):
        with pytest.raises(tloam_b200.RegistrationError) as e:
            call()
        assert e.value.status == _lib.ERR_INVALID_ARG
    g = reg.ground_remove(np.zeros((0, 3)), **VLP)
    assert len(g["ground"]) == 0 and len(g["object"]) == 0 and len(g["intensity"]) == 0
    for raw in (np.zeros((0, 3)), np.full((1000, 3), np.nan), np.ones((1000, 3))):      # empty, all NaN, all within 9 m
        s = reg.segment_raw_scan(raw, ground=VLP)
        assert len(s["ground"]) == 0 and len(s["edge"]) == 0 and len(s["general"]) == 0 and len(s["sizes"]) == 0
        assert len(s["intensity"]) == len(raw) and np.all(np.isnan(s["intensity"]))
    # a later call is unaffected
    assert np.array_equal(reg.ground_remove(scan, **VLP)["ground"], reg.ground_extract(scan, **VLP)["ground"])
    reg.close()


def frame_features(raw, segment, planar_sphere):
    seg = segment(raw)
    edge = np.ascontiguousarray(raw[seg["edge"]])
    general = np.ascontiguousarray(raw[seg["general"]])
    ground = np.ascontiguousarray(raw[seg["ground"]][::4])
    p_scan, p_sub, s_scan, s_sub, s_cand = planar_sphere(general)
    return dict(edge=edge, ground=ground, p_scan=general[p_scan], p_sub=general[p_sub], s_scan=general[s_cand[s_scan]],
                s_sub=general[s_cand[s_sub]])


@pytest.mark.gpu
def test_gpu_vlp16_raw_scan_to_pose_matches_the_oracle_chain(oracle):
    """the analogue of test_front_end_chain.py for the VLP-16: segment_raw_scan -> PCA features of the general cloud ->
    frame 1 registered against frame 0, every stage on the device, against the same chain on the oracle"""
    import tloam_b200
    raw0 = synth.vlp16_raw_scan(seed=31, nonfinite=0.01, near=0.01)
    T = synth.se3_exp([0.4, 0.05, 0.0, 0.0, 0.0, 0.01])
    Ti = np.linalg.inv(T)
    with np.errstate(invalid="ignore"):                                   # the NaN / Inf rows stay non-finite
        raw1 = np.ascontiguousarray((raw0 @ Ti[:3, :3].T + Ti[:3, 3]) + np.random.default_rng(3).normal(0, 0.005, raw0.shape))
    predict = T @ synth.se3_exp(synth.CONFIG1_PERTURB)
    reg = tloam_b200.LocalRegistration()
    g = [frame_features(s, lambda x: reg.segment_raw_scan(x, ground=VLP), lambda c: reg.extract_planar_sphere(c, **FE)) for s in (raw0, raw1)]
    o = [frame_features(s, lambda x: vo.raw_chain(oracle, x), lambda c: oracle.extract_planar_sphere(c, **FE)) for s in (raw0, raw1)]
    for a, b in zip(g, o):
        for k in a:
            assert np.array_equal(a[k], b[k]), k
        assert len(a["edge"]) > 200 and len(a["p_scan"]) > 200 and len(a["p_sub"]) > 200 and len(a["ground"]) > 500
    reg.close()
    reg = tloam_b200.LocalRegistration(factor_num=3)
    reg.set_input_target([g[0]["edge"], g[0]["p_sub"][:16], g[0]["p_sub"], g[0]["ground"]])
    reg.set_input_source([g[1]["edge"], g[1]["p_scan"][:16], g[1]["p_scan"], g[1]["ground"]])
    Tg = reg.scan_matching(predict)
    orc = oracle.Oracle(threads_mode=1, factor_num=3)
    orc.set_input_target([o[0]["edge"], o[0]["p_sub"][:16], o[0]["p_sub"], o[0]["ground"]])
    orc.set_input_source([o[1]["edge"], o[1]["p_scan"][:16], o[1]["p_scan"], o[1]["ground"]])
    rc, To, _ = orc.scan_matching(predict)
    assert rc == 0
    d = np.linalg.inv(To) @ Tg
    dt, dr = np.linalg.norm(d[:3, 3]), np.arccos(np.clip((np.trace(d[:3, :3]) - 1) / 2, -1, 1))
    assert dt < 1e-4 and dr < 1e-5, (dt, dr)
    e = np.linalg.inv(T) @ Tg                                             # against the motion: 5 cm of prediction error shrink
    assert np.linalg.norm(e[:3, 3]) < 5e-2
    reg.close()


@pytest.mark.gpu
def test_gpu_segmentation_shim_vlp16_two_frames_matches_the_oracle_chain(oracle):
    """tloam::SegmentationB200::segmentRawScan on two consecutive VLP-16 frames (the second with the DCVC members
    resetParams() leaves) and GroundExtractB200::groundRemove: the clouds of the oracle chain, and every intensity_ the shim
    writes is the oracle's channel (fractional part for ground points) to <= 8 ulp"""
    from test_cpp_shim import build_driver
    exe = build_driver("vlp16_driver", "segmentation_b200.hpp")
    raw = synth.vlp16_raw_scan(seed=41, nonfinite=0.01, near=0.01)
    keep = host_filter(raw)
    filt = np.ascontiguousarray(raw[keep])
    path = os.path.join(os.path.dirname(exe), "vlp16.bin")
    with open(path, "wb") as f:
        for c in (raw, filt):
            f.write(struct.pack("Q", c.shape[0]))
            f.write(np.ascontiguousarray(c, dtype=np.float64).tobytes())
    res = subprocess.run([exe, path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.strip().split("\n")

    def check(rows, pts, idx, channel, ground):
        assert [int(r[0]) for r in rows] == [int(b) for b in pts[idx, 0].copy().view(np.uint64)]
        got, c = np.array([float(r[1]) for r in rows]), channel[idx]
        want = c - np.trunc(c) if ground else c
        assert np.all(np.abs(got - want) <= 8 * np.spacing(np.maximum(np.abs(c), 1.0)))

    pos = 0
    for init in (5.0, 0.0):
        want = vo.raw_chain(oracle, raw, dcvc=dict(min_polar_init=init, max_polar_init=init))
        channel = np.full(len(raw), np.nan)
        channel[keep] = want["intensity"]
        ng, nb, ne, nn = (int(v) for v in lines[pos].split())
        pos += 1
        assert (ng, nb, ne, nn) == (len(want["ground"]), len(want["sizes"]), len(want["edge"]), len(want["general"]))
        for c in range(nb):
            v = lines[pos + c].split()
            assert int(v[0]) == c + 1 and int(v[1]) == want["sizes"][c] and [float(x) for x in v[2:]] == list(want["boxes"][c])
        pos += nb
        for idx, ground in ((want["ground"], True), (want["edge"], False), (want["general"], False)):
            check([l.split() for l in lines[pos:pos + len(idx)]], raw, idx, channel, ground)
            pos += len(idx)
        assert ne > 20 and nn > 2000
    ge = vo.ground_remove(oracle, filt, **VLP)
    ng, no, ncur = (int(v) for v in lines[pos].split())
    pos += 1
    cur = np.flatnonzero(ge["region"] != 12)
    assert (ng, no, ncur) == (len(ge["ground"]), len(ge["object"]), len(cur))
    for idx, ground in ((ge["ground"], True), (ge["object"], False), (cur, False)):
        check([l.split() for l in lines[pos:pos + len(idx)]], filt, idx, ge["intensity"], ground)
        pos += len(idx)
    assert pos == len(lines)
