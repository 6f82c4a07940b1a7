"""The global map's intensity channel (tloam_b200_global_map_*intensity*, kernels in libtloam_b200_gmi.so): each voxel of
an appended frame gets the reference's AccumulatedPoint average of its rows' intensity (sequential FP64 sum in raw-row
order from +0.0, / count), and the map keeps the channel under PointCloud2::operator+='s rule.

CPU: the restatement (tests/global_map_intensity_oracle.py) against an independent numpy form and on exact cases; the +=
rule table; the new symbols; the shim driver compiles as C++14 -Wall -Wextra clean; the new library holds only its own
kernels, for sm_90a.  GPU: host-pose appends (HDL-64E with NaN / Inf rows and special intensities, VLP-16), a 7-frame
chained loop, the rule on the device, growth, a voxel of more than 10 000 rows, determinism, status codes, the shim."""
import json
import os
import struct
import subprocess

import numpy as np
import pytest

from tloam_b200 import synth
import global_map_oracle as gmo
import global_map_intensity_oracle as gmi
import sass_digest
from test_global_map import hdl_scan, with_nonfinite
from test_process_cloud import FE, moved

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_global_map_append_intensity", "tloam_b200_global_map_append_intensity_chained",
               "tloam_b200_global_map_append_frame_intensity", "tloam_b200_global_map_append_frame_intensity_chained",
               "tloam_b200_global_map_has_intensity", "tloam_b200_global_map_intensity_download"]


def same_bits(a, b):
    """equal bit for bit, except that any NaN equals any NaN (the payload of a propagated NaN is not specified)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    ok = ~np.isnan(a)
    return np.array_equal(a[ok].view(np.uint64), b[ok].view(np.uint64))


def numpy_intensity(registered, intensity, voxel=1.0):
    """independent form: np.unique inverse over the floor indices, a stable argsort, a sequential sum per group"""
    fin = np.isfinite(registered).all(axis=1)
    if not fin.any():
        return np.zeros(0)
    p, v = registered[fin], np.asarray(intensity, dtype=np.float64)[fin]
    idx = np.floor((p - (p.min(0) - 0.5 * voxel)) / voxel).astype(np.int64)
    _, inv, cnt = np.unique(idx, axis=0, return_inverse=True, return_counts=True)
    order = np.argsort(inv.reshape(-1), kind="stable")
    starts = np.concatenate([[0], np.cumsum(cnt)])
    out = np.empty(len(cnt))
    with np.errstate(invalid="ignore"):
        for j in range(len(cnt)):
            grp = v[order[starts[j]:starts[j + 1]]]
            out[j] = np.cumsum(np.concatenate([[0.0], grp]))[-1] / float(cnt[j])   # np.cumsum adds one by one
    return out


def special_intensity(n, seed, finite_rows):
    """uniform intensities with NaN, +-Inf and -0.0 written on some finite rows"""
    rng = np.random.default_rng(seed)
    v = rng.uniform(0.0, 255.0, n)
    rows = rng.choice(np.flatnonzero(finite_rows), 40, replace=False)
    v[rows[:10]] = np.nan
    v[rows[10:20]] = np.inf
    v[rows[20:25]] = -np.inf
    v[rows[25:]] = -0.0
    v[~finite_rows] = rng.uniform(0.0, 255.0, int((~finite_rows).sum()))
    return v


# ---------------------------------------------------------------------------------------------------------------------
def test_restatement_matches_an_independent_numpy_form():
    raw = with_nonfinite(synth.raw_scan(n_az=400), 1)
    reg = gmo.transform(raw, synth.se3_exp([3.0, -1.0, 0.2, 0.01, -0.02, 0.4]))
    fin = np.isfinite(reg).all(axis=1)
    inten = special_intensity(len(reg), 5, fin)
    for voxel in (1.0, 0.37):
        got = gmi.frame_intensity(reg, inten, voxel)
        assert len(got) > 300 and same_bits(got, numpy_intensity(reg, inten, voxel))
        ranks, nv = gmi.voxel_ranks(reg, voxel)
        assert nv == len(got) and np.all(ranks[~fin] == -1) and set(ranks[fin]) == set(range(nv))
    assert np.isnan(got).any() and np.isinf(got).any()
    assert len(gmi.frame_intensity(np.full((10, 3), np.nan), np.ones(10))) == 0


def test_restatement_exact_cases():
    # one voxel per group of rows: (0.1, 0.1, 0.1) + k * 5 m
    def cloud(groups):
        pts, vals = [], []
        for k, g in enumerate(groups):
            for v in g:
                pts.append([0.1 + 5.0 * k, 0.1, 0.1])
                vals.append(v)
        return np.array(pts), np.array(vals, dtype=np.float64)

    pts, vals = cloud([[1.0, 2.0, 4.0], [-0.0, -0.0], [np.nan, 1.0], [np.inf, -np.inf], [np.inf, 3.0], [7.0]])
    got = gmi.frame_intensity(pts, vals)
    assert got[0] == 7.0 / 3.0 and got[5] == 7.0
    assert got[1] == 0.0 and not np.signbit(got[1])                          # +0.0 + -0.0 + -0.0 = +0.0
    assert np.isnan(got[2]) and np.isnan(got[3]) and got[4] == np.inf
    assert same_bits(got, numpy_intensity(pts, vals))
    # the order of the rows matters: the sum is sequential (1e16 + 1 + 1 - 1e16 in row order)
    pts, vals = cloud([[1e16, 1.0, 1.0, -1e16]])
    assert gmi.frame_intensity(pts, vals)[0] == 0.0
    assert gmi.frame_intensity(pts[::-1], vals[::-1])[0] == 0.0
    pts, vals = cloud([[1.0, 1e16, -1e16, 1.0]])
    assert gmi.frame_intensity(pts, vals)[0] == 0.25


RULES = [  # frames: (points the frame adds, frame has intensity) -> the map's channel after each
    ([(5, True), (3, True)], [True, True]),
    ([(5, True), (3, False)], [True, False]),
    ([(5, False), (3, True)], [False, False]),
    ([(0, False), (3, True)], [False, True]),                                 # an all-NaN plain frame adds nothing
    ([(5, True), (0, False)], [True, True]),
    ([(5, True), (3, False), (4, True)], [True, False, False]),               # never regained before a reset
]


def test_append_rule_table():
    for frames, want in RULES:
        m = gmi.MapChannel()
        assert [m.add(n, i).has_intensity() for n, i in frames] == want
    m = gmi.MapChannel().add(5, True).add(3, False)
    assert not m.has_intensity() and m.reset().add(2, True).has_intensity()   # reset re-arms


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


def test_intensity_shim_driver_compiles_as_cpp14_warning_free():
    from tloam_b200 import build
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("front_end_map_intensity_driver", "front_end_b200.hpp"))
    src = os.path.join(ROOT, "tests", "mock", "front_end_map_intensity_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr
    assert os.path.exists(build.GMI_LIB)


def test_intensity_library_holds_only_its_own_kernels_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    got = sass_digest.digests(build.GMI_LIB)
    pinned = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests.json")))
    main = sass_digest.digests()
    assert len(got) >= 5 and all("k_gmi_" in k for k in got)
    assert not set(got) & (set(pinned) | set(main))
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.GMI_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


# ---------------------------------------------------------------------------------------------------------------------
def check_frame(reg, off, f, R, inten, voxel=1.0):
    """frame f's intensity block against the restatement applied to the device's own registered scan R"""
    got = reg.global_map_intensity(int(off[f]), int(off[f + 1] - off[f]))
    want = gmi.frame_intensity(R, inten, voxel)
    assert same_bits(got, want), f


@pytest.mark.gpu
def test_gpu_host_pose_append_matches_the_restatement():
    import tloam_b200
    hdl = hdl_scan()
    vlp = synth.vlp16_raw_scan(seed=31, nonfinite=0.01, near=0.01)
    poses = [synth.se3_exp([5.0, -2.0, 0.3, 0.01, 0.02, 0.7]), synth.se3_exp([-3.0, 4.0, 0.0, 0.0, 0.0, -1.2])]
    intens = [special_intensity(len(hdl), 11, np.isfinite(hdl).all(axis=1)),
              np.random.default_rng(12).uniform(0.0, 100.0, len(vlp))]
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    plain = tloam_b200.LocalRegistration()
    plain.enable_global_map()
    regs = []
    for raw, T, v in zip((hdl, vlp), poses, intens):
        r.global_map_append(raw, T, intensity=v)
        regs.append(r.registered_scan())
        plain.global_map_append(raw, T)
        assert np.array_equal(regs[-1], plain.registered_scan(), equal_nan=True)
    off = r.global_map_frames()
    assert r.global_map_has_intensity() and not plain.global_map_has_intensity()
    assert np.array_equal(r.global_map(), plain.global_map()) and np.array_equal(off, plain.global_map_frames())
    for f in range(2):
        check_frame(r, off, f, regs[f], intens[f])
    inten = r.global_map_intensity()
    assert len(inten) == off[-1] and np.isnan(inten).any() and np.isinf(inten).any()
    # determinism: after a reset, and on a second handle, the same bits
    r.reset_global_map()
    assert not r.global_map_has_intensity()
    other = tloam_b200.LocalRegistration()
    other.enable_global_map()
    for h in (r, other):
        for raw, T, v in zip((hdl, vlp), poses, intens):
            h.global_map_append(raw, T, intensity=v)
        assert same_bits(h.global_map_intensity(), inten) and np.array_equal(h.global_map(), plain.global_map())
    for h in (r, plain, other):
        h.close()


def chained_loop(scans, mapping=None, intens=None):
    """frame 0: process_raw_scan -> submap_init_frame; frames 1..: process_raw_scan -> scan_match_predicted_async ->
    submap_update_frame_chained [-> global_map_append_frame(intensity=...) chained] -> get_result"""
    import tloam_b200
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    if mapping:
        r.enable_global_map()
    r.process_raw_scan(scans[0], feature=FE)
    r.submap_init_frame()
    r.set_pose_history(synth.se3_exp(-np.array([0.3, 0.02, 0, 0, 0, 0.005])), np.eye(4))
    poses, regs = [], []
    for k, s in enumerate(scans[1:]):
        r.process_raw_scan(s, feature=FE)
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        if mapping == "xyz":
            r.global_map_append_frame()
        elif mapping == "intensity":
            r.global_map_append_frame(intensity=intens[k + 1])
            regs.append(r.registered_scan())
        poses.append(r.get_result())
    return poses, r, regs


@pytest.mark.gpu
def test_gpu_chained_loop_keeps_poses_and_xyz_map():
    xis = [np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k + 0.001 * (k % 2)]) for k in range(7)]
    scan0 = synth.raw_scan()
    scans = [with_nonfinite(scan0, 90)] + [with_nonfinite(moved(scan0, xi, 100 + k), 200 + k) for k, xi in enumerate(xis) if k > 0]
    intens = [special_intensity(len(s), 300 + k, np.isfinite(s).all(axis=1)) for k, s in enumerate(scans)]
    plain, a, _ = chained_loop(scans)
    a.close()
    xyz, b, _ = chained_loop(scans, "xyz")
    withi, c, regs = chained_loop(scans, "intensity", intens)
    for k in range(6):
        assert np.array_equal(withi[k], plain[k]) and np.array_equal(xyz[k], plain[k]), k
    off = c.global_map_frames()
    assert np.array_equal(c.global_map(), b.global_map()) and np.array_equal(off, b.global_map_frames())
    assert len(off) == 7 and np.all(np.diff(off) > 1000)
    assert c.global_map_capacity() == (1 << 20, 0)                   # no growth, no synchronisation
    assert c.global_map_has_intensity()
    for k in range(6):
        check_frame(c, off, k, regs[k], intens[k + 1])
    b.close()
    c.close()


@pytest.mark.gpu
def test_gpu_append_rule_on_the_device():
    import tloam_b200
    from tloam_b200 import _lib
    scan = synth.raw_scan(n_az=300)
    nan = np.full((400, 3), np.nan)
    v = np.random.default_rng(2).uniform(0, 50, len(scan))
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    for frames, want in RULES:                                              # n > 0: the scan, n == 0: an all-NaN cloud
        r.reset_global_map()
        got = []
        for n, with_i in frames:
            cloud = scan if n else nan
            r.global_map_append(cloud, np.eye(4), intensity=np.linspace(0, 1, len(cloud)) if with_i else None)
            got.append(r.global_map_has_intensity())
        assert got == want, (frames, got)
    # reset re-arms the channel
    assert not r.global_map_has_intensity()
    r.reset_global_map()
    r.global_map_append(scan, np.eye(4), intensity=v)
    assert r.global_map_has_intensity()
    # a refused frame (VOXEL_RANGE) leaves the flag unchanged, with or without intensity
    r.enable_global_map(voxel=1e-5)
    small = np.random.default_rng(3).uniform(-0.5, 0.5, (3000, 3))
    r.global_map_append(small, np.eye(4), intensity=np.arange(3000.0))
    for with_i in (False, True):
        r.global_map_append(scan, np.eye(4), intensity=v if with_i else None)
        with pytest.raises(tloam_b200.RegistrationError) as e:
            r.global_map_has_intensity()
        assert e.value.status == _lib.ERR_VOXEL_RANGE
        assert r.global_map_has_intensity() and r.global_map_size() == (3000, 1)
    ranks, nv = gmi.voxel_ranks(small, 1e-5)
    want = np.empty(3000)
    want[ranks] = np.arange(3000.0)
    assert nv == 3000 and np.array_equal(r.global_map_intensity(), want)
    r.close()


@pytest.mark.gpu
def test_gpu_launches_nothing_new_without_intensity():
    import tloam_b200
    scan = synth.raw_scan(n_az=200)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()

    def launches(**kw):
        before = r.launch_count()
        r.global_map_append(scan, np.eye(4), **kw)
        return r.launch_count() - before

    fresh = launches()
    r.global_map_append(scan, np.eye(4), intensity=np.ones(len(scan)))
    assert launches() == fresh + 1                                          # the channel is cleared on the device
    r.reset_global_map()
    assert launches() == fresh and not r.global_map_has_intensity()
    r.close()


@pytest.mark.gpu
def test_gpu_growth_gives_the_same_bits():
    import tloam_b200
    sparse = with_nonfinite(np.random.default_rng(6).uniform(-1000, 1000, (20000, 3)), 8)
    scans = [sparse, hdl_scan()] * 3
    poses = [synth.se3_exp([4.0 * k, 1.0 * k, 0.0, 0.0, 0.0, 0.3 * k]) for k in range(6)]
    intens = [np.random.default_rng(40 + k).uniform(0, 255, len(s)) for k, s in enumerate(scans)]
    out = []
    for cap in (1 << 22, 5000):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map(initial_capacity=cap)
        for s, T, v in zip(scans, poses, intens):
            r.global_map_append(s, T, intensity=v)
        out.append((r.global_map(), r.global_map_intensity(), r.global_map_capacity()[1]))
        r.close()
    (m0, i0, g0), (m1, i1, g1) = out
    assert g0 == 0 and g1 >= 2
    assert np.array_equal(m0, m1) and same_bits(i0, i1) and len(i0) == len(m0)


@pytest.mark.gpu
def test_gpu_a_voxel_of_more_than_10000_rows_is_exact():
    import tloam_b200
    rng = np.random.default_rng(8)
    dense = rng.uniform(0.0, 0.45, (15000, 3))                              # one voxel: the min bound is 0, the grid's -0.5 m
    dense[0] = 0.0
    rest = rng.uniform(2.0, 40.0, (5000, 3))
    cloud = np.concatenate([dense, rest])[rng.permutation(20000)]
    v = rng.uniform(0.0, 1e6, 20000) * rng.choice([1.0, 1e-9], 20000)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.global_map_append(cloud, np.eye(4), intensity=v)
    want = gmi.frame_intensity(r.registered_scan(), v)
    assert np.max(np.bincount(gmi.voxel_ranks(r.registered_scan())[0])) > 10000
    assert same_bits(r.global_map_intensity(), want)
    r.close()


@pytest.mark.gpu
def test_gpu_intensity_status_codes():
    import ctypes as C
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    pts = np.ascontiguousarray(synth.raw_scan(n_az=200))
    v = np.ascontiguousarray(np.linspace(0, 1, len(pts)))
    dp = C.POINTER(C.c_double)
    p, pv = pts.ctypes.data_as(dp), v.ctypes.data_as(dp)
    pose = np.ascontiguousarray(np.eye(4)).ctypes.data_as(dp)
    has = C.c_int(7)
    # mapping off: NOT_READY
    assert [L.tloam_b200_global_map_append_intensity(h, pose, p, pv, len(pts)),
            L.tloam_b200_global_map_append_intensity_chained(h, p, pv, len(pts)),
            L.tloam_b200_global_map_append_frame_intensity(h, pose, pv),
            L.tloam_b200_global_map_append_frame_intensity_chained(h, pv),
            L.tloam_b200_global_map_has_intensity(h, C.byref(has)),
            L.tloam_b200_global_map_intensity_download(h, 0, 0, pv)] == [_lib.ERR_NOT_READY] * 6
    r.enable_global_map()
    bad = [L.tloam_b200_global_map_append_intensity(h, pose, p, None, len(pts)),
           L.tloam_b200_global_map_append_intensity(None, pose, p, pv, len(pts)),
           L.tloam_b200_global_map_append_intensity(h, None, p, pv, len(pts)),
           L.tloam_b200_global_map_append_intensity(h, pose, None, pv, len(pts)),
           L.tloam_b200_global_map_append_intensity_chained(h, p, None, len(pts)),
           L.tloam_b200_global_map_append_frame_intensity(h, pose, None),
           L.tloam_b200_global_map_append_frame_intensity(h, None, pv),
           L.tloam_b200_global_map_append_frame_intensity_chained(h, None),
           L.tloam_b200_global_map_has_intensity(h, None), L.tloam_b200_global_map_has_intensity(None, C.byref(has)),
           L.tloam_b200_global_map_intensity_download(h, 0, 1, None)]
    assert bad == [_lib.ERR_INVALID_ARG] * len(bad)
    assert r.global_map_size() == (0, 0)                                      # nothing was appended
    assert L.tloam_b200_global_map_append_frame_intensity_chained(h, pv) == _lib.ERR_NOT_READY   # no process_raw_scan
    with pytest.raises(tloam_b200.RegistrationError) as e:                   # no channel yet
        r.global_map_intensity()
    assert e.value.status == _lib.ERR_NOT_READY
    with pytest.raises(ValueError):
        r.global_map_append(pts, np.eye(4), intensity=v[:-1])
    r.global_map_append(np.zeros((0, 3)), np.eye(4), intensity=np.zeros(0))   # empty: changes nothing
    assert not r.global_map_has_intensity()
    r.global_map_append(pts, np.eye(4), intensity=v)
    n = r.global_map_size()[0]
    assert r.global_map_has_intensity() and L.tloam_b200_global_map_intensity_download(h, n, 1, pv) == _lib.ERR_INVALID_ARG
    assert same_bits(r.global_map_intensity(1, 2), r.global_map_intensity()[1:3])
    # the raw scan of process_raw_scan, with one intensity per row
    scan = synth.raw_scan(n_az=400)
    vs = np.random.default_rng(1).uniform(0, 9, len(scan))
    r.process_raw_scan(scan, feature=FE)
    r.global_map_append_frame(np.eye(4), intensity=vs)
    off = r.global_map_frames()
    assert len(off) == 4                                                     # the empty frame, pts, the raw scan
    check_frame(r, off, 2, r.registered_scan(), vs)
    with pytest.raises(ValueError):
        r.global_map_append_frame(np.eye(4), intensity=vs[1:])
    r.segment_raw_scan(scan)
    with pytest.raises(tloam_b200.RegistrationError) as e:
        r.global_map_append_frame(np.eye(4), intensity=vs)
    assert e.value.status == _lib.ERR_NOT_READY
    r.close()


@pytest.mark.gpu
def test_gpu_front_end_shim_maps_intensity_like_the_python_mirror():
    """FrontEndB200 with raw scans that carry intensity_: the map and its channel of the Python mirror, bit for bit"""
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("front_end_map_intensity_driver", "front_end_b200.hpp")
    reg = tloam_b200.LocalRegistration()
    scan0 = synth.raw_scan(n_az=1200)
    xis = [np.zeros(6), np.array([0.3, 0.02, 0, 0, 0, 0.004]), np.array([0.6, 0.05, 0, 0, 0, 0.009])]
    raws = [with_nonfinite(scan0 if k == 0 else moved(scan0, xi, 50 + k), 60 + k) for k, xi in enumerate(xis)]
    intens = [special_intensity(len(s), 70 + k, np.isfinite(s).all(axis=1)) for k, s in enumerate(raws)]
    frames = []
    for raw in raws:
        s = reg.segment_raw_scan(raw)
        frames.append([np.ascontiguousarray(raw[s[k]]) for k in ("ground", "edge", "general")])
    predicts = [synth.se3_exp(xi) @ synth.se3_exp(synth.CONFIG1_PERTURB) for xi in xis[1:]]
    d = os.path.dirname(exe)
    paths = [os.path.join(d, x) for x in ("fe_int_frames.bin", "fe_int_raw.bin", "fe_int_out.bin")]
    with open(paths[0], "wb") as fh:
        for fr in frames:
            for c in fr:
                fh.write(struct.pack("Q", c.shape[0]))
                fh.write(np.ascontiguousarray(c, dtype=np.float64).tobytes())
        for P in predicts:
            fh.write(np.ascontiguousarray(P.T, dtype=np.float64).tobytes())
    with open(paths[1], "wb") as fh:
        for raw, v in zip(raws, intens):
            fh.write(struct.pack("Q", raw.shape[0]))
            fh.write(np.ascontiguousarray(raw, dtype=np.float64).tobytes())
            fh.write(np.ascontiguousarray(v, dtype=np.float64).tobytes())
    res = subprocess.run([exe] + paths, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert len(res.stdout.strip().split("\n")) == 2
    blob = open(paths[2], "rb").read()
    n_map = struct.unpack_from("Q", blob, 0)[0]
    cpp_map = np.frombuffer(blob, dtype=np.float64, count=3 * n_map, offset=8).reshape(-1, 3)
    o = 8 + 24 * n_map
    n_int = struct.unpack_from("Q", blob, o)[0]
    cpp_int = np.frombuffer(blob, dtype=np.float64, count=n_int, offset=o + 8)
    reg.enable_global_map()
    reg.process_cloud(*frames[0], **FE)
    reg.submap_init_frame()
    for k in (1, 2):
        reg.process_cloud(*frames[k], **FE)
        T = reg.scan_matching(predicts[k - 1])
        reg.submap_update_frame(T)
        reg.global_map_append(raws[k], T if k == 1 else None, intensity=intens[k])
    assert n_map > 1000 and n_int == n_map
    assert np.array_equal(cpp_map, reg.global_map()) and same_bits(cpp_int, reg.global_map_intensity())
    reg.close()
