"""Raw scans in the sensor's packed float32 layout (tloam_packed_scan, the *_packed calls, k_unpack_scan in
libtloam_b200_unpack.so): the records cross PCIe once and are unpacked on the device with (double)float, so every packed
call gives the bits of the FP64 call on f.astype(np.float64).

The layouts are restated here, as the drivers publish them:
  - KITTI .bin: 16-byte records float x, y, z, reflectance;
  - velodyne_pointcloud XYZIR: x, y, z at 0 / 4 / 8, float intensity at 16, uint16 ring at 20, 32 bytes;
  - velodyne_pointcloud XYZIRT: x, y, z, intensity at 0 / 4 / 8 / 12, uint16 ring at 16, float time at 18, 22 bytes (records
    are not 4-byte aligned);
  - an Ouster-like point: x, y, z at 0 / 4 / 8, float intensity at 16, then t / reflectivity / ring / ambient / range, 48 bytes.

CPU: the new symbols, the descriptors packed_scan derives and the arrays it refuses, the shim driver compiles -Wall -Wextra
clean, the new library holds only k_unpack_scan for sm_90a.  GPU: unpack exactness in every layout (and in odd ones: a
17-byte record, a record larger than the kernel's staging window), segmentation and processCloud, a 7-frame chained loop,
intensity precedence and the raw-scan generation rule, status codes, the shim against the Python mirror."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest

from tloam_b200 import synth
import sass_digest
from test_global_map import hdl_scan, with_nonfinite
from test_global_map_intensity import chained_loop, same_bits
from test_process_cloud import FE, FE16, VLP, moved

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_segment_raw_scan_packed", "tloam_b200_process_raw_scan_packed", "tloam_b200_global_map_append_packed",
               "tloam_b200_global_map_append_packed_chained"]

F4 = "<f4"
STRUCTURED = {
    "velodyne_xyzir32": dict(names=["x", "y", "z", "intensity", "ring"], formats=[F4, F4, F4, F4, "<u2"], offsets=[0, 4, 8, 16, 20],
                             itemsize=32),
    "velodyne_xyzirt22": dict(names=["x", "y", "z", "intensity", "ring", "time"], formats=[F4, F4, F4, F4, "<u2", F4],
                              offsets=[0, 4, 8, 12, 16, 18], itemsize=22),
    "ouster48": dict(names=["x", "y", "z", "intensity", "t", "reflectivity", "ring", "ambient", "range"],
                     formats=[F4, F4, F4, F4, "<u4", "<u2", "u1", "<u2", "<u4"], offsets=[0, 4, 8, 16, 20, 24, 26, 28, 32], itemsize=48),
    # not a driver's layout: x / y / z / intensity at odd offsets of a 17-byte record, and a record larger than the staging
    # window with its fields far apart
    "odd17": dict(names=["x", "y", "z", "intensity"], formats=[F4] * 4, offsets=[1, 5, 9, 13], itemsize=17),
    "wide20000": dict(names=["z", "x", "intensity", "y"], formats=[F4] * 4, offsets=[3, 9001, 17000, 19996], itemsize=20000),
}
LAYOUTS = ["kitti16", "velodyne_xyzir32", "velodyne_xyzirt22", "ouster48"]
DESCRIPTORS = {"kitti16": (16, 0, 4, 8, 12), "velodyne_xyzir32": (32, 0, 4, 8, 16), "velodyne_xyzirt22": (22, 0, 4, 8, 12),
               "ouster48": (48, 0, 4, 8, 16), "xyz12": (12, 0, 4, 8, -1)}


def pack(f, inten, layout, seed=0):
    """the float32 scan f (n x 3) and its float32 intensity in `layout`; other fields and padding hold random bytes"""
    if layout == "kitti16":
        return np.ascontiguousarray(np.column_stack([f, inten]).astype(F4))
    if layout == "xyz12":
        return np.ascontiguousarray(f, dtype=F4)
    dt = np.dtype(STRUCTURED[layout])
    a = np.random.default_rng(seed).integers(0, 256, len(f) * dt.itemsize, dtype=np.uint8).view(dt)
    a["x"], a["y"], a["z"] = f[:, 0], f[:, 1], f[:, 2]
    a["intensity"] = inten
    return a


def f32_scan(scan):
    """the scan as the sensor sends it (float32); NaN / Inf rows stay non-finite"""
    with np.errstate(over="ignore", invalid="ignore"):
        return scan.astype(np.float32)


def special_intensity32(n, seed, finite_rows):
    """float32 intensities with +-0, subnormals, NaN, +-Inf and the float32 extremes on some finite rows"""
    rng = np.random.default_rng(seed)
    v = rng.uniform(0.0, 255.0, n).astype(np.float32)
    specials = np.array([0.0, -0.0, 1e-40, -1e-45, 1.1754942e-38, np.nan, np.inf, -np.inf, 3.4028235e38, -3.4028235e38], np.float32)
    rows = rng.choice(np.flatnonzero(finite_rows), 10 * len(specials), replace=False)
    v[rows] = np.repeat(specials, 10)
    return v


def odd_n_hdl():
    """an HDL-64E scan with NaN / Inf rows whose length is not a multiple of any layout's records per block"""
    s = hdl_scan()[:-3]
    assert all(len(s) % r for r in (1024, 512, 744, 341, 963))       # 16 / 32 / 22 / 48 / 17-byte records
    return s


# ---------------------------------------------------------------------------------------------------------------------
def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


@pytest.mark.parametrize("layout", LAYOUTS + ["xyz12"])
def test_packed_scan_derives_the_descriptor(layout):
    import tloam_b200
    f = np.arange(3 * 37, dtype=np.float32).reshape(-1, 3)
    a = pack(f, np.ones(37, np.float32), layout)
    d = tloam_b200.packed_scan(a)
    assert (d.point_step, d.x_offset, d.y_offset, d.z_offset, d.intensity_offset) == DESCRIPTORS[layout]
    assert d.n == 37 and d.data == a.ctypes.data and d._keep is a
    got = np.frombuffer(a.tobytes(), np.uint8).reshape(37, d.point_step)          # the fields are where it says
    for k, o in enumerate((d.x_offset, d.y_offset, d.z_offset)):
        assert np.array_equal(got[:, o:o + 4].copy().view(F4).reshape(-1), f[:, k])


def test_packed_scan_takes_an_organised_cloud_and_a_structured_scan_without_intensity():
    import tloam_b200
    dt = np.dtype(dict(names=["x", "y", "z", "ring"], formats=[F4, F4, F4, "<u2"], offsets=[0, 4, 8, 12], itemsize=16))
    d = tloam_b200.packed_scan(np.zeros((16, 1024), dt))                          # height x width, as an Ouster publishes
    assert (d.n, d.point_step, d.intensity_offset) == (16 * 1024, 16, -1)
    assert tloam_b200.packed_scan(np.zeros(0, np.dtype(STRUCTURED["velodyne_xyzirt22"]))).n == 0


def test_packed_scan_refuses_what_it_cannot_describe():
    import tloam_b200
    good = pack(np.zeros((8, 3), np.float32), np.zeros(8, np.float32), "velodyne_xyzir32")
    big = np.zeros(8, np.dtype(dict(names=["x", "y", "z"], formats=[">f4"] * 3, offsets=[0, 4, 8], itemsize=16)))
    f64 = np.zeros(8, np.dtype(dict(names=["x", "y", "z"], formats=["<f8"] * 3, offsets=[0, 8, 16], itemsize=24)))
    f64_int = np.zeros(8, np.dtype(dict(names=["x", "y", "z", "intensity"], formats=[F4, F4, F4, "<f8"], offsets=[0, 4, 8, 16],
                                        itemsize=24)))
    no_z = np.zeros(8, np.dtype(dict(names=["x", "y", "intensity"], formats=[F4] * 3, offsets=[0, 4, 8], itemsize=16)))
    for bad in (big, f64, f64_int, no_z, good[::2], np.zeros((8, 4)), np.zeros((8, 5), np.float32), np.zeros((8, 4), ">f4"),
                np.zeros(12, np.float32), np.zeros((8, 4), np.float32)[:, :3], np.zeros((4, 8), np.float32).T, [[0.0, 0.0, 0.0]]):
        with pytest.raises(ValueError):
            tloam_b200.packed_scan(bad)


def test_packed_scan_shim_driver_compiles_warning_free():
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("packed_scan_driver", "front_end_b200.hpp"))
    src = os.path.join(ROOT, "tests", "mock", "packed_scan_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


def test_unpack_library_holds_only_k_unpack_scan_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    got = sass_digest.digests(build.UNPACK_LIB)
    assert len(got) == 1 and "k_unpack_scan" in next(iter(got))
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.UNPACK_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


# ---------------------------------------------------------------------------------------------------------------------
def map_state(r):
    has = r.global_map_has_intensity()
    return r.registered_scan(), r.global_map(), r.global_map_frames(), (r.global_map_intensity() if has else None)


def assert_same_map(a, b):
    (ra, ma, fa, ia), (rb, mb, fb, ib) = a, b
    assert same_bits(ra, rb) and same_bits(ma, mb) and np.array_equal(fa, fb)
    assert (ia is None) == (ib is None) and (ia is None or same_bits(ia, ib))


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS + ["odd17", "xyz12"])
def test_gpu_unpack_is_exact(layout):
    """global_map_append_packed against global_map_append[_intensity] of f.astype(float64): registered scan, map, frame table
    and intensity channel bit-identical, NaN / Inf rows and special intensities included"""
    import tloam_b200
    f = f32_scan(odd_n_hdl())
    v = special_intensity32(len(f), 3, np.isfinite(f).all(axis=1))
    a = pack(f, v, layout, seed=9)
    T = synth.se3_exp([5.0, -2.0, 0.3, 0.01, 0.02, 0.7])
    p, q = tloam_b200.LocalRegistration(), tloam_b200.LocalRegistration()
    p.enable_global_map()
    q.enable_global_map()
    p.global_map_append_packed(a, T)
    q.global_map_append(f.astype(np.float64), T, intensity=None if layout == "xyz12" else v.astype(np.float64))
    got, want = map_state(p), map_state(q)
    assert_same_map(got, want)
    assert (got[3] is None) == (layout == "xyz12") and len(got[1]) > 1000
    if got[3] is not None:
        assert np.isnan(got[3]).any() and np.isinf(got[3]).any()
    p.close()
    q.close()


@pytest.mark.gpu
def test_gpu_unpack_a_record_wider_than_the_staging_window():
    import tloam_b200
    f = f32_scan(with_nonfinite(synth.raw_scan(n_az=40), 3))                      # ~2.8k rows of 20000 bytes
    v = special_intensity32(len(f), 4, np.isfinite(f).all(axis=1))
    p, q = tloam_b200.LocalRegistration(), tloam_b200.LocalRegistration()
    for r in (p, q):
        r.enable_global_map()
    p.global_map_append_packed(pack(f, v, "wide20000", seed=2), np.eye(4))
    q.global_map_append(f.astype(np.float64), np.eye(4), intensity=v.astype(np.float64))
    assert_same_map(map_state(p), map_state(q))
    p.close()
    q.close()


@pytest.mark.gpu
def test_gpu_segmentation_and_process_cloud_match_the_fp64_calls():
    import tloam_b200
    cases = [(odd_n_hdl(), {}, FE, "velodyne_xyzirt22"),
             (synth.vlp16_raw_scan(seed=31, nonfinite=0.01, near=0.01), dict(ground=VLP), FE16, "velodyne_xyzir32")]
    r = tloam_b200.LocalRegistration()
    for scan, kw, fe, layout in cases:
        f = f32_scan(scan)
        a = pack(f, np.random.default_rng(1).uniform(0, 100, len(f)).astype(np.float32), layout)
        got, want = r.segment_raw_scan_packed(a, **kw), r.segment_raw_scan(f.astype(np.float64), **kw)
        assert len(want["ground"]) > 100 and len(want["edge"]) > 10 and len(want["sizes"]) > 0
        for k in ("ground", "edge", "general", "sizes", "boxes"):
            assert np.array_equal(got[k], want[k]), k
        assert same_bits(got["intensity"], want["intensity"])
        n_packed = r.process_raw_scan_packed(a, feature=fe, **kw)
        src_packed = [r.source_cloud(c) for c in range(4)]
        assert r.process_raw_scan(f.astype(np.float64), feature=fe, **kw) == n_packed and n_packed[2] > 100 and n_packed[3] > 100
        for c in range(4):
            assert np.array_equal(r.source_cloud(c), src_packed[c]), c
    r.close()


def sorted_rows(a):
    return a[np.lexsort(a.T[::-1])]


def packed_loop(arrs):
    """chained_loop with process_raw_scan_packed and global_map_append_frame() (the packed intensity, if any, read on the device)"""
    import tloam_b200
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()
    r.process_raw_scan_packed(arrs[0], feature=FE)
    r.submap_init_frame()
    r.set_pose_history(synth.se3_exp(-np.array([0.3, 0.02, 0, 0, 0, 0.005])), np.eye(4))
    poses, regs = [], []
    for a in arrs[1:]:
        r.process_raw_scan_packed(a, feature=FE)
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        r.global_map_append_frame()
        regs.append(r.registered_scan())
        poses.append(r.get_result())
    return poses, r, regs


@pytest.mark.gpu
def test_gpu_chained_loop_matches_the_fp64_loop():
    xis = [np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k + 0.001 * (k % 2)]) for k in range(7)]
    scan0 = synth.raw_scan()
    scans = [f32_scan(with_nonfinite(scan0, 90))] + [f32_scan(with_nonfinite(moved(scan0, xi, 100 + k), 200 + k))
                                                     for k, xi in enumerate(xis) if k > 0]
    intens = [special_intensity32(len(s), 300 + k, np.isfinite(s).all(axis=1)) for k, s in enumerate(scans)]
    f64 = [s.astype(np.float64) for s in scans]
    for layout, mapping in (("velodyne_xyzirt22", "intensity"), ("xyz12", "xyz")):
        arrs = [pack(s, v, layout, seed=k) for k, (s, v) in enumerate(zip(scans, intens))]
        got, p, regs_p = packed_loop(arrs)
        want, q, _ = chained_loop(f64, mapping, [v.astype(np.float64) for v in intens])
        for k in range(6):
            assert np.array_equal(got[k], want[k]), (layout, k)
        for c in range(4):                                # the same rows; the submap's voxel emission is unordered
            assert same_bits(sorted_rows(p.submap_cloud(c)), sorted_rows(q.submap_cloud(c))), (layout, c)
        assert np.array_equal(p.global_map(), q.global_map()) and np.array_equal(p.global_map_frames(), q.global_map_frames())
        assert len(p.global_map_frames()) == 7 and p.global_map_capacity() == (1 << 20, 0)
        assert p.global_map_has_intensity() == (mapping == "intensity") == q.global_map_has_intensity()
        if mapping == "intensity":
            assert same_bits(p.global_map_intensity(), q.global_map_intensity())
        assert regs_p[-1].shape == (len(scans[-1]), 3)
        p.close()
        q.close()


@pytest.mark.gpu
def test_gpu_explicit_intensity_takes_precedence_and_the_generation_rule_holds():
    import tloam_b200
    from tloam_b200 import _lib
    f = f32_scan(with_nonfinite(synth.raw_scan(n_az=400), 5))
    v = np.random.default_rng(7).uniform(0, 99, len(f)).astype(np.float32)
    explicit = np.random.default_rng(8).uniform(100, 200, len(f))
    a = pack(f, v, "ouster48")
    T = synth.se3_exp([1.0, 2.0, 0.0, 0.0, 0.0, 0.3])
    p, q = tloam_b200.LocalRegistration(), tloam_b200.LocalRegistration()
    for r in (p, q):
        r.enable_global_map()
    # the packed intensity of process_raw_scan_packed, then an explicit array, against the FP64 calls
    p.process_raw_scan_packed(a, feature=FE)
    p.global_map_append_frame(T)
    p.process_raw_scan_packed(a, feature=FE)
    p.global_map_append_frame(T, intensity=explicit)
    q.process_raw_scan(f.astype(np.float64), feature=FE)
    q.global_map_append_frame(T, intensity=v.astype(np.float64))
    q.process_raw_scan(f.astype(np.float64), feature=FE)
    q.global_map_append_frame(T, intensity=explicit)
    assert_same_map(map_state(p), map_state(q))
    off = p.global_map_frames()
    assert not same_bits(p.global_map_intensity(off[0], off[1] - off[0]), p.global_map_intensity(off[1], off[2] - off[1]))
    # any later segmentation or process call: NOT_READY
    for later in (lambda: p.segment_raw_scan_packed(a), lambda: p.segment_raw_scan(f.astype(np.float64)),
                  lambda: p.process_cloud(f[:500].astype(np.float64), f[500:900].astype(np.float64), f[900:].astype(np.float64), **FE)):
        p.process_raw_scan_packed(a, feature=FE)
        later()
        for append in (lambda: p.global_map_append_frame(T), lambda: p.global_map_append_frame()):
            with pytest.raises(tloam_b200.RegistrationError) as e:
                append()
            assert e.value.status == _lib.ERR_NOT_READY
    # the FP64 process_raw_scan after a packed one: a frame without intensity
    p.process_raw_scan_packed(a, feature=FE)
    p.process_raw_scan(f.astype(np.float64), feature=FE)
    p.reset_global_map()
    p.global_map_append_frame(T)
    assert p.global_map_size()[0] > 0 and not p.global_map_has_intensity()
    p.close()
    q.close()


@pytest.mark.gpu
def test_gpu_packed_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    f = f32_scan(synth.raw_scan(n_az=200))
    a = pack(f, np.ones(len(f), np.float32), "velodyne_xyzir32")
    good = tloam_b200.packed_scan(a)
    pose = np.ascontiguousarray(np.eye(4))
    dp = C.POINTER(C.c_double)
    pp = pose.ctypes.data_as(dp)

    def desc(**kw):
        d = _lib.PackedScan(good.data, good.n, good.point_step, good.x_offset, good.y_offset, good.z_offset, good.intensity_offset)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    # mapping off: NOT_READY
    assert [L.tloam_b200_global_map_append_packed(h, pp, C.byref(good)),
            L.tloam_b200_global_map_append_packed_chained(h, C.byref(good))] == [_lib.ERR_NOT_READY] * 2
    r.enable_global_map()
    bad = [desc(data=None), desc(point_step=11, x_offset=0, y_offset=4, z_offset=7, intensity_offset=-1), desc(x_offset=-1),
           desc(y_offset=29), desc(z_offset=1 << 20), desc(intensity_offset=-2), desc(intensity_offset=29),
           desc(n=(1 << 26) + 1)]
    m = 1 << 12
    idx = [np.zeros(m, np.uintp) for _ in range(3)]
    cnt = [C.c_size_t(0) for _ in range(3)]
    ncl, sizes, boxes, inten = C.c_int(0), np.zeros(m, np.int32), np.zeros((m, 6)), np.zeros(m)
    gc, dc, fc = _lib.GroundConfig(), _lib.DcvcConfig(), r._feature_config(FE)
    L.tloam_b200_ground_default_config(C.byref(gc))
    L.tloam_b200_dcvc_default_config(C.byref(dc))
    szp = C.POINTER(C.c_size_t)
    ns = (C.c_size_t * 4)()

    def segment(d):
        return L.tloam_b200_segment_raw_scan_packed(h, C.byref(gc), C.byref(dc), 131, 3.0, d, idx[0].ctypes.data_as(szp),
                                                    C.byref(cnt[0]), idx[1].ctypes.data_as(szp), C.byref(cnt[1]),
                                                    idx[2].ctypes.data_as(szp), C.byref(cnt[2]), C.byref(ncl),
                                                    sizes.ctypes.data_as(C.POINTER(C.c_int)), boxes.ctypes.data_as(dp),
                                                    inten.ctypes.data_as(dp))

    def process(d):
        return L.tloam_b200_process_raw_scan_packed(h, C.byref(gc), C.byref(dc), 131, 3.0, C.byref(fc), 0.3, 0.1, d, ns)

    calls = [lambda d: L.tloam_b200_global_map_append_packed(h, pp, d), lambda d: L.tloam_b200_global_map_append_packed_chained(h, d),
             segment, process]
    for call in calls:
        assert call(None) == _lib.ERR_INVALID_ARG
        for d in bad:
            assert call(C.byref(d)) == _lib.ERR_INVALID_ARG, (d.point_step, d.x_offset, d.y_offset, d.z_offset, d.intensity_offset)
    assert L.tloam_b200_global_map_append_packed(None, pp, C.byref(good)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_global_map_append_packed(h, None, C.byref(good)) == _lib.ERR_INVALID_ARG
    assert r.global_map_size() == (0, 0)                                      # nothing was appended
    # the limits themselves are valid: a 12-byte record, intensity in the last 4 bytes, n == 0 with no data
    edge = np.ascontiguousarray(f, dtype=F4)
    assert L.tloam_b200_global_map_append_packed(h, pp, C.byref(tloam_b200.packed_scan(edge))) == _lib.OK
    assert L.tloam_b200_global_map_append_packed(h, pp, C.byref(desc(intensity_offset=28))) == _lib.OK
    empty = desc(data=None, n=0)
    for call in calls:
        assert call(C.byref(empty)) == _lib.OK
    assert list(ns) == [0, 0, 0, 0] and [c.value for c in cnt] == [0, 0, 0]
    n, frames = r.global_map_size()
    assert frames == 4 and n > 0 and r.global_map_frames()[-2] == n       # the two empty frames add nothing
    r.close()


@pytest.mark.gpu
def test_gpu_packed_scan_shim_maps_like_the_python_mirror():
    """FrontEndB200::updateGlobalMap[Chained] with the driver's messages: the map and its channel of the Python mirror"""
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("packed_scan_driver", "front_end_b200.hpp")
    reg = tloam_b200.LocalRegistration()
    scan0 = synth.raw_scan(n_az=1200)
    xis = [np.zeros(6), np.array([0.3, 0.02, 0, 0, 0, 0.004]), np.array([0.6, 0.05, 0, 0, 0, 0.009])]
    raws = [f32_scan(with_nonfinite(scan0 if k == 0 else moved(scan0, xi, 50 + k), 60 + k)) for k, xi in enumerate(xis)]
    intens = [special_intensity32(len(s), 70 + k, np.isfinite(s).all(axis=1)) for k, s in enumerate(raws)]
    msgs = [pack(s, v, layout, seed=k) for k, (s, v, layout) in
            enumerate(zip(raws, intens, ("kitti16", "velodyne_xyzir32", "velodyne_xyzirt22")))]
    frames = []
    for raw in raws:
        raw64 = raw.astype(np.float64)
        s = reg.segment_raw_scan(raw64)
        frames.append([np.ascontiguousarray(raw64[s[k]]) for k in ("ground", "edge", "general")])
    predicts = [synth.se3_exp(xi) @ synth.se3_exp(synth.CONFIG1_PERTURB) for xi in xis[1:]]
    d = os.path.dirname(exe)
    paths = [os.path.join(d, x) for x in ("packed_frames.bin", "packed_raw.bin", "packed_out.bin")]
    with open(paths[0], "wb") as fh:
        for fr in frames:
            for c in fr:
                fh.write(struct.pack("Q", c.shape[0]))
                fh.write(np.ascontiguousarray(c, dtype=np.float64).tobytes())
        for P in predicts:
            fh.write(np.ascontiguousarray(P.T, dtype=np.float64).tobytes())
    with open(paths[1], "wb") as fh:
        for m in msgs:
            dsc = tloam_b200.packed_scan(m)
            fh.write(struct.pack("QQQiiii", dsc.n, 1, dsc.point_step, dsc.x_offset, dsc.y_offset, dsc.z_offset, dsc.intensity_offset))
            fh.write(m.tobytes())
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
        reg.global_map_append_packed(msgs[k], T if k == 1 else None)
    assert n_map > 1000 and n_int == n_map
    assert np.array_equal(cpp_map, reg.global_map()) and same_bits(cpp_int, reg.global_map_intensity())
    reg.close()
