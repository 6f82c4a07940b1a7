"""Deskewing (include/tloam_b200.h "Deskewing", the *_timed calls, k_deskew_motion / k_deskew_tend / k_deskew in
libtloam_b200_deskew.so): every row of a raw scan becomes exp(s_i . xi) . p_i with s_i = (t_i - t_end) / P and xi the pose
history's constant-velocity increment, so the scan is expressed in the sensor frame at the end of its sweep.
tests/deskew_oracle.py is the CPU restatement.

The time fields are restated as the drivers publish them:
  - velodyne_pointcloud XYZIRT: float32 `time` (s from the sweep's start) at byte 18 of a 22-byte record;
  - an Ouster-like point: uint32 `t` (ns) at byte 20 of a 48-byte record;
  - a Hesai-like point: float64 `timestamp` (s, absolute) at byte 16 of a 32-byte record.

CPU: the restatement against scipy.linalg.expm (small-angle branch and s = 0 included), its edge cases, packed_time and the
shim's packedTimeOf on those layouts and on refused ones, the symbols, the new library's kernels.  GPU: the kernels against
the restatement in every time form, bit-identity to the untimed loop where nothing moves, determinism, accuracy on a
rolling-shutter sequence, the status codes, the shim against the Python mirror."""
import ctypes as C
import os
import struct
import subprocess

import numpy as np
import pytest
import scipy.linalg

import deskew_oracle as dko
import sass_digest
from tloam_b200 import synth
from test_global_map import with_nonfinite
from test_global_map_intensity import same_bits
from test_packed_scan import STRUCTURED, f32_scan
from test_process_cloud import FE, moved

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_process_raw_scan_timed", "tloam_b200_process_raw_scan_packed_timed"]
F4 = "<f4"
TIMED = {
    "velodyne_xyzirt22": STRUCTURED["velodyne_xyzirt22"],
    "ouster48": STRUCTURED["ouster48"],
    "hesai32": dict(names=["x", "y", "z", "intensity", "timestamp", "ring"], formats=[F4, F4, F4, F4, "<f8", "<u2"],
                    offsets=[0, 4, 8, 12, 16, 24], itemsize=32),
}
TIME_DESCRIPTORS = {"velodyne_xyzirt22": (18, 7, 1.0), "ouster48": (20, 6, 1e-9), "hesai32": (16, 8, 1.0)}
HESAI_EPOCH = 1.7e9                                          # an absolute timestamp: s since 1970
PERIOD = 0.1
# the increment the GPU tests seed: 1.5 m forward and 0.05 rad of yaw over one frame (15 m/s at 10 Hz)
XI_SEED = np.array([1.5, 0.0, 0.0, 0.0, 0.0, 0.05])


def hat(a):
    W = np.zeros((4, 4))
    W[:3, :3] = [[0, -a[5], a[4]], [a[5], 0, -a[3]], [-a[4], a[3], 0]]
    W[:3, 3] = a[:3]
    return W


def pack_timed(f, rel_time, layout, seed=0):
    """float32 rows f (n x 3) with their time in `layout`; rel_time (FP64 s from the sweep's start) becomes the layout's field.
    Returns the records and the FP64 times the device must read from them."""
    dt = np.dtype(TIMED[layout])
    a = np.random.default_rng(seed).integers(0, 256, len(f) * dt.itemsize, dtype=np.uint8).view(dt)
    a["x"], a["y"], a["z"] = f[:, 0], f[:, 1], f[:, 2]
    a["intensity"] = 1.0
    if layout == "velodyne_xyzirt22":
        a["time"] = rel_time.astype(np.float32)
        t = a["time"].astype(np.float64)
    elif layout == "ouster48":
        a["t"] = np.where(np.isfinite(rel_time), np.round(np.nan_to_num(rel_time) * 1e9), 0).astype(np.uint32)
        t = a["t"].astype(np.float64) * 1e-9
    else:
        a["timestamp"] = HESAI_EPOCH + rel_time
        t = a["timestamp"].astype(np.float64)
    return a, t


# ---------------------------------------------------------------------------------------------------------------------
def test_restatement_exp_matches_expm_of_the_twist():
    rng = np.random.default_rng(1)
    cases = [np.zeros(6), np.array([1.5, 0, 0, 0, 0, 0]), np.array([0.3, -0.2, 0.1, 1e-12, -3e-12, 2e-12]),
             np.array([0.3, -0.2, 0.1, 0, 0, 5e-11]), np.array([1.0, 2.0, 3.0, 0.0, 0.0, 1e-10]), XI_SEED, -0.7 * XI_SEED,
             np.array([0.1, 0.2, -0.3, 1.0, -2.0, 0.5])] + [rng.normal(0, 1, 6) for _ in range(20)]
    for a in cases:
        R, t = dko.se3_exp(a)
        want = scipy.linalg.expm(hat(a))
        # below theta = 1e-10 Sophus (and se3.cuh) take V = R, which is off by at most theta |upsilon| / 2
        tol = 1e-13 + np.linalg.norm(a[3:]) * np.linalg.norm(a[:3]) * (np.linalg.norm(a[3:]) < 1e-10)
        assert np.allclose(R, want[:3, :3], rtol=0, atol=1e-13) and np.allclose(t, want[:3, 3], rtol=0, atol=tol), a
    R, t = dko.se3_exp(np.zeros((3, 6)))                          # s = 0: exactly the identity
    assert np.array_equal(R, np.broadcast_to(np.eye(3), (3, 3, 3))) and np.array_equal(t, np.zeros((3, 3)))


def test_restatement_log_inverts_exp():
    rng = np.random.default_rng(2)
    for a in [XI_SEED, np.array([0.2, 0.1, 0.0, 1e-12, 0.0, 0.0])] + [rng.normal(0, 0.5, 6) for _ in range(20)]:
        T = scipy.linalg.expm(hat(a))
        assert np.allclose(dko.se3_log(T), a, rtol=0, atol=1e-12), a
    last = synth.se3_exp([3.0, -1.0, 0.2, 0.01, 0.02, 0.4])
    assert np.allclose(dko.increment(last, last @ scipy.linalg.expm(hat(XI_SEED))), XI_SEED, rtol=0, atol=1e-12)


def test_restatement_edge_cases():
    rng = np.random.default_rng(3)
    p = rng.uniform(-50, 50, (200, 3))
    p[5] = np.nan
    p[6] = [np.inf, 0.0, 1.0]
    t = rng.uniform(0, PERIOD, 200)
    t[[10, 11, 12]] = [np.nan, np.inf, -np.inf]
    t[20] = 0.2                                                  # t_end
    curr = scipy.linalg.expm(hat(XI_SEED))
    out = dko.deskew(p, t, PERIOD, np.eye(4), curr)
    for i in (10, 11, 12, 20):                                   # s = 0: the row itself
        assert same_bits(out[i], p[i])
    assert not np.isfinite(out[5]).any() and not np.isfinite(out[6]).all()
    i = 30
    R, tt = dko.se3_exp((t[i] - 0.2) / PERIOD * XI_SEED)
    assert np.allclose(out[i], R @ p[i] + tt, rtol=0, atol=1e-12) and np.linalg.norm(out[i] - p[i]) > 0.5
    # a row one period before t_end moves by exactly last . curr^-1
    t2 = np.array([0.1, 0.2])
    out2 = dko.deskew(p[:2], t2, PERIOD, np.eye(4), curr)
    back = np.linalg.inv(curr)
    assert np.allclose(out2[0], back[:3, :3] @ p[0] + back[:3, 3], rtol=0, atol=1e-12)
    for times, last, cur in ((np.full(200, np.nan), np.eye(4), curr), (t, np.eye(4), np.eye(4)), (np.full(200, 0.05), np.eye(4), curr)):
        assert same_bits(dko.deskew(p, times, PERIOD, last, cur), p)   # no finite time / identity history / all equal


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)


@pytest.mark.parametrize("layout", sorted(TIMED))
def test_packed_time_derives_the_descriptor(layout):
    import tloam_b200
    a, _ = pack_timed(np.zeros((9, 3), np.float32), np.linspace(0, 0.09, 9), layout)
    d = tloam_b200.packed_time(a)
    assert (d.offset, d.datatype, d.unit) == TIME_DESCRIPTORS[layout]


def refused_time_layouts():
    s = lambda names, formats, offsets, itemsize: np.zeros(4, np.dtype(dict(names=names, formats=formats, offsets=offsets,
                                                                            itemsize=itemsize)))
    return {
        "no_time": s(["x", "y", "z", "intensity", "ring"], [F4, F4, F4, F4, "<u2"], [0, 4, 8, 16, 20], 32),
        "time_f64": s(["x", "y", "z", "time"], [F4, F4, F4, "<f8"], [0, 4, 8, 16], 24),
        "t_f32": s(["x", "y", "z", "t"], [F4, F4, F4, F4], [0, 4, 8, 12], 16),
        "t_u16": s(["x", "y", "z", "t"], [F4, F4, F4, "<u2"], [0, 4, 8, 12], 16),
        "timestamp_f32": s(["x", "y", "z", "timestamp"], [F4, F4, F4, F4], [0, 4, 8, 12], 16),
        "time_big_endian": s(["x", "y", "z", "time"], [F4, F4, F4, ">f4"], [0, 4, 8, 12], 16),
    }


def test_packed_time_refuses_what_it_cannot_describe():
    import tloam_b200
    for bad in list(refused_time_layouts().values()) + [np.zeros((4, 4), np.float32), [[0.0] * 4]]:
        with pytest.raises(ValueError):
            tloam_b200.packed_time(bad)


def test_deskew_driver_compiles_warning_free():
    from test_cpp_shim import build_driver
    assert os.path.exists(build_driver("deskew_driver", "packed_scan_b200.hpp"))
    src = os.path.join(ROOT, "tests", "mock", "deskew_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


_INVALID_ARG = 1
PF_TYPES = {"i1": 1, "u1": 2, "i2": 3, "u2": 4, "i4": 5, "u4": 6, "f4": 7, "f8": 8}


def driver_input(path, arrays, last=np.eye(4), curr=np.eye(4), big_endian=()):
    """the driver's in.bin: the history, the period and one message per structured array (its fields as PointFields)"""
    with open(path, "wb") as fh:
        fh.write(np.ascontiguousarray(last.T, dtype=np.float64).tobytes())
        fh.write(np.ascontiguousarray(curr.T, dtype=np.float64).tobytes())
        fh.write(struct.pack("dI", PERIOD, len(arrays)))
        for k, a in enumerate(arrays):
            fields = a.dtype.fields
            fh.write(struct.pack("I", len(fields)))
            for name, (dt, off) in fields.items():
                fh.write(struct.pack("B", len(name)) + name.encode() + struct.pack("<IBI", off, PF_TYPES[dt.str[1:]], 1))
            fh.write(struct.pack("<BIII", 1 if k in big_endian else 0, a.size, 1, a.dtype.itemsize))
            fh.write(a.tobytes())


def parse_descriptions(text):
    out = []
    for line in text.strip().split("\n"):
        v = line.split()
        out.append((int(v[0]), int(v[1])) + ((int(v[2]), int(v[3]), float(v[4])) if len(v) == 5 else ()))
    return out


def test_shim_describes_the_time_field_like_the_python_mirror():
    """packedTimeOf against packed_time on every layout above; a message flagged big-endian is refused"""
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("deskew_driver", "packed_scan_b200.hpp")
    good = [pack_timed(np.zeros((3, 3), np.float32), np.zeros(3), layout)[0] for layout in sorted(TIMED)]
    refused = [a for name, a in refused_time_layouts().items() if name != "time_big_endian"]   # a per-field byte order is
    arrays = good + refused + [good[0]]                                                         # not a PointCloud2's
    path = os.path.join(os.path.dirname(exe), "deskew_describe.bin")
    driver_input(path, arrays, big_endian=(len(arrays) - 1,))                 # the last: the XYZIRT message, big-endian
    res = subprocess.run([exe, "describe", path], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = parse_descriptions(res.stdout)
    assert len(got) == len(arrays)
    for g, a in zip(got[:len(good)], good):
        d = tloam_b200.packed_time(a)
        assert g == (0, 0, d.offset, d.datatype, d.unit)
    assert [g[1:] for g in got[:len(good)]] == [(0,) + TIME_DESCRIPTORS[layout] for layout in sorted(TIMED)]
    for g, a in zip(got[len(good):-1], refused):
        with pytest.raises(ValueError):
            tloam_b200.packed_time(a)
        assert g == (0, _INVALID_ARG)
    assert got[-1] == (_INVALID_ARG, _INVALID_ARG)                          # big-endian: both descriptors refused


def test_deskew_library_holds_only_the_three_kernels_for_sm90a():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.DESKEW_LIB))
    assert len(names) == 3 and [sum(f"{len(k)}{k}E" in m for m in names) for k in ("k_deskew", "k_deskew_tend", "k_deskew_motion")] == [1, 1, 1]
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.DESKEW_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)


# ---------------------------------------------------------------------------------------------------------------------
def seeded(r):
    """the handle's history set to the seeded increment: last = I, curr = exp(XI_SEED)"""
    curr = scipy.linalg.expm(hat(XI_SEED))
    r.set_pose_history(np.eye(4), curr)
    return np.eye(4), curr


def corrected(r):
    """the scan the device corrected, read back through the global map's registered scan at pose I"""
    r.global_map_append_frame(np.eye(4))
    return r.registered_scan()


def assert_matches_restatement(got, raw, times, last, curr):
    want = dko.deskew(raw, times, PERIOD, last, curr)
    fin = np.isfinite(raw).all(axis=1)
    assert got.shape == raw.shape
    assert np.all(~np.isfinite(got[~fin]).all(axis=1))                     # non-finite rows stay non-finite
    assert np.abs(got[fin] - want[fin]).max() <= 1e-10
    te = dko.t_end(times)
    still = fin & (~np.isfinite(times) | (times == te))                   # s = 0: the raw row, bit for bit
    assert still.sum() >= 1 and same_bits(got[still], raw[still])
    assert np.linalg.norm(got[fin] - raw[fin], axis=1).max() > 1.0        # the correction is not negligible


def scan_times(n, seed, nonfinite=True):
    """times in [0, PERIOD) s with NaN / +-Inf on a few rows"""
    rng = np.random.default_rng(seed)
    t = rng.uniform(0.0, PERIOD * 0.999, n)
    if nonfinite:
        bad = rng.choice(n, 300, replace=False)
        t[bad] = np.tile([np.nan, np.inf, -np.inf], 100)
    return t


@pytest.mark.gpu
def test_gpu_kernels_match_the_restatement():
    """the 116k-point HDL-64E scan with NaN / Inf rows: FP64 times (with non-finite ones), then float32 `time`, uint32-ns `t`
    and float64 `timestamp` fields read from the uploaded records"""
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    raw = with_nonfinite(synth.raw_scan(), 7)
    assert len(raw) > 110_000
    t = scan_times(len(raw), 11)
    last, curr = seeded(r)
    r.process_raw_scan(raw, feature=FE, time=t, frame_period=PERIOD)
    assert_matches_restatement(corrected(r), raw, t, last, curr)
    f = f32_scan(raw)
    for k, layout in enumerate(sorted(TIMED)):
        a, tt = pack_timed(f, scan_times(len(f), 20 + k, nonfinite=layout == "velodyne_xyzirt22"), layout, seed=k)
        seeded(r)
        r.process_raw_scan_packed(a, feature=FE, deskew=True, frame_period=PERIOD)
        assert_matches_restatement(corrected(r), f.astype(np.float64), tt, last, curr)
    r.close()


def loop_scans(frames=7):
    xis = [np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k + 0.001 * (k % 2)]) for k in range(frames)]
    scan0 = synth.raw_scan()
    return [f32_scan(with_nonfinite(scan0, 90))] + [f32_scan(with_nonfinite(moved(scan0, xi, 100 + k), 200 + k))
                                                     for k, xi in enumerate(xis) if k > 0]


def timed_loop(arrs, deskew, history=None, fitness_thres=0.3):
    """frame 0: process_raw_scan_packed -> submap_init_frame; frames 1..: process_raw_scan_packed -> scan_match_predicted_async
    -> submap_update_frame_chained -> global_map_append_frame chained.  history: (last, curr) seeded before frame 0 and after
    the submap's initialisation.  Returns the poses, the source clouds and the registered scan of every frame, and the handle."""
    import tloam_b200
    r = tloam_b200.LocalRegistration(fitness_thres=fitness_thres)
    r.enable_global_map()
    last, curr = history if history is not None else (synth.se3_exp(-np.array([0.3, 0.02, 0, 0, 0, 0.005])), np.eye(4))
    if history is not None:
        r.set_pose_history(last, curr)
    r.process_raw_scan_packed(arrs[0], feature=FE, deskew=deskew, frame_period=PERIOD)
    r.submap_init_frame()
    r.set_pose_history(last, curr)
    poses, sources, regs = [], [], []
    for a in arrs[1:]:
        r.process_raw_scan_packed(a, feature=FE, deskew=deskew, frame_period=PERIOD)
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        r.global_map_append_frame()
        poses.append(r.get_result())
        sources.append([r.source_cloud(c) for c in range(4)])
        regs.append(r.registered_scan())
    return poses, sources, r, regs


def assert_same_loop(a, b):
    (pa, sa, ra, _), (pb, sb, rb, _) = a, b
    for k in range(len(pa)):
        assert np.array_equal(pa[k], pb[k]), k
        for c in range(4):
            assert same_bits(sa[k][c], sb[k][c]), (k, c)
    assert np.array_equal(ra.global_map(), rb.global_map()) and np.array_equal(ra.global_map_frames(), rb.global_map_frames())
    assert same_bits(ra.registered_scan(), rb.registered_scan())


@pytest.mark.gpu
def test_gpu_identity_cases_are_bit_identical_to_the_untimed_loop():
    """all times equal (s = 0 on every row) over a 7-frame chained loop, and a fresh handle's identity history (frame 0 and
    frame 1 are not corrected): poses, source clouds, map and frame table are the untimed loop's bits"""
    scans = loop_scans()
    equal = [pack_timed(s, np.full(len(s), 0.05), "velodyne_xyzirt22", seed=k)[0] for k, s in enumerate(scans)]
    plain = timed_loop(equal, False)
    assert len(plain[0]) == 6 and plain[1][-1][2].shape[0] > 100
    timed = timed_loop(equal, True)
    assert_same_loop(timed, plain)
    timed[2].close()
    import tloam_b200
    varying = [pack_timed(s, scan_times(len(s), 40 + k, nonfinite=False), "ouster48", seed=k)[0] for k, s in enumerate(scans[:2])]
    p, q = tloam_b200.LocalRegistration(), tloam_b200.LocalRegistration()
    for r in (p, q):
        r.enable_global_map()
    for a in varying:
        p.process_raw_scan_packed(a, feature=FE, deskew=True)
        q.process_raw_scan_packed(a, feature=FE)
        for c in range(4):
            assert same_bits(p.source_cloud(c), q.source_cloud(c))
        assert same_bits(corrected(p), corrected(q))
    p.close()
    q.close()
    plain[2].close()


@pytest.mark.gpu
def test_gpu_timed_loop_is_deterministic_and_differs_from_the_untimed_loop():
    scans = loop_scans()
    arrs = [pack_timed(s, scan_times(len(s), 60 + k), "velodyne_xyzirt22", seed=k)[0] for k, s in enumerate(scans)]
    a, b = timed_loop(arrs, True), timed_loop(arrs, True)
    assert_same_loop(a, b)
    plain = timed_loop(arrs, False)
    assert not np.array_equal(a[0][-1], plain[0][-1])
    for r in (a[2], b[2], plain[2]):
        r.close()


# ---- a rolling-shutter sequence ---------------------------------------------------------------------------------------
TWIST = np.array([15.0, 0.0, 0.0, 0.0, 0.0, 0.2])               # body-frame velocity: 15 m/s forward, 0.2 rad/s of yaw
ELEV = np.radians([-24.9 + 0.4 * i + (1.7 if i >= 31 else 0.0) for i in range(64)])


def world_hits(o, d, rng_boxes):
    """ray parameter of the first return of rays o + t d (world frame, unit d; inf: none) in a street along x with cross
    streets every 40 m (their building faces are perpendicular to the road), parked boxes and poles on both kerbs"""
    t = np.full(len(d), np.inf)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        tg = np.where(d[:, 2] < -1e-6, (-1.73 - o[:, 2]) / d[:, 2], np.inf)            # ground
        t = np.minimum(t, tg)
        for yw in (8.0, -8.0):                                                         # kerb-side walls, gaps at cross streets
            tw = np.where((yw - o[:, 1]) * d[:, 1] > 1e-9, (yw - o[:, 1]) / d[:, 1], np.inf)
            x = o[:, 0] + tw * d[:, 0]
            z = o[:, 2] + tw * d[:, 2]
            gap = np.mod(x, 40.0) - 15.0
            t = np.minimum(t, np.where((z < 4.3) & (z > -1.73) & ((gap < 0) | (gap > 10.0)), tw, np.inf))
        for xc in np.arange(-65.0, 185.0, 40.0):                                       # cross-street building faces
            for xw in (xc, xc + 10.0):
                tw = np.where((xw - o[:, 0]) * d[:, 0] > 1e-9, (xw - o[:, 0]) / d[:, 0], np.inf)
                y = o[:, 1] + tw * d[:, 1]
                z = o[:, 2] + tw * d[:, 2]
                ok = (np.abs(y) > 8.0) & (np.abs(y) < 30.0) & (z < 4.3) & (z > -1.73)
                t = np.minimum(t, np.where(ok, tw, np.inf))
        for c, h in rng_boxes:                                                         # boxes: slab test
            t1, t2 = (c - h - o) / d, (c + h - o) / d
            tn, tf = np.nanmax(np.minimum(t1, t2), axis=1), np.nanmin(np.maximum(t1, t2), axis=1)
            t = np.minimum(t, np.where((tn <= tf) & (tn > 0), tn, np.inf))
        a = d[:, 0] ** 2 + d[:, 1] ** 2
        for px in np.arange(-60.0, 180.0, 7.0):                                        # poles, radius 0.15 m, 5 m high
            for py in (6.5, -6.5):
                ox, oy = o[:, 0] - px, o[:, 1] - py
                b = ox * d[:, 0] + oy * d[:, 1]
                disc = b * b - a * (ox * ox + oy * oy - 0.15 ** 2)
                tp = (-b - np.sqrt(np.maximum(disc, 0.0))) / a
                z = o[:, 2] + tp * d[:, 2]
                t = np.minimum(t, np.where((disc > 0) & (tp > 0) & (z < 3.27) & (z > -1.73), tp, np.inf))
    return t


def rolling_shutter_sequence(frames, n_az=1200, seed=5):
    """HDL-64E-shaped scans (beam after beam, each sweeping the azimuth from +x counter-clockwise) taken while the sensor moves
    along exp(tau . TWIST): every column is cast from the pose at its own time.  Returns per frame the float32 rows (sensor
    frame at the column's time), the float32 time from the sweep's start, the pose at the frame's last time and the world
    point every row was cast to."""
    rng = np.random.default_rng(seed)
    boxes = [(np.array([x, s * rng.uniform(3.5, 6.0), -1.73 + 0.75]), np.array([2.2, 0.9, 0.75]))
             for x, s in zip(rng.uniform(-40, 160, 24), rng.choice([-1.0, 1.0], 24))]
    az = (np.arange(n_az) + 0.5) * (2 * np.pi / n_az)
    el, a = np.meshgrid(ELEV, az, indexing="ij")
    d = np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.sin(el)], axis=-1).reshape(-1, 3)
    col = np.tile(np.arange(n_az), len(ELEV))
    out = []
    for k in range(frames):
        tau = k * PERIOD + (np.arange(n_az) + 0.5) / n_az * PERIOD
        Rs, ts = dko.se3_exp(tau[:, None] * TWIST[None, :])
        dw = np.einsum("nij,nj->ni", Rs[col], d)
        t = world_hits(ts[col], dw, boxes)
        keep = np.isfinite(t) & (t < 120.0) & (t > 3.0) & (rng.random(len(t)) >= 0.03)
        p = (d[keep] * t[keep, None] + rng.normal(0, 0.01, (int(keep.sum()), 3))).astype(np.float32)
        world = ts[col][keep] + t[keep, None] * dw[keep]
        rel = (tau[col[keep]] - k * PERIOD).astype(np.float32)
        te = k * PERIOD + float(rel.max())
        R, tt = dko.se3_exp(te * TWIST)
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, tt
        out.append((p, rel, T, world))
    return out


def pose_errors(poses, gts):
    """per frame: translation (m) and rotation (rad) of gt^-1 . estimate"""
    et, er = [], []
    for P, G in zip(poses, gts):
        D = np.linalg.inv(G) @ P
        et.append(float(np.linalg.norm(D[:3, 3])))
        er.append(float(np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1))))
    return np.array(et), np.array(er)


# bounds from the first runs on an H100 80GB HBM3 (400 W power limit), with margin.  Deskewed, the loop's pose errors were
# at most 0.16 m / 0.0056 rad over 8 frames, and the same registration noise (2-5 cm per frame) sets the untimed loop's: at a
# constant velocity every raw frame is warped alike, so the warp largely cancels in scan-to-map odometry.  It does not cancel
# in what the loop maps: the raw rows land up to a sweep's travel (1.5 m) from where they were measured.
TIMED_MAX_TRANSLATION, TIMED_MAX_ROTATION = 0.3, 0.012
TIMED_MAX_MEAN_MAP_ERROR = 0.25


@pytest.mark.gpu
def test_gpu_deskewing_brings_the_rolling_shutter_poses_and_map_to_ground_truth():
    """9 frames at 15 m/s and 0.2 rad/s, 10 Hz, through the packed chained loop with and without deskewing.  The history is
    seeded with the true increment before frame 0 (so frame 0 and the submap it seeds are corrected too) and for frame 1's
    prediction.  Poses are compared with the ground truth at each frame's last time, relative to frame 0's; every registered
    row, placed in the world by frame 0's true pose, with the world point it was cast to."""
    seq = rolling_shutter_sequence(9)
    arrs = [pack_timed(p, rel.astype(np.float64), "velodyne_xyzirt22", seed=k)[0] for k, (p, rel, _, _) in enumerate(seq)]
    T0 = seq[0][2]
    gts = [np.linalg.inv(T0) @ T for _, _, T, _ in seq[1:]]
    step = scipy.linalg.expm(hat(PERIOD * TWIST))
    hist = (np.linalg.inv(step), np.eye(4))
    res = {}
    for deskew in (True, False):
        poses, _, r, regs = timed_loop(arrs, deskew, history=hist)
        err = [np.linalg.norm(reg @ T0[:3, :3].T + T0[:3, 3] - w, axis=1).mean() for reg, (_, _, _, w) in zip(regs, seq[1:])]
        res[deskew] = pose_errors(poses, gts) + (np.array(err),)
        r.close()
    (tt, tr, tm), (ut, ur, um) = res[True], res[False]
    for name, (a, b, c) in (("deskewed", res[True]), ("raw", res[False])):
        print(f"{name}: translation {np.array2string(a, precision=4)} m, rotation {np.array2string(b, precision=5)} rad, "
              f"mean map error {np.array2string(c, precision=3)} m")
    assert tt.max() < TIMED_MAX_TRANSLATION and tr.max() < TIMED_MAX_ROTATION
    assert tm.max() < TIMED_MAX_MEAN_MAP_ERROR and tm.max() < 0.5 * um.min()


# ---- status codes and the shim ---------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_gpu_timed_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    raw = synth.raw_scan(n_az=200)
    a, _ = pack_timed(f32_scan(raw), scan_times(len(raw), 3, nonfinite=False), "velodyne_xyzirt22")
    scan = tloam_b200.packed_scan(a)
    good = tloam_b200.packed_time(a)
    t = scan_times(len(raw), 4, nonfinite=False)
    dp = C.POINTER(C.c_double)
    gc, dc, fc = _lib.GroundConfig(), _lib.DcvcConfig(), r._feature_config(FE)
    L.tloam_b200_ground_default_config(C.byref(gc))
    L.tloam_b200_dcvc_default_config(C.byref(dc))
    ns = (C.c_size_t * 4)()

    def fp64(xyz, time, n, period):
        return L.tloam_b200_process_raw_scan_timed(h, C.byref(gc), C.byref(dc), 131, 3.0, C.byref(fc), 0.3, 0.1, xyz, time, n, period, ns)

    def packed(s, tm, period=PERIOD):
        return L.tloam_b200_process_raw_scan_packed_timed(h, C.byref(gc), C.byref(dc), 131, 3.0, C.byref(fc), 0.3, 0.1, s, tm, period, ns)

    def tdesc(**kw):
        d = _lib.PackedTime(good.offset, good.datatype, good.unit)
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    xyz, tp = raw.ctypes.data_as(dp), t.ctypes.data_as(dp)
    bad_periods = [0.0, -0.1, float("nan"), float("inf"), -float("inf")]
    assert fp64(xyz, None, len(raw), PERIOD) == _lib.ERR_INVALID_ARG
    for p in bad_periods:
        assert fp64(xyz, tp, len(raw), p) == _lib.ERR_INVALID_ARG, p
        assert packed(C.byref(scan), C.byref(good), p) == _lib.ERR_INVALID_ARG, p
    assert packed(C.byref(scan), None) == _lib.ERR_INVALID_ARG
    assert packed(None, C.byref(good)) == _lib.ERR_INVALID_ARG
    bad = [tdesc(offset=-1), tdesc(offset=19), tdesc(datatype=8, offset=15), tdesc(datatype=5), tdesc(datatype=9), tdesc(datatype=0),
           tdesc(unit=0.0), tdesc(unit=-1.0), tdesc(unit=float("nan")), tdesc(unit=float("inf"))]
    for d in bad:
        assert packed(C.byref(scan), C.byref(d)) == _lib.ERR_INVALID_ARG, (d.offset, d.datatype, d.unit)
    bad_scan = _lib.PackedScan(scan.data, scan.n, 11, 0, 4, 7, -1)
    assert packed(C.byref(bad_scan), C.byref(tdesc(offset=0))) == _lib.ERR_INVALID_ARG
    assert list(ns) == [0, 0, 0, 0]
    # the limits are valid: a field in the record's last bytes, an 8-byte field ending there, n == 0 without times
    assert packed(C.byref(scan), C.byref(tdesc(offset=18))) == _lib.OK and ns[3] > 0
    assert packed(C.byref(scan), C.byref(tdesc(offset=14, datatype=8))) == _lib.OK
    assert packed(C.byref(scan), C.byref(tdesc(offset=16, datatype=6, unit=1e-9))) == _lib.OK
    assert fp64(xyz, tp, len(raw), PERIOD) == _lib.OK and ns[3] > 0
    assert fp64(None, None, 0, PERIOD) == _lib.OK and list(ns) == [0, 0, 0, 0]
    empty = _lib.PackedScan(None, 0, 22, 0, 4, 8, 12)
    assert packed(C.byref(empty), None) == _lib.OK
    with pytest.raises(ValueError):
        r.process_raw_scan(raw, time=t[:-1])
    with pytest.raises(ValueError):
        r.process_raw_scan_packed(np.ascontiguousarray(f32_scan(raw)), deskew=True)     # (n, 3) records have no time field
    r.close()


@pytest.mark.gpu
def test_gpu_deskew_shim_matches_the_python_mirror():
    """packedScanOf + packedTimeOf + tloam_b200_process_raw_scan_packed_timed on the driver's messages: the corrected scans
    of the Python mirror, bit for bit"""
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("deskew_driver", "packed_scan_b200.hpp")
    raw = f32_scan(with_nonfinite(synth.raw_scan(n_az=1200), 8))
    arrays = [pack_timed(raw, scan_times(len(raw), 80 + k, nonfinite=layout == "velodyne_xyzirt22"), layout, seed=k)[0]
              for k, layout in enumerate(sorted(TIMED))]
    last = synth.se3_exp([2.0, 1.0, 0.0, 0.0, 0.0, 0.3])
    curr = last @ scipy.linalg.expm(hat(XI_SEED))
    d = os.path.dirname(exe)
    paths = [os.path.join(d, "deskew_in.bin"), os.path.join(d, "deskew_out.bin")]
    driver_input(paths[0], arrays, last, curr)
    res = subprocess.run([exe, "run"] + paths, capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    assert [g[:2] for g in parse_descriptions(res.stdout)] == [(0, 0)] * 3
    blob = open(paths[1], "rb").read()
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    o = 0
    for a in arrays:
        n = struct.unpack_from("Q", blob, o)[0]
        cpp = np.frombuffer(blob, dtype=np.float64, count=3 * n, offset=o + 8).reshape(-1, 3)
        o += 8 + 24 * n
        r.set_pose_history(last, curr)
        r.process_raw_scan_packed(a, feature=FE, deskew=True)
        py = corrected(r)
        assert n == len(raw) and same_bits(cpp, py)
        fin = np.isfinite(raw).all(axis=1)
        assert np.abs(py[fin] - raw[fin]).max() > 1.0
    assert o == len(blob)
    r.close()
