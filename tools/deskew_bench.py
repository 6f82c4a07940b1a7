"""Deskewing cost on the 116k-point synthetic HDL-64E scan (the street scene of synth.raw_scan) as a 32-byte XYZIRT-style
message: x, y, z, intensity at 0 / 4 / 8 / 12, ring at 16, float32 time (s from the sweep's start) at 20.
  (a) one process_raw_scan_packed call;
  (b) one process_raw_scan_packed(deskew=True) call: (a) plus the three deskew kernels and the gathers from the corrected
      scan.
Both calls end in the call's own synchronise (they read the source sizes).  The pose history is seeded with a 1.5 m /
0.05 rad increment so the correction does work.  The forms alternate within one call, `rounds` rounds of `calls` calls
each, after a warm-up.  Then k_deskew_motion, k_deskew_tend (from the packed records) and k_deskew are timed with CUDA
events over back-to-back launches of each, through libtloam_b200_deskew.so's launchers.  Prints the card and its power limit
read in the same call.

    python tools/deskew_bench.py [calls] [rounds]
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import tloam_b200  # noqa: E402
from tloam_b200 import build, synth  # noqa: E402

FE = dict(cvr_submap=0.005, cvr_scan=0.01)        # the street scene has few curvature maxima (tests/test_front_end_chain.py)
XYZIRT32 = np.dtype(dict(names=["x", "y", "z", "intensity", "ring", "time"], formats=["<f4", "<f4", "<f4", "<f4", "<u2", "<f4"],
                         offsets=[0, 4, 8, 12, 16, 20], itemsize=32))
PERIOD = 0.1
XI = [1.5, 0.0, 0.0, 0.0, 0.0, 0.05]


def message():
    raw = synth.raw_scan()
    m = np.zeros(len(raw), XYZIRT32)
    m["x"], m["y"], m["z"] = raw[:, 0], raw[:, 1], raw[:, 2]
    m["intensity"] = np.random.default_rng(5).uniform(0.0, 255.0, len(raw)).astype(np.float32)
    m["ring"] = np.arange(len(raw)) % 64
    az = np.mod(np.arctan2(raw[:, 1], raw[:, 0]), 2 * np.pi)                 # counter-clockwise sweep from +x
    m["time"] = (az / (2 * np.pi) * PERIOD).astype(np.float32)
    return m


def call_ms(r, m, deskew, calls):
    t0 = time.perf_counter()
    for _ in range(calls):
        r.process_raw_scan_packed(m, feature=FE, deskew=deskew, frame_period=PERIOD)
    return 1e3 * (time.perf_counter() - t0) / calls


class Args(C.Structure):                           # tloam_deskew_args (tloam_b200/csrc/deskew.h)
    _fields_ = [("last_pose", C.c_void_p), ("curr_pose", C.c_void_p), ("time", C.c_void_p), ("records", C.c_void_p),
                ("point_step", C.c_ulonglong), ("offset", C.c_int), ("datatype", C.c_int), ("unit", C.c_double),
                ("n", C.c_ulonglong), ("period", C.c_double), ("xyz", C.c_void_p), ("out", C.c_void_p), ("scratch", C.c_void_p),
                ("device", C.c_int), ("stream", C.c_void_p)]


def kernel_ms(m, launches=200):
    """each deskew kernel alone: CUDA events around `launches` back-to-back launches; returns ms per launch (3 windows)"""
    import torch
    lib = C.CDLL(build.DESKEW_LIB)
    n, ps = len(m), m.dtype.itemsize
    dev = torch.cuda.current_device()
    stream = torch.cuda.current_stream()
    rec = torch.from_numpy(m.view(np.uint8).reshape(-1).copy()).cuda()
    xyz = torch.from_numpy(np.column_stack([m["x"], m["y"], m["z"]]).astype(np.float64).reshape(-1)).cuda()
    out = torch.empty_like(xyz)
    last = torch.eye(4, dtype=torch.float64, device="cuda")
    curr = torch.from_numpy(np.ascontiguousarray(synth.se3_exp(XI).T)).cuda()    # column-major
    scratch = torch.zeros(8, dtype=torch.float64, device="cuda")
    a = Args(last.data_ptr(), curr.data_ptr(), None, rec.data_ptr(), ps, 20, 7, 1.0, n, PERIOD, xyz.data_ptr(), out.data_ptr(),
             scratch.data_ptr(), dev, stream.cuda_stream)
    fns = {"k_deskew_motion": lib.tloam_deskew_motion, "k_deskew_tend": lib.tloam_deskew_tend, "k_deskew": lib.tloam_deskew_apply}
    for f in fns.values():
        f.argtypes = [C.POINTER(Args)]
        assert f(C.byref(a)) == 0
    res = {}
    for name, f in fns.items():
        if name == "k_deskew_tend":
            launch = lambda: (lib.tloam_deskew_motion(C.byref(a)), f(C.byref(a)))   # noqa: E731  (t_end is cleared by motion)
        else:
            launch = lambda f=f: f(C.byref(a))                                         # noqa: E731
        for _ in range(10):
            launch()
        per = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(launches):
                launch()
            e1.record(stream)
            e1.synchronize()
            per.append(round(e0.elapsed_time(e1) / launches, 4))
        res[name] = per
    motion = res["k_deskew_motion"]
    res["k_deskew_tend"] = [round(x - y, 4) for x, y in zip(res["k_deskew_tend"], motion)] + ["net of k_deskew_motion"]
    return res


def main():
    args = [int(a) for a in sys.argv[1:]]
    calls = args[0] if args else 20
    rounds = args[1] if len(args) > 1 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    m = message()
    r = tloam_b200.LocalRegistration()
    T = synth.se3_exp(XI)
    r.set_pose_history(np.eye(4), T)
    res = {"gpu": card, "raw_points": len(m), "point_step": m.dtype.itemsize, "calls": calls, "rounds": rounds}
    call_ms(r, m, False, 5)                                   # warm-up: modules, staging threads, buffers, the deskew library
    call_ms(r, m, True, 5)
    runs = {False: [], True: []}
    for _ in range(rounds):
        for deskew in (False, True):                          # alternating: the shared card drifts
            runs[deskew].append(round(call_ms(r, m, deskew, calls), 3))
    r.close()
    res["packed_ms_per_call"] = runs[False]
    res["packed_timed_ms_per_call"] = runs[True]
    res["packed_median_ms"] = float(np.median(runs[False]))
    res["packed_timed_median_ms"] = float(np.median(runs[True]))
    res["kernel_ms"] = kernel_ms(m)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
