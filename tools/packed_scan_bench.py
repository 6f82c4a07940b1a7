"""Raw scans in the sensor's packed float32 layout against the FP64 form, on the 116k-point synthetic HDL-64E scan (the street
scene of synth.raw_scan) as the driver would publish it: velodyne-style 32-byte XYZI records (x, y, z at 0 / 4 / 8,
intensity at 16, ring at 20).  The per-frame loop with mapping on, frames 1 .. `frames`:
  (a) the message converted with numpy (what a caller does today: every float to a double, xyz and intensity in two
      arrays), then process_raw_scan + global_map_append_frame(intensity=...) chained;
  (b) process_raw_scan_packed(message) + global_map_append_frame() chained: one upload, unpacked on the device;
  (c) (b) with the scan as a KITTI .bin (16-byte records x, y, z, reflectance).
Each loop also runs scan_match_predicted_async, submap_update_frame_chained and get_result, so every frame ends in a
synchronise.  The forms alternate within one call, `rounds` rounds each; the first round checks that (a), (b) and (c) give
the same poses, map and intensity channel bit for bit.  One k_unpack_scan launch of the 32-byte message is timed with CUDA
events over back-to-back launches.  Prints the card and its power limit read in the same call, and the bytes each form
moves over PCIe per frame.

    python tools/packed_scan_bench.py [frames] [rounds]
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
XYZIR32 = np.dtype(dict(names=["x", "y", "z", "intensity", "ring"], formats=["<f4", "<f4", "<f4", "<f4", "<u2"],
                        offsets=[0, 4, 8, 16, 20], itemsize=32))


def messages(frames):
    """frames + 1 scans of a sensor moving along the street, each as a 32-byte XYZI message and as a KITTI (n, 4) array"""
    raw = synth.raw_scan()
    rng = np.random.default_rng(5)
    out = []
    for k in range(frames + 1):
        Ti = np.linalg.inv(synth.se3_exp([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k]))
        f = (raw @ Ti[:3, :3].T + Ti[:3, 3]).astype(np.float32)
        m = np.zeros(len(f), XYZIR32)
        m["x"], m["y"], m["z"] = f[:, 0], f[:, 1], f[:, 2]
        m["intensity"] = rng.uniform(0.0, 255.0, len(f)).astype(np.float32)
        m["ring"] = np.arange(len(f)) % 64
        kitti = np.ascontiguousarray(np.column_stack([f, m["intensity"]]))
        out.append((m, kitti))
    return out


def run(form, msgs):
    """one loop; returns ms per frame (frames 1 ..) and the handle"""
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()

    def process(k):
        m, kitti = msgs[k]
        if form == "a_fp64":
            xyz = np.column_stack([m["x"], m["y"], m["z"]]).astype(np.float64)
            inten = m["intensity"].astype(np.float64)
            r.process_raw_scan(xyz, feature=FE)
            return inten
        r.process_raw_scan_packed(m if form == "b_packed32" else kitti, feature=FE)
        return None

    process(0)
    r.submap_init_frame()
    r.set_pose_history(synth.se3_exp(-np.array([0.3, 0.02, 0, 0, 0, 0.004])), np.eye(4))
    poses = []
    t0 = time.perf_counter()
    for k in range(1, len(msgs)):
        inten = process(k)
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        r.global_map_append_frame(intensity=inten)
        poses.append(r.get_result())
    ms = 1e3 * (time.perf_counter() - t0) / (len(msgs) - 1)
    return ms, r, poses


def unpack_kernel_ms(m, launches=200):
    """k_unpack_scan alone on the 32-byte message: CUDA events around `launches` back-to-back launches"""
    import torch
    lib = C.CDLL(build.UNPACK_LIB)
    lib.tloam_unpack_scan.argtypes = [C.c_void_p, C.c_ulonglong, C.c_ulonglong, C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_int,
                                      C.c_void_p]
    n, ps = len(m), m.dtype.itemsize
    src = torch.zeros((n * ps + 15) // 16 * 16, dtype=torch.uint8, device="cuda")
    src[:n * ps].copy_(torch.from_numpy(m.view(np.uint8).reshape(-1)))
    xyz = torch.empty(3 * n, dtype=torch.float64, device="cuda")
    inten = torch.empty(n, dtype=torch.float64, device="cuda")
    off = (C.c_int * 4)(0, 4, 8, 16)
    stream = torch.cuda.current_stream()

    def launch():
        rc = lib.tloam_unpack_scan(src.data_ptr(), n, ps, off, xyz.data_ptr(), inten.data_ptr(), torch.cuda.current_device(),
                                   stream.cuda_stream)
        assert rc == 0, rc

    for _ in range(10):
        launch()
    per = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(launches):
            launch()
        b.record(stream)
        b.synchronize()
        per.append(a.elapsed_time(b) / launches)
    f = np.column_stack([m["x"], m["y"], m["z"]]).astype(np.float64).reshape(-1)
    exact = np.array_equal(xyz.cpu().numpy(), f) and np.array_equal(inten.cpu().numpy(), m["intensity"].astype(np.float64))
    return per, exact, 32 * n + 32 * n                    # bytes read (records) + written (xyz + intensity, FP64)


def main():
    args = [int(a) for a in sys.argv[1:]]
    frames = args[0] if args else 8
    rounds = args[1] if len(args) > 1 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    msgs = messages(frames)
    n = len(msgs[0][0])
    res = {"gpu": card, "raw_points": n, "frames": frames, "rounds": rounds,
           "pcie_bytes_per_frame": {"a_fp64": 32 * n, "b_packed32": 32 * n, "c_packed16": 16 * n}}
    forms = ("a_fp64", "b_packed32", "c_packed16")
    runs = {f: [] for f in forms}
    run("a_fp64", msgs[:3])[1].close()                    # warm-up: modules, staging threads, buffers
    run("b_packed32", msgs[:3])[1].close()
    for rd in range(rounds):
        outs = {}
        for form in forms:                                # alternating: the shared card drifts
            ms, r, poses = run(form, msgs)
            runs[form].append(round(ms, 3))
            if rd == 0:
                outs[form] = (poses, r.global_map(), r.global_map_frames(), r.global_map_intensity())
            r.close()
        if rd == 0:
            ref = outs["a_fp64"]
            res["same_bits"] = all(
                all(np.array_equal(x, y) for x, y in zip(o[0], ref[0])) and np.array_equal(o[1], ref[1]) and np.array_equal(o[2], ref[2])
                and np.array_equal(o[3].view(np.uint64), ref[3].view(np.uint64)) for o in outs.values())
    for form in forms:
        res[f"{form}_ms_per_frame"] = runs[form]
        res[f"{form}_median_ms"] = float(np.median(runs[form]))
    per, exact, nbytes = unpack_kernel_ms(msgs[0][0])
    res["k_unpack_scan_ms"] = [round(x, 4) for x in per]
    res["k_unpack_scan_exact"] = bool(exact)
    res["k_unpack_scan_GB_per_s"] = round(nbytes / (float(np.median(per)) * 1e-3) / 1e9, 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
