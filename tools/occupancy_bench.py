"""Occupancy grid (include/tloam_b200.h "Occupancy grid"): the cost of a capture, of a build, and of the same build in numpy.
  - capture: one global_map_append of a 116 k-row HDL-64E scan (tloam_b200.synth.raw_scan) on a handle with the grid on
    against one with it off, alternated: device time from the handle's CUDA events and host clock to a synchronise.
  - build: a seq-00-shaped drive, 4 541 frames at the poses of tests/test_pose_graph.seq_graph("00"), each appending the
    HDL-64E scan, at the defaults: occupancy_build's host clock (the C call synchronises), its kernels' device time from
    the CUDA events, the counted window-cell tests per second, the bytes the build must move at least (each frame's 2D
    scan and pose read once, the two counters written and read, the values written) per second, and the 2D-scan bytes
    k_occ_free's blocks read (every block of a frame loads the frame's records; from HBM or from L2, which this does not
    tell apart).
  - numpy: the restatement (tests/occupancy_oracle.py) on the host over the first `numpy_frames` frames, scaled to the
    drive by frame count.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/occupancy_bench.py [frames] [numpy_frames]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tloam_b200  # noqa: E402
from tloam_b200 import _lib, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def device_ms(r):
    return sum(v for _, v in r.get_profile().values())


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 4541
    numpy_frames = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    print(card(), flush=True)
    scan = synth.raw_scan()

    # ---- capture: on against off, alternated
    res = {}
    handles = {}
    for mode in ("on", "off"):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map(initial_capacity=1 << 24)
        if mode == "on":
            r.occupancy_enable()
        handles[mode] = r
        res[mode] = ([], [])
    for rnd in range(60):
        for mode in ("on", "off") if rnd % 2 == 0 else ("off", "on"):
            r = handles[mode]
            r.set_profiling(True)
            t0 = time.perf_counter()
            r.global_map_append(scan, np.eye(4))
            r.global_map_size()                                     # a read-back: ends in a synchronise
            host = (time.perf_counter() - t0) * 1e3
            dev = device_ms(r)
            r.set_profiling(False)
            if rnd >= 4:
                res[mode][0].append(host)
                res[mode][1].append(dev)
    med = {m: (float(np.median(res[m][0])), float(np.median(res[m][1]))) for m in res}
    print(json.dumps(dict(case=f"global_map_append of an HDL-64E scan ({len(scan)} rows), grid on against off",
                          host_ms_on=round(med["on"][0], 4), host_ms_off=round(med["off"][0], 4),
                          device_ms_on=round(med["on"][1], 4), device_ms_off=round(med["off"][1], 4),
                          capture_device_ms=round(med["on"][1] - med["off"][1], 4))), flush=True)
    for r in handles.values():
        r.close()

    # ---- build of a seq-00-shaped drive
    from test_pose_graph import seq_graph
    G = seq_graph("00")[0][:frames]
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 25)
    r.occupancy_enable()
    t0 = time.perf_counter()
    for P in G:
        r.global_map_append(scan, P)
    r.global_map_size()
    append_s = time.perf_counter() - t0
    r.occupancy_build()                                             # warm
    info = _lib.OccupancyInfo()
    host, dev = [], []
    for _ in range(5):
        r.set_profiling(True)
        t0 = time.perf_counter()
        assert r._L.tloam_b200_occupancy_build(r._h, C.byref(info)) == 0
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(device_ms(r))
        r.set_profiling(False)
    cells = info.width * info.height
    n_cols = 1024
    moved = info.frames * (n_cols * 32 + 128) + cells * (4 + 4) * 2 + cells * 1
    window = info.cell_tests // info.frames                         # nwin^2 candidates per frame
    tiles = -(-window // (256 * 16))                                # k_occ_free's blocks per frame (occupancy.cu)
    block_reads = info.frames * tiles * n_cols * 32
    d = float(np.median(dev))
    print(json.dumps(dict(case=f"occupancy_build of {info.frames} frames at the defaults", grid=[info.width, info.height],
                          host_ms=[round(x, 2) for x in host], device_ms=[round(x, 2) for x in dev],
                          cell_tests=info.cell_tests, cell_tests_per_s=float(f"{info.cell_tests / (d * 1e-3):.3e}"),
                          bytes_min=moved, bytes_min_per_s=float(f"{moved / (d * 1e-3):.3e}"), blocks_per_frame=tiles,
                          record_bytes_read_by_blocks=block_reads, dropped=info.dropped,
                          appends_s=round(append_s, 2))), flush=True)

    # ---- numpy restatement of the same build, over the first numpy_frames frames
    import occupancy_oracle as oo
    cfg = oo.config()
    ob, fl, _ = r.occupancy_scans(0, numpy_frames)
    g = r.occupancy_build()
    D = oo.sco.boundaries(cfg["n_cols"])
    ox, oy = g.origin
    h, w = g.cells.shape
    occ, free = np.zeros((h, w), dtype=np.uint32), np.zeros((h, w), dtype=np.uint32)
    t0 = time.perf_counter()
    for k in range(numpy_frames):
        oo.free_counts(ob[k], fl[k], G[k], cfg, ox, oy, w, h, D, free)
        oo.hit_counts(ob[k], G[k], cfg, ox, oy, w, h, occ)
    s = time.perf_counter() - t0
    print(json.dumps(dict(case=f"the same build in numpy on the host ({numpy_frames} frames timed, scaled to {info.frames})",
                          seconds_timed=round(s, 2), seconds_scaled=round(s * info.frames / numpy_frames, 1))), flush=True)
    r.close()


if __name__ == "__main__":
    main()
