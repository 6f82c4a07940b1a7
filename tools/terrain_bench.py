"""Terrain map (include/tloam_b200.h "Terrain"): the cost of a build on a seq-00-shaped drive, and of the same build in numpy.
  - drive: 4 541 frames at the poses of tests/test_pose_graph.seq_graph("00"), each appending the HDL-64E scan
    (tloam_b200.synth.raw_scan) to a map of voxel 0.2 m (or the finest of 0.3 and 0.5 m that fits the device), the
    occupancy grid on.
  - build: terrain_build at the defaults with combine_occupancy (on the occupancy build's grid): host clock around the C
    call (it synchronises) and its kernels' device time from the handle's CUDA events, median over the builds after a
    warm-up; the bytes it must move at least (the rows read twice, the cell layers written: the values, three FP64 layers,
    four encodings and two counts) against 3.35 TB/s; the occupancy build's own time in the same call.
  - numpy: tests/terrain_oracle.build on the host over the map rows within a stated crop around the first pose, with the
    device's build of the same rows and whether their values agree.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/terrain_bench.py [frames] [crop_m]
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

PEAK_BPS = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def device_ms(r):
    return sum(v for _, v in r.get_profile().values())


def drive(G, scan, voxel):
    """a handle with the drive appended at this map voxel; None (the handle closed) when the map does not fit"""
    r = tloam_b200.LocalRegistration()
    try:
        r.enable_global_map(voxel=voxel, initial_capacity=1 << 26)
        r.occupancy_enable()
        for P in G:
            r.global_map_append(scan, P)
        r.global_map_size()                                         # a read-back: raises if an append was refused
    except (tloam_b200.RegistrationError, MemoryError):
        r.close()
        return None
    return r


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 4541
    crop = float(sys.argv[2]) if len(sys.argv) > 2 else 60.0
    print(card(), flush=True)
    from test_pose_graph import seq_graph
    G = seq_graph("00")[0][:frames]
    scan = synth.raw_scan()
    r, voxel = None, None
    for v in (0.2, 0.3, 0.5):
        r, voxel = drive(G, scan, v), v
        if r is not None:
            break
    if r is None:
        raise SystemExit("the drive does not fit the device at a map voxel of 0.5 m")
    rows = r.global_map_size()[0]
    t0 = time.perf_counter()
    g = r.occupancy_build()
    occ_host = (time.perf_counter() - t0) * 1e3
    cfg = _lib.TerrainConfig()
    r._L.tloam_b200_terrain_default_config(C.byref(cfg))
    cfg.combine_occupancy = 1
    info = _lib.TerrainInfo()
    assert r._L.tloam_b200_terrain_build(r._h, C.byref(cfg), C.byref(info)) == 0     # warm
    host, dev = [], []
    for _ in range(10):
        r.set_profiling(True)
        t0 = time.perf_counter()
        assert r._L.tloam_b200_terrain_build(r._h, C.byref(cfg), C.byref(info)) == 0
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(device_ms(r))
        r.set_profiling(False)
    r.set_profiling(True)
    r.occupancy_build()
    occ_dev = device_ms(r)
    r.set_profiling(False)
    cells = info.width * info.height
    moved = 2 * rows * 24 + cells * (1 + 3 * 8 + 4 * 8 + 2 * 4)
    d = float(np.median(dev))

    # the numpy restatement on a crop around the first pose, against the device's build of the same rows
    import terrain_oracle as to
    mp = r.global_map(0, min(rows, 4_000_000))                    # the drive's first frames
    c0 = G[0][:2, 3]
    sel = mp[(np.abs(mp[:, 0] - c0[0]) < crop / 2) & (np.abs(mp[:, 1] - c0[1]) < crop / 2)]
    t0 = time.perf_counter()
    want = to.build(sel, to.config())
    numpy_s = time.perf_counter() - t0
    got = r.terrain_build(sel)
    from test_global_map_intensity import same_bits                # bit for bit, any NaN equal to any NaN
    same = all(same_bits(getattr(got, k), want[k]) for k in ("values", "ground", "elevation", "step", "slope", "roughness",
                                                             "points"))
    case = f"terrain_build of a seq-00-shaped drive ({len(G)} frames), defaults, combined with the occupancy grid"
    print(json.dumps(dict(case=case,
                          map_voxel=voxel, rows=rows, grid=[info.width, info.height], cells=cells, known=info.known,
                          lethal=info.lethal, overhang=info.overhang, dropped=info.dropped,
                          host_ms=round(float(np.median(host)), 3), device_ms=round(d, 3),
                          bytes_min=moved, bound_share=round(moved / PEAK_BPS / (d * 1e-3), 3),
                          occupancy_build_host_ms=round(occ_host, 2), occupancy_build_device_ms=round(occ_dev, 3),
                          occupancy_grid=list(g.cells.shape[::-1]),
                          numpy_crop_m=crop, numpy_rows=len(sel), numpy_cells=int(want["values"].size),
                          numpy_s=round(numpy_s, 2), numpy_equals_device=same)), flush=True)
    r.close()


if __name__ == "__main__":
    main()
