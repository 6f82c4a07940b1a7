"""Distance field and costmap (include/tloam_b200.h "Distance field and costmap"): the cost of a build and of a query on a
seq-00-shaped occupancy grid, against scipy's EDT of the same grid on the host.
  - grid: the occupancy build of a seq-00-shaped drive, 4 541 frames at the poses of tests/test_pose_graph.seq_graph("00"),
    each appending the HDL-64E scan (tloam_b200.synth.raw_scan), at the occupancy defaults, as tools/occupancy_bench.py
    builds it.
  - build: distance_build at the defaults, after warm-up: the C call's host clock (it synchronises) and its kernels'
    device time from the CUDA events; the bytes the passes must move at least (the grid read by the three passes that
    classify cells, the column distance and sq written and read once, sd, cost and value written) and their share of
    3.35 TB/s.  The occupancy build's own time is printed beside it.
  - kernels: the split by kernel from torch.profiler, in a separate run.
  - query: one distance_query of 10^6 points (host clock, device time).
  - scipy: scipy.ndimage.distance_transform_edt of the grid's obstacles and of its other cells, on the host.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/distance_bench.py [frames] [builds]
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

KERNELS = ("k_dist_bands", "k_dist_cols", "k_dist_rows", "k_dist_cost", "k_dist_query")
HBM_BYTES_PER_S = 3.35e12       # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def device_ms(r):
    return sum(v for _, v in r.get_profile().values())


def timed(r, call):
    r.set_profiling(True)
    t0 = time.perf_counter()
    call()
    host = (time.perf_counter() - t0) * 1e3
    dev = device_ms(r)
    r.set_profiling(False)
    return host, dev


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 4541
    builds = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    print(card(), flush=True)
    from test_pose_graph import seq_graph
    scan = synth.raw_scan()
    G = seq_graph("00")[0][:frames]
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=1 << 25)
    r.occupancy_enable()
    for P in G:
        r.global_map_append(scan, P)
    r.global_map_size()
    occ = r.occupancy_build()
    h, w = occ.cells.shape
    occ_host, occ_dev = timed(r, lambda: r.occupancy_build())

    cfg = _lib.DistanceConfig()
    r._L.tloam_b200_distance_default_config(C.byref(cfg))
    info = _lib.DistanceInfo()

    def build():
        assert r._L.tloam_b200_distance_build(r._h, C.byref(cfg), C.byref(info)) == 0

    for _ in range(3):
        build()                                                     # warm: loads the library, allocates
    host, dev = [], []
    for _ in range(builds):
        a, b = timed(r, build)
        host.append(a)
        dev.append(b)
    cells = w * h
    moved = cells * (3 * 1 + 2 * 4 + 2 * 4 + 4 + 1 + 1)
    d = float(np.median(dev))
    f = r.distance_build()
    print(json.dumps(dict(case=f"distance_build of the occupancy grid of {frames} frames at the defaults", grid=[w, h],
                          cells=cells, obstacles=int(info.obstacles),
                          host_ms_median=round(float(np.median(host)), 3), device_ms_median=round(d, 3),
                          device_ms_min=round(min(dev), 3), device_ms_max=round(max(dev), 3),
                          bytes_min=moved, bytes_min_share_of_3_35_TBps=round(moved / HBM_BYTES_PER_S / (d * 1e-3), 3),
                          occupancy_build_host_ms=round(occ_host, 2), occupancy_build_device_ms=round(occ_dev, 2),
                          finite_cells=int(np.isfinite(f.signed).sum()), max_distance_m=float(f.signed.max()))), flush=True)

    rng = np.random.default_rng(0)
    ox, oy = f.origin
    xy = np.column_stack([rng.uniform(ox, ox + w * f.resolution, 1_000_000), rng.uniform(oy, oy + h * f.resolution, 1_000_000)])
    r.distance_query(xy)
    qh, qd = timed(r, lambda: r.distance_query(xy))
    print(json.dumps(dict(case="distance_query of 10^6 points", host_ms=round(qh, 3), device_ms=round(qd, 4))), flush=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            build()
        r.distance_query(xy)
        torch.cuda.synchronize()
    seen = {}
    for e in prof.events():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = getattr(e, "cuda_time_total", 0.0)
        for k in KERNELS:
            if k in e.name:
                seen[k] = seen.get(k, 0.0) + dt / 1e3
    per = {k: round(v / (5 if k != "k_dist_query" else 1), 4) for k, v in sorted(seen.items())}
    print(json.dumps(dict(case="distance_build by kernel (torch.profiler, mean of 5 builds; k_dist_query of one call), ms",
                          kernels_ms=per)), flush=True)

    from scipy.ndimage import distance_transform_edt as edt
    ob = occ.cells.astype(np.int16) >= 65
    t0 = time.perf_counter()
    e1 = edt(~ob)
    e2 = edt(ob)
    s = time.perf_counter() - t0
    sq = np.where(ob, np.round(e2 ** 2), np.round(e1 ** 2))
    print(json.dumps(dict(case="scipy.ndimage.distance_transform_edt of the same grid on the host (both classes)",
                          seconds=round(s, 2), sq_equal=bool(np.array_equal(sq.astype(np.uint32), f.sq)))), flush=True)
    r.close()


if __name__ == "__main__":
    main()
