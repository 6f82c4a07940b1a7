"""Frontiers (include/tloam_b200.h "Frontiers"): the cost of a frontier search on a seq-00-shaped costmap, against the
numpy restatement on the host.
  - costmap and plan: the occupancy grid of a seq-00-shaped drive, 4 541 frames at the poses of
    tests/test_pose_graph.seq_graph("00"), each appending the HDL-64E scan (tloam_b200.synth.raw_scan), as
    tools/plan_bench.py builds it; the distance build at the defaults and plan_build at the defaults with the goal at the
    last pose (the robot).
  - search: frontier_search at the defaults after warm-up: the kernels' device time from the CUDA events and the C call's
    host clock (it synchronises), median over the searches; the frontier cells, the frontiers before and after the
    filter; the bytes the search must move (the codes read, the labels written, read by the compaction and read again,
    the frontier cells' keys, rows and statistics) against 3.35 TB/s.
  - split: the device time of each kernel from a separate torch.profiler run of one search.
  - host: tests/frontier_oracle.search on the same costs and potential, its time and whether it equals the device's.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/frontier_bench.py [frames] [searches]
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
import frontier_oracle as fo  # noqa: E402

HBM = 3.35e12                                                       # H100 SXM HBM3, bytes per second (data sheet)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def device_ms(r):
    return sum(v for _, v in r.get_profile().values())


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 4541
    searches = int(sys.argv[2]) if len(sys.argv) > 2 else 20
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
    r.occupancy_build()
    f = r.distance_build()
    h, w = f.costs.shape
    p = r.plan_build(G[-1][:2, 3])

    cfg = _lib.FrontierConfig()
    r._L.tloam_b200_frontier_default_config(C.byref(cfg))
    info = _lib.FrontierInfo()

    def search():
        assert r._L.tloam_b200_frontier_search(r._h, C.byref(cfg), C.byref(info)) == 0

    for _ in range(3):
        search()                                                    # warm: loads the library, allocates
    host, dev = [], []
    for _ in range(searches):
        r.set_profiling(True)
        t0 = time.perf_counter()
        search()
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(device_ms(r))
        r.set_profiling(False)
    d = float(np.median(dev))
    n, m = w * h, int(info.cells)
    # codes 1 B read, labels 4 B written by k_fr_tile, read by k_fr_flatten and k_fr_compact; per frontier cell the
    # (root, cell) pairs (12 B) written, the sort's passes (2 x 12 B read, 12 B written each), the head scan's keys
    # (2 x 8 B), the stats' rows, codes and potentials of 4 neighbours (4 + 4 x 9 B) and the labels (4 B)
    passes = 4 if n > 1 << 24 else 3
    nbytes = n * (1 + 4 + 4 + 4) + m * (12 + passes * 36 + 16 + 4 + 36 + 4) + 64 * int(info.components)
    print(json.dumps(dict(case=f"frontier_search on the costmap of {frames} frames at the defaults, plan at the last pose",
                          grid=[w, h], cells=n, frontier_cells=m, frontiers=int(info.components), kept=int(info.kept),
                          reachable=int(info.reachable), host_ms_median=round(float(np.median(host)), 3),
                          device_ms_median=round(d, 3), device_ms_min=round(min(dev), 3), device_ms_max=round(max(dev), 3),
                          counted_bytes=nbytes, bytes_bound_ms=round(nbytes / HBM * 1e3, 3),
                          share_of_hbm_bound=round(nbytes / HBM * 1e3 / d, 3))), flush=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        search()
        torch.cuda.synchronize()
    split = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = next((k for k in ("k_fr_tile", "k_fr_border", "k_fr_flatten", "k_fr_compact", "k_fr_stats",
                                     "k_gmm_hist", "k_gmm_offsets", "k_gmm_scatter", "k_gmm_head_count",
                                     "k_gmm_head_scatter") if k in e.name), None)
            if name:
                split[name] = split.get(name, 0.0) + e.device_time / 1e3
    print(json.dumps(dict(case="the split of one search by kernel (torch.profiler, ms)",
                          kernels={k: round(v, 4) for k, v in split.items()})), flush=True)

    info_py, got = r.frontier_search()
    lab = r.frontier_labels()
    t0 = time.perf_counter()
    want = fo.search(f.costs, p.potential, f.origin, f.resolution)
    s = time.perf_counter() - t0
    same = (np.array_equal(lab, want["labels"]) and [q.id for q in got] == want["frontiers"]["id"].tolist() and
            [q.cost for q in got] == want["frontiers"]["cost"].tolist())
    print(json.dumps(dict(case="tests/frontier_oracle.search of the same costs on the host", seconds=round(s, 2),
                          equal=bool(same))), flush=True)
    r.close()


if __name__ == "__main__":
    main()
