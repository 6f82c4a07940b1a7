"""Path planning (include/tloam_b200.h "Path planning"): the cost of a plan build and of paths on a seq-00-shaped costmap,
against scipy's Dijkstra on the same costs on the host.
  - costmap: the distance build at the defaults of the occupancy grid of a seq-00-shaped drive, 4 541 frames at the poses
    of tests/test_pose_graph.seq_graph("00"), each appending the HDL-64E scan (tloam_b200.synth.raw_scan), as
    tools/distance_bench.py builds it.
  - build: plan_build at the defaults to the first pose, after warm-up: the C call's host clock (it synchronises) and its
    kernels' device time from the CUDA events, the rounds, the tiles relaxed and the cells of those tiles per second of
    device time.
  - paths: plan_paths from 1 and from 1 024 poses sampled evenly along the trajectory (host clock, device time).
  - scipy: scipy.sparse.csgraph.dijkstra on the same costs (tests/plan_oracle.scipy_potential), on the 2 048 x 2 048 crop
    of the occupancy grid around the goal (its own distance and plan build on the device beside it) and on the full grid
    when the host has the memory for it, with the host time and whether the potentials are equal.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/plan_bench.py [frames] [builds]
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
import plan_oracle as po  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def device_ms(r):
    return sum(v for _, v in r.get_profile().values())


def timed(r, call):
    r.set_profiling(True)
    t0 = time.perf_counter()
    out = call()
    host = (time.perf_counter() - t0) * 1e3
    dev = device_ms(r)
    r.set_profiling(False)
    return host, dev, out


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def scipy_case(name, t, goal, P):
    t0 = time.perf_counter()
    S = po.scipy_potential(t, goal)
    s = time.perf_counter() - t0
    print(json.dumps(dict(case=name, cells=int(t.size), seconds=round(s, 2), potential_equal=bool(np.array_equal(S, P)))),
          flush=True)


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 4541
    builds = int(sys.argv[2]) if len(sys.argv) > 2 else 10
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
    f = r.distance_build()
    h, w = f.costs.shape
    goal_xy = G[0][:2, 3]

    cfg = _lib.PlanConfig()
    r._L.tloam_b200_plan_default_config(C.byref(cfg))
    info = _lib.PlanInfo()

    def build():
        assert r._L.tloam_b200_plan_build(r._h, C.byref(cfg), float(goal_xy[0]), float(goal_xy[1]), C.byref(info)) == 0

    for _ in range(2):
        build()                                                     # warm: loads the library, allocates
    host, dev = [], []
    for _ in range(builds):
        a, b, _ = timed(r, build)
        host.append(a)
        dev.append(b)
    d = float(np.median(dev))
    print(json.dumps(dict(case=f"plan_build on the costmap of {frames} frames at the defaults, goal at the first pose",
                          grid=[w, h], cells=w * h, reachable=int(info.reachable), rounds=int(info.rounds),
                          tiles=int(info.tiles), host_ms_median=round(float(np.median(host)), 3),
                          device_ms_median=round(d, 3), device_ms_min=round(min(dev), 3), device_ms_max=round(max(dev), 3),
                          tile_cells_relaxed_per_s=float(f"{info.tiles * 1024 / (d * 1e-3):.3g}"))), flush=True)
    p = r.plan_build(goal_xy)
    t = po.cell_costs(f.costs)
    print(json.dumps(dict(case="the potential's Bellman certificate (tests/plan_oracle.bellman_holds)",
                          holds=po.bellman_holds(p.potential, t, p.goal))), flush=True)

    idx = np.linspace(0, len(G) - 1, 1024).astype(int)
    starts = np.array([G[k][:2, 3] for k in idx])
    for n in (1, 1024):
        s = starts[-1:] if n == 1 else starts
        r.plan_paths(s)
        a, b, paths = timed(r, lambda: r.plan_paths(s))
        cells = [len(q.cells) for q in paths]
        print(json.dumps(dict(case=f"plan_paths from {n} trajectory pose(s)", host_ms=round(a, 3), device_ms=round(b, 3),
                              reached=sum(q.status == 0 for q in paths), cells_total=int(sum(cells)),
                              cells_max=int(max(cells)))), flush=True)

    # the 2 048 x 2 048 crop of the occupancy grid around the goal, planned on the device and by scipy
    gi, gj = p.goal
    i0, j0 = max(0, min(gi - 1024, w - 2048)), max(0, min(gj - 1024, h - 2048))
    crop = np.ascontiguousarray(occ.cells[j0:j0 + 2048, i0:i0 + 2048])
    origin = (f.origin[0] + i0 * f.resolution, f.origin[1] + j0 * f.resolution)
    fc = r.distance_build(crop, origin, f.resolution)
    r.plan_build(goal_xy)
    a, b, pc = timed(r, lambda: r.plan_build(goal_xy))
    print(json.dumps(dict(case="plan_build of the 2048 x 2048 crop around the goal", shape=list(crop.shape),
                          host_ms=round(a, 3), device_ms=round(b, 3), rounds=pc.rounds, tiles=pc.tiles)), flush=True)
    scipy_case("scipy.sparse.csgraph.dijkstra of the 2048 x 2048 crop on the host", po.cell_costs(fc.costs), pc.goal,
               pc.potential)
    need = t.size * 8 * 60                                          # the move graph's arrays, with room for scipy's copies
    if mem_available() > need:
        scipy_case("scipy.sparse.csgraph.dijkstra of the full grid on the host", t, p.goal, p.potential)
    else:
        print(json.dumps(dict(case="scipy.sparse.csgraph.dijkstra of the full grid on the host", seconds="not measured",
                              reason=f"needs about {need / 1e9:.0f} GB of host memory, {mem_available() / 1e9:.0f} GB "
                                     "available")), flush=True)
    r.close()


if __name__ == "__main__":
    main()
