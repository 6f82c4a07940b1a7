"""Robust pose-graph cost (include/tloam_b200.h "Robust pose graph"), default configurations, on the seq-00-shaped graph of
tests/test_pose_graph.py (4 541 nodes, 183 loop edges) with 10 % family-(b) outliers of tests/test_pose_graph_robust.py
(18 true loops' measurements moved by 2-10 m / 5-30 degrees).
  (a) one tloam_b200_pose_graph_optimize_robust: host clock per call (it returns once the result is home) and the device
      time of its launches from the handle's CUDA events (class "submap"); its stages, Gauss-Newton steps and launches.
  (b) the plain tloam_b200_pose_graph_optimize on the same graph, for scale.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/pose_graph_robust_bench.py [calls]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tloam_b200  # noqa: E402,F401
from test_pose_graph import device_graph, loop_pair_error, seq_graph  # noqa: E402
from test_pose_graph_robust import outliers  # noqa: E402


def timed(r, fn, calls):
    fn()                                                            # warm-up (and the scratch allocation)
    host = []
    for _ in range(calls):
        t0 = time.perf_counter()
        res = fn()
        host.append(1e3 * (time.perf_counter() - t0))
    n0 = r.launch_count()
    fn()
    launches = r.launch_count() - n0
    r.set_profiling(True)
    for _ in range(calls):
        fn()
    dev = r.get_profile()["submap"][1] / calls
    r.set_profiling(False)
    return res, host, dev, launches


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    G, O, loops = seq_graph("00")
    bad = outliers(G, loops, 0.1, "b")
    r = device_graph(O, loops + bad)
    res, host, dev, launches = timed(r, r.pose_graph_optimize_robust, calls)
    stages = 1 + res.outer_iterations
    err = loop_pair_error(r.pose_graph_poses(), G, loops)
    print(f"(a) optimize_robust, {len(O)} nodes, {len(loops)} loops + {len(bad)} outliers: {stages} stages, "
          f"{res.pg.iterations} Gauss-Newton steps, {launches} launches, termination {res.gnc_termination}, "
          f"{res.rejected} rejected, loop-pair error {err:.4f} m: {np.median(host):.1f} ms host clock median "
          f"(min {np.min(host):.1f}), {dev:.1f} ms device (CUDA events)")
    pres, phost, pdev, plaunches = timed(r, r.pose_graph_optimize, calls)
    perr = loop_pair_error(r.pose_graph_poses(), G, loops)
    print(f"(b) plain optimize on the same graph: {pres.iterations} steps, {plaunches} launches, loop-pair error "
          f"{perr:.4f} m: {np.median(phost):.1f} ms host clock median, {pdev:.1f} ms device")
    r.close()
    print(json.dumps(dict(card=card, nodes=len(O), loops=len(loops), outliers=len(bad), stages=stages,
                          steps=res.pg.iterations, launches=launches, outer_iterations=res.outer_iterations,
                          rejected=res.rejected, loop_pair_error=err, host_ms_median=float(np.median(host)),
                          host_ms_min=float(np.min(host)), device_ms=dev, plain_steps=pres.iterations,
                          plain_host_ms_median=float(np.median(phost)), plain_device_ms=pdev, plain_loop_pair_error=perr)))


if __name__ == "__main__":
    main()
