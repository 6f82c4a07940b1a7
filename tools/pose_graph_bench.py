"""Pose-graph cost (include/tloam_b200.h "Pose graph"), default configuration, on the seq-00-shaped graph of
tests/test_pose_graph.py (4 541 nodes from T-LOAM's recorded KITTI 00 motion with seeded drift, 183 loop edges).
  (a) one tloam_b200_pose_graph_optimize: host clock per call (it returns once the result is home), and the device time of
      its launches from the handle's CUDA events (class "submap").
  (b) the device time per kernel (k_pg_*), from torch.profiler's CUDA activity in a run of its own.
  (c) the same optimisation through the numpy restatement (tests/pose_graph_oracle.py) on the host, for scale.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/pose_graph_bench.py [calls] [seq]
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
import tloam_b200  # noqa: E402
import pose_graph_oracle as pgo  # noqa: E402
from test_pose_graph import device_graph, seq_graph  # noqa: E402


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    seq = sys.argv[2] if len(sys.argv) > 2 else "00"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    G, O, loops = seq_graph(seq)
    r = device_graph(O, loops)
    res = r.pose_graph_optimize()                                  # warm-up (and the scratch allocation)
    host = []
    for _ in range(calls):
        t0 = time.perf_counter()
        res = r.pose_graph_optimize()
        host.append(1e3 * (time.perf_counter() - t0))
    r.set_profiling(True)
    for _ in range(calls):
        r.pose_graph_optimize()
    prof = r.get_profile()["submap"]
    r.set_profiling(False)
    dev = prof[1] / calls
    print(f"(a) optimize, {len(O)} nodes, {len(loops)} loops, {res.iterations} iterations, termination {res.termination}: "
          f"{np.median(host):.2f} ms host clock median (min {np.min(host):.2f}), {dev:.2f} ms device (CUDA events)")
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for _ in range(3):
            r.pose_graph_optimize()
        torch.cuda.synchronize()
    kern = {}
    for ev in p.events():
        if "k_pg_" in ev.name:
            name = ev.name[ev.name.index("k_pg_"):].split("(")[0].split("E")[0].rstrip("0123456789")
            n, t = kern.get(name, (0, 0.0))
            kern[name] = (n + 1, t + ev.device_time_total / 1e3)
    for name, (n, t) in sorted(kern.items(), key=lambda x: -x[1][1]):
        print(f"(b) {name}: {t / 3:.3f} ms per optimise over {n // 3} launches")
    r.close()
    t0 = time.perf_counter()
    o = pgo.optimize(O, loops, pgo.config())
    oms = 1e3 * (time.perf_counter() - t0)
    print(f"(c) numpy restatement on the host: {oms:.0f} ms ({o['iterations']} iterations)")
    print(json.dumps(dict(card=card, seq=seq, nodes=len(O), loops=len(loops), iterations=res.iterations,
                          host_ms_median=float(np.median(host)), host_ms_min=float(np.min(host)), device_ms=dev,
                          kernels_ms={k: t / 3 for k, (n, t) in kern.items()}, oracle_ms=oms)))


if __name__ == "__main__":
    main()
