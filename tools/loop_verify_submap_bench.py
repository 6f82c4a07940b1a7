"""Cost of loop verification against a submap (include/tloam_b200.h "Loop verification against a submap"), default
configuration, on two workloads:
  route: the revisit pair of the ray-cast 16-beam world (tests/test_loop_closure.py), the window placed by the route's poses;
  hdl:   twelve views of the 116k-point synthetic HDL-64E scan 1 m apart (keyframes of about 5 000 points, a target of
         eleven of them), the last against the sixth.
Per workload, in alternating rounds against tloam_b200_loop_verify on the same pair: the host clock to the result and the
device time of the launches (the handle's profiling, CUDA events).  Then, in a run of its own, the per-kernel times of
k_lvs_normals and of the passes' kernels from torch.profiler's CUDA activities.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/loop_verify_submap_bench.py [rounds] [verifies]
"""
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tloam_b200  # noqa: E402
from tloam_b200 import synth  # noqa: E402
from test_loop_closure import route_scans  # noqa: E402


def pose(x, y, yaw):
    T = np.eye(4)
    T[:2, :2] = [[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]]
    T[:2, 3] = x, y
    return T


def workloads():
    poses, scans = route_scans()
    yield "route", scans, [pose(*p) for p in poses], len(scans) - 1, 10, pose(0, 0, math.radians(-96.0))
    raw = synth.raw_scan()
    raw = raw[np.isfinite(raw).all(axis=1)]
    P = [pose(1.0 * k, 0.0, 0.0) for k in range(11)] + [pose(5.3, 0.2, 0.02)]
    yield "hdl", [(raw - T[:3, 3]) @ T[:3, :3] for T in P], P, 11, 5, np.eye(4)


def timed(r, call, verifies):
    """(host ms median, host ms min, device ms per call, the result)"""
    v = call()                                                     # warm-up
    host = []
    for _ in range(verifies):
        t0 = time.perf_counter()
        v = call()
        host.append(1e3 * (time.perf_counter() - t0))
    r.set_profiling(True)
    for _ in range(verifies):
        call()
    prof = r.get_profile()["submap"]
    r.set_profiling(False)
    return float(np.median(host)), float(np.min(host)), prof[1] / verifies, v


def kernel_times(call, verifies):
    """{kernel: (launches per call, device us per call)} of the k_lvs_* kernels"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(verifies):
            call()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if "k_lvs_" in e.key:
            name = e.key[e.key.index("k_lvs_"):].split("(")[0]
            out[name] = (e.count / verifies, getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / verifies)
    return out


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    verifies = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    report = dict(card=card)
    for name, scans, P, q, c, guess in workloads():
        r = tloam_b200.LocalRegistration()
        r.loop_enable()
        r.loop_verify_enable()
        r.loop_verify_submap_enable()
        r.pose_graph_enable()
        for p, T in zip(scans, P):
            r.loop_add(p)
            r.pose_graph_add_node(T)
        sub = lambda: r.loop_verify_submap(q, c, guess)            # noqa: E731
        old = lambda: r.loop_verify(q, c, guess)                   # noqa: E731
        rows = dict(submap=[], scan=[])
        for _ in range(rounds):
            rows["submap"].append(timed(r, sub, verifies))
            rows["scan"].append(timed(r, old, verifies))
        vs, vo = rows["submap"][0][3], rows["scan"][0][3]
        for k, v in (("submap", vs), ("scan", vo)):
            t = np.array([x[:3] for x in rows[k]])
            print(f"{name} {k}: {v.n_query_points} x {v.n_candidate_points} points, {v.iterations} iterations, termination "
                  f"{v.termination}, fitness {v.fitness:.4f}: host clock median {np.round(t[:, 0], 3)} ms (min {np.round(t[:, 1], 3)}), "
                  f"device {np.round(t[:, 2], 3)} ms")
        kt = kernel_times(sub, verifies)
        for k in sorted(kt):
            print(f"{name} {k}: {kt[k][0]:.0f} launches, {kt[k][1]:.1f} us per verification")
        n = vs.n_candidate_points
        if "k_lvs_normals" in kt:
            pairs = 2.0 * n * n
            print(f"{name} k_lvs_normals: {pairs:.3g} pair tests in two sweeps, {pairs / (kt['k_lvs_normals'][1] * 1e-6):.3g} per second")
        report[name] = dict(rows=n, n_query=vs.n_query_points, iterations=vs.iterations,
                            submap=[x[:3] for x in rows["submap"]], scan=[x[:3] for x in rows["scan"]], kernels=kt)
        r.close()
    print(json.dumps(report))


if __name__ == "__main__":
    main()
