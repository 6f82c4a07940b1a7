"""Global registration (include/tloam_b200.h "Global registration"): the cost of one global_register of two HDL-64E scans
at the defaults (0.5 m keypoints, 65 536 hypotheses), against the numpy restatement on the same keypoints.
  - scans: tloam_b200.synth.raw_scan, and the same street seen from a sensor moved by 135 deg and 7.2 m with 2 cm noise
    (the GPU test's "scan" case).
  - call: after warm-up, the C call's host clock (it synchronises) and the device time of its kernels from the library's
    CUDA events, median over the calls.
  - stages: torch.profiler with CUDA activities over 3 more calls, in a run of its own: device time per kernel name per call
    (the down-sample, the index, and every k_gr_* kernel).
  - FP64 operations: k_gr_match does 33 x (sub, mul, add) per (source feature, target feature) pair, both ways; k_gr_hyp
    does 26 per (valid hypothesis, pair) (R p + t: 9 mul + 9 add; the squared distance: 3 sub, 3 mul, 2 add), not counting
    the construction of each hypothesis.  Rates are those counts over the kernel's device time.
  - numpy: tests/global_registration_oracle.run on the device's keypoints (host time), and whether T is the device's.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/global_registration_bench.py [calls]
"""
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import tloam_b200  # noqa: E402
from tloam_b200 import synth  # noqa: E402
import global_registration_oracle as gro  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def scans():
    P = synth.raw_scan()
    P = P[np.isfinite(P).all(1)]
    a = math.radians(135)
    T = np.eye(4)
    T[:2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
    T[:3, 3] = (6.0, -4.0, 0.2)
    Ti = np.linalg.inv(T)
    src = P @ Ti[:3, :3].T + Ti[:3, 3] + np.random.default_rng(8).normal(0, 0.02, P.shape)
    return src, P


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    print(card())
    src, tgt = scans()
    r = tloam_b200.LocalRegistration()
    r.global_registration_enable()
    for _ in range(2):
        res = r.global_register(src, tgt)
    host, dev = [], []
    for _ in range(calls):
        r.set_profiling(True)
        t0 = time.perf_counter()
        res = r.global_register(src, tgt)
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(sum(v for _, v in r.get_profile().values()))
        r.set_profiling(False)
    S, T = r.global_registration_side(0), r.global_registration_side(1)

    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            r.global_register(src, tgt)
    stages = {}
    for e in prof.key_averages():
        if e.device_type == torch.autograd.DeviceType.CUDA and e.count:
            stages[e.key] = stages.get(e.key, 0.0) + e.device_time_total / 1e3 / 3
    named = {}
    for k, v in stages.items():
        short = next((w for w in k.replace("(", " ").replace("<", " ").split() if w.split("::")[-1].startswith("k_")), k)
        short = short.split("::")[-1]
        named[short] = named.get(short, 0.0) + v
    match_ops = 2 * 99 * int(S["has_feature"].sum()) * int(T["has_feature"].sum())
    hyp_ops = 26 * res.n_valid_hypotheses * res.n_correspondences

    t0 = time.perf_counter()
    want = gro.run(S["xyz"], T["xyz"], gro.config())
    numpy_s = time.perf_counter() - t0
    out = dict(
        keypoints=[res.n_source_points, res.n_target_points], features=[res.n_source_features, res.n_target_features],
        correspondences=res.n_correspondences, valid_hypotheses=res.n_valid_hypotheses, inliers=res.inliers,
        fitness=res.fitness, accepted=res.accepted, calls=calls,
        host_ms_median=statistics.median(host), device_ms_median=statistics.median(dev),
        stage_ms={k: round(v, 4) for k, v in sorted(named.items(), key=lambda kv: -kv[1])},
        match_fp64_ops=match_ops, hyp_fp64_ops=hyp_ops,
        match_gflops=match_ops / (named.get("k_gr_match", float("nan")) * 1e6),
        hyp_gflops=hyp_ops / (named.get("k_gr_hyp", float("nan")) * 1e6),
        numpy_s=numpy_s, numpy_T_equal=bool(np.array_equal(want["T"], res.T)))
    print(json.dumps(out))
    r.close()


if __name__ == "__main__":
    main()
