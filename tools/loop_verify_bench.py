"""Loop-verification cost (include/tloam_b200.h "Loop verification"), default configuration.
  (a) one loop add (loop_add_frame of the 116k-point synthetic HDL-64E scan process_raw_scan left on the device) with
      verification on against off, in alternating rounds, at keyframe voxels 0.5 and 1.0 m, with the keyframe size.  Host
      clock over `adds` adds ending in the result's synchronise, and the device time of the launches (the handle's
      profiling, class "submap").
  (b) one loop_verify of the revisit pair of the ray-cast world (tests/test_loop_closure.py: the return frame against its
      candidate, guess Rz(yaw)): host clock ending in the result, and the CUDA-event time of the k_lv_* launches.
  (c) the same verification through the numpy restatement (tests/loop_verify_oracle.py) on the host, for scale.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/loop_verify_bench.py [adds] [rounds] [verifies]
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
from tloam_b200 import synth  # noqa: E402
import loop_verify_oracle as lvo  # noqa: E402
from test_loop_closure import route_scans  # noqa: E402

FE = dict(cvr_submap=0.005, cvr_scan=0.01)        # the street scene has few curvature maxima (tests/test_front_end_chain.py)


def add_time(raw, voxel, adds):
    """(host ms, device ms, launches per add, keyframe size) of loop_add_frame; voxel None: verification off"""
    r = tloam_b200.LocalRegistration()
    r.loop_enable()
    if voxel is not None:
        r.loop_verify_enable(voxel=voxel, initial_capacity_points=(adds + 2) * len(raw))
    r.process_raw_scan(raw, feature=FE)
    r.loop_add_frame()                                             # warm-up
    r.loop_result()
    r.set_profiling(True)
    t0 = time.perf_counter()
    for _ in range(adds):
        r.loop_add_frame()
    r.loop_result()
    host = 1e3 * (time.perf_counter() - t0) / adds
    prof = r.get_profile()["submap"]
    r.set_profiling(False)
    size = len(r.loop_keyframe(0)) if voxel is not None else 0
    r.close()
    return host, prof[1] / adds, prof[0] / adds, size


def main():
    adds = int(sys.argv[1]) if len(sys.argv) > 1 else 50
    rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    verifies = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    raw = synth.raw_scan()
    a = {}
    for voxel in (None, 0.5, 1.0):
        add_time(raw, voxel, 3)                                    # warm-up of every shape
    for _ in range(rounds):
        for voxel in (None, 0.5, 1.0):
            a.setdefault(str(voxel), []).append(add_time(raw, voxel, adds))
    for k, v in a.items():
        v = np.array(v)
        print(f"(a) verification {'off' if k == 'None' else 'on, voxel ' + k}: add {np.round(v[:, 0], 3)} ms host clock, "
              f"{np.round(v[:, 1], 3)} ms device, {v[0, 2]:.0f} launches, keyframe {int(v[0, 3])} points ({len(raw)} rows)")
    _, scans = route_scans()
    r = tloam_b200.LocalRegistration()
    r.loop_enable()
    r.loop_verify_enable()
    for p in scans:
        r.loop_add(p)
    lr = r.loop_result()
    v = r.loop_verify(lr.query, lr.candidate, yaw=lr.yaw)          # warm-up
    host = []
    for _ in range(verifies):
        t0 = time.perf_counter()
        v = r.loop_verify(lr.query, lr.candidate, yaw=lr.yaw)
        host.append(1e3 * (time.perf_counter() - t0))
    r.set_profiling(True)
    for _ in range(verifies):
        r.loop_verify(lr.query, lr.candidate, yaw=lr.yaw)
    prof = r.get_profile()["submap"]
    r.set_profiling(False)
    kq, km = r.loop_keyframe(lr.query), r.loop_keyframe(lr.candidate)
    r.close()
    dev = prof[1] / verifies
    print(f"(b) loop_verify {lr.query} -> {lr.candidate} ({len(kq)} x {len(km)} points, {v.iterations} iterations, termination "
          f"{v.termination}, accepted {v.accepted}): {np.median(host):.3f} ms host clock median (min {np.min(host):.3f}), "
          f"{dev:.3f} ms device (k_lv_* launches, CUDA events)")
    t0 = time.perf_counter()
    o = lvo.run(kq, km, tloam_b200.registration.rz(lr.yaw), lvo.config())
    oms = 1e3 * (time.perf_counter() - t0)
    print(f"(c) numpy restatement on the host: {oms:.0f} ms ({o['iterations']} iterations)")
    print(json.dumps(dict(card=card, add={k: np.array(v).tolist() for k, v in a.items()},
                          verify=dict(query=lr.query, candidate=lr.candidate, n_query=len(kq), n_candidate=len(km),
                                      iterations=v.iterations, host_ms_median=float(np.median(host)), host_ms_min=float(np.min(host)),
                                      device_ms=dev), oracle_ms=oms)))


if __name__ == "__main__":
    main()
