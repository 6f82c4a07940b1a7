"""Dynamic-point removal cost (include/tloam_b200.h "Dynamic-point removal") at a ~1 M-point map and at a seq-00-sized map
(about 9 M points, as tools/map_correct_bench.py builds it: frames of `points_per_frame` distinct points, one per 1 m voxel,
at the odometry poses of tests/test_pose_graph.py's seq_graph("00")).
  (a) the device time of one append with removal on against off: two maps built alike, one with removal on; rounds of
      appends of an HDL-64E-sized scan (120 000 rows) alternate between them; the device time of the class "submap" launches
      (CUDA events) per append, and their difference.  The difference is the vote's four kernels; their algorithmic bytes are
      24 B of xyz + 8 B of counters read + 8 B written per map point, against 3.35 TB/s.
  (b) one tloam_b200_global_map_static_download: device time of its two kernels and the host clock of the call (which
      includes copying the static map home).
Prints the card and its power limit read in the same call, then one JSON line per map size.

    python tools/map_dynamic_bench.py [rounds] [points_per_frame]
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
from test_pose_graph import seq_graph  # noqa: E402

HBM = 3.35e12


def hdl64_scan(rng, n_az=1875):
    """64 beams x n_az azimuths (120 000 rows) in a street-like world: the ground 1.73 m below and a wall 25 m around, so
    that an append adds a few thousand voxels and the map keeps its size over the rounds"""
    el, az = np.meshgrid(np.radians(np.linspace(-24.9, 2.0, 64)), (np.arange(n_az) + 0.5) * (2 * np.pi / n_az), indexing="ij")
    d = np.stack([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)], axis=-1).reshape(-1, 3)
    with np.errstate(divide="ignore"):
        t = np.where(d[:, 2] < 0, -1.73 / d[:, 2], np.inf)
    t = np.minimum(t, 25.0 / np.hypot(d[:, 0], d[:, 1]))
    return d * t[:, None] + rng.normal(0, 0.02, d.shape)


def build(O, pts, dynamic, seed=7):
    rng = np.random.default_rng(seed)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=len(O) * pts + 200 * pts)
    if dynamic:
        r.global_map_dynamic_enable()
    for T in O:
        r.global_map_append(rng.uniform(-60.0, 60.0, (pts, 3)), T)
    r.global_map_size()
    return r


def measure(O, pts, rounds, card):
    maps = {d: build(O, pts, d) for d in (True, False)}
    n_pts = maps[True].global_map_size()[0]
    rng = np.random.default_rng(3)
    scans = [(hdl64_scan(rng), O[len(O) // 2 + k]) for k in range(8)]
    dev = {True: [], False: []}
    for k in range(rounds + 1):                                    # round 0 warms up
        for d in ((True, False) if k % 2 else (False, True)):
            r = maps[d]
            r.global_map_size()
            r.set_profiling(True)
            for p, T in scans:
                r.global_map_append(p, T)
            r.global_map_size()
            ms = r.get_profile()["submap"][1] / len(scans)
            r.set_profiling(False)
            if k:
                dev[d].append(ms)
    on, off = float(np.median(dev[True])), float(np.median(dev[False]))
    vote_ms = on - off
    nbytes = n_pts * 40
    bw = nbytes / (max(vote_ms, 1e-9) * 1e-3)
    r = maps[True]
    r.global_map_static()                                          # warm-up (the scratch allocation)
    n_now = r.global_map_size()[0]
    r.set_profiling(True)
    t0 = time.perf_counter()
    xyz, _ = r.global_map_static()
    host = 1e3 * (time.perf_counter() - t0)
    static_dev = r.get_profile()["submap"][1]
    r.set_profiling(False)
    print(f"map of {n_pts} points: append device {on:.3f} ms on, {off:.3f} ms off (medians of {rounds} alternating rounds "
          f"of {len(scans)}); votes {vote_ms:.3f} ms = {bw / 1e9:.0f} GB/s of {nbytes / 1e6:.0f} MB ({100 * bw / HBM:.0f} % "
          f"of 3.35 TB/s); static download of {n_now} points {static_dev:.3f} ms device, {host:.1f} ms host clock, "
          f"{len(xyz)} points kept")
    for m in maps.values():
        m.close()
    print(json.dumps(dict(card=card, points=int(n_pts), append_ms_on=on, append_ms_off=off, rounds_on=dev[True],
                          rounds_off=dev[False], vote_ms=vote_ms, vote_bytes=int(nbytes), static_device_ms=static_dev,
                          static_host_ms=host, static_map_points=int(n_now), static_points=int(len(xyz)))))


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 6
    pts = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    G, O, loops = seq_graph("00")
    O = np.array(O)
    measure(O[:1_000_000 // pts], pts, rounds, card)
    measure(O, pts, rounds, card)


if __name__ == "__main__":
    main()
