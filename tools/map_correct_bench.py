"""Loop-corrected global map cost (include/tloam_b200.h "Loop-corrected global map") on a seq-00-sized map: the graph of
tests/test_pose_graph.py's seq_graph("00") (4 541 nodes, 183 loop edges), a frame of about 2 000 voxels appended at every
node's odometry pose (about 9 M points).
  (a) one tloam_b200_global_map_correct that moves every frame: the device time of its launches from the handle's CUDA
      events (class "submap"), and the host clock of the call (it synchronises).  Calls alternate between the optimised
      node table and an all -1 table, so that every call moves every frame.
  (b) the per-append cost of tracking: rounds of appends on a tracked and an untracked map, alternating, host clock to a
      synchronise at the end of each round.
  (c) the same correction through the numpy restatement (tests/map_correct_oracle.py) on the host, for scale.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/map_correct_bench.py [calls] [points_per_frame]
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
import map_correct_oracle as mco  # noqa: E402
from test_pose_graph import loop_result, seq_graph  # noqa: E402


def append_rounds(frames, rounds=5):
    """(b): per-append ms of the tracked and the untracked map, alternating rounds of len(frames) appends"""
    maps = {}
    for track in (True, False):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map(initial_capacity=(rounds + 1) * sum(len(p) for p, _ in frames))
        if track:
            r.global_map_correction_enable()
        maps[track] = r
    times = {True: [], False: []}
    for k in range(rounds + 1):                                     # round 0 warms up
        for track in ((True, False) if k % 2 else (False, True)):
            r = maps[track]
            r.global_map_size()
            t0 = time.perf_counter()
            for p, T in frames:
                r.global_map_append(p, T)
            r.global_map_size()
            if k:
                times[track].append(1e3 * (time.perf_counter() - t0) / len(frames))
    for r in maps.values():
        r.close()
    return times


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    pts = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    G, O, loops = seq_graph("00")
    rng = np.random.default_rng(7)
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=len(O) * pts)
    r.global_map_correction_enable()
    r.pose_graph_enable()
    for T in O:
        r.pose_graph_add_node(T)
        r.global_map_append(rng.uniform(-60.0, 60.0, (pts, 3)), T)
    for i, j, Z in loops:
        r.pose_graph_add_loop(loop_result(i, j, Z))
    res = r.pose_graph_optimize()
    n_pts, n_frames = r.global_map_size()
    nodes = np.arange(n_frames)
    none = np.full(n_frames, -1)
    before = r.global_map()
    off = r.global_map_frames()
    Of, Pf = r.global_map_frame_poses()
    T_opt = r.pose_graph_poses()
    r.global_map_correct(nodes)                                    # warm-up (and the scratch allocation)
    r.global_map_correct(none)
    host = []
    for k in range(calls):
        t0 = time.perf_counter()
        r.global_map_correct(nodes if k % 2 == 0 else none)
        host.append(1e3 * (time.perf_counter() - t0))
    r.set_profiling(True)
    for k in range(calls):
        r.global_map_correct(nodes if k % 2 == 0 else none)
    dev = r.get_profile()["submap"][1] / calls
    r.set_profiling(False)
    nbytes = n_pts * 48 + n_frames * (3 * 128 + 8 + 8 + 4)          # points read + written, the tables, offsets, node, moved
    print(f"(a) correct, {n_frames} frames, {n_pts} points, termination {res.termination}: {dev:.3f} ms device (CUDA "
          f"events), {np.median(host):.2f} ms host clock median (min {np.min(host):.2f}); {nbytes / 1e9:.2f} GB moved, "
          f"{nbytes / dev / 1e6:.0f} GB/s")
    r.close()
    frames = [(rng.uniform(-60.0, 60.0, (pts, 3)), O[k]) for k in range(200)]
    t = append_rounds(frames)
    on, offm = float(np.median(t[True])), float(np.median(t[False]))
    print(f"(b) append of {pts} rows: {on:.4f} ms tracked, {offm:.4f} ms untracked (medians of {len(t[True])} alternating "
          f"rounds of {len(frames)}); tracking {1e3 * (on - offm):.1f} us per append")
    t0 = time.perf_counter()
    mco.correct(before, off, Of, Pf, nodes, T_opt, np.array(O))
    oms = 1e3 * (time.perf_counter() - t0)
    print(f"(c) numpy restatement on the host: {oms:.0f} ms")
    print(json.dumps(dict(card=card, frames=int(n_frames), points=int(n_pts), device_ms=dev,
                          host_ms_median=float(np.median(host)), host_ms_min=float(np.min(host)), bytes=int(nbytes),
                          append_ms_tracked=on, append_ms_untracked=offm, append_rounds_tracked=t[True],
                          append_rounds_untracked=t[False], oracle_ms=oms)))


if __name__ == "__main__":
    main()
