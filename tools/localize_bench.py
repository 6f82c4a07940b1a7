"""Localization in a prior map (include/tloam_b200.h "Localization in a prior map"): the cost of a load and of a frame.
  - set_map: the seq-00-sized map tools/global_map_merge_bench.py builds (4 541 frames of 2 000 points at the seq 00
    odometry poses, about 9.08 M rows), merged at 1.0 and 0.5 m and loaded with tloam_b200_localize_set_map_merged; and the
    same map unmerged (every row, a denser map: up to a few hundred rows within 1 m).  Host clock of the call (it ends in a
    synchronise), the map's rows and cells, the share of rows with a valid normal, the largest neighbourhood, and the
    device memory the load took (cudaMemGetInfo before and after).
  - per frame: HDL-64E scans (tloam_b200.synth.raw_scan, about 120 000 rows) moved along a straight line, each localized
    with tloam_b200_localize_frame from its true pose after process_raw_scan, against the merged map of the same scans;
    host clock of the call, with its device time from the handle's CUDA events.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/localize_bench.py [frames]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tloam_b200  # noqa: E402
from tloam_b200 import synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def free_bytes():
    import torch
    return torch.cuda.mem_get_info()[0]


def load_case(r, what, n_rows, set_map):
    f0 = free_bytes()
    t0 = time.perf_counter()
    set_map()
    ms = (time.perf_counter() - t0) * 1e3
    used = f0 - free_bytes()
    _, valid, cnt = r.localize_map_normals()
    _, keys, _ = r.localize_cells(n_rows)
    print(json.dumps(dict(case=what, rows=n_rows, cells=int(len(keys)), set_map_ms=round(ms, 2), valid=round(float(valid.mean()), 4),
                          max_neighbours=int(cnt.max()), mean_neighbours=round(float(cnt.mean()), 1),
                          device_bytes_per_row=round(used / n_rows, 1))), flush=True)


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    print(card(), flush=True)
    from global_map_merge_bench import build
    from test_pose_graph import seq_graph
    O = seq_graph("00")[0]
    r = build(O, 2000, False)
    r.localize_enable()
    for voxel in (1.0, 0.5):
        xyz, _ = r.global_map_merged(voxel)
        for k in range(2):                                          # the first load allocates; the second is the steady cost
            load_case(r, f"seq-00 map merged at {voxel} m" + (" (first load)" if k == 0 else ""), len(xyz), r.localize_set_map_merged)
    raw = r.global_map()
    load_case(r, "seq-00 map unmerged", len(raw), lambda: r.localize_set_map(raw))
    r.close()

    from test_process_cloud import FE
    scan0 = synth.raw_scan()
    steps = [synth.se3_exp(np.array([0.5 * k, 0.0, 0.0, 0.0, 0.0, 0.002 * k])) for k in range(frames)]
    scans = [(scan0 - T[:3, 3]) @ T[:3, :3] for T in steps]
    m = tloam_b200.LocalRegistration()
    m.enable_global_map(voxel=0.5)
    for T, s in zip(steps, scans):
        m.global_map_append(s, T)
    prior, _ = m.global_map_merged(0.5)
    m.close()
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.localize_enable()
    r.localize_set_map(prior)
    host, dev, acc = [], [], 0
    for k, s in enumerate(scans):
        r.process_raw_scan(s, feature=FE)
        r.set_profiling(True)
        t0 = time.perf_counter()
        x = r.localize_frame(steps[k])                             # no odometry here: the true pose as the guess
        host.append((time.perf_counter() - t0) * 1e3)
        prof = r.get_profile()
        dev.append(sum(ms for _, ms in prof.values()))
        r.set_profiling(False)
        acc += int(x.accepted)
    print(json.dumps(dict(case=f"localize_frame, HDL-64E scans ({len(scans[0])} rows) against {len(prior)} map rows",
                          query_rows=int(x.n_query_points), host_ms_median=round(float(np.median(host[1:])), 3),
                          device_ms_median=round(float(np.median(dev[1:])), 3), accepted=acc, frames=len(scans),
                          iterations_last=x.iterations)), flush=True)
    r.close()


if __name__ == "__main__":
    main()
