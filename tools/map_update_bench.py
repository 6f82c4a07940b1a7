"""Updating a prior map (include/tloam_b200.h "Updating a prior map"): the cost of an add, of its two vote calls, of a build,
and of the localize loop with updating on and off.
  - The prior map is the seq-00-sized map tools/global_map_merge_bench.py builds, merged at 0.5 m (about 8.9 M rows), with
    the merged map of HDL-64E scans (tloam_b200.synth.raw_scan moved along a straight line) placed 2 km away, so that the
    scans localize from their true poses.
  - per add: process_raw_scan, localize_frame from the true pose, then map_update_add: host clock of the add to a
    synchronise after it, and its device time from the handle's CUDA events.  The kernels of the two tloam_gmd_vote calls
    (k_gmd_clear / _bin / _window / _vote over the prior rows, then over the additions) from torch.profiler in a run of
    their own.
  - per build: map_update_build at about 0, 1e5 and 1e6 addition rows (novel_radius 0.01 m, min_frames 1, so that nearly
    every query row is new), host clock of the C call (it synchronises), and with the download of the cloud that
    LocalRegistration.map_update_build adds.
  - the localize loop (process_raw_scan, localize_frame(NULL)) with and without map_update_add, alternated in rounds.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/map_update_bench.py [frames]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import tloam_b200  # noqa: E402
from tloam_b200 import _lib, synth  # noqa: E402

FAR = np.array([2000.0, 0.0, 0.0])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def sync_ms(r, f):
    t0 = time.perf_counter()
    out = f()
    r.map_update_size()                                             # a read-back: ends in a synchronise
    return out, (time.perf_counter() - t0) * 1e3


def main():
    frames = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    print(card(), flush=True)
    from global_map_merge_bench import build
    from test_pose_graph import seq_graph
    from test_process_cloud import FE
    O = seq_graph("00")[0]
    g = build(O, 2000, False)
    seq, _ = g.global_map_merged(0.5)
    g.close()
    scan0 = synth.raw_scan()
    steps = [synth.se3_exp(np.array([0.5 * k, 0.0, 0.0, 0.0, 0.0, 0.002 * k])) for k in range(frames)]
    scans = [(scan0 - T[:3, 3]) @ T[:3, :3] for T in steps]        # sensor frame
    for T in steps:                                                 # the poses in the map, 2 km from the seq-00 part
        T[:3, 3] += FAR
    m = tloam_b200.LocalRegistration()
    m.enable_global_map(voxel=0.5)
    for T, s in zip(steps, scans):
        m.global_map_append(s, T)
    local, _ = m.global_map_merged(0.5)
    m.close()
    prior = np.vstack([seq, local])

    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.localize_enable()
    r.localize_set_map(prior)
    r.map_update_enable()
    host, dev, used = [], [], 0
    for k, s in enumerate(scans):
        r.process_raw_scan(s, feature=FE)
        r.localize_frame(steps[k])
        r.set_profiling(True)
        a, ms = sync_ms(r, r.map_update_add)
        prof = r.get_profile()
        r.set_profiling(False)
        host.append(ms)
        dev.append(sum(v for _, v in prof.values()))
        used += int(a.used)
    print(json.dumps(dict(case=f"map_update_add, HDL-64E scans ({len(scans[0])} rows) on {len(prior)} prior rows",
                          host_ms_median=round(float(np.median(host[1:])), 3), device_ms_median=round(float(np.median(dev[1:])), 3),
                          used=used, frames=len(scans), additions=r.map_update_size()[1])), flush=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        for k, s in enumerate(scans[:8]):
            r.process_raw_scan(s, feature=FE)
            r.localize_frame(steps[k])
            r.map_update_add()
        torch.cuda.synchronize()
    ev = [(e.name, e.time_range.elapsed_us()) for e in p.events() if "k_gmd_" in e.name or "k_mu_" in e.name]
    votes = [[], []]
    i = 0
    while i + 4 <= len(ev):                                         # per add: 4 kernels over the prior, 4 over the additions
        if "k_gmd_clear" in ev[i][0]:
            votes[len(votes[0]) > len(votes[1])].append(sum(us for _, us in ev[i:i + 4]) / 1e3)
            i += 4
        else:
            i += 1
    print(json.dumps(dict(case="the two tloam_gmd_vote calls of an add (torch.profiler kernel time)",
                          prior_votes_ms_median=round(float(np.median(votes[0][1:])), 4) if len(votes[0]) > 1 else None,
                          addition_votes_ms_median=round(float(np.median(votes[1][1:])), 4) if len(votes[1]) > 1 else None,
                          adds=len(votes[0]))), flush=True)

    # the loop with and without the add, alternated
    rates = {"on": [], "off": []}
    for rnd in range(6):
        mode = "on" if rnd % 2 == 0 else "off"
        r.localize_set_map(prior)
        r.process_raw_scan(scans[0], feature=FE)
        r.localize_frame(steps[0])
        t0 = time.perf_counter()
        for k in range(1, len(scans)):
            r.process_raw_scan(scans[k], feature=FE)
            r.localize_frame(steps[k])
            if mode == "on":
                r.map_update_add()
        r.map_update_size()
        rates[mode].append((len(scans) - 1) / (time.perf_counter() - t0))
    print(json.dumps(dict(case="localize loop (process_raw_scan + localize_frame), frames/s", updating_on=[round(x, 1) for x in rates["on"]],
                          updating_off=[round(x, 1) for x in rates["off"]])), flush=True)

    # builds at about 0, 1e5 and 1e6 addition rows
    r.map_update_enable(novel_radius=0.01, min_frames=1)
    r.localize_set_map(prior)
    targets, k = [0, 100_000, 1_000_000], 0
    for target in targets:
        while r.map_update_size()[1] < target:
            j = k % len(scans)
            r.process_raw_scan(scans[j], feature=FE)
            r.localize_frame(steps[j])
            r.map_update_add()
            k += 1
        r.map_update_build()                                        # warm
        n = _lib.MapUpdateResult()
        t0 = time.perf_counter()
        assert r._L.tloam_b200_map_update_build(r._h, C.byref(n)) == 0     # the build alone, without the download
        ms = (time.perf_counter() - t0) * 1e3
        t0 = time.perf_counter()
        r.map_update_build()
        ms_dl = (time.perf_counter() - t0) * 1e3
        print(json.dumps(dict(case=f"map_update_build at {n.n_additions} addition rows", build_ms=round(ms, 2),
                              build_and_download_ms=round(ms_dl, 2), prior_rows=n.n_prior, voxels=n.n_voxels,
                              total=n.n_total)), flush=True)
    r.close()


if __name__ == "__main__":
    main()
