"""Loop-closure cost (include/tloam_b200.h "Loop closure"), default Scan Context configuration (20 x 60, exclude_recent 50).
  (a) one add (loop_add_frame of the 116k-point synthetic HDL-64E scan process_raw_scan left on the device: descriptor
      and exact search) at database sizes 1 000, 4 541 (KITTI 00) and 20 000.  The database is filled with real adds of
      small clouds; at each size `adds` adds run back to back.  Reported: the host clock over them ending in the result's
      synchronise, and the device time of the loop launches from CUDA events (the handle's profiling, class "submap").
  (b) frames/s of the four-call mapping loop (process_raw_scan -> scan_match_predicted_async -> submap_update_frame_chained
      -> global_map_append_frame_chained -> get_result) with and without loop_add_frame, in alternating rounds.
  (c) the same exhaustive search through the numpy restatement (tests/scan_context_oracle.py) on the host, for scale.
Prints the card and its power limit read in the same call, then one JSON line.

    python tools/loop_bench.py [adds] [frames] [rounds]
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
import scan_context_oracle as sco  # noqa: E402

FE = dict(cvr_submap=0.005, cvr_scan=0.01)        # the street scene has few curvature maxima (tests/test_front_end_chain.py)
SIZES = (1000, 4541, 20000)


def small_cloud(rng):
    return np.column_stack([rng.uniform(-70, 70, (1500, 2)), rng.uniform(-2.0, 4.0, 1500)])


def add_times(raw, adds):
    r = tloam_b200.LocalRegistration()
    r.loop_enable()
    r.process_raw_scan(raw, feature=FE)
    rng = np.random.default_rng(1)
    clouds = [small_cloud(rng) for _ in range(64)]
    out = {}
    for size in SIZES:
        while r.loop_size() < size - adds // 2:
            r.loop_add(clouds[r.loop_size() % 64])
        r.loop_add_frame()                                         # warm-up at this size
        r.loop_result()
        r.set_profiling(True)
        t0 = time.perf_counter()
        for _ in range(adds):
            r.loop_add_frame()
        res = r.loop_result()
        host = 1e3 * (time.perf_counter() - t0) / adds
        prof = r.get_profile()["submap"]
        r.set_profiling(False)
        out[size] = dict(host_ms=host, device_ms=prof[1] / adds, launches=prof[0], frames=r.loop_size(), last=res.candidate)
    r.close()
    return out


def mapping_fps(scans, loop, frames):
    r = tloam_b200.LocalRegistration(fitness_thres=0.3)
    r.enable_global_map()
    if loop:
        r.loop_enable()
    r.process_raw_scan(scans[0], feature=FE)
    r.submap_init_frame()
    t0 = time.perf_counter()
    for k in range(frames):
        r.process_raw_scan(scans[1 + k % (len(scans) - 1)], feature=FE)
        r.scan_matching_predicted_async()
        r.submap_update_frame_chained()
        r.global_map_append_frame()
        if loop:
            r.loop_add_frame()
        r.get_result()
    fps = frames / (time.perf_counter() - t0)
    r.close()
    return fps


def oracle_ms(n_db):
    rng = np.random.default_rng(2)
    cfg = sco.config()
    descs = [sco.descriptor(small_cloud(rng), cfg) for _ in range(8)]
    db = [descs[k % 8] for k in range(n_db + 50)]
    t0 = time.perf_counter()
    sco.query(db, n_db + 49, 50)
    return 1e3 * (time.perf_counter() - t0)


def main():
    adds = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    frames = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    raw = synth.raw_scan()
    a = add_times(raw, adds)
    for size, v in a.items():
        print(f"(a) database {v['frames']:6d}: add {v['host_ms']:.3f} ms host clock, {v['device_ms']:.3f} ms device "
              f"({v['launches']} launches)")
    scans = [raw]
    for k in range(1, 7):                                          # the scan seen from a sensor moved along the street
        Ti = np.linalg.inv(synth.se3_exp([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k]))
        scans.append(np.ascontiguousarray(raw @ Ti[:3, :3].T + Ti[:3, 3] + np.random.default_rng(k).normal(0, 0.005, raw.shape)))
    mapping_fps(scans, False, 3)                                   # warm-up
    mapping_fps(scans, True, 3)
    fps = {False: [], True: []}
    for _ in range(rounds):
        for loop in (False, True):
            fps[loop].append(mapping_fps(scans, loop, frames))
    print(f"(b) mapping loop frames/s without loop_add_frame {np.round(fps[False], 1)}, with {np.round(fps[True], 1)}")
    o = {n: oracle_ms(n) for n in (1000, 4541)}
    print(f"(c) numpy exhaustive search on the host: {o[1000]:.0f} ms at 1 000 frames, {o[4541]:.0f} ms at 4 541")
    print(json.dumps(dict(card=card, add={str(k): v for k, v in a.items()}, fps_without=fps[False], fps_with=fps[True],
                          oracle_ms={str(k): v for k, v in o.items()})))


if __name__ == "__main__":
    main()
