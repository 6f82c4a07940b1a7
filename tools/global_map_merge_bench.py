"""Merged global map cost (include/tloam_b200.h "Merged global map") on a seq-00-sized map, built as
tools/map_correct_bench.py builds it: a frame of `points_per_frame` points uniform in +-60 m (one per 1 m voxel, about
2 000 voxels) appended with intensity at every odometry pose of tests/test_pose_graph.py's seq_graph("00") (4 541 frames,
about 9.08 M points), with dynamic-point removal on so that static_only can run.  The "parked" variant adds to every frame
the same 200 world points of a 4.5 x 1.8 x 1.5 m box (a parked vehicle): one row per frame in the same voxels, so its voxels
are thousands of rows long.
For each map, merges at 1.0 and 0.5 m, with and without static_only:
  - device time of the merge's launches from the handle's CUDA events (class "submap"), and host clock to the merge's
    last synchronise (tloam_b200_global_map_merge; the download is not included)
  - n_vox and the longest voxel
  - the bytes the pipeline moves, counted from the shapes (below), against 3.35 TB/s
  - the numpy restatement's host time (tests/global_map_merge_oracle.py), and whether the device result equals it bit for
    bit
Prints the card and its power limit read in the same call, then one JSON line per merge.

Counted bytes per selected map row: bounds 24 (+ 8 of counters with static_only), keys 24 (+ 8) read and 12 written,
32 per radix pass (the histogram reads the 8-byte key, the scatter reads and writes key and row index), 16 for the
heads (each key and its predecessor), 4 + 24 (+ 8 intensity) gathered by the averages; per voxel 8 of starts and 32 (24
without intensity) written.

    python tools/global_map_merge_bench.py [calls] [points_per_frame]
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
import tloam_b200  # noqa: E402
import global_map_merge_oracle as gmo  # noqa: E402
import map_dynamic_oracle as mdo  # noqa: E402
from test_pose_graph import seq_graph  # noqa: E402

HBM = 3.35e12


def build(O, pts, parked):
    rng = np.random.default_rng(7)
    box = rng.uniform(-1.0, 1.0, (200, 3)) * np.array([2.25, 0.9, 0.75]) + np.array([O[len(O) // 2][0, 3] + 5.0,
                                                                                      O[len(O) // 2][1, 3], 0.0])
    r = tloam_b200.LocalRegistration()
    r.enable_global_map(initial_capacity=len(O) * (pts + 250))
    r.global_map_dynamic_enable()
    for T in O:
        p = rng.uniform(-60.0, 60.0, (pts, 3))
        if parked:                                                 # the box's world points in this frame's sensor frame
            p = np.concatenate([p, (box - T[:3, 3]) @ T[:3, :3]])
        r.global_map_append(p, T, intensity=rng.uniform(0.0, 255.0, len(p)))
    r.global_map_size()
    return r


def counted_bytes(n_sel, n_vox, passes, static, inten):
    sel = 8 if static else 0
    per_row = (24 + sel) + (24 + sel + 12) + 32 * passes + 16 + 4 + 24 + (8 if inten else 0)
    per_vox = 8 + 24 + (8 if inten else 0)
    return n_sel * per_row + n_vox * per_vox


def measure(r, name, voxel, static, calls, card):
    m, inten = r.global_map(), r.global_map_intensity()
    if static:
        t, h = r.global_map_votes()
        m, inten = mdo.static_map(m, inten, t, h, mdo.config())
    key, _ = gmo.keys(m, voxel)
    bits = sum(int(b).bit_length() for b in np.floor(((m.max(0) - (m.min(0) - voxel * 0.5)) / voxel)).astype(np.int64))
    passes = (bits + (1 if static else 0) + 7) // 8
    got = r.global_map_merged(voxel, static=static)                # warm-up (and the buffers' allocation)
    host = []
    L = r._L
    nv = C.c_size_t(0)
    for _ in range(calls):
        t0 = time.perf_counter()
        rc = L.tloam_b200_global_map_merge(r._h, voxel, 1 if static else 0, C.byref(nv))
        host.append(1e3 * (time.perf_counter() - t0))
        assert rc == 0, rc
    r.set_profiling(True)
    for _ in range(calls):
        L.tloam_b200_global_map_merge(r._h, voxel, 1 if static else 0, C.byref(nv))
    dev = r.get_profile()["submap"][1] / calls
    r.set_profiling(False)
    t0 = time.perf_counter()
    want = gmo.merge(m, voxel, inten)
    oracle_ms = 1e3 * (time.perf_counter() - t0)
    exact = bool(np.array_equal(got[0].view(np.uint64), want[0].view(np.uint64)) and
                 np.array_equal(np.isnan(got[1]), np.isnan(want[1])) and
                 np.array_equal(got[1][~np.isnan(got[1])].view(np.uint64), want[1][~np.isnan(want[1])].view(np.uint64)))
    longest = int(np.unique(key, return_counts=True)[1].max())
    nbytes = counted_bytes(len(m), nv.value, passes, static, True)
    print(f"{name}: voxel {voxel} static {static}: {len(m)} rows -> {nv.value} voxels (longest {longest} rows), "
          f"{passes} passes; {dev:.3f} ms device (CUDA events), {np.median(host):.2f} ms host clock median; "
          f"{nbytes / 1e9:.3f} GB counted = {nbytes / (dev * 1e-3) / 1e9:.0f} GB/s ({100 * nbytes / (dev * 1e-3) / HBM:.0f} % "
          f"of 3.35 TB/s); numpy restatement {oracle_ms:.0f} ms; exact {exact}")
    print(json.dumps(dict(card=card, map=name, voxel=voxel, static_only=static, rows=int(len(m)), n_vox=int(nv.value),
                          longest_voxel=longest, passes=passes, device_ms=dev, host_ms_median=float(np.median(host)),
                          host_ms_min=float(np.min(host)), bytes=int(nbytes), oracle_ms=oracle_ms, exact=exact)))


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    pts = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print("card:", card)
    G, O, loops = seq_graph("00")
    O = np.array(O)
    for name, parked in (("seq00", False), ("parked", True)):
        r = build(O, pts, parked)
        print(f"{name}: {r.global_map_size()[0]} map points in {r.global_map_size()[1]} frames")
        for voxel in (1.0, 0.5):
            for static in (False, True):
                measure(r, name, voxel, static, calls, card)
        r.close()


if __name__ == "__main__":
    main()
