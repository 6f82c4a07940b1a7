"""FrontEnd::processCloud on the device, on a 116k-point synthetic HDL-64E raw scan (the street scene of synth.raw_scan):
  (a) one tloam_b200_process_cloud call on the scan's segmented ground / edge / general clouds (host clouds in);
  (b) one tloam_b200_process_raw_scan call (raw scan in, nothing but counts out);
  (c) the host-glue path (b) replaces: segment_raw_scan, numpy gathers, voxel_down_sample x 2, extract_planar_sphere, numpy
      gathers, set_input_source;
  (d) frames/s of the per-frame loop process_raw_scan -> scan_match_predicted_async -> submap_update_frame_chained ->
      get_result against the same loop with the host glue of (c) and submap_update_chained.
It checks that (b) and (c) give the same source apart from the voxel order and the fixed-point voxel averages (planar /
sphere bit-identical, ground / edge the same rows to 1e-10 m), and prints the card and its power limit with the numbers.

With --mapping it measures the global map instead: frames/s of the loop (d) with global_map_append_frame_chained after the
submap update against the same loop without it, three alternating runs each, the voxels appended per frame, and the time
per frame of the same work on the CPU (numpy: transform, finite rows, VoxelDownSample(1.0) by np.unique and a group mean).

With --mapping --intensity it times one global_map_append_frame of the raw scan with and without its intensity channel
(two handles, alternating rounds of back-to-back appends) and checks that the xyz map is the same.

    python tools/process_cloud_bench.py [reps] [--mapping [--intensity]]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import tloam_b200  # noqa: E402
from tloam_b200 import synth  # noqa: E402

FE = dict(cvr_submap=0.005, cvr_scan=0.01)        # the street scene has few curvature maxima (tests/test_front_end_chain.py)


def host_glue(reg, raw):
    """(c): what a caller does today to turn a raw scan into the registration source; returns the planar-submap selection"""
    s = reg.segment_raw_scan(raw)
    ground, edge, general = (np.ascontiguousarray(raw[s[k]]) for k in ("ground", "edge", "general"))
    g = reg.voxel_down_sample(ground, 0.3)
    e = reg.voxel_down_sample(edge, 0.1)
    p_scan, p_sub, s_scan, s_sub, _ = reg.extract_planar_sphere(general, **FE)
    reg.set_input_source([e, general[:len(s_scan)], general[p_scan], g])          # sphere: the rank list taken literally (Q12)
    return general[p_sub]


def timed(fn, reps):
    fn()
    passes = []
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        passes.append(1e3 * (time.perf_counter() - t0) / reps)           # every call ends in a synchronisation
    return float(np.median(passes)), passes


def sorted_rows(a):
    return a[np.lexsort(a.T[::-1])]


def moved_scans(raw, reps):
    xis = [np.array([0.3 * k, 0.02 * k, 0.0, 0.0, 0.0, 0.004 * k]) for k in range(reps + 1)]
    scans = [raw]
    for k in range(1, reps + 1):
        Ti = np.linalg.inv(synth.se3_exp(xis[k]))
        scans.append(np.ascontiguousarray(raw @ Ti[:3, :3].T + Ti[:3, 3]))
    return scans, synth.se3_exp(-xis[1])


def cpu_map_frame(raw, T, voxel=1.0):
    """what a caller without the device map does per frame: T.p, finite rows, VoxelDownSample(voxel) of the frame"""
    reg = raw @ T[:3, :3].T + T[:3, 3]
    fin = reg[np.isfinite(reg).all(axis=1)]
    idx = np.floor((fin - (fin.min(0) - 0.5 * voxel)) / voxel).astype(np.int64)
    uniq, inv, cnt = np.unique(idx, axis=0, return_inverse=True, return_counts=True)
    out = np.zeros((cnt.size, 3))
    np.add.at(out, inv.reshape(-1), fin)
    return out / cnt[:, None]


def mapping_main(reps, card):
    raw = synth.raw_scan()
    scans, prev = moved_scans(raw, reps)
    res = {"gpu": card, "raw_points": int(len(raw)), "frames": reps, "voxel": 1.0}
    runs = {"without_mapping": [], "with_mapping": []}
    for _ in range(3):
        for mode in ("without_mapping", "with_mapping"):                 # alternating: the shared card drifts
            r = tloam_b200.LocalRegistration(fitness_thres=0.3)
            if mode == "with_mapping":
                r.enable_global_map()
            r.process_raw_scan(scans[0], feature=FE)
            r.submap_init_frame()
            r.set_pose_history(prev, np.eye(4))
            t0 = time.perf_counter()
            for sc in scans[1:]:
                r.process_raw_scan(sc, feature=FE)
                r.scan_matching_predicted_async()
                r.submap_update_frame_chained()
                if mode == "with_mapping":
                    r.global_map_append_frame()
                T = r.get_result()
            runs[mode].append(reps / (time.perf_counter() - t0))
            if mode == "with_mapping":
                n, f = r.global_map_size()
                res["voxels_per_frame"] = n / f
                res["growths"] = r.global_map_capacity()[1]
            r.close()
    for mode, v in runs.items():
        res[f"{mode}_frames_per_s"] = [round(x, 1) for x in v]
    res["mapping_ms_per_frame"] = [round(1e3 / w - 1e3 / wo, 3) for wo, w in zip(runs["without_mapping"], runs["with_mapping"])]
    # the append alone: back-to-back global_map_append_frame calls on one processed scan, ending in a synchronise
    r = tloam_b200.LocalRegistration()
    r.enable_global_map()
    r.process_raw_scan(raw, feature=FE)
    T = synth.se3_exp([1.0, 0.5, 0.0, 0.0, 0.0, 0.1])
    r.global_map_append_frame(T)
    r.global_map_size()
    per = []
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(50):
            r.global_map_append_frame(T)
        r.global_map_size()
        per.append(round(1e3 * (time.perf_counter() - t0) / 50, 3))
    res["append_frame_ms"] = per
    r.close()
    cpu_map_frame(raw, T)
    t0 = time.perf_counter()
    for _ in range(5):
        cpu_map_frame(raw, T)
    res["cpu_numpy_ms_per_frame"] = round(1e3 * (time.perf_counter() - t0) / 5, 2)
    print(json.dumps(res))


def intensity_main(card, rounds=5, calls=50):
    """one global_map_append_frame on the 116k-point raw scan with and without the intensity channel: two handles (one never
    sees intensity), `calls` back-to-back appends each ending in a synchronise, `rounds` alternating rounds"""
    raw = synth.raw_scan()
    inten = np.random.default_rng(1).uniform(0.0, 255.0, len(raw))
    T = synth.se3_exp([1.0, 0.5, 0.0, 0.0, 0.0, 0.1])
    handles = {}
    for mode in ("without_intensity", "with_intensity"):
        r = tloam_b200.LocalRegistration()
        r.enable_global_map()
        r.process_raw_scan(raw, feature=FE)
        handles[mode] = r
    kw = {"without_intensity": {}, "with_intensity": {"intensity": inten}}
    per = {m: [] for m in handles}
    for _ in range(rounds):
        for mode, r in handles.items():                                  # alternating: the shared card drifts
            r.reset_global_map()
            r.global_map_append_frame(T, **kw[mode])
            r.global_map_size()
            t0 = time.perf_counter()
            for _ in range(calls):
                r.global_map_append_frame(T, **kw[mode])
            r.global_map_size()
            per[mode].append(round(1e3 * (time.perf_counter() - t0) / calls, 4))
    r = handles["with_intensity"]
    n, f = r.global_map_size()
    assert r.global_map_has_intensity() and len(r.global_map_intensity()) == n
    a = handles["without_intensity"]
    same = np.array_equal(a.global_map(), r.global_map())
    res = {"gpu": card, "raw_points": int(len(raw)), "voxels_per_frame": n / f, "xyz_map_identical": bool(same),
           "calls_per_round": calls}
    for mode, v in per.items():
        res[f"append_frame_{mode}_ms"] = v
    res["added_ms"] = [round(w - wo, 4) for wo, w in zip(per["without_intensity"], per["with_intensity"])]
    for h in handles.values():
        h.close()
    print(json.dumps(res))


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    reps = int(args[0]) if args else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    if "--mapping" in sys.argv and "--intensity" in sys.argv:
        return intensity_main(card)
    if "--mapping" in sys.argv:
        return mapping_main(reps, card)
    raw = synth.raw_scan()
    reg = tloam_b200.LocalRegistration()
    s = reg.segment_raw_scan(raw)
    clouds = [np.ascontiguousarray(raw[s[k]]) for k in ("ground", "edge", "general")]
    res = {"gpu": card, "raw_points": int(len(raw)), "ground": len(clouds[0]), "edge": len(clouds[1]), "general": len(clouds[2])}
    res["a_process_cloud_ms"], _ = timed(lambda: reg.process_cloud(*clouds, **FE), reps)
    res["b_process_raw_scan_ms"], _ = timed(lambda: reg.process_raw_scan(raw, feature=FE), reps)
    res["source_sizes"] = reg.process_raw_scan(raw, feature=FE)
    dev = [reg.source_cloud(c) for c in range(4)]
    res["c_host_glue_ms"], _ = timed(lambda: host_glue(reg, raw), reps)
    host_glue(reg, raw)
    host = [reg.source_cloud(c) for c in range(4)]
    same = np.array_equal(dev[1], host[1]) and np.array_equal(dev[2], host[2])
    for c in (0, 3):
        a, b = sorted_rows(dev[c]), sorted_rows(host[c])
        same = same and a.shape == b.shape and bool(np.allclose(a, b, rtol=0, atol=1e-10))
    res["b_equals_c_up_to_voxel_order"] = bool(same)

    # (d) the per-frame loop over rigid motions of the scan, seeded from frame 0
    scans, prev = moved_scans(raw, reps)
    for mode in ("device", "host_glue"):
        r = tloam_b200.LocalRegistration(fitness_thres=0.3)
        if mode == "device":
            r.process_raw_scan(scans[0], feature=FE)
            r.submap_init_frame()
        else:
            s0 = r.segment_raw_scan(scans[0])
            ground, edge, general = (np.ascontiguousarray(scans[0][s0[k]]) for k in ("ground", "edge", "general"))
            p_scan, p_sub, s_scan, s_sub, _ = r.extract_planar_sphere(general, **FE)
            r.submap_init(edge, ground, general[p_sub], general[:len(s_sub)])
        r.set_pose_history(prev, np.eye(4))
        t0 = time.perf_counter()
        for sc in scans[1:]:
            if mode == "device":
                r.process_raw_scan(sc, feature=FE)
                r.scan_matching_predicted_async()
                r.submap_update_frame_chained()
            else:
                planar_sub = host_glue(r, sc)
                r.scan_matching_predicted_async()
                r.submap_update_chained(planar_sub)
            T = r.get_result()
        res[f"d_{mode}_frames_per_s"] = reps / (time.perf_counter() - t0)
        res[f"d_{mode}_last_pose_t"] = [float(v) for v in T[:3, 3]]
        r.close()
    reg.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
