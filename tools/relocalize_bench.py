"""Relocalization in a prior map (include/tloam_b200.h "Relocalization in a prior map"): the cost of one relocalization
against a seq-00-sized session, and of the same hypotheses as sequential localizations.
  - map: the seq-00-sized map tools/global_map_merge_bench.py builds (4 541 frames of 2 000 points at the seq 00 odometry
    poses), plus an HDL-64E scan (tloam_b200.synth.raw_scan, about 120 000 rows) appended at the poses of 8 frames spread
    along the route, merged at 0.5 m and loaded with tloam_b200_localize_set_map_merged.
  - places: 4 541, one per frame, made by tloam_b200_loop_add on the same handle (the 8 frames above get the HDL-64E
    scan, the others a cloud of 2 000 points uniform in +-60 m) and loaded with tloam_b200_relocalize_set_places_loop at
    the odometry poses.  The query is the HDL-64E scan with new noise, so the 8 scan places are the top_k 8 hypotheses,
    each converging on its own copy of the scan (the result is ambiguous: the timing is that of 8 full runs).
  - timed, alternated in one run: tloam_b200_relocalize (host clock of the call, which ends in a synchronise, and its
    device time from the handle's CUDA events), and the same 8 guesses as 8 sequential tloam_b200_localize calls.
  - the split of the relocalization's device time into the search (k_sc_bin, k_sc_finish, k_rl_search, k_rl_topk,
    k_rl_guess) and the ICP (k_rl_match, k_rl_reduce, k_rl_step, k_rl_final, k_rl_select), from the kernels' device
    timestamps in a separate torch.profiler run.
Prints the card and its power limit read in the same call, then one JSON line per case.

    python tools/relocalize_bench.py [calls]
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

SEARCH = ("k_sc_bin", "k_sc_finish", "k_rl_search", "k_rl_topk", "k_rl_guess")
ICP = ("k_rl_match", "k_rl_reduce", "k_rl_step", "k_rl_final", "k_rl_select")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def device_ms(r, call):
    r.set_profiling(True)
    t0 = time.perf_counter()
    out = call()
    host = (time.perf_counter() - t0) * 1e3
    dev = sum(ms for _, ms in r.get_profile().values())
    r.set_profiling(False)
    return out, host, dev


def main():
    calls = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    print(card(), flush=True)
    from global_map_merge_bench import build
    from test_pose_graph import seq_graph
    O = seq_graph("00")[0]
    scan = synth.raw_scan()
    scan = scan[np.isfinite(scan).all(axis=1)]
    chosen = set(np.linspace(200, len(O) - 200, 8).astype(int).tolist())
    r = build(O, 2000, False)
    for j in sorted(chosen):
        r.global_map_append(scan, O[j])
    prior, _ = r.global_map_merged(0.5)
    r.localize_enable()
    r.localize_set_map_merged()
    r.relocalize_enable()
    r.loop_enable(initial_capacity_frames=len(O))
    rng = np.random.default_rng(5)
    for j in range(len(O)):
        r.loop_add(scan + rng.normal(0, 0.01, scan.shape) if j in chosen else rng.uniform(-60.0, 60.0, (2000, 3)))
    r.loop_result()
    t0 = time.perf_counter()
    r.relocalize_set_places_loop(O)
    load_ms = (time.perf_counter() - t0) * 1e3
    query = scan + rng.normal(0, 0.01, scan.shape)

    rel, _, _ = device_ms(r, lambda: r.relocalize(query))                                # warm-up
    guesses = [h[3].guess for h in r.relocalize_hypotheses()]
    for G in guesses:
        r.localize(query, G)
    rh, rd, sh, sd = [], [], [], []
    for _ in range(calls):
        rel, h, d = device_ms(r, lambda: r.relocalize(query))
        rh.append(h)
        rd.append(d)
        h, d = 0.0, 0.0
        for G in guesses:
            _, hh, dd = device_ms(r, lambda: r.localize(query, G))
            h += hh
            d += dd
        sh.append(h)
        sd.append(d)
    hyps = r.relocalize_hypotheses()
    print(json.dumps(dict(case=f"relocalize, HDL-64E scan ({len(query)} rows, {hyps[0][3].n_query_points} after the down-sample) "
                          f"against {len(O)} places and {len(prior)} map rows", top_k=len(hyps),
                          places=sorted(int(h[0]) for h in hyps) == sorted(chosen), iterations=[h[3].iterations for h in hyps],
                          set_places_loop_ms=round(load_ms, 2), relocalize_host_ms_median=round(float(np.median(rh)), 3),
                          relocalize_device_ms_median=round(float(np.median(rd)), 3),
                          sequential_8_localize_host_ms_median=round(float(np.median(sh)), 3),
                          sequential_8_localize_device_ms_median=round(float(np.median(sd)), 3),
                          ambiguous=bool(rel.ambiguous), calls=calls)), flush=True)

    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            r.relocalize(query)
        torch.cuda.synchronize()
    tot = {"search": 0.0, "icp": 0.0}
    seen = {}
    for e in prof.events():
        name = e.name
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = getattr(e, "cuda_time_total", 0.0)
        for k in SEARCH + ICP:
            if k in name:
                seen[k] = seen.get(k, 0.0) + dt / 1e3 / 5
                tot["search" if k in SEARCH else "icp"] += dt / 1e3 / 5
    print(json.dumps(dict(case="relocalize device time by kernel (torch.profiler, mean of 5 calls)",
                          search_ms=round(tot["search"], 3), icp_ms=round(tot["icp"], 3),
                          kernels_ms={k: round(v, 3) for k, v in sorted(seen.items())})), flush=True)
    r.close()


if __name__ == "__main__":
    main()
