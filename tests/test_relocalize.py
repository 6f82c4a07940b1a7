"""Relocalization in a prior map (include/tloam_b200.h "Relocalization in a prior map"; k_rl_* in libtloam_b200_reloc.so):
a Scan Context search over a saved session's places, the best candidates refined by the localization's ICP in one batch.
tests/relocalize_oracle.py is the CPU restatement.

CPU: the place search and the top-K against a brute force over np.roll (ties between places and between shifts), the
guess of a scan turned by whole sectors, a kidnapped second drive, an off-route query, the symbols, the library's kernels
and the side libraries' unchanged SASS.  GPU: the query descriptor, the candidates, every guess and every hypothesis's run
against the restatement, places from the loop database, the prediction after a relocalization, the status codes."""
import ctypes as C
import json
import math
import os
import subprocess

import numpy as np
import pytest

import localize_oracle as lo
import loop_verify_oracle as lvo
import relocalize_oracle as ro
import sass_digest
import scan_context_oracle as sco
from test_global_map_intensity import same_bits
from test_localize import ACCURACY_BOUND, check_run
from test_loop_verify import apply4, se3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["tloam_b200_loop_descriptors_download", "tloam_b200_relocalize_default_config", "tloam_b200_relocalize_enable",
               "tloam_b200_relocalize_set_places", "tloam_b200_relocalize_set_places_loop", "tloam_b200_relocalize_frame",
               "tloam_b200_relocalize", "tloam_b200_relocalize_hypotheses", "tloam_b200_relocalize_matches"]
KERNELS = ("k_rl_search", "k_rl_topk", "k_rl_guess", "k_rl_match", "k_rl_reduce", "k_rl_step", "k_rl_final", "k_rl_select")


def small_cfg():
    return ro.config(n_ring=6, n_sector=12, max_radius=20.0)


def random_desc(rng, R, S, zero_cols=()):
    """(bins, ring key, norms) of random bins, the columns zero_cols empty"""
    bins = rng.uniform(0.0, 3.0, (R, S))
    bins[:, list(zero_cols)] = 0.0
    return bins, bins.sum(1) / S, np.sqrt((bins * bins).sum(0))


# ---- CPU: the restatement -------------------------------------------------------------------------------------------------
def test_oracle_place_search_and_top_k_are_a_brute_force_over_rolls():
    rng = np.random.default_rng(3)
    cfg = small_cfg()
    R, S = cfg["n_ring"], cfg["n_sector"]
    q = random_desc(rng, R, S, zero_cols=(2,))
    periodic = np.tile(rng.uniform(0.0, 3.0, (R, S // 2)), (1, 2))              # equal distances at shifts s and s + S/2
    places = [random_desc(rng, R, S) for _ in range(9)] + [(periodic, periodic.sum(1) / S, np.sqrt((periodic ** 2).sum(0)))]
    places += [places[4], places[1]]                                             # ties between places
    dist, shift = ro.place_search(q, places)
    for j, p in enumerate(places):
        d = [sco.distance_literal(q, (np.roll(p[0], s, axis=1), p[1], np.roll(p[2], s)), 0) for s in range(S)]
        want = min(range(S), key=lambda s: (d[s], s))
        assert shift[j] == want and dist[j] == d[want], j
    assert shift[9] < S // 2
    top = ro.top_k(dist, 5, 2.0)
    want = sorted(range(len(places)), key=lambda j: (dist[j], j))[:5]
    assert list(top) == want
    assert list(ro.top_k(dist, 20, np.sort(dist)[3])) == sorted(range(len(places)), key=lambda j: (dist[j], j))[:3]
    assert list(ro.top_k(np.array([0.2, 0.1, 0.2, 0.1]), 3, 1.0)) == [1, 3, 0]


def test_oracle_guess_of_a_scan_turned_by_whole_sectors_is_its_places_pose():
    from test_loop_closure import cast, make_world
    cfg = ro.config()
    S = cfg["n_sector"]
    world = make_world()
    scan = cast(world, 10.0, 0.0, 0.0, seed=5)
    P = se3([12.0, -4.0, 0.3, 0.01, -0.02, 0.6])
    place = sco.descriptor(scan, cfg)
    for m in (0, 1, 7, 31, 59):
        yaw = 2.0 * math.pi * m / S
        Rz = np.eye(4)
        Rz[:2, :2] = [[math.cos(yaw), -math.sin(yaw)], [math.sin(yaw), math.cos(yaw)]]
        query = apply4(np.linalg.inv(Rz), scan)                                 # p_place = Rz(yaw) p_query
        dist, shift = ro.place_search(sco.descriptor(query, cfg), [place])
        assert (-int(shift[0])) % S == m and dist[0] < 0.05, (m, shift[0], dist[0])
        G = ro.guess(P, shift[0], S)
        assert np.abs(G - P @ Rz).max() < 1e-12 and np.array_equal(G[3], [0, 0, 0, 1]) and same_bits(G[:3, 3], P[:3, 3])


# ---- CPU: a kidnapped second drive against the first drive's places and map ------------------------------------------------
KIDNAPPED = range(0, 50, 5)


def first_session(frames):
    """the first drive's places (descriptor tuples, true poses) over `frames` and its map merged at 0.5 m"""
    from oracle import pyoracle
    from test_loop_closure import cast, make_world, route
    from test_loop_verify import pose4
    pyoracle.build()
    world = make_world()
    P = [pose4(p) for p in route()]
    scans = {k: cast(world, *route()[k], seed=k) for k in frames}
    prior = lvo.keyframe(pyoracle, np.vstack([apply4(P[k], scans[k]) for k in frames]), 0.5)
    cfg = ro.config()
    return [sco.descriptor(scans[k], cfg) for k in frames], [P[k] for k in frames], prior, world, P


def kidnapped_queries():
    """(per query: the scan, its down-sample, the true pose) of every 5th frame of the second drive (0.6 m to the left)"""
    from oracle import pyoracle
    from test_loop_closure import cast
    places, poses, prior, world, P = first_session(range(50))
    side = np.eye(4)
    side[1, 3] = 0.6
    out = []
    for k in KIDNAPPED:
        Pk = P[k] @ side
        scan = cast(world, Pk[0, 3], Pk[1, 3], math.atan2(Pk[1, 0], Pk[0, 0]), seed=1000 + k)
        out.append((scan, lvo.keyframe(pyoracle, scan, lo.config()["voxel"]), Pk))
    return places, poses, prior, out


def test_oracle_relocalizes_a_kidnapped_second_drive():
    cfg, lcfg = ro.config(), lo.config()
    places, poses, prior, queries = kidnapped_queries()
    g = lo.grid(prior, lcfg["cell"])
    nrm, valid, _ = lo.normals(g, lcfg)
    acc, errs = 0, []
    for scan, Q, truth in queries:
        r = ro.relocalize(scan, Q, places, poses, g, nrm, valid, cfg, lcfg)
        if r["accepted"]:
            acc += 1
            errs.append(lvo.relative_error(r["runs"][r["winner"]]["T"], truth))
        print(f"kidnapped: {len(r['top'])} hypotheses, winner {r['winner']}, distance "
              f"{r['distance'][r['top'][r['winner']]] if r['winner'] >= 0 else math.inf:.3f}, accepted {r['accepted']}, "
              f"ambiguous {r['ambiguous']}")
    print(f"kidnapped: {acc} / {len(queries)} accepted, worst {max(e[0] for e in errs):.4f} m "
          f"{math.degrees(max(e[1] for e in errs)):.4f} deg")
    assert acc >= 0.9 * len(queries)
    assert all(e[0] < ACCURACY_BOUND[0] and e[1] < ACCURACY_BOUND[1] for e in errs)


def test_oracle_off_route_query_is_not_accepted():
    from oracle import pyoracle
    from test_loop_closure import cast, route
    cfg, lcfg = ro.config(), lo.config()
    places, poses, prior, world, P = first_session(range(0, 50, 2))
    g = lo.grid(prior, lcfg["cell"])
    nrm, valid, _ = lo.normals(g, lcfg)
    xy = np.array([p[:2] for p in route()])
    far = np.array([xy[:, 0].mean(), xy[:, 1].max() + 45.0])
    assert np.min(np.linalg.norm(np.array([p[:2, 3] for p in poses]) - far, axis=1)) >= 40.0
    scan = cast(world, far[0], far[1], 0.3, seed=77)
    r = ro.relocalize(scan, lvo.keyframe(pyoracle, scan, lcfg["voxel"]), places, poses, g, nrm, valid, cfg, lcfg)
    assert not r["accepted"], r["winner"]


def aliasing_case():
    """the world, the map and the places duplicated 300 m along x (nothing of one copy is within 80 m of the other's
    route, so a scan cast in one copy is the scan of the other): (places, poses, map, query scan, its true pose)"""
    from test_loop_closure import cast
    places, poses, prior, world, P = first_session(range(0, 30, 3))
    X = np.eye(4)
    X[0, 3] = 300.0
    side = np.eye(4)
    side[1, 3] = 0.6
    truth = P[12] @ side
    scan = cast(world, truth[0, 3], truth[1, 3], math.atan2(truth[1, 0], truth[0, 0]), seed=2012)
    return places + places, poses + [X @ p for p in poses], np.vstack([prior, prior + X[:3, 3]]), scan, truth


def test_oracle_aliasing_is_ambiguous_and_not_accepted():
    from oracle import pyoracle
    cfg, lcfg = ro.config(), lo.config()
    places, poses, prior, scan, truth = aliasing_case()
    g = lo.grid(prior, lcfg["cell"])
    nrm, valid, _ = lo.normals(g, lcfg)
    r = ro.relocalize(scan, lvo.keyframe(pyoracle, scan, lcfg["voxel"]), places, poses, g, nrm, valid, cfg, lcfg)
    n = len(places) // 2
    acc = [k for k, run in enumerate(r["runs"]) if run["accepted"]]
    copies = {int(r["top"][k]) % n for k in acc if int(r["top"][k]) >= n} & {int(r["top"][k]) for k in acc if int(r["top"][k]) < n}
    print(f"aliasing: hypotheses {list(r['top'])}, accepted {acc}, winner {r['winner']}, ambiguous {r['ambiguous']}")
    assert copies, "a place and its copy are both accepted hypotheses"
    assert r["ambiguous"] and not r["accepted"]
    X = poses[n] @ np.linalg.inv(poses[0])                                       # the 300 m shift
    w = r["runs"][r["winner"]]
    assert w["accepted"] and min(lvo.relative_error(w["T"], T)[0] for T in (truth, X @ truth)) < ACCURACY_BOUND[0]
    # without the copy the same query is accepted: the duplicate alone makes it ambiguous
    g1 = lo.grid(prior[:len(prior) // 2], lcfg["cell"])
    n1, v1, _ = lo.normals(g1, lcfg)
    one = ro.relocalize(scan, lvo.keyframe(pyoracle, scan, lcfg["voxel"]), places[:n], poses[:n], g1, n1, v1, cfg, lcfg)
    assert one["accepted"] and not one["ambiguous"]


def test_oracle_select_rule():
    cfg = ro.config()
    T = np.eye(4)
    far, turned, near = T.copy(), T.copy(), T.copy()
    far[0, 3] = 2.5
    a = math.radians(12.0)
    turned[:2, :2] = [[math.cos(a), -math.sin(a)], [math.sin(a), math.cos(a)]]
    near[0, 3] = 1.9
    run = lambda T, f, ok=True: dict(T=T, fitness=f, accepted=ok)                  # noqa: E731
    assert ro.select([run(T, 0.10), run(far, 0.15)], cfg) == (0, True, False)      # distinct, fitness within 1.5x
    assert ro.select([run(T, 0.10), run(far, 0.151)], cfg) == (0, False, True)     # distinct, fitness above 1.5x
    assert ro.select([run(far, 0.12), run(T, 0.10)], cfg) == (1, True, False)      # the winner by fitness, not rank
    assert ro.select([run(T, 0.10), run(turned, 0.11)], cfg) == (0, True, False)   # distinct by rotation
    assert ro.select([run(T, 0.10), run(near, 0.11)], cfg) == (0, False, True)     # the same pose
    assert ro.select([run(T, 0.10), run(far, 0.11, False)], cfg) == (0, False, True)   # only accepted runs count
    assert ro.select([run(T, 0.3, False), run(far, 0.2, False)], cfg) == (1, False, False)
    assert ro.select([run(T, 0.1), run(far, 0.1)], cfg) == (0, True, False)        # a tie: the lower rank wins
    assert ro.select([], cfg) == (-1, False, False)


REVISIT_PLACES = range(92)


def test_oracle_reverse_revisit_is_accepted():
    """the places are frames 0 .. 91 (three legs); the return leg's last frame, heading -97 deg against its place's 0 deg,
    relocalizes within ACCURACY_BOUND"""
    from oracle import pyoracle
    from test_loop_closure import REVISIT_OF, cast, route
    cfg, lcfg = ro.config(), lo.config()
    places, poses, prior, world, P = first_session(REVISIT_PLACES)
    last = len(route()) - 1
    truth = P[last]
    scan = cast(world, *route()[last], seed=3000)
    g = lo.grid(prior, lcfg["cell"])
    nrm, valid, _ = lo.normals(g, lcfg)
    r = ro.relocalize(scan, lvo.keyframe(pyoracle, scan, lcfg["voxel"]), places, poses, g, nrm, valid, cfg, lcfg)
    w = r["winner"]
    e = lvo.relative_error(r["runs"][w]["T"], truth)
    print(f"reverse revisit: place {int(r['top'][w])} shift {int(r['shift'][r['top'][w]])} distance "
          f"{r['distance'][r['top'][w]]:.4f}, accepted {r['accepted']}, error {e[0]:.4f} m {math.degrees(e[1]):.4f} deg")
    assert abs(int(r["top"][w]) - REVISIT_OF) <= 2
    assert r["accepted"] and e[0] < ACCURACY_BOUND[0] and e[1] < ACCURACY_BOUND[1]


# ---- CPU: the library -------------------------------------------------------------------------------------------------------
def test_relocalize_driver_compiles_warning_free():
    src = os.path.join(ROOT, "tests", "mock", "relocalize_driver.cpp")
    res = subprocess.run(["/usr/bin/g++", "-std=c++14", "-O2", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I",
                          os.path.join(ROOT, "tests", "mock"), src], capture_output=True, text=True)
    assert res.returncode == 0 and res.stderr == "", res.stderr


def test_new_symbols_are_declared_and_bound():
    from tloam_b200 import _lib
    from test_abi import declared_symbols
    assert set(NEW_SYMBOLS) <= set(declared_symbols()) and set(NEW_SYMBOLS) <= set(_lib.EXPORTS)
    c = _lib.RelocalizeConfig()
    _lib.load().tloam_b200_relocalize_default_config(C.byref(c))
    assert {k: getattr(c, k) for k, _ in c._fields_} == ro.config()


def test_reloc_library_holds_only_its_kernels_for_sm90a_and_match_does_not_spill():
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    names = sorted(sass_digest.digests(build.RELOC_LIB))
    assert len(names) == len(KERNELS) and [sum(f"{len(k)}{k}E" in m for m in names) for k in KERNELS] == [1] * len(KERNELS)
    elf = subprocess.run([sass_digest.cuobjdump(), "-lelf", build.RELOC_LIB], capture_output=True, text=True, check=True).stdout
    cubins = [l for l in elf.splitlines() if l.strip()]
    assert cubins and all(l.rstrip().endswith(".sm_90a.cubin") for l in cubins)
    res = subprocess.run([sass_digest.cuobjdump(), "-res-usage", build.RELOC_LIB], capture_output=True, text=True, check=True).stdout
    lines = res.splitlines()
    usage = [lines[i + 1] for i, l in enumerate(lines) if "10k_rl_matchE" in l]
    assert len(usage) == 1 and " LOCAL:0 " in usage[0] and " STACK:0 " in usage[0], usage


def test_localization_and_loop_libraries_keep_their_sass():
    """the ICP bodies moved to localize_icp.cuh and the Scan Context distance to scan_context.cuh: the digests of every
    kernel of libtloam_b200_loc.so and libtloam_b200_loop.so are those of the commit before"""
    from tloam_b200 import build
    if sass_digest.cuobjdump() is None:
        pytest.skip("cuobjdump not available")
    build.build()
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "sass_digests_side.json")))
    for lib in ("libtloam_b200_loc.so", "libtloam_b200_loop.so"):
        assert sass_digest.digests(os.path.join(ROOT, "tloam_b200", lib)) == want[lib], lib


# ---- GPU ------------------------------------------------------------------------------------------------------------------
def handle(**cfg):
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    r.localize_enable()
    r.relocalize_enable(**cfg)
    return r


def device_query(rq, scan):
    """the device's down-sample of scan (relocalization's query is the localization's): from a localization on handle rq"""
    rq.localize(scan, np.eye(4))
    return rq.localize_query()


def check_against_restatement(r, rq, scan, places, poses, g, nrm, valid, cfg, name):
    """r.relocalize(scan) against the restatement on the device's query: the candidates, distances, shifts and guesses bit
    for bit; every hypothesis's iterations, termination, inliers and accepted, T within 1e-9, every pass's matches; the
    selection"""
    lcfg = lo.config()
    got = r.relocalize(scan)
    Q = device_query(rq, scan)
    want = ro.relocalize(scan, Q, places, poses, g, nrm, valid, cfg, lcfg)
    hyps = r.relocalize_hypotheses()
    assert [h[0] for h in hyps] == list(want["top"]), name
    assert [h[1] for h in hyps] == [int(want["shift"][j]) for j in want["top"]], name
    assert same_bits(np.array([h[2] for h in hyps]), want["distance"][want["top"]]), name
    for k, (_, _, _, res) in enumerate(hyps):
        assert same_bits(res.guess, want["guesses"][k]), (name, k)
        w = want["runs"][k]
        assert (res.iterations, res.termination, res.inliers, res.accepted) == \
            (w["iterations"], w["termination"], w["inliers"], w["accepted"]), (name, k)
        if w["termination"] == lo.EMPTY:
            continue
        assert np.abs(res.T - w["T"]).max() < 1e-9, (name, k)
        assert len(w["passes"]) == res.iterations + 1, (name, k)
        for p, (idx, d2) in enumerate(w["passes"]):
            gi, gd = r.relocalize_matches(k, p)
            assert np.array_equal(gi, idx), (name, k, p)
            if p == 0:
                assert same_bits(gd, d2), (name, k)
    # the selection rule over the device's own runs gives the device's selection bit for bit; the restatement's fitness
    # sums in another order, so a tie between hypotheses converged to one pose may break the other way
    runs = [dict(T=res.T, fitness=res.fitness, accepted=res.accepted) for _, _, _, res in hyps]
    assert (got.winner, got.ambiguous, got.accepted) == ro.select(runs, cfg), name
    assert (got.ambiguous, got.accepted) == (want["ambiguous"], want["accepted"]), name
    if want["winner"] >= 0:
        f = want["runs"][want["winner"]]["fitness"]
        assert abs(got.result.fitness - f) <= 1e-9 * abs(f), name
        assert same_bits(got.result.T_map_odom, lo.map_odom(got.result.T, np.eye(4))), name
    print(f"relocalize {name}: {len(hyps)} hypotheses, winner {got.winner}, ambiguous {got.ambiguous}, accepted {got.accepted}")
    return got, want


@pytest.mark.gpu
def test_gpu_relocalization_matches_the_restatement():
    cfg, lcfg = ro.config(), lo.config()
    places, poses, prior, queries = kidnapped_queries()
    g = lo.grid(prior, lcfg["cell"])
    nrm, valid, _ = lo.normals(g, lcfg)
    r, rq = handle(), handle()
    r.localize_set_map(prior)
    rq.localize_set_map(prior)
    r.relocalize_set_places(np.stack([ro.pack(d) for d in places]), poses)
    n_acc = 0
    for qi, (scan, _, truth) in enumerate(queries):
        got, _ = check_against_restatement(r, rq, scan, places, poses, g, nrm, valid, cfg, f"kidnapped {qi}")
        n_acc += got.accepted
        if got.accepted:
            e = lvo.relative_error(got.result.T, truth)
            assert e[0] < ACCURACY_BOUND[0] and e[1] < ACCURACY_BOUND[1], (qi, e)
    assert n_acc >= 0.9 * len(queries)
    scan = queries[0][0]
    rq.loop_enable()
    rq.loop_add(scan)
    assert same_bits(rq.loop_descriptors()[0], ro.pack(sco.descriptor(scan, cfg)))     # the descriptor loop_add gives


@pytest.mark.gpu
def test_gpu_aliasing_is_ambiguous_bit_for_bit_with_the_restatement():
    cfg, lcfg = ro.config(), lo.config()
    places, poses, prior, scan, _ = aliasing_case()
    g = lo.grid(prior, lcfg["cell"])
    nrm, valid, _ = lo.normals(g, lcfg)
    r, rq = handle(), handle()
    r.localize_set_map(prior)
    rq.localize_set_map(prior)
    r.relocalize_set_places(np.stack([ro.pack(d) for d in places]), poses)
    got, want = check_against_restatement(r, rq, scan, places, poses, g, nrm, valid, cfg, "aliasing")
    assert got.ambiguous and not got.accepted and want["ambiguous"]
    with pytest.raises(Exception):
        r.localize(scan)                                                # rejected: still no prediction memory


@pytest.mark.gpu
def test_gpu_places_from_the_loop_database_are_the_downloaded_places():
    from test_loop_closure import cast, make_world, route
    from test_loop_verify import pose4
    world = make_world()
    P = [pose4(p) for p in route()]
    scans = [cast(world, *route()[k], seed=k) for k in range(0, 30, 3)]
    prior = np.vstack([apply4(P[3 * i], s) for i, s in enumerate(scans)])
    r = handle()
    r.loop_enable()
    for s in scans:
        r.loop_add(s)
    r.localize_set_map(prior)
    poses = [P[3 * i] for i in range(len(scans))]
    r.relocalize_set_places_loop(poses)
    a = r.relocalize(scans[4])
    ha = r.relocalize_hypotheses()
    d = r.loop_descriptors()
    assert d.shape[0] == len(scans) and all(same_bits(d[i], r.loop_descriptors(i, 1)[0]) for i in range(len(scans)))
    r.relocalize_set_places(d, poses)
    b = r.relocalize(scans[4])
    hb = r.relocalize_hypotheses()
    assert (a.winner, a.accepted, a.place, a.shift) == (b.winner, b.accepted, b.place, b.shift)
    assert same_bits(a.result.T, b.result.T) and len(ha) == len(hb)
    for x, y in zip(ha, hb):
        assert x[:3] == y[:3] and same_bits(x[3].T, y[3].T)


@pytest.mark.gpu
def test_gpu_accepted_relocalization_feeds_the_prediction_and_a_rejected_one_does_not():
    from test_loop_closure import cast, make_world, route
    from test_loop_verify import pose4
    world = make_world()
    P = [pose4(p) for p in route()]
    frames = range(0, 40, 4)
    scans = {k: cast(world, *route()[k], seed=k) for k in frames}
    prior = np.vstack([apply4(P[k], scans[k]) for k in frames])
    cfg = ro.config()
    places = np.stack([ro.pack(sco.descriptor(scans[k], cfg)) for k in frames])
    r = handle()
    r.localize_set_map(prior)
    r.relocalize_set_places(places, [P[k] for k in frames])
    bad = r.relocalize(scans[8] + np.array([0.0, 0.0, 50.0]))        # the map's places, but 50 m above the map
    assert not bad.accepted
    with pytest.raises(Exception):
        r.localize(scans[8])                                            # still no previous localization: NOT_READY
    got = r.relocalize(scans[8])
    assert got.accepted
    nxt = r.localize(scans[8])
    assert same_bits(nxt.guess, lo.predict(got.result.T, np.eye(4), np.eye(4)))


@pytest.mark.gpu
def test_gpu_chained_flow_relocalizes_the_first_frame_and_moves_nothing_else():
    """process_raw_scan_packed -> (submap_init_frame | scan_match_predicted_async -> submap_update_frame_chained ->
    global_map_append_frame) -> loop_add_frame, against the merged map and the loop places of a first session over the same
    scans: frame 0 is relocalized instead of given a guess, every later frame localized from the prediction.  A rejected
    relocalization leaves localize_frame(None) NOT_READY; after the accepted one its guess is lo.predict(T_reloc, O_0, O_1)
    bit for bit.  The odometry, sources, submap, global map, registered scan, loop database and the launch counts of
    those calls are those of a handle without relocalization, with it enabled and loaded but unused, and with it running."""
    import tloam_b200
    from tloam_b200 import _lib
    from test_deskew import loop_scans
    from test_loop_closure import assert_same_odometry, process_packed
    scans = loop_scans()
    runs = {}
    prior = places = None
    for mode in ("off", "enabled", "running"):
        r = tloam_b200.LocalRegistration(fitness_thres=0.3)
        r.enable_global_map(voxel=0.5)
        r.loop_enable(exclude_recent=2)
        if mode != "off":
            r.localize_enable()
            r.localize_set_map(prior)
            r.relocalize_enable()
            r.relocalize_set_places(*places)
        poses, sources, launches, results, loops = [], [], [], [], []
        for k, a in enumerate(scans):
            n0 = r.launch_count()
            process_packed(r, a)
            if k == 0:
                r.submap_init_frame()
            else:
                r.scan_matching_predicted_async()
                r.submap_update_frame_chained()
                r.global_map_append_frame()
            r.loop_add_frame()
            launches.append(r.launch_count() - n0)
            loops.append(r.loop_result())
            if mode == "running":
                if k == 0:
                    res = _lib.LocalizeResult()
                    bad = r.relocalize(np.random.default_rng(0).uniform(-30.0, 30.0, (5000, 3)) + np.array([0.0, 0.0, 50.0]))
                    assert not bad.accepted
                    assert r._L.tloam_b200_localize_frame(r._h, None, C.byref(res)) == _lib.ERR_NOT_READY
                    results.append(r.relocalize_frame())
                else:
                    results.append(r.localize_frame(None))
            if k:
                poses.append(r.get_result())
            sources.append([r.source_cloud(c) for c in range(4)])
        runs[mode] = dict(poses=poses, sources=sources, submap=[r.submap_cloud(c) for c in range(4)], map=r.global_map(),
                          frames=r.global_map_frames(), reg=r.registered_scan(), launches=launches, loc=results, loop=loops,
                          desc=r.loop_descriptors())
        if mode == "off":
            prior, _ = r.global_map_merged(0.5)
            places = (r.loop_descriptors(), [np.eye(4)] + poses)
        r.close()
    off = runs["off"]
    for mode in ("enabled", "running"):
        assert_same_odometry(off, runs[mode])
        assert runs[mode]["launches"] == off["launches"], mode
        assert runs[mode]["loop"] == off["loop"] and same_bits(runs[mode]["desc"], off["desc"]), mode
    O = [np.eye(4)] + runs["running"]["poses"]
    res = runs["running"]["loc"]
    rel = res[0]
    assert rel.accepted and rel.n_hypotheses >= 1, rel
    assert same_bits(rel.result.T_map_odom, lo.map_odom(rel.result.T, O[0]))
    assert same_bits(res[1].guess, lo.predict(rel.result.T, O[0], O[1]))
    for k in range(2, len(res)):
        prev = res[k - 1]
        assert same_bits(res[k].guess, lo.predict(prev.T if prev.accepted else prev.guess, O[k - 1], O[k])), k
    print("chained: relocalized at place %d (distance %.4f), then %s" %
          (rel.place, rel.distance, ", ".join(f"{x.termination}/{x.fitness:.4f}" for x in res[1:])))


@pytest.mark.gpu
def test_gpu_relocalize_shim_matches_the_python_mirror():
    import struct
    import tloam_b200
    from test_cpp_shim import build_driver
    exe = build_driver("relocalize_driver", "front_end_b200.hpp")
    places, poses, prior, queries = kidnapped_queries()
    D = np.stack([ro.pack(d) for d in places])
    scans = [queries[1][0], queries[4][0], queries[1][0] + np.array([0.0, 0.0, 50.0])]
    d = os.path.dirname(exe)
    with open(os.path.join(d, "reloc_map.bin"), "wb") as fh:
        fh.write(struct.pack("Q", len(prior)) + np.ascontiguousarray(prior).tobytes())
    with open(os.path.join(d, "reloc_places.bin"), "wb") as fh:
        fh.write(struct.pack("QQ", *D.shape) + D.tobytes() + np.stack([P.ravel(order="F") for P in poses]).tobytes())
    with open(os.path.join(d, "reloc_scans.bin"), "wb") as fh:
        fh.write(struct.pack("Q", len(scans)))
        for p in scans:
            fh.write(struct.pack("Q", len(p)) + np.ascontiguousarray(p).tobytes())
    res = subprocess.run([exe] + [os.path.join(d, f) for f in ("reloc_map.bin", "reloc_places.bin", "reloc_scans.bin")],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    got = [l.split() for l in res.stdout.strip().split("\n")]
    r = handle()
    r.localize_set_map(prior)
    r.relocalize_set_places(D, poses)
    assert len(got) == len(scans)
    for k, p in enumerate(scans):
        x = r.relocalize(p)
        g = got[k]
        assert [int(v) for v in g[:6]] == [x.n_hypotheses, x.winner, x.place, x.shift, int(x.ambiguous), int(x.accepted)], k
        assert float(g[6]) == x.result.fitness
        assert np.array_equal(np.array([float(v) for v in g[7:23]]), x.result.T.ravel(order="F")), k
        want = r.localize(p).guess.ravel(order="F") if x.accepted else np.zeros(16)
        assert np.array_equal(np.array([float(v) for v in g[23:39]]), want), k
    assert sum(int(g[5]) for g in got) == 2
    r.close()


@pytest.mark.gpu
def test_gpu_status_codes():
    import tloam_b200
    from tloam_b200 import _lib
    r = tloam_b200.LocalRegistration()
    L, h = r._L, r._h
    cfg = _lib.RelocalizeConfig()
    L.tloam_b200_relocalize_default_config(C.byref(cfg))
    res = _lib.RelocalizeResult()
    assert L.tloam_b200_relocalize_enable(h, C.byref(cfg)) == _lib.ERR_NOT_READY                 # localization off
    r.localize_enable()
    bad = _lib.RelocalizeConfig()
    L.tloam_b200_relocalize_default_config(C.byref(bad))
    bad.top_k = 0
    assert L.tloam_b200_relocalize_enable(h, C.byref(bad)) == _lib.ERR_INVALID_ARG
    assert L.tloam_b200_relocalize(h, None, 0, C.byref(res)) == _lib.ERR_NOT_READY                 # relocalization off
    r.relocalize_enable()
    assert L.tloam_b200_relocalize(h, None, 0, C.byref(res)) == _lib.ERR_NOT_READY                 # no map, no places
    assert L.tloam_b200_relocalize_frame(h, C.byref(res)) == _lib.ERR_NOT_READY                     # no scan
    from test_loop_verify import structured_cloud
    M = structured_cloud(3)
    r.localize_set_map(M)
    assert L.tloam_b200_relocalize(h, None, 0, C.byref(res)) == _lib.ERR_NOT_READY                 # no places
    slot = 20 * 60 + 20 + 60
    d = np.zeros((1, slot))
    d[0, 5] = np.nan
    eye = np.eye(4).ravel(order="F").copy()
    dp = C.POINTER(C.c_double)
    assert L.tloam_b200_relocalize_set_places(h, d.ctypes.data_as(dp), eye.ctypes.data_as(dp), 1) == _lib.ERR_INVALID_ARG
    shear = np.eye(4)
    shear[0, 1] = 0.5
    s = shear.ravel(order="F").copy()
    d[0, 5] = 0.0
    assert L.tloam_b200_relocalize_set_places(h, d.ctypes.data_as(dp), s.ctypes.data_as(dp), 1) == _lib.ERR_BAD_POSE
    assert L.tloam_b200_relocalize_set_places_loop(h, eye.ctypes.data_as(dp), 1) == _lib.ERR_NOT_READY   # loop closure off
    r.relocalize_set_places(d, [np.eye(4)])                              # an empty place: distance 1 everywhere
    got = r.relocalize(M)
    assert (got.n_hypotheses, got.place, got.winner, got.accepted) == (0, -1, -1, False)
    r.close()
