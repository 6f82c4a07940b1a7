"""The correspondence search is exact (DESIGN section 3: cell edge = the cloud's radius, so the 27 cells around a query hold
every point with d2 < r2; results ordered by (d2, original index)).  These tests pin that claim where a grid search can
break -- cell faces, distance ties, path thresholds, hash wrap-around and key aliasing, odd sizes -- against the
brute-force restatement in search_edges_oracle.py, for every device path: tloam_b200_knn (knn_search), the lane-pair
search of build_factors (knn_search_pair), the dense staged search, the two-level search and the batched frame kernels.

CPU tests check the restatement itself (the fma chain, exactness on dyadic scenes), that the CPU oracle's KD-tree and
brute force equal it on every scene (which is what makes the build_factors comparisons below valid) and the coverage
of each scene.  GPU tests compare the device bit for bit."""
import os
from fractions import Fraction

import numpy as np
import pytest

import search_edges_oracle as so

BIG = 10 ** 9
CAPS = dict(edge_maxnum=BIG, sphere_maxnum=BIG, planar_maxnum=BIG, ground_maxnum=BIG)

_MAKERS = {}
for _r in so.RADII:
    _MAKERS[f"faces_r{_r}"] = (lambda r: lambda: so.scene_faces(r, seed=1))(_r)
    _MAKERS[f"corners_r{_r}"] = (lambda r: lambda: so.scene_corners(r, seed=2))(_r)
_MAKERS.update({
    "dyadic_faces_r0.5": lambda: so.scene_dyadic_faces(0.5, seed=3),
    "ties_r0.5": lambda: so.scene_ties(0.5, seed=4),
    "ties_r0.3": lambda: so.scene_ties(0.3, seed=5),
    "thresholds_r0.5": lambda: so.scene_thresholds(0.5, seed=6),
    "hash_r0.5": lambda: so.scene_hash(0.5, seed=7),
    "hash_r1.1": lambda: so.scene_hash(1.1, seed=8, n=1021),
    "sizes_r0.3": lambda: so.scene_sizes(0.3, seed=9),
})
NAMES = list(_MAKERS)
_CACHE = {}


def scene(name):
    if name not in _CACHE:
        _CACHE[name] = _MAKERS[name]()
    return _CACHE[name]


def below(r):
    return float(np.nextafter(r, 0.0))


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def fma_chain(dx, dy, dz):
    """fma(dz, dz, fma(dy, dy, dx * dx)), each fma rounded once (written out independently of the restatement)."""
    inner = float(Fraction(dy) ** 2 + Fraction(dx * dx))
    return float(Fraction(dz) ** 2 + Fraction(inner))


def assert_same_knn(name, got, ref, k, what):
    idx, d2, cnt = got
    ri, rd, rc = ref["idx"][:, :k], ref["d2"][:, :k], np.minimum(ref["n_within"], k)
    bad = np.nonzero((cnt != rc) | np.any(idx != ri, 1) | np.any(bits(d2) != bits(rd), 1))[0]
    assert bad.size == 0, (f"{name} {what}: {bad.size} queries differ, first {bad[:5]}: "
                           f"got {idx[bad[0]]} {d2[bad[0]]} {cnt[bad[0]]}, want {ri[bad[0]]} {rd[bad[0]]} {rc[bad[0]]}")


# ------------------------------------------------------------------------------------------------------------------
# CPU: the restatement, the CPU oracle and the coverage
@pytest.mark.parametrize("name", NAMES)
def test_reference_d2_is_the_fma_chain(name):
    s = scene(name)
    ref = s.reference()
    m = s.map_rel.astype(np.float64)
    rng = np.random.default_rng(0)
    qs = rng.permutation(len(s.rx))[:2000]
    n = 0
    for i in qs:
        for j in range(int(ref["count"][i])):
            dd = m[ref["idx"][i, j]] - s.rx[i]
            d = ref["d2"][i, j]
            assert d == fma_chain(*dd), (name, i, j)
            e = so.d2_exact(m[ref["idx"][i, j]], s.rx[i])
            if s.dyadic:
                assert Fraction(d) == e, (name, i, j)                 # every subtraction and product is exact
            else:
                assert abs(Fraction(d) - e) <= 2 * Fraction(float(np.spacing(d))), (name, i, j)
            n += 1
    print(f"{name}: {n} neighbours recomputed{' (dyadic: d2 == exact distance^2)' if s.dyadic else ''}")
    assert n > 0


@pytest.mark.parametrize("name", NAMES)
def test_oracle_knn_equals_reference(oracle, name):
    """oracle.knn (KD-tree and brute force, world coordinates) == the device-frame restatement: idx, d2 bits, count."""
    s = scene(name)
    for radius in (s.cell, below(s.cell)):
        ref = s.reference(radius)
        for brute in (False, True):
            got = oracle.knn(s.map_world, s.queries, radius, so.KMAX, brute_force=brute)
            assert_same_knn(name, got, ref, so.KMAX, f"oracle.knn(brute_force={brute}, r={radius!r})")


@pytest.mark.parametrize("name", NAMES)
def test_reference_matches_scipy_away_from_the_radius(name):
    """Queries with no point within 1e-9 r2 of the radius must agree with plain geometry (scipy's ball query)."""
    from scipy.spatial import cKDTree
    s = scene(name)
    ref = s.reference()
    m = s.map_rel.astype(np.float64)
    r2 = s.cell * s.cell
    tree = cKDTree(m)
    wide = tree.query_ball_point(s.rx, s.cell * (1 + 1e-6))
    n = 0
    for i, c in enumerate(wide):
        c = np.asarray(c, dtype=np.int64)
        d = ((m[c] - s.rx[i]) ** 2).sum(1) if c.size else np.zeros(0)
        if np.any(np.abs(d - r2) <= 1e-9 * r2):
            continue
        inside = set(c[d < r2].tolist())
        got = ref["idx"][i, :ref["count"][i]].tolist()
        assert ref["count"][i] == min(len(inside), so.KMAX) and set(got) <= inside, (name, i)
        if len(inside) <= so.KMAX:
            assert set(got) == inside
        n += 1
    print(f"{name}: {n} of {len(s.rx)} queries away from the radius agree with scipy")
    assert n > 0


def test_scene_coverage():
    """Minimum counts of the edges each scene exists for: an edit that drops them fails here."""
    tot = {}
    for name in NAMES:
        s = scene(name)
        st = dict(s.reference()["stats"])
        st.update(so.grid_stats(s))
        tot[name] = st
        print(name, {k: v for k, v in sorted(st.items()) if v})
    need = {
        "corners_r0.5": dict(pairs_within_4ulp_of_r=500, neighbours_one_cell_away_on_3_axes=30, neighbours_with_d2_within_4ulp_of_r2=30,
                             tie_groups_cut_by_K=100, queries_on_a_cell_face=500, queries_on_a_cell_edge=100, queries_on_a_cell_corner=100),
        "dyadic_faces_r0.5": dict(pairs_within_4ulp_of_r=500, tie_groups_larger_than_K=100, queries_on_a_cell_corner=300),
        "ties_r0.5": dict(tie_groups_larger_than_K=10, tie_groups_across_cells=5, tie_groups_across_bricks=5,
                          tie_groups_across_lane_pair_z_layers=5),
        "ties_r0.3": dict(tie_groups_larger_than_K=10, tie_groups_across_cells=5, tie_groups_across_lane_pair_z_layers=5),
        "thresholds_r0.5": {"cells_with_15_points": 1, "cells_with_16_points": 1, "cells_with_17_points": 1, "cells_with_63_points": 1,
                            "cells_with_64_points": 1, "cells_with_65_points": 1, "queries_behind_a_kFineMin_cell": 3,
                            "neighbourhoods_of_kDenseCap-1": 1, "neighbourhoods_of_kDenseCap+0": 1, "neighbourhoods_of_kDenseCap+1": 1,
                            "lanes_with_kPairCells_cells": 1, "queries_with_no_neighbour": 1, "queries_with_fewer_than_K": 4},
        "hash_r0.5": dict(probe_sequences_wrapping_the_table=100, brick_lookups_aliasing_a_populated_brick=50),
        "hash_r1.1": dict(probe_sequences_wrapping_the_table=100, brick_lookups_aliasing_a_populated_brick=50),
    }
    for r in so.RADII:
        need[f"corners_r{r}"] = {**need.get(f"corners_r{r}", {}), "pairs_within_4ulp_of_r": 500, "neighbours_one_cell_away_on_3_axes": 30,
                                 "tie_groups_cut_by_K": 100, "queries_with_fewer_than_K": 100}
        need[f"faces_r{r}"] = dict(tie_groups_larger_than_K=100, queries_on_a_cell_face=200, lanes_with_kPairCells_cells=50)
    for name, mins in need.items():
        for k, v in mins.items():
            assert tot[name].get(k, 0) >= v, f"{name}: {k} = {tot[name].get(k, 0)} < {v}"
    # the aliased queries (2^21 bricks away) find nothing
    h = scene("hash_r0.5")
    assert np.all(h.reference()["count"][-64:] == 0)


# ------------------------------------------------------------------------------------------------------------------
# GPU
def make_reg(cell, path="pair", **cfg):
    import tloam_b200
    env = {"pair": {}, "dense": {"TLOAM_B200_DENSE": "1", "TLOAM_B200_FINE": "0", "TLOAM_B200_DENSE_CHECK": "1"},
           "fine": {"TLOAM_B200_DENSE": "0", "TLOAM_B200_FINE": "1", "TLOAM_B200_DENSE_CHECK": "1"}}[path]
    os.environ.update(env)
    try:
        return tloam_b200.LocalRegistration(edge_dist_thres=cell, sphere_dist_thres=cell, planar_dist_thres=cell,
                                            ground_dist_thres=cell, **cfg)
    finally:
        for k in env:
            os.environ.pop(k, None)


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_knn_abi_bit_identical(name):
    s = scene(name)
    r = make_reg(s.cell)
    r.set_input_target([s.map_world] * 4)
    assert np.array_equal(r.map_origin(), s.origin)
    try:
        for radius in (s.cell, below(s.cell)):
            ref = s.reference(radius)
            for cloud in range(4):
                for k in (1, 3, 5):
                    assert_same_knn(name, r.knn(cloud, s.queries, radius, k), ref, k, f"cloud {cloud} k {k} r {radius!r}")
            if name.startswith("sizes"):
                for nq in (1, 127, 128, 129):
                    sub = dict(idx=ref["idx"][:nq], d2=ref["d2"][:nq], n_within=ref["n_within"][:nq])
                    assert_same_knn(name, r.knn(2, s.queries[:nq], radius, 5), sub, 5, f"{nq} queries")
        st = ref["stats"]
        print(f"{name}: {len(s.queries)} queries bit-identical; near-r pairs {st['pairs_within_4ulp_of_r']}, "
              f"3-axis neighbours {st['neighbours_one_cell_away_on_3_axes']}, ties cut by K {st['tie_groups_cut_by_K']}")
    finally:
        r.close()


def _eigenvalues(nb):
    return np.linalg.eigvalsh(np.cov(nb.T, bias=True)) if len(nb) >= 2 else np.zeros(3)


# The fits form the covariance from raw cumulants of world coordinates (|x| ~ 1e3 m here), whose cancellation leaves
# ~1e-9 m^2 of noise: neighbours within a few float32 ulps of one lattice point (the face scenes) are fitted to that
# noise, and the device and the oracle may then disagree without any search being wrong.
SPREAD_MIN = 1e-6


def _fit_is_geometric(nb, principal):
    """The fitted direction (largest eigenvector for a line, smallest for a plane) is determined by the geometry."""
    ev = _eigenvalues(nb)
    gap = ev[2] - ev[1] if principal else ev[1] - ev[0]
    return ev[2] > SPREAD_MIN and gap > 1e-3 * ev[2]


BF_NAMES = [n for n in NAMES if not n.startswith("hash")] + ["hash_r0.5"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["pair", "dense", "fine"])
@pytest.mark.parametrize("name", BF_NAMES)
def test_build_factors_at_identity(oracle, name, path):
    """build_factors(cloud, x = 0): se3_exp(0) is exactly I, so the queries are the source points as given."""
    s = scene(name)
    src = [s.queries] * 4
    if name.startswith("sizes"):
        src = [s.queries[:0], s.queries[:1], s.queries[:129], s.queries]   # 0, 1, 129 and 4097 features
    r = make_reg(s.cell, path, **CAPS)
    r.set_input_target([s.map_world] * 4)
    r.set_input_source(src)
    o = oracle.Oracle(edge_dist_thres=s.cell, sphere_dist_thres=s.cell, planar_dist_thres=s.cell, ground_dist_thres=s.cell, **CAPS)
    o.set_input_target([s.map_world] * 4)
    o.set_input_source(src)
    x = np.zeros(6)
    ref = s.reference()
    n_cmp = n_fit_by_rounding = 0
    try:
        for cloud in range(4):
            v, p = r.build_factors(cloud, x)
            nq = len(src[cloud])
            if cloud == 1:       # sphere, K = 1: prim[0:3] is the nearest neighbour (valid when d2 <= 0.2)
                cnt, d0, i0 = ref["count"][:nq], ref["d2"][:nq, 0], ref["idx"][:nq, 0]
                want = (cnt >= 1) & (d0 <= 0.2)
                assert np.array_equal(v.astype(bool), want), f"{name} {path}: {np.sum(v.astype(bool) != want)} sphere validity flips"
                assert np.array_equal(bits(p[want, :3]), bits(s.map_world[i0[want]])), f"{name} {path}: sphere neighbour differs"
                continue
            vo, po = o.build_factors(cloud, x)
            # validity follows the neighbour count (edge: > 3, plane: 5) and then the fit; where the fit of the (same)
            # neighbours is decided by rounding, the device and the oracle may differ without any search being wrong
            cnt = ref["count"][:nq]
            decided = np.array([cnt[i] < (4 if cloud == 0 else 5) or _eigenvalues(s.map_world[ref["idx"][i, :cnt[i]]])[2] > SPREAD_MIN
                                for i in range(nq)], dtype=bool)
            flips = np.nonzero((v != vo) & decided)[0]
            assert flips.size == 0, f"{name} {path} cloud {cloud}: {flips.size} validity flips, first {flips[:5]}"
            n_fit_by_rounding += int((~decided).sum())
            for i in np.nonzero(v.astype(bool) & decided)[0]:
                nb = s.map_world[ref["idx"][i, :ref["count"][i]]]
                if not _fit_is_geometric(nb, cloud == 0):
                    continue
                if cloud == 0:
                    same, swapped = np.abs(p[i] - po[i]).max(), np.abs(p[i] - po[i, [3, 4, 5, 0, 1, 2]]).max()
                    assert min(same, swapped) < 1e-7, (name, path, cloud, i)
                else:
                    assert np.allclose(p[i], po[i], rtol=0, atol=1e-9), (name, path, cloud, i, p[i], po[i])
                n_cmp += 1
        if path != "pair":
            cnt = r.dense_check_counters()
            assert cnt[1] == 0, f"{name} {path}: {cnt[1]} of {cnt[0]} queries differ from knn_search on the device"
            assert cnt[0] > 0, f"{name} {path}: the {path} search did not run"
        st = ref["stats"]
        print(f"{name} {path}: validity equal on 4 clouds ({n_fit_by_rounding} factors fitted to ulp-sized neighbourhoods left out), {n_cmp} primitives compared; near-r pairs {st['pairs_within_4ulp_of_r']}, "
              f"3-axis neighbours {st['neighbours_one_cell_away_on_3_axes']}, ties cut by K {st['tie_groups_cut_by_K']}")
    finally:
        r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("pair", [("corners_r0.5", "ties_r0.5"), ("thresholds_r0.5", "corners_r0.5")])
def test_batched_scan_match_bit_identical(pair):
    """Two scenes through BatchRegistration (S = 2): every pose bit-identical to the single-handle scan_match."""
    import tloam_b200
    sc = [scene(n) for n in pair]
    cfg = dict(edge_dist_thres=0.5, sphere_dist_thres=0.5, planar_dist_thres=0.5, ground_dist_thres=0.5)
    srcs = [[s.queries[:3000]] * 4 for s in sc]
    singles = []
    for s, src in zip(sc, srcs):
        r = tloam_b200.LocalRegistration(**cfg)
        r.set_input_target([s.map_world] * 4)
        r.set_input_source(src)
        singles.append(r.scan_matching(np.eye(4)))
        r.close()
    b = tloam_b200.BatchRegistration(2, **cfg)
    try:
        b.set_input_target(b.pack_host([[s.map_world] * 4 for s in sc]))
        b.set_input_source(b.pack_host(srcs))
        T, st = b.scan_matching(np.stack([np.eye(4)] * 2))
        assert np.all(st == 0), st
        for i in range(2):
            assert np.array_equal(T[i], singles[i]), (pair[i], T[i] - singles[i])
        print(f"{pair}: batched poses bit-identical to the single handle")
    finally:
        b.close()
