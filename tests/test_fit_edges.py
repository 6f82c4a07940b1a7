"""The registration's primitive fits (fit_neighbours: sphere / edge / plane decisions and primitives) and its SE(3) maps
against the exact / 50-digit restatement in fit_edges_oracle.py, at degenerate neighbourhoods, decision thresholds and
branch edges.

Every feature of the crafted scenes owns a cluster of map points; clusters sit further apart than the cloud's search
radius, so the k neighbours of each feature are known in advance.  The map is origin + float32 with origin 0 (two far
sentinels in the edge cloud centre its bounding box), and the threshold families run at x = 0, where se3_exp(0) = I and
T p = p exactly.  Outside each decision's error band the exact verdict is the contract; inside it, agreement with the CPU
oracle (oracle.Oracle.build_factors).  The tests print the in-band counts and the worst errors seen."""
from fractions import Fraction

import mpmath as mp
import numpy as np
import pytest

import fit_edges_oracle as fo
from test_gpu_parity import bbox_origin, quantize_map

BIG = 10 ** 9
CAPS = dict(edge_maxnum=BIG, sphere_maxnum=BIG, planar_maxnum=BIG, ground_maxnum=BIG)
RADIUS = (1.0, 0.5, 0.5, 0.5)             # default edge / sphere / planar / ground search radius
SPACING = 4.0                             # sites are further apart than twice the largest radius plus a cluster
SENTINEL = 3.0e4
POSE_X = np.array([3.0, -2.0, 0.5, 0.1, -0.2, 0.3])


def f32(a):
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


class Sites:
    """Lattice sites near the origin (4 m apart, |x|, |y| < 40 m) and far families at a given distance along x."""

    def __init__(self):
        self.i = 0

    def next(self, far=0.0):
        i = self.i
        self.i += 1
        # integer coordinates 4 j + 2: none is 0, so a neighbour's difference to its query is exact on every axis
        c = SPACING * np.array([i % 18 - 9, (i // 18) % 18 - 9, i // 324 - 4], dtype=np.float64) + 2.0
        if far:
            c[0] += far
        return c


# ----------------------------------------------------------------------------------------------------------------------
# FP64 screening (numpy, vectorised) used only to choose near-threshold candidates; the verdicts come from fit_edges_oracle
def _edge_margins(P):
    m = P.mean(1, keepdims=True)
    D = P - m
    C = np.einsum("nki,nkj->nij", D, D) / P.shape[1]
    w, V = np.linalg.eigh(C)
    return w[:, 2] - 3 * w[:, 1], np.abs(V[:, 2, 2]) - fo.EDGE_DIR_THRES, w


def _plane_margin(P):
    m = P.mean(1, keepdims=True)
    D = P - m
    C = np.einsum("nki,nkj->nij", D, D) / P.shape[1]
    xx, xy, xz, yy, yz, zz = C[:, 0, 0], C[:, 0, 1], C[:, 0, 2], C[:, 1, 1], C[:, 1, 2], C[:, 2, 2]
    w = np.zeros((len(P), 3))
    for det, ax in ((yy * zz - yz * yz, (yy * zz - yz * yz, xz * yz - xy * zz, xy * yz - xz * yy)),
                    (xx * zz - xz * xz, (xz * yz - xy * zz, xx * zz - xz * xz, xy * xz - yz * xx)),
                    (xx * yy - xy * xy, (xy * yz - xz * yy, xy * xz - yz * xx, xx * yy - xy * xy))):
        a = np.stack(ax, 1)
        wgt = det * det * np.where((w * a).sum(1) < 0, -1.0, 1.0)
        w = w + a * wgt[:, None]
    n = w / np.linalg.norm(w, axis=1, keepdims=True)
    dist = np.einsum("nki,ni->nk", D, n)
    return dist.max(1) - fo.PLANE_THRES


def _rot(axis, ang):
    axis = np.asarray(axis, float) / np.linalg.norm(axis)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * K @ K


def _pick(cands, margins, target):
    j = int(np.argmin(np.abs(margins - target)))
    return cands[j]


def _tune(rng, make, margin, p0, width, target, n=3000, jitter=2e-6):
    """A coarse sweep of one scalar parameter finds the threshold crossing; then many candidates at that parameter, each
    moved by a random sub-micrometre jitter before the float32 rounding, sample the quantisation until one candidate's
    margin lands near `target`."""
    ps = p0 + np.linspace(-width, width, n)
    mg = margin(f32(make(ps)))
    best = ps[int(np.argmin(np.abs(mg - target)))]
    base = make(np.full(8 * n, best))
    P = f32(base + rng.normal(0, jitter, base.shape))
    return P[int(np.argmin(np.abs(margin(P) - target)))]


# ----------------------------------------------------------------------------------------------------------------------
# scene
class Case:
    __slots__ = ("cloud", "family", "q", "nb", "ref", "pose")

    def __init__(self, cloud, family, q, nb, pose=False):
        self.cloud, self.family, self.q, self.nb, self.pose = cloud, family, np.asarray(q, float), nb, pose
        self.ref = None


def _edge_cases(rng, S):
    out = []
    L = np.array([-2, -1, 0, 1, 2], float) * 0.12

    def line(c, d, perp):
        e1 = np.cross(d, [0.3, 0.5, 0.1]); e1 /= np.linalg.norm(e1)
        e2 = np.cross(d, e1)
        return c + L[:, None] * d + perp[:, :1] * e1 + perp[:, 1:] * e2

    # |dir.z| = 0.85 +- delta and l2 / l1 = 3 +- delta, chosen among quantised candidates by FP64 screening
    deltas = [s * 10.0 ** -e for e in range(3, 11) for s in (1, -1)]
    for target in deltas:
        for rep in range(6):
            c = S.next()
            psi = rng.uniform(0, 2 * np.pi)
            perp = rng.normal(0, 0.01, (5, 2))
            d0 = np.array([np.sin(0.55) * np.cos(psi), np.sin(0.55) * np.sin(psi), np.cos(0.55)])
            e1 = np.cross(d0, [0.3, 0.5, 0.1]); e1 /= np.linalg.norm(e1)
            e2 = np.cross(d0, e1)

            def make(phi, c=c, psi=psi, perp=perp, e1=e1, e2=e2):
                d = np.stack([np.sin(phi) * np.cos(psi), np.sin(phi) * np.sin(psi), np.cos(phi)], 1)
                return c + L[None, :, None] * d[:, None, :] + perp[None, :, :1] * e1 + perp[None, :, 1:] * e2
            P = _tune(rng, make, lambda P: _edge_margins(P)[1], np.arccos(fo.EDGE_DIR_THRES + target), 1e-3, target)
            out.append(Case(0, "edge_dir", c, list(map(tuple, P))))
    for target in deltas:
        for rep in range(6):
            c = S.next()
            R = _rot(rng.normal(size=3), rng.uniform(0, 0.2))
            d = R @ np.array([0.0, 0.0, 1.0])
            e1 = np.cross(d, [0.3, 0.5, 0.1]); e1 /= np.linalg.norm(e1)
            e2 = np.cross(d, e1)
            base = rng.normal(0, 1, (5, 2))
            base -= base.mean(0)
            s0 = np.sqrt(np.var(L) / (3 * np.var(base[:, 0])))

            def make(sc, c=c, d=d, e1=e1, e2=e2, base=base):
                sc = sc[:, None, None]
                return c + L[None, :, None] * d + base[None, :, :1] * sc * e1 + base[None, :, 1:] * 0.2 * sc * e2

            def rel(P):
                mr, _, w = _edge_margins(P)
                return mr / w[:, 2]
            P = _tune(rng, make, rel, s0, 0.2 * s0, target)
            out.append(Case(0, "edge_ratio", c, list(map(tuple, P))))
    a = 1.0 / 16
    for rep in range(24):
        c = S.next()
        out.append(Case(0, "edge_ratio_exactly_3", c, [tuple(c + a * np.array(p)) for p in ((1, 0, 1), (-1, 0, 1), (0, 0, 0), (0, 0, -2))]))
        e, h = a, a * (1.25 + 0.25 * (rep % 4))            # h^2 > 1.5 e^2: kept; ties l0 = l1 below l2
        out.append(Case(0, "edge_tie_l0_l1", S.next(), None))
        out[-1].nb = [tuple(out[-1].q + p) for p in ((e, 0, h), (-e, 0, h), (0, e, -h), (0, -e, -h))]
        out.append(Case(0, "edge_tie_l1_l2", S.next(), None))
        out[-1].nb = [tuple(out[-1].q + p) for p in ((h, 0, e), (-h, 0, e), (0, h, -e), (0, -h, -e))]
        c = S.next()
        # coincident: dyadic coordinates make every raw cumulant exact, so the covariance is exactly 0 on the device too
        # and 0 > 3 * 0 decides; the last few use float32 coordinates whose cumulants round (then the oracle decides)
        off = [0.125, -0.25, 0.375 + rep * 0.0625] if rep < 20 else [0.1, -0.2, 0.3 + rep * 0.01]
        out.append(Case(0, "edge_coincident", c, [tuple(f32(c + off))] * 5))
        c = S.next()
        p = tuple(f32(c + [0.1, 0.05, -0.1]))
        out.append(Case(0, "edge_four_coincident_plus_one", c, [p] * 4 + [tuple(f32(c + [0.1, 0.05, 0.2 + 0.01 * rep]))]))
        for k in range(5):
            c = S.next()
            out.append(Case(0, f"edge_{k}_neighbours", c, [tuple(f32(c + [0.01 * j, 0.02, 0.1 * j - 0.2])) for j in range(k)]))
    # covariances a few Jacobi sweeps from diagonal: clustered spectra, small and generic rotations
    for rep in range(400):
        c = S.next()
        lam = [(1.0, 1.001, 12.0), (1.0, 2.0, 30.0), (0.2, 1.0, 1.02), (1.0, 1.0 + 1e-6, 20.0)][rep % 4]
        ang = [1e-3, 1e-2, 0.3, 1.0][(rep // 4) % 4]
        R = _rot(rng.normal(size=3), ang)
        Z = rng.normal(size=(5, 3))
        Z -= Z.mean(0)
        U_, s_, Vt = np.linalg.svd(Z, full_matrices=False)
        Z = U_ @ Vt * np.sqrt(5)                                   # identity covariance
        P = f32(c + (Z * np.sqrt(np.array(lam)) * 0.03) @ R.T)
        out.append(Case(0, "edge_jacobi", c, list(map(tuple, P)), pose=True))
    # far from the origin: the raw cumulants cancel
    for far in (1e2, 1e3, 1e4):
        for rep in range(64):
            c = S.next(far)
            phi = rng.uniform(0, 0.7) if rep % 2 == 0 else rng.uniform(0.7, 1.4)
            d = np.array([np.sin(phi), 0, np.cos(phi)])
            P = f32(line(c, d, rng.normal(0, 0.01, (5, 2))))
            out.append(Case(0, f"edge_far_{far:g}", c, list(map(tuple, P)), pose=True))
    return out


def _plane_cases(rng, S, cloud):
    out = []
    name = "planar" if cloud == 2 else "ground"
    grid = np.array([[0, 0], [1, 0], [0, 1], [-1, 0], [0, -1]], float) * 0.125
    for rep in range(12):
        for ax in range(3):                                            # normal along x, y, z: two dets vanish
            c = S.next()
            P = np.insert(grid * (1 + rep % 3), ax, 0.0, axis=1) + c
            out.append(Case(cloud, f"{name}_axis_{'xyz'[ax]}", c, list(map(tuple, f32(P)))))
        for n in ((1, 0, 1), (1, 0, -1), (1, 1, 0), (1, -1, 0), (0, 1, 1), (0, 1, -1), (1, 1, 1), (1, -1, 1)):
            c = S.next()                                               # 45 degree planes: the dot < 0 sign flip
            n = np.array(n, float)
            e1 = np.cross(n, [1.0, 0, 0] if abs(n[0]) < 0.9 else [0, 1.0, 0])
            e1 /= np.abs(e1).max()
            e2 = np.cross(n, e1)
            e2 /= np.abs(e2).max()
            P = c + grid[:, :1] * e1 + grid[:, 1:] * e2 * (1 + rep % 2)
            out.append(Case(cloud, f"{name}_diagonal", c, list(map(tuple, f32(P)))))
        for d in ((1, 0, 0), (0, 0, 1), (1, 1, 0), (1, 2, 3)):
            c = S.next()                                               # collinear (symmetric, dyadic): the zero plane
            P = c + np.outer(np.arange(-2, 3) * 0.03125 * (1 + rep % 2), d)
            out.append(Case(cloud, f"{name}_collinear", c, list(map(tuple, f32(P)))))
        c = S.next()
        out.append(Case(cloud, f"{name}_coincident", c, [tuple(f32(c + [0.1, 0.2, -0.1]))] * 5))
        for k in (3, 4):
            c = S.next()
            out.append(Case(cloud, f"{name}_{k}_neighbours", c, [tuple(f32(c + [0.05 * j, 0.01, -0.05 * j])) for j in range(k)]))
    # one neighbour at a signed distance 0.2 +- delta from the fitted plane, above (rejects) and below (one-sided: kept)
    for side in (1, -1):
        for target in [0.0] + [s * 10.0 ** -e for e in range(3, 11) for s in (1, -1)]:
            for rep in range(2):
                c = S.next()
                R = _rot(rng.normal(size=3), rng.uniform(0, 0.5))
                base = np.array([[0.15, 0.15, 0], [-0.15, 0.15, 0], [0.15, -0.15, 0], [-0.15, -0.15, 0], [0, 0, 0]], float)
                base[0, 2] = rng.normal(0, 1e-3)
                q = c + R @ np.array([0.0, 0.0, 0.1 * side])

                def make(h, c=c, R=R, base=base):
                    P = np.repeat(base[None], len(h), 0)
                    P[:, 4, 2] = h
                    return c + P @ R.T
                if side < 0:   # the one below never rejects (one-sided), however far below
                    P = f32(make(np.array([-0.32 - 0.01 * rep]))[0])
                    out.append(Case(cloud, f"{name}_below", q, list(map(tuple, P))))
                else:
                    P = _tune(rng, make, _plane_margin, 0.32, 0.03, target)
                    out.append(Case(cloud, f"{name}_at_0.2", q, list(map(tuple, P))))
    for far in (1e2, 1e3, 1e4):
        for rep in range(24):
            c = S.next(far)
            R = _rot(rng.normal(size=3), rng.uniform(0, np.pi))
            P = rng.uniform(-0.2, 0.2, (5, 3)) * [1, 1, 0.01 if rep % 2 == 0 else 0.4]
            out.append(Case(cloud, f"{name}_far_{far:g}", c, list(map(tuple, f32(c + P @ R.T))), pose=True))
    for rep in range(650):
        c = S.next()
        R = _rot(rng.normal(size=3), rng.uniform(0, np.pi))
        P = rng.uniform(-0.25, 0.25, (5, 3)) * [1, 1, rng.choice([0.0, 0.01, 0.3])]
        out.append(Case(cloud, f"{name}_generic", c, list(map(tuple, f32(c + P @ R.T))), pose=True))
    return out


def _sphere_d2_case(c, target):
    """Query q = c + (b, e, a) 2^-28 with the nearest neighbour at c and a^2 + b^2 + e^2 = target 2^56, b and e small:
    dx * dx and fma(dy, dy, .) stay far below 2^53 units and the last fma(dz, dz, .) rounds an exactly representable
    value, so every step of the device's d2 is exact and the exact squared distance IS `target`."""
    from math import isqrt
    M = Fraction(target) * 2 ** 56
    assert M.denominator == 1
    M = M.numerator
    a = isqrt(M)
    while a > 0:
        r = M - a * a
        for b in range(isqrt(r) + 1):
            e = isqrt(r - b * b)
            if e * e == r - b * b:
                return c + np.array([b, e, a], dtype=np.float64) * 2.0 ** -28
        a -= 1
    raise AssertionError("no exact d2 construction")


def _sphere_cases(rng, S):
    out = []
    ulp = np.spacing(0.2)
    for k in (0, 1, 2, 2 ** 20):
        for s in ((1, -1) if k else (1,)):
            for rep in range(6):
                c = S.next()
                q = _sphere_d2_case(c, 0.2 + s * k * ulp)
                out.append(Case(1, f"sphere_d2_0.2{'+-'[s < 0]}{k}ulp", q, [tuple(c)]))
    for rep in range(40):
        c = S.next()
        out.append(Case(1, "sphere_at_radius", c + [0.5, 0, 0], [tuple(c)]))        # d2 == r^2: not found
        out.append(Case(1, "sphere_no_neighbour", S.next(), []))
    for rep in range(840):
        c = S.next()
        d = rng.normal(size=3)
        d *= rng.choice([0.2, 0.4, 0.46]) / np.linalg.norm(d)
        out.append(Case(1, "sphere_generic", c + d, [tuple(c)], pose=True))
    for far in (1e2, 1e3, 1e4):
        for rep in range(16):
            c = S.next(far)
            d = rng.normal(size=3)
            d *= rng.choice([0.3, 0.47]) / np.linalg.norm(d)
            out.append(Case(1, f"sphere_far_{far:g}", c + d, [tuple(f32(c))], pose=True))
    return out


def _reference(case):
    if case.cloud == 1:
        nb = case.nb[0] if case.nb and sum((case.q[i] - case.nb[0][i]) ** 2 for i in range(3)) < 0.25 else None
        if nb is not None and fo.sphere_exact(case.q, nb)["d2"] >= Fraction(0.25):
            nb = None
        return fo.sphere_exact(case.q, nb)
    if case.cloud == 0:
        return fo.edge_exact(case.nb)
    return fo.plane_exact(case.nb)


class Scene:
    def __init__(self, seed=2026):
        rng = np.random.default_rng(seed)
        S = Sites()
        self.cases = [[], [], [], []]
        for c in _edge_cases(rng, S):
            self.cases[0].append(c)
        for c in _sphere_cases(rng, S):
            self.cases[1].append(c)
        for cl in (2, 3):
            for c in _plane_cases(rng, S, cl):
                self.cases[cl].append(c)
        mp_ = []
        for cl in range(4):
            pts = [p for c in self.cases[cl] for p in c.nb]
            if cl == 0:
                pts += [(-SENTINEL,) * 3, (SENTINEL,) * 3]
            mp_.append(np.asarray(pts, dtype=np.float64).reshape(-1, 3))
        self.origin = bbox_origin(mp_)
        self.map = quantize_map(mp_, self.origin)
        for cl in range(4):
            assert np.array_equal(self.map[cl], mp_[cl]), "map points must be origin + float32 exactly"
            for c in self.cases[cl]:
                c.ref = _reference(c)
        self.T = fo.quat_rot(fo.so3_exp_quat([fo.mpf(fo.fr(t)) for t in POSE_X[3:]]))

    def source(self, cl, pose=False):
        qs = np.array([c.q for c in self.cases[cl] if (c.pose or not pose)]).reshape(-1, 3)
        if not pose:
            return qs
        from tloam_b200 import synth
        T = synth.se3_exp(POSE_X)
        return (qs - T[:3, 3]) @ T[:3, :3]                  # T^-1 q: the device's T p lands within 1e-13 of q

    def pose_cases(self, cl):
        return [c for c in self.cases[cl] if c.pose]


_SCENE = None


def scene():
    global _SCENE
    if _SCENE is None:
        _SCENE = Scene()
    return _SCENE


def families(cases):
    out = {}
    for c in cases:
        out.setdefault(c.family, []).append(c)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# CPU: the restatement itself
def test_edge_restatement_matches_numpy_eigh():
    rng = np.random.default_rng(1)
    for _ in range(60):
        P = f32(rng.normal(0, 0.2, (5, 3)) * rng.uniform(0.1, 2, 3) + rng.uniform(-50, 50, 3))
        r = fo.edge_exact(list(map(tuple, P)))
        D = P - P.mean(0)
        w, V = np.linalg.eigh(D.T @ D / 5)
        assert np.allclose([float(t) for t in r["ev"]], w, rtol=1e-9, atol=1e-13)
        v = np.array([float(t) for t in r["v"]])
        if w[2] - w[1] > 1e-3 * w[2]:
            assert min(np.abs(v - V[:, 2]).max(), np.abs(v + V[:, 2]).max()) < 1e-9


def test_plane_restatement_matches_svd_on_coplanar_points():
    rng = np.random.default_rng(2)
    for _ in range(60):
        n = rng.normal(size=3)
        n /= np.linalg.norm(n)
        e1 = np.cross(n, rng.normal(size=3)); e1 /= np.linalg.norm(e1)
        e2 = np.cross(n, e1)
        ab = rng.uniform(-0.3, 0.3, (5, 2))
        c = rng.uniform(-20, 20, 3)
        P = c + ab[:, :1] * e1 + ab[:, 1:] * e2          # coplanar in FP64 to 1e-15; the restatement sees these doubles
        r = fo.plane_exact(list(map(tuple, P)))
        svd_n = np.linalg.svd(P - P.mean(0))[2][2]
        assert min(np.abs(r["n"] - svd_n).max(), np.abs(r["n"] + svd_n).max()) < 1e-9
        assert max(abs(float(t)) for t in r["dist"]) < 1e-12 and r["verdict"]


def test_restatement_documented_degenerate_behaviour():
    c = np.array([5.0, -7.0, 9.0])
    line = [tuple(c + t * np.array([1.0, 2.0, 3.0]) * 0.03125) for t in range(-2, 3)]
    r = fo.plane_exact(line)
    assert r["zero"] and r["B_n"] == 0.0 and np.all(r["n"] == 0) and r["d"] == 0 and r["verdict"] and r["decided"]
    r = fo.plane_exact([tuple(c)] * 5)
    assert r["zero"] and r["verdict"]
    assert not fo.plane_exact(line[:4])["verdict"] and fo.plane_exact(line[:4])["decided"]           # k <= 4
    for k in range(4):
        r = fo.edge_exact(line[:k])
        assert not r["verdict"] and r["decided"]                                                       # k <= 3
    a = 1.0 / 16
    r = fo.edge_exact([tuple(c + a * np.array(p)) for p in ((1, 0, 1), (-1, 0, 1), (0, 0, 0), (0, 0, -2))])
    assert r["m_ratio"] == 0 and r["B_ratio"] == 0.0 and not r["verdict"] and r["decided"]         # l2 == 3 l1 exactly
    r = fo.edge_exact([tuple(c + [0.125, -0.25, 0.375])] * 5)                   # coincident, exact cumulants: 0 > 3 * 0
    assert r["m_ratio"] == 0 and r["B_ratio"] == 0.0 and not r["verdict"] and r["decided"]
    q = c + np.array([0.375, 0.25, 0.0])                                          # d2 = 0.203125, computed exactly
    assert fo.sphere_exact(q, tuple(c))["B"] == 0.0 and fo.sphere_exact(q, tuple(c))["decided"]
    r = fo.edge_exact(line)                                  # l0 = l1 = 0: the ratio passes, |v.z| = 3 / sqrt(14) fails
    assert r["m_ratio"] > 0 and abs(float(r["v"][2]) - 3 / np.sqrt(14)) < 1e-15 and not r["verdict"] and r["decided"]
    assert fo.sphere_exact(c, None)["verdict"] is False


def test_se3_restatement_round_trips():
    rng = np.random.default_rng(3)
    for _ in range(20):
        ax = rng.normal(size=3)
        a = np.concatenate([rng.normal(0, 5, 3), ax / np.linalg.norm(ax) * rng.uniform(0, 3)])
        q, R, t = fo.se3_exp(a)
        T = np.eye(4)
        T[:3, :3] = np.array(R.tolist(), dtype=float)
        T[:3, 3] = np.array(t.T.tolist()[0], dtype=float)
        xi, th, w, _ = fo.se3_log(T)
        assert np.allclose([float(v) for v in xi], a, atol=1e-12)
        from scipy.spatial.transform import Rotation
        assert np.allclose(Rotation.from_rotvec(a[3:]).as_matrix(), T[:3, :3], atol=1e-14)


def _count_band(cases):
    return sum(1 for c in cases if not c.ref["decided"])


def test_scene_coverage():
    """The families exist, the in-band share stays small, and the edges are reached (margins near each threshold)."""
    s = scene()
    tot = sum(len(c) for c in s.cases)
    band = sum(_count_band(c) for c in s.cases)
    for cl in range(4):
        fam = families(s.cases[cl])
        print(f"cloud {cl}: {len(s.cases[cl])} features, " +
              ", ".join(f"{k} {len(v)} (band {_count_band(v)})" for k, v in sorted(fam.items())))
    e = s.cases[0]
    dirm = sorted(abs(float(c.ref["m_dir"])) for c in e if c.family == "edge_dir")
    ratm = sorted(abs(float(c.ref["m_ratio"] / c.ref["ev"][2])) for c in e if c.family == "edge_ratio")
    pm = sorted(abs(float(c.ref["margin"])) for cl in (2, 3) for c in s.cases[cl] if c.family.endswith("at_0.2"))
    print(f"{tot} features, {band} in band; closest |dir.z| - 0.85: {dirm[:3]}, closest ratio margin / l2: {ratm[:3]}, "
          f"closest plane distance - 0.2: {pm[:3]}")
    assert all(len(cl) >= 1000 for cl in s.cases) and band <= 12
    assert all(_count_band(v) <= 6 for cl in s.cases for v in families(cl).values())
    # the exact ties are decided by the exact reference: B = 0 and a margin of exactly 0
    ties = [c for c in e if c.family in ("edge_ratio_exactly_3", "edge_coincident")]
    ties += [c for c in s.cases[1] if c.family.startswith("sphere_d2_0.2") and "1048576" not in c.family]
    assert len(ties) >= 70 and sum(1 for c in ties if c.ref["decided"] and c.ref.get("B", c.ref.get("B_ratio")) == 0.0) >= 70
    assert sum(1 for c in s.cases[1] if c.family == "sphere_d2_0.2+0ulp" and c.ref["margin"] == 0 and c.ref["verdict"]) == 6
    assert dirm[0] < 1e-8 and ratm[0] < 1e-8 and pm[0] < 1e-8
    assert sum(1 for c in e if c.ref.get("m_ratio") == 0) >= 24
    assert sum(1 for cl in (2, 3) for c in s.cases[cl] if c.ref.get("zero")) >= 60
    # both sign-flip branches of fitBestPlane are taken by the 45 degree planes
    dots = [d for cl in (2, 3) for c in s.cases[cl] if c.family.endswith("diagonal") for d in c.ref["dots"][1:]]
    assert sum(1 for d in dots if d < 0) >= 20 and sum(1 for d in dots if d > 0) >= 20


def _oracle_run(oracle, s, x, pose):
    o = oracle.Oracle(**CAPS)
    o.set_input_target(s.map)
    o.set_input_source([s.source(cl, pose) for cl in range(4)])
    return [o.build_factors(cl, x) for cl in range(4)]


def _check(cases, v, p, vo, what):
    """valid == exact verdict outside the band and == oracle inside it; primitives within their bounds."""
    bad, band, worst = [], 0, {}
    for i, c in enumerate(cases):
        r = c.ref
        if r["decided"]:
            if bool(v[i]) != r["verdict"]:
                bad.append((c.family, i, int(v[i]), r["verdict"]))
        else:
            band += 1
            if v[i] != vo[i]:
                bad.append((c.family, i, int(v[i]), "oracle", int(vo[i])))
        if not v[i]:
            continue
        assert np.all(np.isfinite(p[i])), (what, c.family, i, p[i])
        if not r["verdict"]:
            continue
        if c.cloud == 0 and r["decided"]:
            e = min(max(np.abs(p[i, :3] - r["a"]).max(), np.abs(p[i, 3:] - r["b"]).max()),
                    max(np.abs(p[i, :3] - r["b"]).max(), np.abs(p[i, 3:] - r["a"]).max()))
            assert e <= r["B_end"], (what, c.family, i, e, r["B_end"], p[i], r["a"], r["b"])
            worst[c.family] = max(worst.get(c.family, 0.0), e)
        elif c.cloud >= 2 and r["decided"]:
            en = np.abs(p[i, :3] - r["n"]).max()
            ed = abs(p[i, 3] - r["d"])
            assert en <= r["B_n"] and ed <= r["B_d"], (what, c.family, i, en, r["B_n"], ed, r["B_d"], p[i], r["n"], r["d"])
            worst[c.family] = max(worst.get(c.family, 0.0), en)
        elif c.cloud == 1:
            assert np.array_equal(p[i, :3], np.asarray(c.nb[0])), (what, i)
    return bad, band, worst


@pytest.mark.parametrize("pose", [False, True])
def test_oracle_matches_restatement_outside_the_band(oracle, pose):
    s = scene()
    x = POSE_X if pose else np.zeros(6)
    res = _oracle_run(oracle, s, x, pose)
    for cl in range(4):
        cases = s.pose_cases(cl) if pose else s.cases[cl]
        vo, po = res[cl]
        bad, band, worst = _check(cases, vo, po, vo, f"oracle cloud {cl}")
        print(f"oracle cloud {cl} pose={pose}: {len(cases)} features, {band} in band, worst prim error by family {worst}")
        assert not bad, f"cloud {cl}: {len(bad)} verdicts differ from the exact restatement, first {bad[:5]}"


def _cap_scene():
    """Sphere features whose only observable difference is the `counted` flag (sphere_sum++ of the reference): a
    neighbour at d2 == r^2 exactly is not found (counted), one an ulp-scale step inside the radius is found and rejected by
    d2 > 0.2 (not counted), no neighbour at all is counted.  Ten valid features follow; with sphere_maxnum = CAP_COUNTED
    + 4 only the first four survive if and only if exactly the at-radius and empty ones were counted."""
    S = Sites()
    cases = []
    for kind in ("at_radius", "inside_radius", "no_neighbour", "valid"):
        for rep in range(10 if kind == "valid" else 6):
            c = S.next()
            if kind == "no_neighbour":
                cases.append(Case(1, kind, c, []))
                continue
            dx = {"at_radius": 0.5, "inside_radius": 0.5 - 2.0 ** -28, "valid": 0.375}[kind]
            cases.append(Case(1, kind, c + [dx, 0, 0], [tuple(c)]))
    for c in cases:
        c.ref = _reference(c)
    pts = [p for c in cases for p in c.nb]
    far = np.array([[-SENTINEL] * 3, [SENTINEL] * 3])
    return cases, [far, np.asarray(pts, float), far, far]


CAP = 12 + 4


def _cap_expected(cases, cap):
    """The reference's capped loop (registration.cpp:531-551): a candidate stops the loop once the counter reaches the
    cap; every candidate and every feature without a neighbour advances the counter."""
    out, counter = [], 0
    for c in cases:
        found = "d2" in c.ref
        cand = c.ref["verdict"]
        if cand and counter >= cap:
            return out + [0] * (len(cases) - len(out))
        out.append(int(cand))
        counter += int(cand or not found)
    return out


def _cap_run(z, cases, mp_):
    z.set_input_target(mp_)
    z.set_input_source([np.zeros((0, 3)), np.array([c.q for c in cases]), np.zeros((0, 3)), np.zeros((0, 3))])
    return z.build_factors(1, np.zeros(6))[0]


def test_sphere_counted_flag_through_the_cap_oracle(oracle):
    cases, mp_ = _cap_scene()
    want = _cap_expected(cases, CAP)
    assert sum(want) == 4 and all(c.ref["decided"] for c in cases)
    assert [("d2" in c.ref) for c in cases[:12]] == [False] * 6 + [True] * 6     # d2 == r^2 is outside the search
    v = _cap_run(oracle.Oracle(sphere_maxnum=CAP), cases, mp_)
    assert list(v) == want, (list(v), want)


@pytest.mark.gpu
def test_sphere_counted_flag_through_the_cap():
    import tloam_b200
    cases, mp_ = _cap_scene()
    want = _cap_expected(cases, CAP)
    r = tloam_b200.LocalRegistration(sphere_maxnum=CAP)
    try:
        v = _cap_run(r, cases, mp_)
        assert list(v) == want, (list(v), want)
        print(f"sphere cap {CAP}: {int(v.sum())} of 10 valid features kept after 6 at-radius, 6 inside-radius, 6 empty")
    finally:
        r.close()


# ----------------------------------------------------------------------------------------------------------------------
# GPU: tloam_b200_build_factors
@pytest.mark.gpu
@pytest.mark.parametrize("pose", [False, True])
def test_build_factors_at_fit_edges(oracle, pose):
    import tloam_b200
    s = scene()
    x = POSE_X if pose else np.zeros(6)
    r = tloam_b200.LocalRegistration(**CAPS)
    try:
        r.set_input_target(s.map)
        assert np.array_equal(r.map_origin(), s.origin)
        r.set_input_source([s.source(cl, pose) for cl in range(4)])
        res_o = _oracle_run(oracle, s, x, pose)
        fails = []
        for cl in range(4):
            cases = s.pose_cases(cl) if pose else s.cases[cl]
            v, p = r.build_factors(cl, x)
            vo, _ = res_o[cl]
            bad, band, worst = _check(cases, v, p, vo, f"device cloud {cl}")
            fam = families(cases)
            print(f"device cloud {cl} pose={pose}: {len(cases)} features, {int(v.sum())} valid, {band} in band "
                  f"({', '.join(f'{k} {_count_band(vv)}' for k, vv in sorted(fam.items()) if _count_band(vv))}); "
                  f"worst prim error by family {worst}")
            fails += [(cl,) + b for b in bad]
        assert not fails, f"{len(fails)} verdicts differ, first {fails[:8]}"
    finally:
        r.close()


# ----------------------------------------------------------------------------------------------------------------------
# GPU: the SE(3) maps through the k_se3 kernel
def _mp_to_np(x):
    return np.array([float(t) for t in x])


@pytest.fixture(scope="module")
def reg():
    import tloam_b200
    r = tloam_b200.LocalRegistration()
    yield r
    r.close()


@pytest.mark.gpu
def test_se3_exp_at_the_taylor_switch(reg):
    rng = np.random.default_rng(11)
    worst = [0.0, 0.0]
    n = 0
    for k in list(range(1, 53, 4)) + [None]:
        for base in (1e-10, 1e-9, 1e-7, 1e-5):
            if k is None and base != 1e-10:
                continue
            for sgn in (1, -1):
                th = base * (1 + sgn * 2.0 ** -k) if k is not None else (base if sgn > 0 else 0.0)
                ax = rng.normal(size=3)
                ax /= np.linalg.norm(ax)
                a = np.concatenate([rng.normal(0, 20, 3), ax * th])
                T = reg.se3_exp(a)
                q, R, t = fo.se3_exp(a)
                BR, Bt = fo.exp_bounds(a)
                eR = np.abs(T[:3, :3] - np.array(R.tolist(), dtype=float)).max()
                et = np.abs(T[:3, 3] - _mp_to_np(t)).max()
                assert eR <= BR and et <= Bt, (k, base, sgn, th, eR, BR, et, Bt)
                worst = [max(worst[0], eR / BR), max(worst[1], et / Bt)]
                n += 1
    print(f"se3_exp: {n} samples around theta = 1e-10; worst error / bound: rotation {worst[0]:.3g}, translation {worst[1]:.3g}")


def _rt(R, t):
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def _axis_angle(axis, ang):
    axis = [fo.mpf(fo.fr(t)) for t in axis]
    nrm = mp.sqrt(sum(t * t for t in axis))
    om = [t / nrm * ang for t in axis]
    R = fo.quat_rot(fo.so3_exp_quat(om))
    return np.array([[float(R[i, j]) for j in range(3)] for i in range(3)])


def _check_log(reg, T, what, stats):
    xi, th, w, br = fo.se3_log(T)
    Bw, Bu = fo.log_bounds(xi, th, w, float(np.linalg.norm(T[:3, 3])))
    got = reg.se3_log(T)
    ew = np.abs(got[3:] - _mp_to_np(xi[3:])).max()
    eu = np.abs(got[:3] - _mp_to_np(xi[:3])).max()
    assert ew <= Bw and eu <= Bu, (what, br, float(th), float(w), got, _mp_to_np(xi), ew, Bw, eu, Bu)
    stats["n"] += 1
    stats["branch"][br] = stats["branch"].get(br, 0) + 1
    stats["worst"] = max(stats["worst"], ew / Bw, eu / Bu)
    stats["w0"] += int(w == 0)
    stats["wneg"] += int(w < 0)


@pytest.mark.gpu
def test_se3_log_near_pi_and_quaternion_branches(reg):
    rng = np.random.default_rng(12)
    stats = dict(n=0, branch={}, worst=0.0, w0=0, wneg=0)
    axes = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, -1, 0), (0, 1, 1), (0, 1, -1), (1, 0, 1), (1, 0, -1),
            (1, 1, 1), (1, -1, 1), (-1, 1, 1)] + [tuple(rng.normal(size=3)) for _ in range(6)]
    for ax in axes:
        for eps in (1e-3, 1e-6, 1e-9, 0.0):
            for sgn in (1, -1):
                ang = sgn * (mp.pi - eps)
                R = _axis_angle(ax, ang)
                if eps == 0.0:
                    R = 0.5 * (R + R.T)                       # a rotation by pi is symmetric: qw comes out as +0
                _check_log(reg, _rt(R, rng.normal(0, 10, 3)), (ax, eps, sgn), stats)
    # exact diagonal ties: rotations by pi / 2 and pi about axes whose matrices repeat diagonal entries
    for ax, ang in (((1, 1, 0), mp.pi), ((1, -1, 0), mp.pi), ((0, 1, -1), mp.pi), ((1, 0, -1), mp.pi), ((1, 1, 1), mp.pi),
                    ((1, 0, 0), mp.pi / 2), ((0, 1, 0), mp.pi / 2), ((0, 0, 1), -mp.pi / 2), ((1, 1, 1), 2 * mp.pi / 3)):
        R = _axis_angle(ax, ang)
        R[np.abs(R) < 1e-15] = 0.0
        R = np.round(R * 2 ** 40) / 2 ** 40 if ang in (mp.pi / 2, -mp.pi / 2) else R
        if ang == mp.pi:
            R = 0.5 * (R + R.T)
        _check_log(reg, _rt(R, [1.0, -2.0, 3.0]), (ax, float(ang)), stats)
    # generic rotations on each branch of the quaternion extraction, with w < 0 from the non-trace branches
    for _ in range(40):
        ax = rng.normal(size=3)
        _check_log(reg, _rt(_axis_angle(ax, mp.mpf(rng.uniform(1.6, 3.1))), rng.normal(0, 30, 3)), "generic", stats)
    print(f"se3_log: {stats['n']} matrices within bounds, branches {stats['branch']}, w == 0: {stats['w0']}, "
          f"w < 0: {stats['wneg']}, worst error / bound {stats['worst']:.3g}")
    assert all(stats["branch"].get(b, 0) >= 5 for b in (-1, 0, 1, 2)) and stats["w0"] >= 10 and stats["wneg"] >= 10


@pytest.mark.gpu
def test_se3_log_diagonal_tie_picks_the_first_index(reg):
    """A rotation by pi about (1, -1, 0): diagonal (0, 0, -1), a tie between entries 0 and 1.  Eigen's strict `>` keeps
    i = 0, so v = (+, -, 0) and, w being +0, Sophus returns -pi * v / |v|."""
    R = np.array([[0.0, -1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, -1.0]])
    got = reg.se3_log(_rt(R, [0.0, 0.0, 0.0]))
    want = -np.pi * np.array([1.0, -1.0, 0.0]) / np.sqrt(2.0)
    assert np.allclose(got[3:], want, atol=1e-15), (got, want)


@pytest.mark.gpu
def test_se3_plus_with_negative_w(reg):
    rng = np.random.default_rng(13)
    n = wneg = 0
    worst = 0.0
    for _ in range(40):
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        x = np.concatenate([rng.normal(0, 10, 3), ax * rng.uniform(3.3, 6.0)])      # |omega| > pi: w = cos(theta / 2) < 0
        d = np.concatenate([rng.normal(0, 0.5, 3), rng.normal(0, 0.1, 3) * rng.choice([0.0, 1e-11, 1.0])])
        xi, th, w = fo.se3_plus(x, d)
        B = fo.plus_bound(x, d, th, w)
        got = reg.se3_plus(x, d)
        e = np.abs(got - _mp_to_np(xi)).max()
        assert e <= B, (x, d, got, _mp_to_np(xi), e, B)
        worst = max(worst, e / B)
        n += 1
        wneg += int(w < 0)
    print(f"se3_plus: {n} samples within bounds ({wneg} with w < 0), worst error / bound {worst:.3g}")
    assert wneg >= 20


@pytest.mark.gpu
def test_pose_orthogonality_tolerance(reg):
    import tloam_b200
    rng = np.random.default_rng(14)
    n_ok = n_bad = 0
    for _ in range(6):
        R0 = _axis_angle(rng.normal(size=3), mp.mpf(rng.uniform(0.1, 3.0)))
        for rel in (-1e-3, -1e-5, 1e-5, 1e-3):
            target = 1e-9 * (1 + rel)
            # scale row 0 by (1 + e): (R R^T)_00 = (1 + e)^2 |r0|^2, the largest deviation from I
            e = np.sqrt(1 + target) - 1
            R = R0.copy()
            R[0] *= 1 + e
            err = fo.ortho_error(R)
            margin = Fraction(1e-9) - err
            assert abs(float(margin)) > 64 * fo.U, "construction too close to the tolerance"
            T = _rt(R, [1.0, 2.0, 3.0])
            if margin > 0:
                reg.se3_log(T)
                n_ok += 1
            else:
                with pytest.raises(tloam_b200.RegistrationError) as ei:
                    reg.se3_log(T)
                assert ei.value.status == 3
                n_bad += 1
    R = np.diag([1.0, 1.0, -1.0])                                      # a reflection is not a pose
    with pytest.raises(tloam_b200.RegistrationError):
        reg.se3_log(_rt(R, [0, 0, 0]))
    print(f"orthogonality: {n_ok} accepted just below 1e-9, {n_bad} refused just above")
    assert n_ok >= 10 and n_bad >= 10
