"""Brute-force restatement of the device's radius-truncated kNN (map_grid.cuh knn_search / knn_search_pair, the dense
and two-level paths) and seeded scenes that put map points and queries where a grid search can go wrong.

The restatement works on the map AS THE DEVICE STORES IT: float32 coordinates relative to the map origin (integer-rounded
centre of the bounding box of the first non-empty cloud), the query taken as rx = fl(q - origin).  d2 is the device's
operation sequence fma(ddz, ddz, fma(ddy, ddy, ddx * ddx)) with dd = (double)m - rx, every fma rounded once (exact
Fraction arithmetic, then one correctly rounded conversion); a neighbour is kept when d2 < fl(r * r); results are
ordered by (d2, original index), truncated to K and padded with -1 / +inf.

Every scene also carries coverage counts (pairs whose EXACT distance lies within 4 ulps of r, pairs one cell apart on
all three axes, tie groups cut by the truncation, cells at the path thresholds, probe sequences that wrap ...) so that
the tests can assert that the edges are really there.
"""
from collections import Counter
from fractions import Fraction

import numpy as np
from scipy.spatial import cKDTree

# thresholds of the device search paths (map_grid.cuh, dense_search.cuh)
K_MERGE_MAX = 16
K_PAIR_CELLS = 18
K_FINE_MIN = 64
K_DENSE_CAP = 9216
KMAX = 5
M64 = (1 << 64) - 1
# world frame of the scenes: the origin is an integer (the origin rule), the scenes span negative and positive cells
# around it, and every world query stays in the origin's binade so that q - origin is exact -- the CPU oracle works in
# world coordinates and then sees the same differences as the device
ORIGIN = np.array([1234.0, -568.0, 40.0])


# ---------------------------------------------------------------------------------------------------------------------
# device arithmetic
def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def d2_device(dd):
    """dd: the three (already rounded) differences (double)m - rx."""
    return fma(dd[2], dd[2], fma(dd[1], dd[1], dd[0] * dd[0]))


def d2_exact(m, rx):
    """Unrounded squared distance between a stored map point and the query (both exact in the world frame)."""
    return sum((Fraction(float(a)) - Fraction(float(b))) ** 2 for a, b in zip(m, rx))


def cell_key(bx, by, bz):
    ux, uy, uz = ((int(v) + (1 << 20)) & 0x1FFFFF for v in (bx, by, bz))
    return (1 << 63) | (ux << 42) | (uy << 21) | uz


def hash_key(k):
    k = (k * 0x9E3779B97F4A7C15) & M64
    k ^= k >> 32
    k = (k * 0xD6E8FEB86659FD93) & M64
    k ^= k >> 29
    return k & 0xFFFFFFFF


def table_size(n):
    p = 256
    while p < n + 1:
        p <<= 1
    return p


def cells_of(v, cell):
    return np.floor(np.asarray(v, dtype=np.float64) * (1.0 / cell)).astype(np.int64)


def bbox_origin(world):
    return np.rint(0.5 * (world.min(0) + world.max(0)))


# ---------------------------------------------------------------------------------------------------------------------
class Scene:
    """map_rel: (n,3) float32 in the device frame; queries: (nq,3) float64 world; cell: the grid's cell edge (= radius)."""

    def __init__(self, name, cell, map_rel, queries, origin=ORIGIN, dyadic=False):
        self.name, self.cell, self.dyadic = name, float(cell), dyadic
        self.map_rel = np.ascontiguousarray(map_rel, dtype=np.float32).reshape(-1, 3)
        self.origin = np.asarray(origin, dtype=np.float64)
        self.map_world = self.origin + self.map_rel.astype(np.float64)
        assert np.array_equal((self.map_world - self.origin).astype(np.float32), self.map_rel), name
        if len(self.map_rel):
            assert np.array_equal(bbox_origin(self.map_world), self.origin), (name, bbox_origin(self.map_world))
        self.queries = np.ascontiguousarray(queries, dtype=np.float64).reshape(-1, 3)
        self.rx = self.queries - self.origin
        o = np.broadcast_to(self.origin, self.queries.shape).ravel().tolist()
        assert all(Fraction(q) - Fraction(oo) == Fraction(r)
                   for q, oo, r in zip(self.queries.ravel().tolist(), o, self.rx.ravel().tolist())), f"{name}: q - origin inexact"
        self._ref = {}

    def reference(self, radius=None):
        radius = self.cell if radius is None else float(radius)
        if radius not in self._ref:
            self._ref[radius] = search(self, radius)
        return self._ref[radius]

    def __repr__(self):
        return f"Scene({self.name}, cell={self.cell}, n={len(self.map_rel)}, nq={len(self.queries)})"


def search(scene, radius, K=KMAX):
    """Brute-force SearchHybrid of every query (see the module docstring).  Returns dict(idx, d2, count, n_within,
    stats) -- idx / d2 / count as tloam_b200_knn returns them for K; prefixes give K = 1 and 3."""
    m = scene.map_rel.astype(np.float64)
    rx = scene.rx
    nq = len(rx)
    r2 = radius * radius
    idx = np.full((nq, K), -1, dtype=np.int32)
    d2 = np.full((nq, K), np.inf)
    n_within = np.zeros(nq, dtype=np.int64)
    st = Counter()
    if len(m) == 0 or nq == 0:
        return dict(idx=idx, d2=d2, count=np.zeros(nq, dtype=np.int32), n_within=n_within, stats=st)
    lists = cKDTree(m).query_ball_point(rx, radius * (1 + 1e-9) + 1e-300)
    lo, hi = r2 * (1 - 1e-12), r2 * (1 + 1e-12)
    inv = 1.0 / scene.cell
    mc = np.floor(m * inv)
    qc = np.floor(rx * inv)
    ulp = np.spacing(radius)
    r_lo2, r_hi2 = (Fraction(radius) - 4 * Fraction(ulp)) ** 2, (Fraction(radius) + 4 * Fraction(ulp)) ** 2
    fr2 = Fraction(radius) ** 2
    for i in range(nq):
        c = np.asarray(lists[i], dtype=np.int64)
        if c.size == 0:
            continue
        dd = m[c] - rx[i]                      # the device's rounded differences
        approx = (dd * dd).sum(1)
        keep = approx < hi
        c, dd, approx = c[keep], dd[keep], approx[keep]
        if c.size == 0:
            continue
        border = approx >= lo                  # decided only by the exact computation
        for j in np.nonzero(np.abs(approx - r2) <= 1e-9 * r2)[0]:
            e = d2_exact(m[c[j]], rx[i])
            if r_lo2 <= e <= r_hi2:
                st["pairs_within_4ulp_of_r"] += 1
            if (e < fr2) != (d2_device(dd[j]) < r2):
                st["pairs_decided_by_rounding"] += 1
        exact_in = [d2_device(dd[j]) < r2 for j in np.nonzero(border)[0]]
        n_within[i] = int((~border).sum()) + sum(exact_in)
        sel = np.ones(c.size, dtype=bool)
        if c.size > K:
            sel = approx <= np.partition(approx, K - 1)[K - 1] * (1 + 1e-12)
        cand = sorted((d, int(ci)) for d, ci in ((d2_device(dd[j]), c[j]) for j in np.nonzero(sel)[0]) if d < r2)
        top = cand[:K]
        for j, (d, ci) in enumerate(top):
            idx[i, j], d2[i, j] = ci, d
        if len(cand) > K and cand[K][0] == cand[K - 1][0]:
            st["tie_groups_cut_by_K"] += 1
        groups = Counter(d for d, _ in cand)
        for d in (d for d, n in groups.items() if n > 1):
            cs = mc[[ci for dd_, ci in cand if dd_ == d]].astype(np.int64)
            if len({tuple(v) for v in cs}) > 1:
                st["tie_groups_across_cells"] += 1
            if len({tuple(v) for v in cs >> 1}) > 1:
                st["tie_groups_across_bricks"] += 1
            if len(set((cs[:, 2] >> 1).tolist())) > 1:
                st["tie_groups_across_lane_pair_z_layers"] += 1
        if groups and max(groups.values()) > 1:
            st["queries_with_tied_neighbours"] += 1
        if groups and max(groups.values()) > K:
            st["tie_groups_larger_than_K"] += 1
        for d, ci in top:
            if np.all(np.abs(mc[ci] - qc[i]) == 1):
                st["neighbours_one_cell_away_on_3_axes"] += 1
            if r2 - d <= 4 * np.spacing(r2):
                st["neighbours_with_d2_within_4ulp_of_r2"] += 1
    count = np.minimum(n_within, K).astype(np.int32)
    st["queries_with_no_neighbour"] = int((n_within == 0).sum())
    st["queries_with_fewer_than_K"] = int(((n_within > 0) & (n_within < K)).sum())
    on = (rx * inv == np.floor(rx * inv)).sum(1)
    st["queries_on_a_cell_face"] = int((on == 1).sum())
    st["queries_on_a_cell_edge"] = int((on == 2).sum())
    st["queries_on_a_cell_corner"] = int((on == 3).sum())
    return dict(idx=idx, d2=d2, count=count, n_within=n_within, stats=st)


def grid_stats(scene):
    """Occupancy of the device grid: cells at the path thresholds, neighbourhood totals, lane-pair list lengths, hash
    probe sequences that wrap around the end of the table, and queries whose brick keys alias a populated brick."""
    st = Counter()
    cell = scene.cell
    mc = cells_of(scene.map_rel.astype(np.float64), cell)
    occ = Counter(map(tuple, mc.tolist()))
    sizes = Counter(occ.values())
    for n in (8, 9, 15, 16, 17, 63, 64, 65):
        st[f"cells_with_{n}_points"] = sizes.get(n, 0)
    qc = cells_of(scene.rx, cell)
    offs = [(a, b, c) for c in (-1, 0, 1) for b in (-1, 0, 1) for a in (-1, 0, 1)]
    for q in map(tuple, qc.tolist()):
        tot = sum(occ.get((q[0] + a, q[1] + b, q[2] + c), 0) for a, b, c in offs)
        for d in (-1, 0, 1):
            if tot == K_DENSE_CAP + d:
                st[f"neighbourhoods_of_kDenseCap{d:+d}"] += 1
        bz0 = (q[2] - 1) >> 1
        for half in (0, 1):
            zs = [z for z in (2 * (bz0 + half), 2 * (bz0 + half) + 1) if abs(z - q[2]) <= 1]
            n = sum(1 for a in (-1, 0, 1) for b in (-1, 0, 1) for z in zs if occ.get((q[0] + a, q[1] + b, z), 0))
            if n == K_PAIR_CELLS:
                st["lanes_with_kPairCells_cells"] += 1
        # a kFineMin-sized sub-cell ahead of another dense sub-cell of the same brick (second-level table index)
        bx, by, bz = q[0] >> 1, q[1] >> 1, q[2] >> 1
        s_q = (q[0] & 1) | ((q[1] & 1) << 1) | ((q[2] & 1) << 2)
        cnt = [occ.get((2 * bx + (s & 1), 2 * by + ((s >> 1) & 1), 2 * bz + (s >> 2)), 0) for s in range(8)]
        if cnt[s_q] >= K_FINE_MIN and any(cnt[s] == K_FINE_MIN for s in range(s_q)):
            st["queries_behind_a_kFineMin_cell"] += 1
    # hash table: linear probing; the set of occupied slots does not depend on the insertion order, the table built
    # in input order stands for all of them
    bricks = list(dict.fromkeys(map(tuple, (mc >> 1).tolist())))
    tsize = table_size(len(scene.map_rel))
    mask = tsize - 1
    table = {}
    for b in bricks:
        k = cell_key(*b)
        s = hash_key(k) & mask
        while s in table:
            s = (s + 1) & mask
        table[s] = k
    st["bricks"] = len(bricks)
    st["table_slots"] = tsize
    keys = {cell_key(*b): b for b in bricks}
    for q in map(tuple, qc.tolist()):
        b0 = [(v - 1) >> 1 for v in q]
        for ib in range(8):
            b = (b0[0] + (ib & 1), b0[1] + ((ib >> 1) & 1), b0[2] + (ib >> 2))
            k = cell_key(*b)
            if k in keys and keys[k] != b:
                st["brick_lookups_aliasing_a_populated_brick"] += 1
            s = hash_key(k) & mask
            while s in table and table[s] != k:
                if s == mask:
                    st["probe_sequences_wrapping_the_table"] += 1
                s = (s + 1) & mask
    return st


# ---------------------------------------------------------------------------------------------------------------------
# scene generators (deterministic)
def _f32_steps(v, steps):
    """float32 neighbours of v; at 0 (whose float32 neighbours are subnormal and vanish next to a world coordinate of
    the origin's size) steps of 2^-40 instead."""
    v = np.float32(v)
    if v == 0:
        return [np.float32(s * 2.0 ** -40) for s in steps]
    out = []
    for s in steps:
        w = v
        for _ in range(abs(s)):
            w = np.nextafter(w, np.float32(np.inf if s > 0 else -np.inf), dtype=np.float32)
        out.append(w)
    return out


def _world(rel, origin=ORIGIN):
    return origin + np.asarray(rel, dtype=np.float64)


def _shuffle(rng, pts):
    return pts[rng.permutation(len(pts))]


def scene_faces(r, seed=0):
    """A. Cell faces: the lattice k r (k = -3..3 on every axis) and, along every axis, its float32 neighbours +-1 and
    +-2 ulps; queries on the lattice points (cell corners) and on cell faces and edges."""
    rng = np.random.default_rng(seed)
    ks = np.arange(-3, 4)
    base = np.array([np.float32(k * r) for k in ks], dtype=np.float32)
    g = np.stack(np.meshgrid(base, base, base, indexing="ij"), -1).reshape(-1, 3)
    pts = [g]
    for ax in range(3):
        for s in (-2, -1, 1, 2):
            p = g.copy()
            p[:, ax] = [_f32_steps(v, [s])[0] for v in p[:, ax]]
            pts.append(p)
    mp = _shuffle(rng, np.concatenate(pts))
    gq = g.astype(np.float64)
    half = np.float32(0.5 * r)
    faces = gq + np.array([0.0, half, half])[rng.permutation(3)]
    edges = gq + np.array([0.0, 0.0, half])[rng.permutation(3)]
    q = np.concatenate([gq, faces, edges, gq[rng.permutation(len(gq))[:200]] + rng.uniform(-r, r, (200, 3))])
    return Scene(f"faces_r{r}", r, mp, _world(q))


def _directions():
    d = []
    for v in ((1, 0, 0), (1, 1, 0), (1, 1, 1)):
        base = np.array(v, dtype=np.float64)
        for perm in {tuple(np.roll(base, s)) for s in range(3)} | {tuple(base[[0, 2, 1]])}:
            for sg in np.array(np.meshgrid([-1, 1], [-1, 1], [-1, 1])).T.reshape(-1, 3):
                w = np.array(perm) * sg
                if not any(np.array_equal(w, x) for x in d):
                    d.append(w)
    return [w / np.linalg.norm(w) for w in d]          # 6 axis, 12 face-diagonal, 8 body-diagonal


def scene_corners(r, seed=0, n_centres=9):
    """A. Neighbours at distance ~r: isolated clusters (a lattice corner k r and its float32 neighbours +-1, +-2 ulps
    along each axis, clusters 3 cells apart) and queries displaced from the corner by r (1 - 2^-j), j = 20..52, by
    exactly r and by nextafter(r), along the 26 axis / face-diagonal / body-diagonal directions -- the query sits one
    cell away from the neighbour on one, two or three axes and the exact distance crosses r.  The origin is 0 here: world
    coordinates of the size of ORIGIN would round the displacements to 2^-42 and no distance could land within a few
    ulps of a non-dyadic r."""
    rng = np.random.default_rng(seed)
    ks = np.array([-3, 0, 3])
    cen = np.stack(np.meshgrid(ks, ks, ks, indexing="ij"), -1).reshape(-1, 3)
    cen = cen[rng.permutation(len(cen))[:n_centres]]
    pts = []
    for k in cen:
        c = np.array([np.float32(v * r) for v in k], dtype=np.float32)
        pts.append(c)
        for ax in range(3):
            for s in (-2, -1, 1, 2):
                p = c.copy()
                p[ax] = _f32_steps(p[ax], [s])[0]
                pts.append(p)
    pts += [np.full(3, np.float32(-5 * r)), np.full(3, np.float32(5 * r))]          # bbox: origin 0
    mp = _shuffle(rng, np.array(pts, dtype=np.float32))
    mags = [r * (1.0 - 2.0 ** -j) for j in range(20, 53)] + [r, float(np.nextafter(r, np.inf))]
    q = []
    for k in cen:
        c = np.array([np.float32(v * r) for v in k], dtype=np.float64)
        for u in _directions():
            for a in mags:
                q.append(c + a * u)
    return Scene(f"corners_r{r}", r, mp, np.array(q), origin=np.zeros(3))


def scene_ties(r, seed=0):
    """B. Ties, dyadic (2^-20 grid, integer origin: every subtraction and every d2 is exact): shells of +-a on the axes
    (6), the face diagonals (12), the body diagonals (8) and the 30 points of d2 = 9 u^2 ((3,0,0) and (2,2,1) with signs
    and permutations); one point duplicated 1..40 times; groups centred on cell faces, brick faces and the z face that
    splits the two lanes of a pair; the input order shuffled."""
    rng = np.random.default_rng(seed)
    u = 2.0 ** -5 if r >= 0.3 else 2.0 ** -6
    shells = []
    for v in ((1, 0, 0), (1, 1, 0), (1, 1, 1)):
        shells.append(np.unique(np.array([np.roll(np.array(v) * s, k) for k in range(3)
                                          for s in np.array(np.meshgrid([-1, 1], [-1, 1], [-1, 1])).T.reshape(-1, 3)]), axis=0))
    s9 = [np.roll(np.array(v) * s, k) for v in ((3, 0, 0), (2, 2, 1), (2, 1, 2), (1, 2, 2)) for k in range(3)
          for s in np.array(np.meshgrid([-1, 1], [-1, 1], [-1, 1])).T.reshape(-1, 3)]
    shells.append(np.unique(np.array(s9), axis=0))
    assert [len(s) for s in shells] == [6, 12, 8, 30]

    def grid(v):                                   # the 2^-20 grid
        return np.round(np.asarray(v, dtype=np.float64) * 2 ** 20) / 2 ** 20

    cell_i = lambda x: grid(x * r)                  # noqa: E731  (on the face only when r is dyadic)
    centres = []
    spots = [(-5, -5, -5), (-5, 4, 3), (2, -3, 6), (5, 5, -6), (-3, 0, 1), (0, 6, -3), (6, -6, 0), (-6, 2, 5)]
    for i, (cx, cy, cz) in enumerate(spots):
        # cell face in x (odd cell index: inside a brick), brick face in y (even index), lane split in z (even index)
        base = np.array([cell_i(cx if cx % 2 else cx + 1), cell_i(cy if cy % 2 == 0 else cy + 1), cell_i(cz if cz % 2 == 0 else cz + 1)])
        centres.append(base + grid(u / 2 * np.array([1, -1, 1]) * (i % 3 == 0)))
    pts, q = [], []
    for i, c in enumerate(centres):
        for sh in shells:
            pts.append(grid(c + (i + 1) * u / 4 * sh) if i % 2 else grid(c + u * sh))
        dup = [1, 2, 5, 6, 7, 17, 40, 3][i]
        pts.append(np.repeat(grid(c + np.array([0, 0, r / 2]))[None], dup, 0))
        q.append(c)
        q.append(grid(c + np.array([0, 0, r / 2])))
    mp = _shuffle(rng, np.concatenate([np.atleast_2d(p) for p in pts]))
    return Scene(f"ties_r{r}", r, mp.astype(np.float32), _world(np.array(q)), dyadic=True)


def scene_dyadic_faces(r=0.5, seed=0):
    """A on the 2^-20 grid: the lattice and its neighbours 2^-20 apart, queries on faces, edges and corners and at
    dyadic offsets up to r; every d2 is exact, so the reference must equal the real distance."""
    rng = np.random.default_rng(seed)
    step = 2.0 ** -20
    ks = np.arange(-3, 4) * r
    g = np.stack(np.meshgrid(ks, ks, ks, indexing="ij"), -1).reshape(-1, 3)
    pts = [g] + [g + s * step * np.eye(3)[ax] for ax in range(3) for s in (-2, -1, 1, 2)]
    mp = _shuffle(rng, np.concatenate(pts))
    dirs = np.array([w * np.linalg.norm(w) ** 0 for w in _directions()])
    offs = np.round(np.outer(np.array([r, r - step, r + step, r / 2]), np.ones(3)) * 2 ** 20) / 2 ** 20
    q = [g]
    for o in offs:
        q.append(g[rng.permutation(len(g))[:40]] - np.sign(dirs[rng.integers(0, 6, 40)]) * o)
    return Scene(f"dyadic_faces_r{r}", r, mp.astype(np.float32), _world(np.concatenate(q)), dyadic=True)


def _fill_cell(rng, c, n, r):
    return (np.asarray(c, dtype=np.float64) + rng.uniform(0.02, 0.98, (n, 3))) * r


def scene_thresholds(r=0.5, seed=0):
    """C. Path thresholds: cells of 15 / 16 / 17 and 63 / 64 / 65 points; neighbouring sub-cells of one brick whose runs
    merge into 16 points or just do not (kMergeMax); a 64-point sub-cell ahead of another dense sub-cell of the same
    brick (second-level table index); 3 x 3 x 3 neighbourhoods of kDenseCap - 1, kDenseCap and kDenseCap + 1 points;
    a brick z-layer with all 18 cells non-empty (kPairCells); fewer than K points inside r; empty neighbourhoods; a
    query in an empty brick next to a full one."""
    rng = np.random.default_rng(seed)
    pts, q = [], []
    # isolated cells at the thresholds (one every 4 cells along x, y = -8)
    for i, n in enumerate((15, 16, 17, 63, 64, 65)):
        c = (-12 + 4 * i, -8, -1)
        pts.append(_fill_cell(rng, c, n, r))
        q.append(_fill_cell(rng, c, 4, r))
        q.append((np.array(c) + [1.2, 0.5, 0.5]) * r)       # next cell: the dense one is a neighbour
    # merge runs: sub-cells 0 / 1 of one brick (x even / odd)
    for i, (a, b) in enumerate(((8, 8), (8, 9), (7, 8), (1, 15), (1, 16))):
        c0 = (-10 + 4 * i, -4, 2)
        pts += [_fill_cell(rng, c0, a, r), _fill_cell(rng, (c0[0] + 1, c0[1], c0[2]), b, r)]
        q.append((np.array(c0) + [1.0, 0.5, 0.5]) * r)
    # second level: a dense sub-cell (count 63 / 64 / 65) ahead of another dense sub-cell in the same brick
    for i, a in enumerate((63, 64, 65)):
        c0 = (-10 + 4 * i, 0, -4)
        pts += [_fill_cell(rng, c0, a, r), _fill_cell(rng, (c0[0] + 1, c0[1], c0[2]), 90, r)]
        q.append(_fill_cell(rng, (c0[0] + 1, c0[1], c0[2]), 6, r))
    # dense neighbourhoods of kDenseCap + d points around a centre cell
    for i, d in enumerate((-1, 0, 1)):
        c = np.array((3 + 5 * i, 6, 1))
        lo = (c - 1) * r
        pts.append(lo + rng.uniform(0.0, 3.0 * r, (K_DENSE_CAP + d, 3)))
        q.append(_fill_cell(rng, c, 8, r))
    # kPairCells: 27 cells of 17 points around a cell with an odd z index (lane 0 holds 3 x 3 x 2 cells)
    c = np.array((6, -8, 5))
    for o in np.array(np.meshgrid([-1, 0, 1], [-1, 0, 1], [-1, 0, 1])).T.reshape(-1, 3):
        pts.append(_fill_cell(rng, c + o, 17, r))
    q.append((c + 0.5) * r)
    q.append(_fill_cell(rng, c, 5, r))
    # fewer than K inside r
    for i, n in enumerate((1, 2, 3, 4)):
        c = np.array((12, -12 + 4 * i, -6))
        pts.append((c + 0.5) * r + rng.normal(0, 0.05 * r, (n, 3)))
        q.append((c + 0.5) * r)
    # empty neighbourhoods and a query in an empty brick next to a full one
    q.append(np.array([[12.5, 10.5, 6.5]]) * r)
    full = np.array((-2, 8, 6))                              # brick (-1, 4, 3): cells -2..-1, 8..9, 6..7
    for o in np.array(np.meshgrid([0, 1], [0, 1], [0, 1])).T.reshape(-1, 3):
        pts.append(_fill_cell(rng, full + o, 12, r))
    q.append((np.array([[0.1, 8.5, 6.5], [-2.5, 10.2, 6.5], [-1.5, 8.5, 8.1]])) * r)
    mp = _shuffle(rng, np.concatenate(pts)).astype(np.float32)
    mp = np.concatenate([mp, np.array([[-16, -16, -16], [16, 16, 16]], dtype=np.float32) * np.float32(r)])   # bbox: origin
    return Scene(f"thresholds_r{r}", r, mp, _world(np.concatenate([np.atleast_2d(x) for x in q])))


def scene_hash(r=0.5, seed=0, n=509):
    """D. Hash table: n + 2 points in n + 2 distinct bricks (tsize = next_pow2(n + 3): the table is nearly full, probe sequences
    are long and wrap at mask); queries on and between them; queries 2^21 bricks (2^22 cells) away from populated bricks
    on one and on all three axes: their cell_key aliases the populated brick, and they must find no neighbour."""
    rng = np.random.default_rng(seed)
    span = 12
    b = set()
    while len(b) < n:
        b.add(tuple(int(v) for v in rng.integers(-span, span, 3)))
    b = np.array(sorted(b))
    mp = (2 * b + rng.integers(0, 2, (n, 3)) + rng.uniform(0.1, 0.9, (n, 3))) * r
    mp = np.concatenate([mp, np.array([[-2 * span, -2 * span, -2 * span], [2 * span, 2 * span, 2 * span]]) * r])
    mp = _shuffle(rng, mp).astype(np.float32)
    m64 = mp.astype(np.float64)
    q = [m64[:200], m64[200:400] + rng.uniform(-r, r, (200, 3))]
    far = 2.0 ** 22 * r
    for sh in ([far, 0, 0], [0, -far, 0], [0, 0, far], [far, -far, far]):
        q.append(m64[:16] + np.array(sh))
    return Scene(f"hash_r{r}", r, mp, _world(np.concatenate(q)))


def scene_sizes(r=0.3, seed=0, nq=4097):
    """E. Sizes: a clustered random map; the tests slice 1, 127, 128, 129 and 4097 queries (and source clouds of 0 and
    1 feature) out of these."""
    rng = np.random.default_rng(seed)
    cen = rng.uniform(-4, 4, (40, 3))
    mp = np.clip(cen[rng.integers(0, 40, 6000)] + rng.normal(0, 0.4, (6000, 3)), -5.5, 5.5)
    mp = np.concatenate([mp, [[-6.0, -6.0, -6.0], [6.0, 6.0, 6.0]]]).astype(np.float32)     # bbox: origin
    q = cen[rng.integers(0, 40, nq)] + rng.normal(0, 0.45, (nq, 3))
    return Scene(f"sizes_r{r}", r, mp, _world(q))


RADII = (0.5, 0.3, 0.7, 1.1)


def all_scenes():
    out = []
    for r in RADII:
        out += [scene_faces(r, seed=1), scene_corners(r, seed=2)]
    out += [scene_dyadic_faces(0.5, seed=3), scene_ties(0.5, seed=4), scene_ties(0.3, seed=5), scene_thresholds(0.5, seed=6),
            scene_hash(0.5, seed=7), scene_hash(1.1, seed=8, n=1021), scene_sizes(0.3, seed=9)]
    return out
