"""numpy restatement of path planning on the costmap (include/tloam_b200.h "Path planning"; k_plan_* in
tloam_b200/csrc/plan.cu), bit for bit.

The potential is the unique solution of P(goal) = 0, P(v) = min over the allowed moves v -> u of (k t(u) + P(u)), so any
exact shortest-path search gives its bits: `potential` is an integer Dijkstra with heapq, and the CPU tests pin it to a
brute-force Bellman-Ford and to scipy.sparse.csgraph.dijkstra (exact in float64 because every finite P is below 2^53).
`bellman_holds` checks the equations themselves, cell by cell in uint64, which proves a potential exact at any size
without a search.  Grids are (height, width) arrays, row j along y and column i along x; cells are (i, j)."""
import heapq

import numpy as np

INF = np.uint64(0xFFFFFFFFFFFFFFFF)
SIDE, DIAG = 70, 99
MOVES = ((1, 0), (0, 1), (-1, 0), (0, -1), (1, 1), (-1, 1), (-1, -1), (1, -1))   # the path rule's order
DEFAULT = dict(neutral_cost=50, cost_factor=3, allow_unknown=1)


def config(**overrides):
    c = dict(DEFAULT)
    c.update(overrides)
    return c


def config_valid(neutral_cost, cost_factor, allow_unknown):
    return neutral_cost >= 1 and neutral_cost + 252 * cost_factor <= 65535 and allow_unknown in (0, 1)


def cell_costs(costs, neutral_cost=50, cost_factor=3, allow_unknown=1):
    """t (uint16): neutral_cost + cost_factor c at codes 0 .. 252, at 255 with c = 252 when allow_unknown, else 0"""
    c = np.asarray(costs).astype(np.int64)
    passable = (c <= 252) | ((c == 255) & bool(allow_unknown))
    return np.where(passable, neutral_cost + cost_factor * np.where(c == 255, 252, c), 0).astype(np.uint16)


def _allowed(t, i, j, di, dj):
    """move (i, j) -> (i + di, j + dj) allowed: both ends passable and, on a diagonal, both corner cells"""
    H, W = t.shape
    ui, uj = i + di, j + dj
    if not (0 <= ui < W and 0 <= uj < H) or not t[j, i] or not t[uj, ui]:
        return False
    return not (di and dj) or (t[j, ui] and t[uj, i])


def potential(t, goal):
    """P (uint64) by Dijkstra from the goal over the reversed moves, in Python integers"""
    H, W = t.shape
    tl = t.tolist()
    gi, gj = goal
    P = [[None] * W for _ in range(H)]
    P[gj][gi] = 0
    heap = [(0, gi, gj)]
    done = set()
    while heap:
        p, i, j = heapq.heappop(heap)
        if (i, j) in done:
            continue
        done.add((i, j))
        step = tl[j][i]
        for di, dj in MOVES:                       # v = (i - di, j - dj) moves to (i, j) by (di, dj)
            vi, vj = i - di, j - dj
            if not (0 <= vi < W and 0 <= vj < H) or not tl[vj][vi]:
                continue
            if di and dj and not (tl[vj][i] and tl[j][vi]):
                continue
            c = p + (DIAG if di and dj else SIDE) * step
            if P[vj][vi] is None or c < P[vj][vi]:
                P[vj][vi] = c
                heapq.heappush(heap, (c, vi, vj))
    out = np.full((H, W), INF, dtype=np.uint64)
    for j in range(H):
        for i in range(W):
            if P[j][i] is not None and tl[j][i]:
                out[j, i] = P[j][i]
    return out


def brute(t, goal):
    """Bellman-Ford by full sweeps until nothing changes (tiny grids)"""
    H, W = t.shape
    P = {(goal[0], goal[1]): 0}
    changed = True
    while changed:
        changed = False
        for j in range(H):
            for i in range(W):
                if (i, j) == tuple(goal) or not t[j, i]:
                    continue
                best = P.get((i, j))
                for di, dj in MOVES:
                    if not _allowed(t, i, j, di, dj) or (i + di, j + dj) not in P:
                        continue
                    c = (DIAG if di and dj else SIDE) * int(t[j + dj, i + di]) + P[(i + di, j + dj)]
                    if best is None or c < best:
                        best = c
                if best is not None and best != P.get((i, j)):
                    P[(i, j)] = best
                    changed = True
    out = np.full((H, W), INF, dtype=np.uint64)
    for (i, j), p in P.items():
        out[j, i] = p
    return out


def scipy_potential(t, goal):
    """the same potential from scipy.sparse.csgraph.dijkstra (float64) on the reversed move graph"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import dijkstra
    H, W = t.shape
    tt = t.astype(np.float64)
    jj, ii = np.mgrid[0:H, 0:W]
    rows, cols, w = [], [], []
    for di, dj in MOVES:
        ui, uj = ii + di, jj + dj
        inside = (ui >= 0) & (ui < W) & (uj >= 0) & (uj < H)
        ok = inside & (t > 0)
        ok[inside] &= t[uj[inside], ui[inside]] > 0
        if di and dj:
            ok[inside] &= (t[jj[inside], ui[inside]] > 0) & (t[uj[inside], ii[inside]] > 0)
        v = (jj * W + ii)[ok]
        u = (uj * W + ui)[ok]
        rows.append(u)                              # reversed: u -> v, weight k t(u)
        cols.append(v)
        w.append((DIAG if di and dj else SIDE) * tt[uj[ok], ui[ok]])
    g = coo_matrix((np.concatenate(w), (np.concatenate(rows), np.concatenate(cols))), shape=(H * W, H * W)).tocsr()
    d = dijkstra(g, directed=True, indices=goal[1] * W + goal[0])
    out = np.full(H * W, INF, dtype=np.uint64)
    fin = np.isfinite(d)
    out[fin] = d[fin].astype(np.uint64)
    return out.reshape(H, W)


def _shifted(a, di, dj, fill):
    """a[j + dj, i + di] at every (i, j), fill outside"""
    H, W = a.shape
    p = np.full((H + 2, W + 2), fill, dtype=a.dtype)
    p[1:-1, 1:-1] = a
    return p[1 + dj:1 + dj + H, 1 + di:1 + di + W]


def bellman_holds(P, t, goal):
    """True iff P(goal) = 0, every impassable cell holds INF and every other cell equals the min over its allowed moves of
    k t(u) + P(u) (INF without one), in uint64; since the solution is unique this proves P exact"""
    P = np.asarray(P, dtype=np.uint64)
    gi, gj = goal
    if P[gj, gi] != 0 or not t[gj, gi]:
        return False
    imp = t == 0
    if (P[imp] != INF).any():
        return False
    best = np.full(P.shape, INF, dtype=np.uint64)
    for di, dj in MOVES:
        tu = _shifted(t, di, dj, 0)
        pu = _shifted(P, di, dj, INF)
        ok = (t > 0) & (tu > 0) & (pu != INF)
        if di and dj:
            ok &= (_shifted(t, di, 0, 0) > 0) & (_shifted(t, 0, dj, 0) > 0)
        c = np.where(ok, pu, 0) + np.uint64(DIAG if di and dj else SIDE) * tu.astype(np.uint64)
        np.minimum(best, np.where(ok, c, INF), out=best)
    best[gj, gi] = 0
    return bool(np.array_equal(best[~imp], P[~imp]))


def cells_of(xy, origin, resolution, shape):
    """(i, j) (n x 2 int64) of points by the occupancy build's hit rule, and whether each lies inside the grid (finite)"""
    p = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    with np.errstate(invalid="ignore"):
        u = np.floor((p[:, 0] - origin[0]) / resolution)
        v = np.floor((p[:, 1] - origin[1]) / resolution)
        ok = np.isfinite(u) & np.isfinite(v) & (u >= 0) & (u < shape[1]) & (v >= 0) & (v < shape[0])
    ij = np.zeros((len(p), 2), dtype=np.int64)
    ij[ok, 0], ij[ok, 1] = u[ok].astype(np.int64), v[ok].astype(np.int64)
    return ij, ok


def paths(P, t, starts_ij, inside=None):
    """the path rule from each start cell, all walkers stepped together: [(status, cost, cells (m, 2) int32)]"""
    P = np.asarray(P, dtype=np.uint64)
    H, W = t.shape
    s = np.asarray(starts_ij, dtype=np.int64).reshape(-1, 2)
    n = len(s)
    inside = np.ones(n, dtype=bool) if inside is None else np.asarray(inside)
    status = np.where(inside, 0, 1)
    si, sj = np.where(inside, s[:, 0], 0), np.where(inside, s[:, 1], 0)
    status = np.where(inside & (t[sj, si] == 0), 2, status)
    status = np.where((status == 0) & (P[sj, si] == INF), 3, status)
    cost = np.where(status == 0, P[sj, si], INF)
    tracks = [[(int(si[k]), int(sj[k]))] if status[k] == 0 else [] for k in range(n)]
    ci, cj = si.copy(), sj.copy()
    active = np.flatnonzero((status == 0) & (P[sj, si] != 0))
    while len(active):
        i, j = ci[active], cj[active]
        best = np.full(len(active), INF, dtype=np.uint64)
        bi, bj = i.copy(), j.copy()
        for di, dj in MOVES:
            ui, uj = i + di, j + dj
            ok = (ui >= 0) & (ui < W) & (uj >= 0) & (uj < H)
            uic, ujc = np.clip(ui, 0, W - 1), np.clip(uj, 0, H - 1)
            tu = t[ujc, uic]
            ok &= tu > 0
            if di and dj:
                ok &= (t[j, uic] > 0) & (t[ujc, i] > 0)
            pu = P[ujc, uic]
            ok &= pu != INF
            c = np.where(ok, pu, 0) + np.uint64(DIAG if di and dj else SIDE) * tu.astype(np.uint64)
            better = ok & (c < best)
            best = np.where(better, c, best)
            bi, bj = np.where(better, ui, bi), np.where(better, uj, bj)
        assert (best == P[j, i]).all(), "not a fixed point"
        ci[active], cj[active] = bi, bj
        for k, a in enumerate(active):
            tracks[a].append((int(bi[k]), int(bj[k])))
        active = active[P[bj, bi] != 0]
    return [(int(status[k]), int(cost[k]), np.array(tracks[k], dtype=np.int32).reshape(-1, 2)) for k in range(n)]


def centres(cells, origin, resolution):
    """xy of cells (m, 2): origin + (i + 0.5) resolution, each operation rounded on its own"""
    c = np.asarray(cells, dtype=np.float64).reshape(-1, 2)
    return np.column_stack([origin[0] + (c[:, 0] + 0.5) * resolution, origin[1] + (c[:, 1] + 0.5) * resolution])
