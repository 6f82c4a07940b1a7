"""CPU restatement of localization in a prior map (include/tloam_b200.h, "Localization in a prior map"; k_loc_* in
libtloam_b200_loc.so), step by step in FP64:

    grid:     mb = min per axis; cell index floor((x - mb) / cell); key = ix << (by + bz) | iy << bz | iz; the rows sorted
              stably by key; the occupied cells' keys and their starts
    search:   the nearest row with d2 <= r * r by (d2, row index), over the cells between those of p - rr and p + rr
    normals:  loop_verify_submap_oracle's rule with the neighbourhood taken from the grid
    passes:   loop_verify_submap_oracle.run with the grid search: pass k within the pass's radius, the final pass within
              corr_dist_coarse; fitness = mean min(d2, coarse^2), a row without a match counting coarse^2
    predict:  G = L . (O_prev^-1 . O_now), the products in the header's order

The cells this restatement visits per axis may be one more than the device's (np.nextafter stands in for the directed
roundings); both sets hold every row within r, so the results are the same."""
import numpy as np

import loop_verify_oracle as lvo
import loop_verify_submap_oracle as lso
from loop_verify_oracle import CONVERGED, ITERATION_LIMIT, FEW_INLIERS, SINGULAR, EMPTY  # noqa: F401

KEY_BITS = 21
INFLATE = 1.0 + 1e-7


def config(**overrides):
    """tloam_b200_localize_default_config, with overrides"""
    c = dict(voxel=0.5, cell=1.0, normal_radius=1.0, min_normal_neighbours=5, max_planarity=0.1, corr_dist_coarse=2.0,
             corr_dist_fine=0.5, max_iterations=30, eps_translation=1e-4, eps_rotation=1e-5, max_fitness=0.5)
    c.update(overrides)
    return c


def grid(M, cell):
    """the index of map M: dict(M, mb, cell, top, bits, srow, sxyz, ckey, cstart); ValueError past 2^21 cells"""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    if not np.isfinite(M).all():
        raise ValueError("non-finite row")
    n = len(M)
    mb = M.min(0) if n else np.zeros(3)
    idx = np.floor((M - mb) / cell).astype(np.int64)
    top = idx.max(0) if n else np.zeros(3, dtype=np.int64)
    if (top >= 2 ** KEY_BITS).any() or (n and not np.abs(M).max() * 2.0 ** -52 < 1e-6 * cell):
        raise ValueError("extent of 2^21 cells, or coordinates too large for the cell")
    bits = [int(t).bit_length() for t in top]
    key = (idx[:, 0].astype(np.uint64) << np.uint64(bits[1] + bits[2])) | (idx[:, 1].astype(np.uint64) << np.uint64(bits[2])) | \
        idx[:, 2].astype(np.uint64)
    order = np.argsort(key, kind="stable")
    skey = key[order]
    heads = np.r_[True, skey[1:] != skey[:-1]] if n else np.zeros(0, dtype=bool)
    return dict(M=M, mb=mb, cell=cell, top=top, bits=bits, srow=order.astype(np.uint32), sxyz=M[order], ckey=skey[heads],
                cstart=np.r_[np.flatnonzero(heads), n].astype(np.uint32))


def _key(g, ix, iy, iz):
    b = g["bits"]
    return (ix.astype(np.uint64) << np.uint64(b[1] + b[2])) | (iy.astype(np.uint64) << np.uint64(b[2])) | iz.astype(np.uint64)


def pairs(g, P, r):
    """(query, sorted position) of every map row in the cells visited for radius r"""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    if len(P) == 0 or len(g["M"]) == 0:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    rr = np.nextafter(r * INFLATE, np.inf)
    lo = np.floor((np.nextafter(P - rr, -np.inf) - g["mb"]) / g["cell"])
    hi = np.floor((np.nextafter(P + rr, np.inf) - g["mb"]) / g["cell"])
    lo = np.maximum(lo, 0).astype(np.int64)
    hi = np.minimum(hi, g["top"]).astype(np.int64)
    span = int(max(1, (hi - lo + 1).max()))
    qs, ps = [], []
    for a in range(span):
        for b in range(span):
            ix, iy = lo[:, 0] + a, lo[:, 1] + b
            ok = (ix <= hi[:, 0]) & (iy <= hi[:, 1]) & (lo[:, 2] <= hi[:, 2])
            q = np.flatnonzero(ok)
            if len(q) == 0:
                continue
            c0 = np.searchsorted(g["ckey"], _key(g, ix[q], iy[q], lo[q, 2]), "left")
            c1 = np.searchsorted(g["ckey"], _key(g, ix[q], iy[q], hi[q, 2]), "right")
            s, e = g["cstart"][c0].astype(np.int64), g["cstart"][c1].astype(np.int64)
            cnt = e - s
            qq = np.repeat(q, cnt)
            off = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
            qs.append(qq)
            ps.append(np.repeat(s, cnt) + off)
    if not qs:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    return np.concatenate(qs), np.concatenate(ps)


def search(g, P, r):
    """per row of P the nearest map row with d2 <= r * r by (d2, row index): (index (-1: none), d2 (+inf: none))"""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    idx, d2 = np.full(len(P), -1, dtype=np.int64), np.full(len(P), np.inf)
    q, pos = pairs(g, P, r)
    d = lso._d2(P[q], g["sxyz"][pos])
    keep = d <= r * r
    q, row, d = q[keep], g["srow"][pos[keep]].astype(np.int64), d[keep]
    o = np.lexsort((row, d, q))
    q, row, d = q[o], row[o], d[o]
    first = np.r_[True, q[1:] != q[:-1]] if len(q) else np.zeros(0, dtype=bool)
    idx[q[first]], d2[q[first]] = row[first], d[first]
    return idx, d2


def neighbours(g, radius, rows=None):
    """lso.neighbours's (padded ascending indices, counts) of every map row (or of the given rows), from the grid"""
    M = g["M"] if rows is None else g["M"][rows]
    q, pos = pairs(g, M, radius)
    keep = lso._d2(M[q], g["sxyz"][pos]) <= radius * radius
    q, row = q[keep], g["srow"][pos[keep]].astype(np.int64)
    o = np.lexsort((row, q))
    q, row = q[o], row[o]
    cnt = np.bincount(q, minlength=len(M))
    width = int(cnt.max()) if len(M) else 0
    idx = np.full((len(M), width), -1, dtype=np.int64)
    slot = np.arange(len(q)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    idx[q, slot] = row
    return idx, cnt


def normals(g, cfg, rows=None):
    """(normal (n x 3), valid (n,), counts (n,)) of every map row (or of the given rows)"""
    M = g["M"] if rows is None else g["M"][rows]
    if len(M) == 0:
        return np.zeros((0, 3)), np.zeros(0, dtype=bool), np.zeros(0, dtype=np.int64)
    idx, cnt = neighbours(g, cfg["normal_radius"], rows)
    ok = idx >= 0
    P = g["M"][np.maximum(idx, 0)]
    n = cnt.astype(np.float64)
    mean = np.column_stack([lso._seq_sum(np.where(ok, P[:, :, a], 0.0)) / n for a in range(3)])
    D = [np.where(ok, P[:, :, a] - mean[:, None, a], 0.0) for a in range(3)]
    cov = np.column_stack([lso._seq_sum(D[a] * D[b]) / n for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))])
    eig, nrm = lso.jacobi3(cov)
    valid = (cnt >= cfg["min_normal_neighbours"]) & (eig[:, 0] <= cfg["max_planarity"] * eig[:, 1])
    return nrm, valid, cnt


def predict(L, O_prev, O_now):
    """G = L . (O_prev^-1 . O_now) in the header's order"""
    D = lso.relative(np.asarray(O_prev, dtype=np.float64), np.asarray(O_now, dtype=np.float64))
    L = np.asarray(L, dtype=np.float64)
    G = np.eye(4)
    for r in range(3):
        for c in range(3):
            G[r, c] = lso._dot3(L[r, 0], D[0, c], L[r, 1], D[1, c], L[r, 2], D[2, c])
        G[r, 3] = lso._dot3(L[r, 0], D[0, 3], L[r, 1], D[1, 3], L[r, 2], D[2, 3]) + L[r, 3]
    return G


def map_odom(T, O):
    """T . O^-1 in the header's order"""
    M = np.eye(4)
    for r in range(3):
        for c in range(3):
            M[r, c] = lso._dot3(T[r, 0], O[c, 0], T[r, 1], O[c, 1], T[r, 2], O[c, 2])
    for r in range(3):
        M[r, 3] = T[r, 3] - lso._dot3(M[r, 0], O[0, 3], M[r, 1], O[1, 3], M[r, 2], O[2, 3])
    return M


def run(Q, g, nrm, valid, guess, cfg):
    """the localization of query Q (already down-sampled) from guess: dict(T, iterations, termination, inliers, rmse,
    fitness, accepted, passes)"""
    Q = np.asarray(Q, dtype=np.float64).reshape(-1, 3)
    guess = np.asarray(guess, dtype=np.float64)
    R, t = guess[:3, :3].copy(), guess[:3, 3].copy()
    out = dict(T=guess.copy(), iterations=0, termination=EMPTY, inliers=0, rmse=0.0, fitness=np.inf, accepted=False, passes=[])
    if len(Q) == 0 or len(g["M"]) == 0:
        return out
    M, coarse, fine = g["M"], cfg["corr_dist_coarse"], cfg["corr_dist_fine"]
    r, it, term, passes = coarse, 0, ITERATION_LIMIT, []
    while True:
        P = lvo.transform(Q, R, t)
        idx, d2 = search(g, P, r)
        passes.append((idx, d2))
        use = (idx >= 0) & (d2 <= r * r)
        use[use] = valid[idx[use]]
        if use.sum() < 6:
            term = FEW_INLIERS
            break
        delta = lso.gauss_newton_step(P[use], M[idx[use]], nrm[idx[use]])
        if delta is None:
            term = SINGULAR
            break
        R, t = lvo.apply(delta, R, t)
        it += 1
        if np.sqrt(np.sum(delta[:3] ** 2)) < cfg["eps_translation"] and np.sqrt(np.sum(delta[3:] ** 2)) < cfg["eps_rotation"]:
            if r == fine:
                term = CONVERGED
                break
            r = max(r * 0.5, fine)
        if it >= cfg["max_iterations"]:
            break
    P = lvo.transform(Q, R, t)
    fin = search(g, P, coarse)                                     # the final pass searches within coarse
    if term in (CONVERGED, ITERATION_LIMIT):
        passes.append(fin)
    else:
        passes[-1] = fin
    idx, d2 = fin
    use = (idx >= 0) & (d2 <= fine * fine)
    use[use] = valid[idx[use]]
    n = int(use.sum())
    e, _ = lso.plane_rows(P[use], M[idx[use]], nrm[idx[use]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    fitness = float(np.mean(np.where(idx >= 0, d2, coarse * coarse)))
    out.update(T=T, iterations=it, termination=term, inliers=n, rmse=float(np.sqrt(np.sum(e * e) / n)) if n else 0.0,
               fitness=fitness, accepted=term == CONVERGED and fitness <= cfg["max_fitness"], passes=passes)
    return out
