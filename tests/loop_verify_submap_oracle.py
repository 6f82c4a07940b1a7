"""CPU restatement of loop verification against a submap (include/tloam_b200.h, "Loop verification against a submap";
k_lvs_* in libtloam_b200_loopvs.so), step by step in FP64:

    window:   frames lo = max(0, c - k) .. hi = min(c + k, F - 1), without the query
    target:   A_j = O_c^-1 O_j;  the rows A_j p of every window keyframe, frame order then row order (keyframe c copied)
    normals:  per target row i the rows j with d2(i, j) <= normal_radius^2 in ascending j: n_i, the mean and the covariance
              about it, both summed sequentially in that order; cyclic Jacobi; normal = eigenvector of the least eigenvalue;
              valid iff n_i >= min_normal_neighbours and l0 <= max_planarity * l1
    pass:     as loop_verify_oracle: p = R q + t, the exact nearest target row by (d2, index), inlier iff d2 <= r * r
    step:     over the inliers whose match has a valid normal: e = n . (p - m), J = [n, p x n];  H = sum J^T J,
              g = sum J^T e;  delta = -H^-1 g (LDL^T);  T <- exp(delta) . T
    result:   one more pass at r = fine: fitness = mean d2 over all of Q, rmse over the contributing rows' e

Every sum that the header calls sequential is a cumulative sum here (numpy's accumulate adds left to right), every other
operation one rounded numpy operation, so the target, the neighbour counts, the covariances, the normals and the first
pass are the device's bits.  The candidate sets come from a k-d tree with an inflated radius and are then decided by the
exactly rounded d2, so the tree only saves time."""
import numpy as np
from scipy.spatial import cKDTree

import loop_verify_oracle as lvo
from loop_verify_oracle import CONVERGED, ITERATION_LIMIT, FEW_INLIERS, SINGULAR, EMPTY  # noqa: F401


def config(**overrides):
    """tloam_b200_loop_verify_submap_default_config, with overrides"""
    c = dict(half_window=5, normal_radius=1.0, min_normal_neighbours=5, max_planarity=0.1, corr_dist_coarse=4.0,
             corr_dist_fine=1.0, max_iterations=40, eps_translation=1e-4, eps_rotation=1e-5, max_fitness=0.5)
    c.update(overrides)
    return c


def window(candidate, query, k, frames):
    """(lo, hi, the window's frames in order)"""
    lo, hi = max(0, candidate - k), min(candidate + k, frames - 1)
    return lo, hi, [j for j in range(lo, hi + 1) if j != query]


def _dot3(a0, b0, a1, b1, a2, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def relative(Oc, Oj):
    """A_j = O_c^-1 O_j:  R(r, c) = sum_k R_c(k, r) R_j(k, c),  t(r) = sum_k R_c(k, r) (t_j(k) - t_c(k))"""
    A = np.zeros((4, 4))
    d = [Oj[k, 3] - Oc[k, 3] for k in range(3)]
    for r in range(3):
        for c in range(3):
            A[r, c] = _dot3(Oc[0, r], Oj[0, c], Oc[1, r], Oj[1, c], Oc[2, r], Oj[2, c])
        A[r, 3] = _dot3(Oc[0, r], d[0], Oc[1, r], d[1], Oc[2, r], d[2])
    A[3, 3] = 1.0
    return A


def target(keyframes, poses, candidate, query, k):
    """the submap of `candidate` in its sensor frame: keyframes[j] (n_j x 3) and poses[j] (4 x 4) for every loop frame j (only
    the window's are read)"""
    _, _, frames = window(candidate, query, k, len(keyframes))
    blocks = []
    for j in frames:
        p = np.asarray(keyframes[j], dtype=np.float64).reshape(-1, 3)
        if j != candidate and len(p):
            A = relative(np.asarray(poses[candidate], dtype=np.float64), np.asarray(poses[j], dtype=np.float64))
            p = lvo.transform(p, A[:3, :3], A[:3, 3])
        blocks.append(p)
    return np.vstack(blocks) if blocks else np.zeros((0, 3))


def _d2(a, b):
    dx, dy, dz = a[..., 0] - b[..., 0], a[..., 1] - b[..., 1], a[..., 2] - b[..., 2]
    return (dx * dx + dy * dy) + dz * dz


def neighbours(M, radius):
    """per row the ascending indices j with d2(i, j) <= radius * radius, as a padded (n, width) index array and the counts"""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    cand = cKDTree(M).query_ball_point(M, radius * (1.0 + 1e-9) + 1e-12, return_sorted=True)
    cnt = np.array([len(c) for c in cand], dtype=np.int64)
    width = int(cnt.max()) if len(M) else 0
    idx = np.full((len(M), width), -1, dtype=np.int64)
    for i, c in enumerate(cand):
        idx[i, :len(c)] = c
    ok = idx >= 0
    ok &= _d2(M[:, None, :], M[np.maximum(idx, 0)]) <= radius * radius
    # keep the ascending order, move the refused candidates to the end
    order = np.argsort(~ok, axis=1, kind="stable")
    idx = np.where(np.take_along_axis(ok, order, 1), np.take_along_axis(idx, order, 1), -1)
    return idx, ok.sum(axis=1)


def _seq_sum(x):
    """left-to-right sum of each row, from 0.0"""
    return np.cumsum(x, axis=1)[:, -1] if x.shape[1] else np.zeros(len(x))


def moments(M, radius):
    """(counts, mean (n x 3), covariance (n x 6: xx, xy, xz, yy, yz, zz)) of every row's neighbourhood"""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    idx, cnt = neighbours(M, radius)
    ok = idx >= 0
    P = M[np.maximum(idx, 0)]
    n = cnt.astype(np.float64)
    mean = np.column_stack([_seq_sum(np.where(ok, P[:, :, a], 0.0)) / n for a in range(3)])
    D = [np.where(ok, P[:, :, a] - mean[:, None, a], 0.0) for a in range(3)]
    cov = np.column_stack([_seq_sum(D[a] * D[b]) / n for a, b in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))])
    return cnt, mean, cov


def jacobi3(c):
    """cyclic Jacobi on n symmetric matrices (n x 6: xx, xy, xz, yy, yz, zz): at most 32 sweeps over (0,1), (0,2), (1,2),
    each rotation skipped when its entry is 0, a matrix done once off <= 1e-32 * diag; the eigenvalues ascending (ties keep
    the lower axis first) and the eigenvector of the least one.  Operation for operation the device's lvs_jacobi3."""
    c = np.asarray(c, dtype=np.float64).reshape(-1, 6)
    n = len(c)
    a = np.zeros((3, 3, n))
    for (p, q), k in zip(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)), range(6)):
        a[p, q] = a[q, p] = c[:, k]
    v = np.zeros((3, 3, n))
    for k in range(3):
        v[k, k] = 1.0
    live = np.ones(n, dtype=bool)
    with np.errstate(all="ignore"):
        for _ in range(32):
            off = (a[0, 1] * a[0, 1] + a[0, 2] * a[0, 2]) + a[1, 2] * a[1, 2]
            diag = (a[0, 0] * a[0, 0] + a[1, 1] * a[1, 1]) + a[2, 2] * a[2, 2]
            live &= ~((off <= 1e-32 * diag) | (off == 0.0))
            if not live.any():
                break
            for p in range(2):
                for q in range(p + 1, 3):
                    rot = live & (a[p, q] != 0.0)
                    theta = (a[q, q] - a[p, p]) / (2.0 * a[p, q])
                    t = np.where(theta >= 0, 1.0, -1.0) / (np.abs(theta) + np.sqrt(theta * theta + 1.0))
                    cs = 1.0 / np.sqrt(t * t + 1.0)
                    sn = t * cs
                    for k in range(3):
                        akp, akq = a[k, p].copy(), a[k, q].copy()
                        a[k, p] = np.where(rot, cs * akp - sn * akq, akp)
                        a[k, q] = np.where(rot, sn * akp + cs * akq, akq)
                    for k in range(3):
                        apk, aqk = a[p, k].copy(), a[q, k].copy()
                        a[p, k] = np.where(rot, cs * apk - sn * aqk, apk)
                        a[q, k] = np.where(rot, sn * apk + cs * aqk, aqk)
                    for k in range(3):
                        vkp, vkq = v[k, p].copy(), v[k, q].copy()
                        v[k, p] = np.where(rot, cs * vkp - sn * vkq, vkp)
                        v[k, q] = np.where(rot, sn * vkp + cs * vkq, vkq)
    d = [a[0, 0].copy(), a[1, 1].copy(), a[2, 2].copy()]
    vec = [v[:, 0].copy(), v[:, 1].copy(), v[:, 2].copy()]

    def cswap(x, y):
        s = d[y] < d[x]
        d[x], d[y] = np.where(s, d[y], d[x]), np.where(s, d[x], d[y])
        vec[x], vec[y] = np.where(s, vec[y], vec[x]), np.where(s, vec[x], vec[y])

    cswap(0, 1)
    cswap(1, 2)
    cswap(0, 1)
    return np.column_stack(d), vec[0].T.copy()


def normals(M, cfg):
    """(normal (n x 3), valid (n,), neighbour counts (n,), eigenvalues (n x 3), covariance (n x 6)) of the target M"""
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    if len(M) == 0:
        return np.zeros((0, 3)), np.zeros(0, dtype=bool), np.zeros(0, dtype=np.int64), np.zeros((0, 3)), np.zeros((0, 6))
    cnt, _, cov = moments(M, cfg["normal_radius"])
    eig, nrm = jacobi3(cov)
    valid = (cnt >= cfg["min_normal_neighbours"]) & (eig[:, 0] <= cfg["max_planarity"] * eig[:, 1])
    return nrm, valid, cnt, eig, cov


def nearest(P, M, tree=None):
    """loop_verify_oracle.nearest's result ((d2, index) order over all of M), the candidates from a k-d tree"""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    tree = tree if tree is not None else cKDTree(M)
    dist, _ = tree.query(P)
    cand = tree.query_ball_point(P, dist * (1.0 + 1e-9) + 1e-12, return_sorted=True)
    idx = np.zeros(len(P), dtype=np.int64)
    d2 = np.zeros(len(P))
    for i, c in enumerate(cand):
        c = np.asarray(c, dtype=np.int64)
        d = _d2(P[i][None, :], M[c])
        j = int(np.argmin(d))                                      # the first minimum: the lowest index
        idx[i], d2[i] = c[j], d[j]
    return idx, d2


def plane_rows(P, Mm, N):
    """e = n . (p - m) = (nx dx + ny dy) + nz dz and J = [n, p x n] of the pairs"""
    dx, dy, dz = P[:, 0] - Mm[:, 0], P[:, 1] - Mm[:, 1], P[:, 2] - Mm[:, 2]
    e = (N[:, 0] * dx + N[:, 1] * dy) + N[:, 2] * dz
    J = np.column_stack([N[:, 0], N[:, 1], N[:, 2],
                         P[:, 1] * N[:, 2] - P[:, 2] * N[:, 1],
                         P[:, 2] * N[:, 0] - P[:, 0] * N[:, 2],
                         P[:, 0] * N[:, 1] - P[:, 1] * N[:, 0]])
    return e, J


def gauss_newton_step(P, Mm, N):
    """delta = -H^-1 g of the point-to-plane rows; None when the solve fails"""
    e, J = plane_rows(P, Mm, N)
    y = lvo.ldlt_solve(J.T @ J, J.T @ e)
    return None if y is None else -y


def run(Q, M, nrm, valid, guess, cfg):
    """the verification of keyframe Q against the target M with its normals: loop_verify_oracle.run's dict (inliers and rmse
    over the contributing rows)"""
    Q = np.asarray(Q, dtype=np.float64).reshape(-1, 3)
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    guess = np.asarray(guess, dtype=np.float64)
    R, t = guess[:3, :3].copy(), guess[:3, 3].copy()
    out = dict(T=guess.copy(), iterations=0, termination=EMPTY, inliers=0, rmse=0.0, fitness=np.inf, accepted=False, passes=[])
    if len(Q) == 0 or len(M) == 0:
        return out
    tree = cKDTree(M)
    fine = cfg["corr_dist_fine"]
    r, it, term, passes = cfg["corr_dist_coarse"], 0, ITERATION_LIMIT, []
    while True:
        P = lvo.transform(Q, R, t)
        idx, d2 = nearest(P, M, tree)
        passes.append((idx, d2))
        use = (d2 <= r * r) & valid[idx]
        if use.sum() < 6:
            term = FEW_INLIERS
            break
        delta = gauss_newton_step(P[use], M[idx[use]], nrm[idx[use]])
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
    if term in (CONVERGED, ITERATION_LIMIT):                       # a stop without a step already searched at this T
        passes.append(nearest(P, M, tree))
    idx, d2 = passes[-1]
    use = (d2 <= fine * fine) & valid[idx]
    n = int(use.sum())
    e, _ = plane_rows(P[use], M[idx[use]], nrm[idx[use]])
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    fitness = float(np.mean(d2))
    out.update(T=T, iterations=it, termination=term, inliers=n, rmse=float(np.sqrt(np.sum(e * e) / n)) if n else 0.0,
               fitness=fitness, accepted=term == CONVERGED and fitness <= cfg["max_fitness"], passes=passes)
    return out


def verify(keyframes, poses, query, candidate, guess, cfg):
    """target, normals and run; returns (result, target, normals, valid, counts)"""
    M = target(keyframes, poses, candidate, query, cfg["half_window"])
    nrm, valid, cnt, _, _ = normals(M, cfg)
    return run(keyframes[query], M, nrm, valid, guess, cfg), M, nrm, valid, cnt
