"""CPU restatement of global registration (include/tloam_b200.h, "Global registration"; k_gr_* in libtloam_b200_greg.so),
step by step in FP64 with every operation rounded on its own, as the device does it:

    side:        localize_oracle's grid and normals (max_planarity 1), n <- -n when n . p > 0
    SPFH:        per row with a valid normal, integer counts of (theta, alpha, phi) bins over its neighbours (valid normals,
                 0 < d2 <= r^2, not itself), the roles of each pair swapped when |n1 . d| < |n2 . d|
    FPFH:        SPFH(p) + per 11-bin block 100 acc / sum, acc = sum over the neighbours with pairs, in ascending sorted
                 position of the index, of SPFH(k) / d2
    matches:     nearest feature by the squared L2 summed in bin order, lower index on a tie; the mutual pairs
    hypotheses:  splitmix64 draws, Open3D's edge-length check, the cross-product area check, T from Gram-Schmidt frames
    refinement:  alternation of Horn's fit (cyclic Jacobi on 4 x 4) and the inliers within tau
    fitness:     the fraction of source keypoints with a target keypoint at d2 < tau^2 under T

Sums the device runs in order are np.cumsum (strictly sequential) or Python loops here."""
import math

import numpy as np

import localize_oracle as lo

BINS = 33
CONVERGED, ITERATION_LIMIT, FEW_INLIERS, FEW_CORRESPONDENCES, NO_HYPOTHESIS, EMPTY = range(6)
M64 = (1 << 64) - 1


def config(**overrides):
    """tloam_b200_global_registration_default_config, with overrides"""
    c = dict(voxel=0.5, cell=1.0, normal_radius=1.0, min_normal_neighbours=5, feature_radius=2.5, max_correspondence_distance=0.75,
             n_hypotheses=65536, seed=0, edge_similarity=0.9, min_triangle_area=1.0, max_refine_iterations=10, min_inliers=30,
             min_fitness=0.3)
    c.update(overrides)
    return c


def theta_table():
    """(cos, sin) of beta_k = (2k / 11 - 1) pi, k = 1 .. 10, from the C library as the host computes them"""
    b = [(2.0 * (k + 1) / 11.0 - 1.0) * math.pi for k in range(10)]
    return np.array([[math.cos(x), math.sin(x)] for x in b])


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _d2(p, q):
    d = p - q
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def lin_bin(f):
    return np.clip(np.floor(11.0 * ((f + 1.0) * 0.5)), 0, 10).astype(np.int64)


def theta_bin(x, y, cs=None):
    """the device's sign-test binning of atan2(y, x) into 11 bins of [-pi, pi]"""
    cs = theta_table() if cs is None else cs
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    upper = (y > 0) | ((y == 0) & (x < 0))
    b = np.zeros(np.broadcast(x, y).shape, dtype=np.int64)
    for k in range(10):
        s = (cs[k, 0] * y - cs[k, 1] * x) >= 0
        b += ((y >= 0) | s) if k < 5 else (upper & s)
    return b


def pair_bins(p1, n1, p2, n2, d2, cs=None):
    """(bins (m x 3) at 0 / 11 / 22, ok (m,)) of the pairs (p1, n1) -> (p2, n2)"""
    d = p2 - p1
    a1, a2 = _dot(n1, d), _dot(n2, d)
    swap = np.abs(a1) < np.abs(a2)
    u = np.where(swap[:, None], n2, n1)
    m = np.where(swap[:, None], n1, n2)
    d = np.where(swap[:, None], -d, d)
    phi = np.where(swap, -a2, a1) / np.sqrt(d2)
    v = _cross(d, u)
    vn = np.sqrt(_dot(v, v))
    ok = vn != 0
    with np.errstate(invalid="ignore", divide="ignore"):
        v = v / vn[:, None]
    w = _cross(u, v)
    b = np.column_stack([theta_bin(_dot(u, m), _dot(w, m), cs), 11 + lin_bin(_dot(v, m)), 22 + lin_bin(phi)])
    return b, ok


def neighbour_pairs(g, xyz, valid, r):
    """(i, v, d2) of every neighbour pair, i ascending and each row's neighbours in ascending sorted position"""
    q, pos = lo.pairs(g, xyz, r)
    v = g["srow"][pos].astype(np.int64)
    d2 = _d2(xyz[q], g["sxyz"][pos])
    keep = (v != q) & valid[q] & valid[v] & (d2 <= r * r) & (d2 != 0)
    q, pos, v, d2 = q[keep], pos[keep], v[keep], d2[keep]
    o = np.lexsort((pos, q))
    return q[o], v[o], d2[o]


def side(xyz, cfg, cs=None):
    """one cloud's keypoints through index, oriented normals, SPFH and FPFH: a dict"""
    xyz = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    n = len(xyz)
    g = lo.grid(xyz, cfg["cell"])
    nrm, valid, _ = lo.normals(g, dict(normal_radius=cfg["normal_radius"], min_normal_neighbours=cfg["min_normal_neighbours"],
                                       max_planarity=1.0))
    nrm = np.where((_dot(nrm, xyz) > 0)[:, None], -nrm, nrm)
    i, v, d2 = neighbour_pairs(g, xyz, valid, cfg["feature_radius"])
    b, ok = pair_bins(xyz[i], nrm[i], xyz[v], nrm[v], d2, cs)
    spfh = np.zeros((n, BINS), dtype=np.int64)
    for k in range(3):
        np.add.at(spfh, (i[ok], b[ok, k]), 1)
    pairs = np.bincount(i[ok], minlength=n)
    keep = pairs[v] > 0
    i, v, d2 = i[keep], v[keep], d2[keep]
    feat = np.zeros((n, BINS))
    has = pairs > 0
    cnt = np.bincount(i, minlength=n)
    width = int(cnt.max()) if len(i) else 0
    slot = np.arange(len(i)) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    own = (spfh * 100.0) / np.maximum(pairs, 1)[:, None]
    for lo_r in range(0, n, 1024):
        rows = slice(lo_r, min(n, lo_r + 1024))
        sel = (i >= rows.start) & (i < rows.stop)
        val = np.zeros((rows.stop - rows.start, max(width, 1), BINS))
        val[i[sel] - rows.start, slot[sel]] = ((spfh[v[sel]] * 100.0) / pairs[v[sel]][:, None]) / d2[sel][:, None]
        acc = np.cumsum(val, axis=1)[:, -1, :]
        F = np.zeros_like(acc)
        for blk in range(3):
            s = np.cumsum(val[:, :, 11 * blk:11 * blk + 11].reshape(len(val), -1), axis=1)[:, -1]
            a = acc[:, 11 * blk:11 * blk + 11]
            with np.errstate(invalid="ignore", divide="ignore"):
                F[:, 11 * blk:11 * blk + 11] = np.where((s != 0)[:, None], (a * 100.0) / s[:, None], a)
        feat[rows] = np.where(has[rows, None], F + own[rows], 0.0)
    return dict(xyz=xyz, grid=g, normal=nrm, valid=valid, spfh=spfh, pairs=pairs, feature=feat, has_feature=has)


def nearest_feature(A, has_a, B, has_b):
    """per row of A with a feature the row of B with a feature nearest by the in-order squared L2 (-1: none)"""
    out = np.full(len(A), -1, dtype=np.int64)
    if not has_b.any():
        return out
    for s in range(0, len(A), 512):
        a = A[s:s + 512]
        d = np.zeros((len(a), len(B)))
        for j in range(BINS):
            t = a[:, j, None] - B[None, :, j]
            d = d + t * t
        d[:, ~has_b] = np.inf
        out[s:s + 512] = np.argmin(d, axis=1)
    out[~has_a] = -1
    return out


def mutual(S, T):
    a = nearest_feature(S["feature"], S["has_feature"], T["feature"], T["has_feature"])
    b = nearest_feature(T["feature"], T["has_feature"], S["feature"], S["has_feature"])
    i = np.flatnonzero(a >= 0)
    i = i[b[a[i]] == i]
    return np.column_stack([i, a[i]]).astype(np.int64)


def splitmix64(x):
    x = np.asarray(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = x + np.uint64(0x9e3779b97f4a7c15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return z ^ (z >> np.uint64(31))


def draws(seed, h, nc):
    """the three distinct pair indices of hypotheses h (array) over nc >= 3 pairs"""
    h = np.asarray(h, dtype=np.uint64)
    r = [splitmix64(np.uint64(seed) ^ splitmix64((h << np.uint64(2)) | np.uint64(d))) for d in range(3)]
    i0 = r[0] % np.uint64(nc)
    i1 = r[1] % np.uint64(nc - 1)
    i1 = i1 + (i1 >= i0)
    lo_, hi_ = np.minimum(i0, i1), np.maximum(i0, i1)
    i2 = r[2] % np.uint64(nc - 2)
    i2 = i2 + (i2 >= lo_)
    i2 = i2 + (i2 >= hi_)
    return np.column_stack([i0, i1, i2]).astype(np.int64)


def frame(x):
    """(area, E (h x 3 x 3: rows e1, e2, e3)) of triangles x (h x 3 x 3)"""
    a, u = x[:, 1] - x[:, 0], x[:, 2] - x[:, 0]
    c = _cross(a, u)
    area = np.sqrt(_dot(c, c))
    with np.errstate(invalid="ignore", divide="ignore"):
        e1 = a / np.sqrt(_dot(a, a))[:, None]
        b = u - _dot(u, e1)[:, None] * e1
        e2 = b / np.sqrt(_dot(b, b))[:, None]
    return area, np.stack([e1, e2, _cross(e1, e2)], axis=1)


def hypotheses(P, Q, corr, h, cfg):
    """(live (h,), R (h x 3 x 3), t (h x 3)) of hypotheses h"""
    nc = len(corr)
    idx = draws(cfg["seed"], h, nc)
    p, q = P[corr[idx, 0]], Q[corr[idx, 1]]
    sim = cfg["edge_similarity"]
    live = np.ones(len(idx), dtype=bool)
    for u, v in ((0, 1), (0, 2), (1, 2)):
        ds, dt = np.sqrt(_d2(p[:, u], p[:, v])), np.sqrt(_d2(q[:, u], q[:, v]))
        live &= ~((ds < dt * sim) | (dt < ds * sim))
    ap, E = frame(p)
    aq, F = frame(q)
    live &= (ap >= cfg["min_triangle_area"]) & (aq >= cfg["min_triangle_area"])
    R = np.empty((len(idx), 3, 3))
    for r in range(3):
        for c in range(3):
            R[:, r, c] = (F[:, 0, r] * E[:, 0, c] + F[:, 1, r] * E[:, 1, c]) + F[:, 2, r] * E[:, 2, c]
    cp = ((p[:, 0] + p[:, 1]) + p[:, 2]) / 3.0
    cq = ((q[:, 0] + q[:, 1]) + q[:, 2]) / 3.0
    t = cq - np.stack([(R[:, r, 0] * cp[:, 0] + R[:, r, 1] * cp[:, 1]) + R[:, r, 2] * cp[:, 2] for r in range(3)], axis=1)
    return live, R, t


def transform(R, t, P):
    """R p + t as ((R_r0 px + R_r1 py) + R_r2 pz) + t_r for one T (R 3 x 3) or a batch (h x 3 x 3) over rows P"""
    R, t = np.asarray(R), np.asarray(t)
    if R.ndim == 2:
        return np.column_stack([((R[r, 0] * P[:, 0] + R[r, 1] * P[:, 1]) + R[r, 2] * P[:, 2]) + t[r] for r in range(3)])
    return np.stack([((R[:, r, 0, None] * P[None, :, 0] + R[:, r, 1, None] * P[None, :, 1]) + R[:, r, 2, None] * P[None, :, 2])
                     + t[:, r, None] for r in range(3)], axis=-1)


def score(P, Q, corr, cfg, chunk=2048):
    """every hypothesis's inliers (-1: rejected or fewer than 3 pairs)"""
    H, nc = cfg["n_hypotheses"], len(corr)
    out = np.full(H, -1, dtype=np.int64)
    if nc < 3:
        return out
    tau2 = cfg["max_correspondence_distance"] * cfg["max_correspondence_distance"]
    p, q = P[corr[:, 0]], Q[corr[:, 1]]
    for s in range(0, H, chunk):
        h = np.arange(s, min(H, s + chunk))
        live, R, t = hypotheses(P, Q, corr, h, cfg)
        with np.errstate(invalid="ignore"):
            cnt = (_d2(transform(R, t, p), q[None]) < tau2).sum(1)
        out[h] = np.where(live, cnt, -1)
    return out


def jacobi4(N):
    """nf_jacobi3's cyclic Jacobi on the symmetric 4 x 4 N: the eigenvector of the largest eigenvalue (lower index on a tie)"""
    a = [[float(N[i][j]) for j in range(4)] for i in range(4)]
    v = [[1.0 if i == j else 0.0 for j in range(4)] for i in range(4)]
    prs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    for _ in range(32):
        off = 0.0
        for p, r in prs:
            off = off + a[p][r] * a[p][r]
        diag = 0.0
        for p in range(4):
            diag = diag + a[p][p] * a[p][p]
        if off <= 1e-32 * diag or off == 0.0:
            break
        for p, r in prs:
            if a[p][r] == 0.0:
                continue
            theta = (a[r][r] - a[p][p]) / (2.0 * a[p][r])
            tt = (1.0 if theta >= 0 else -1.0) / (abs(theta) + math.sqrt(theta * theta + 1.0))
            cs = 1.0 / math.sqrt(tt * tt + 1.0)
            sn = tt * cs
            for k in range(4):
                akp, akr = a[k][p], a[k][r]
                a[k][p], a[k][r] = cs * akp - sn * akr, sn * akp + cs * akr
            for k in range(4):
                apk, ark = a[p][k], a[r][k]
                a[p][k], a[r][k] = cs * apk - sn * ark, sn * apk + cs * ark
            for k in range(4):
                vkp, vkr = v[k][p], v[k][r]
                v[k][p], v[k][r] = cs * vkp - sn * vkr, sn * vkp + cs * vkr
    b = 0
    for k in range(1, 4):
        if a[k][k] > a[b][b]:
            b = k
    return [v[k][b] for k in range(4)]


def fit(p, q):
    """Horn's least-squares (R, t) with q ~ R p + t, every sum in row order"""
    n = float(len(p))
    cp, cq = [0.0] * 3, [0.0] * 3
    for k in range(len(p)):
        for c in range(3):
            cp[c] = cp[c] + float(p[k, c])
            cq[c] = cq[c] + float(q[k, c])
    cp, cq = [x / n for x in cp], [x / n for x in cq]
    S = [0.0] * 9
    for k in range(len(p)):
        dp = [float(p[k, c]) - cp[c] for c in range(3)]
        dq = [float(q[k, c]) - cq[c] for c in range(3)]
        for u in range(3):
            for v in range(3):
                S[3 * u + v] = S[3 * u + v] + dp[u] * dq[v]
    xx, xy, xz, yx, yy, yz, zx, zy, zz = S
    N = [[(xx + yy) + zz, yz - zy, zx - xz, xy - yx],
         [yz - zy, (xx - yy) - zz, xy + yx, zx + xz],
         [zx - xz, xy + yx, (yy - xx) - zz, yz + zy],
         [xy - yx, zx + xz, yz + zy, (zz - xx) - yy]]
    qv = jacobi4(N)
    qn = math.sqrt(((qv[0] * qv[0] + qv[1] * qv[1]) + qv[2] * qv[2]) + qv[3] * qv[3])
    w, x, y, z = (c / qn for c in qv)
    ww, x2, y2, z2 = w * w, x * x, y * y, z * z
    wx, wy, wz, xy_, xz_, yz_ = w * x, w * y, w * z, x * y, x * z, y * z
    R = np.array([[((ww + x2) - y2) - z2, 2.0 * (xy_ - wz), 2.0 * (xz_ + wy)],
                  [2.0 * (xy_ + wz), ((ww - x2) + y2) - z2, 2.0 * (yz_ - wx)],
                  [2.0 * (xz_ - wy), 2.0 * (yz_ + wx), ((ww - x2) - y2) + z2]])
    t = np.array([cq[r] - ((R[r, 0] * cp[0] + R[r, 1] * cp[1]) + R[r, 2] * cp[2]) for r in range(3)])
    return R, t


def refine(p, q, R, t, cfg):
    """the truncated-least-squares alternation from (R, t): (R, t, inlier mask, fits, termination, [cost per step])"""
    tau = cfg["max_correspondence_distance"]
    tau2 = tau * tau
    r2 = _d2(transform(R, t, p), q)
    S = r2 < tau2
    costs = [float(np.minimum(r2, tau2).sum())]
    it = 0
    while True:
        if it >= cfg["max_refine_iterations"]:
            term = ITERATION_LIMIT
            break
        if S.sum() < 3:
            term = FEW_INLIERS
            break
        R, t = fit(p[S], q[S])
        it += 1
        r2 = _d2(transform(R, t, p), q)
        costs.append(float(np.minimum(r2, tau2).sum()))
        S2 = r2 < tau2
        same = np.array_equal(S2, S)
        S = S2
        if same:
            term = CONVERGED
            break
    return R, t, S, it, term, costs


def run(src_xyz, tgt_xyz, cfg):
    """the whole call on two keypoint sets: a dict of every stage and the result"""
    cs = theta_table()
    out = dict(T=np.eye(4), n_correspondences=0, n_valid_hypotheses=0, best_hypothesis=-1, best_inliers=0, inliers=0,
               inlier_rmse=0.0, fitness=0.0, refine_iterations=0, termination=EMPTY, hyp=np.zeros(0, dtype=np.int64),
               corr=np.zeros((0, 2), dtype=np.int64))
    src_xyz, tgt_xyz = np.asarray(src_xyz, dtype=np.float64).reshape(-1, 3), np.asarray(tgt_xyz, dtype=np.float64).reshape(-1, 3)
    if len(src_xyz) == 0 or len(tgt_xyz) == 0:
        out["accepted"] = False
        return out
    S, T = side(src_xyz, cfg, cs), side(tgt_xyz, cfg, cs)
    corr = mutual(S, T)
    hyp = score(S["xyz"], T["xyz"], corr, cfg)
    out.update(src=S, tgt=T, corr=corr, hyp=hyp, n_correspondences=len(corr), n_valid_hypotheses=int((hyp >= 0).sum()))
    R, t = np.eye(3), np.zeros(3)
    if len(corr) < 3:
        out["termination"] = FEW_CORRESPONDENCES
    elif out["n_valid_hypotheses"] == 0:
        out["termination"] = NO_HYPOTHESIS
    else:
        best = int(np.argmax(hyp))
        live, Rb, tb = hypotheses(S["xyz"], T["xyz"], corr, np.array([best]), cfg)
        p, q = S["xyz"][corr[:, 0]], T["xyz"][corr[:, 1]]
        R, t, mask, it, term, costs = refine(p, q, Rb[0], tb[0], cfg)
        e = 0.0
        r2 = _d2(transform(R, t, p), q)
        for k in np.flatnonzero(mask):
            e = e + float(r2[k])
        n = int(mask.sum())
        out.update(best_hypothesis=best, best_inliers=int(hyp[best]), inliers=n, inlier_rmse=math.sqrt(e / n) if n else 0.0,
                   refine_iterations=it, termination=term, costs=costs)
    Tm = np.eye(4)
    Tm[:3, :3], Tm[:3, 3] = R, t
    out["T"] = Tm
    tau = cfg["max_correspondence_distance"]
    TP = transform(R, t, S["xyz"])
    qi, pos = lo.pairs(T["grid"], TP, tau)
    hit = np.zeros(len(TP), dtype=bool)
    hit[qi[_d2(TP[qi], T["grid"]["sxyz"][pos]) < tau * tau]] = True
    out["fitness"] = float(hit.sum()) / float(len(TP))
    out["accepted"] = out["inliers"] >= cfg["min_inliers"] and out["fitness"] >= cfg["min_fitness"]
    return out
