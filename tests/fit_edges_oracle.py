"""Exact / extended-precision restatement of the registration's primitive fits and of its SE(3) maps, with an FP64 error
model.  Test infrastructure for test_fit_edges.py; nothing here uses the FP64 code paths it checks.

Neighbours are given exactly as the device sees them (origin + float32, i.e. Python floats); every rational quantity is a
fractions.Fraction, every square root / eigenproblem / trigonometric value an mpmath number at 50 digits.

Fits (fit_neighbours in tloam_b200/csrc/frame_kernels.cuh, ref: registration.cpp:445-493, 536-551, 589-625, 732-768):
  sphere  valid iff a neighbour exists and d2 <= 0.2 (d2 = exact squared distance query - nearest neighbour);
  edge    k > 3, covariance C = mean((p - m)(p - m)^T), eigenvalues l0 <= l1 <= l2 and top unit eigenvector v;
          valid iff l2 > 3 l1 and |v.z| > thres; the line is m +- 0.1 v;
  plane   k > 4, fitBestPlane evaluated exactly (det^2-weighted axes, sign flip when dot < 0, zero plane when the
          weighted sum is zero), valid iff no neighbour has n.p + d > 0.2 (one-sided).

Error model.  u = 2^-53; k neighbours; M = largest |coordinate|; S = largest |p - m|.  Each bound B is on the FP64
evaluation of one decision or output; |margin| > B makes the exact verdict the contract, otherwise the case is counted as
"in band" and only has to agree with the CPU oracle (oracle.Oracle.build_factors).  The constants are generous first-order
bounds (FMA contraction only removes roundings, so it stays inside them):
  edge   the covariance comes from raw cumulants, so each entry carries dC = 4 (k + 3) u M^2 (zero when every FP64
         operation of that sequence is exact on these inputs); Jacobi adds 64 u |C|_F; E = 3 dC + 64 u |C|_F bounds every
         eigenvalue.  ratio margin l2 - 3 l1: B = 5 E.  Direction (Davis-Kahan): B_dir = 2 E / (l2 - l1) + 64 u, infinite
         on a tie l1 = l2.  |v.z| margin: B_dir.  Endpoints: 0.1 B_dir + 4 (k + 2) u M.
  plane  each centred covariance entry carries dC = 4 (k + 2) u M S (zero when exact).  The normal's bound B_n is twice
         the sum over the six entries of the largest change of the formula's unit normal under a +-dC change of that
         entry, plus 64 u (a sign flip inside that range makes B_n ~ 2: the normal is then undecided).  Signed distances:
         B_dist = 2 B_n S + 16 u M; offset d: B_n M + 8 u M.
  sphere B = 8 u d2 + 4 |q - p| u max(|q|, |p|) (the difference of the two points rounds once per axis), and B = 0
         when every step of the device's difference / fma chain is exact on the inputs.
  A bound of exactly 0 means the device evaluates that decision without rounding: the exact verdict then holds even at a
  margin of 0, which is how the strict `>` of each test is pinned against the exact reference.
  SE(3)  exp: rotation entries 64 u; translation 64 u |upsilon| (1 + theta), plus theta |upsilon| below the Taylor switch
         theta < 1e-10, where Sophus uses V = R instead of the left Jacobian.  log: omega 64 u (1 + 1 / (pi - theta)),
         upsilon 256 u |t| (1 + 1 / (pi - theta)), plus 2 |w| on omega when |w| < 1e-10 (Sophus returns exactly +-pi there).
         plus: 1024 u (1 + |upsilon_x| + |upsilon_delta|) (1 + 1 / (pi - theta)).  pi - theta is floored at 1e-3: the
         quaternion extraction and the atan form do not amplify rounding at pi itself, and a bound that grew without
         limit there would hide a wrong sign of omega at theta = pi.
"""
from fractions import Fraction

import mpmath as mp
import numpy as np

mp.mp.dps = 50
U = 2.0 ** -53
EDGE_DIR_THRES = 0.85
PLANE_THRES = 0.2
SPHERE_THRES = 0.2
LIE_EPS = 1e-10


def fr(x):
    return Fraction(float(x))


def mpf(q):
    q = Fraction(q)
    return mp.mpf(q.numerator) / q.denominator


def _mean_cov(nb):
    k = len(nb)
    P = [[fr(c) for c in p] for p in nb]
    m = [sum(p[i] for p in P) / k for i in range(3)]
    C = [[sum((p[i] - m[i]) * (p[j] - m[j]) for p in P) / k for j in range(3)] for i in range(3)]
    return P, m, C


def _fp_exact(ops):
    """True when every (float result, exact Fraction) pair agrees: the FP64 sequence rounded nowhere."""
    return all(Fraction(float(a)) == b for a, b in ops)


def _edge_cumulants_exact(nb):
    """Whether the device's raw-cumulant sequence (frame_kernels.cuh fit_neighbours) is exact in FP64 on these inputs."""
    k = len(nb)
    cu = [0.0] * 9
    cx = [Fraction(0)] * 9
    ops = []
    for p in nb:
        x, y, z = (float(c) for c in p)
        X, Y, Z = fr(x), fr(y), fr(z)
        vals = (x, y, z, x * x, x * y, x * z, y * y, y * z, z * z)
        exs = (X, Y, Z, X * X, X * Y, X * Z, Y * Y, Y * Z, Z * Z)
        for j in range(9):
            ops.append((vals[j], exs[j]))
            cu[j] += vals[j]
            cx[j] += exs[j]
            ops.append((cu[j], cx[j]))
    for j in range(9):
        cu[j] /= k
        cx[j] /= k
        ops.append((cu[j], cx[j]))
    for a, b in ((3, (0, 0)), (4, (0, 1)), (5, (0, 2)), (6, (1, 1)), (7, (1, 2)), (8, (2, 2))):
        ops.append((cu[b[0]] * cu[b[1]], cx[b[0]] * cx[b[1]]))
        ops.append((cu[a] - cu[b[0]] * cu[b[1]], cx[a] - cx[b[0]] * cx[b[1]]))
    return _fp_exact(ops)


def eig_sym(C):
    """Eigenvalues (ascending) and unit eigenvectors (columns) of an exact symmetric 3x3 matrix, mpmath.eigsy."""
    A = mp.matrix([[mpf(C[i][j]) for j in range(3)] for i in range(3)])
    E, Q = mp.eigsy(A)
    order = sorted(range(3), key=lambda i: E[i])
    return [E[i] for i in order], [[Q[r, i] for r in range(3)] for i in order]


def edge_exact(nb, thres=EDGE_DIR_THRES):
    """Edge fit of k neighbours.  Returns a dict: k, cov (Fractions), ev (asc), v (top eigenvector), gap, margins
    m_ratio = l2 - 3 l1 and m_dir = |v.z| - thres, their bounds, the endpoints a / b, the exact verdict and `decided`."""
    k = len(nb)
    out = dict(k=k, verdict=False, decided=True, kind="edge")
    if k <= 3:
        return out
    P, m, C = _mean_cov(nb)
    ev, vecs = eig_sym(C)
    v = vecs[2]
    M = max(abs(float(c)) for p in nb for c in p)
    S = max(float(mp.sqrt(sum((p[i] - m[i]) ** 2 for i in range(3)))) for p in P)
    dC = 0.0 if _edge_cumulants_exact(nb) else 4 * (k + 3) * U * M * M
    normC = float(mp.sqrt(sum(mpf(C[i][j]) ** 2 for i in range(3) for j in range(3))))
    diag = all(C[i][j] == 0 for i in range(3) for j in range(3) if i != j)
    E = 3 * dC + (0.0 if diag and dC == 0 else 64 * U * normC)
    gap = ev[2] - ev[1]
    m_ratio = ev[2] - 3 * ev[1]
    m_dir = abs(v[2]) - mp.mpf(thres)
    B_ratio = 5 * E + (0.0 if diag and dC == 0 and Fraction(float(3 * C[0][0])) == 3 * C[0][0] else 8 * U * normC)
    if diag and dC == 0:
        # the device sees a diagonal matrix, Jacobi does not rotate and every eigenvalue is exact: only 3.0 * ev[1] rounds
        lam = sorted(C[i][i] for i in range(3))
        B_ratio = 0.0 if Fraction(float(3 * lam[1])) == 3 * lam[1] else 4 * U * float(lam[1])
        B_dir = 0.0 if gap > 0 else float("inf")
    else:
        B_dir = float("inf") if gap == 0 else 2 * E / float(gap) + 64 * U
    B_end = 0.1 * B_dir + 4 * (k + 2) * U * M
    verdict = bool(m_ratio > 0 and m_dir > 0)
    # a condition is certain when its margin clears its bound, or when the bound is 0 (the device's evaluation is exact,
    # so even a margin of exactly 0 -- a tie that `>` rejects -- is decided)
    ratio_sure = abs(m_ratio) > B_ratio or B_ratio == 0
    dir_sure = abs(m_dir) > B_dir or B_dir == 0
    decided = (ratio_sure and not m_ratio > 0) or (dir_sure and not m_dir > 0) or (ratio_sure and dir_sure)
    mean = [mpf(c) for c in m]
    a = [mean[i] + mp.mpf("0.1") * v[i] for i in range(3)]
    b = [mean[i] - mp.mpf("0.1") * v[i] for i in range(3)]
    out.update(cov=C, ev=ev, v=v, gap=gap, m_ratio=m_ratio, m_dir=m_dir, B_ratio=B_ratio, B_dir=B_dir, B_end=B_end,
               a=np.array([float(t) for t in a]), b=np.array([float(t) for t in b]), verdict=verdict, decided=decided, M=M, S=S,
               mean=m)
    return out


def _best_plane_formula(xx, xy, xz, yy, yz, zz):
    """fitBestPlane's weighted axis sum (ref: registration.cpp:303-368), exact on Fractions or FP64 on floats.
    Returns (w, flips) with flips the signed dot products of the two decisions after the first."""
    w = [0 * xx, 0 * xx, 0 * xx]
    dots = []
    for det, ax in ((yy * zz - yz * yz, (yy * zz - yz * yz, xz * yz - xy * zz, xy * yz - xz * yy)),
                    (xx * zz - xz * xz, (xz * yz - xy * zz, xx * zz - xz * xz, xy * xz - yz * xx)),
                    (xx * yy - xy * xy, (xy * yz - xz * yy, xy * xz - yz * xx, xx * yy - xy * xy))):
        wgt = det * det
        d = w[0] * ax[0] + w[1] * ax[1] + w[2] * ax[2]
        dots.append(d)
        if d < 0:
            wgt = -wgt
        w = [w[i] + ax[i] * wgt for i in range(3)]
    return w, dots


def _unit(w):
    n = float(np.sqrt(sum(float(c) ** 2 for c in w)))
    return np.zeros(3) if n == 0 else np.array([float(c) for c in w]) / n


def _plane_cov_exact(nb):
    """Whether fit_best_plane's centroid / centred-product sequence is exact in FP64 on these inputs."""
    k = len(nb)
    ops = []
    c = [0.0, 0.0, 0.0]
    cx = [Fraction(0)] * 3
    for p in nb:
        for i in range(3):
            c[i] += float(p[i])
            cx[i] += fr(p[i])
            ops.append((c[i], cx[i]))
    c = [t / k for t in c]
    cx = [t / k for t in cx]
    ops += list(zip(c, cx))
    s = [0.0] * 6
    sx = [Fraction(0)] * 6
    for p in nb:
        d = [float(p[i]) - c[i] for i in range(3)]
        dx = [fr(p[i]) - cx[i] for i in range(3)]
        ops += list(zip(d, dx))
        for j, (a, b) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
            ops.append((d[a] * d[b], dx[a] * dx[b]))
            s[j] += d[a] * d[b]
            sx[j] += dx[a] * dx[b]
            ops.append((s[j], sx[j]))
    ops += [(t / k, tx / k) for t, tx in zip(s, sx)]
    return _fp_exact(ops)


def plane_exact(nb, thres=PLANE_THRES):
    """Plane fit of k neighbours.  Returns a dict: normal n, offset d (floats of the exact values), exact signed
    distances, margin m = max(n.p + d) - thres (> 0 rejects), bounds, verdict, decided, zero (the zero plane)."""
    k = len(nb)
    out = dict(k=k, verdict=False, decided=True, kind="plane")
    if k <= 4:
        return out
    P, m, C = _mean_cov(nb)
    xx, xy, xz, yy, yz, zz = C[0][0], C[0][1], C[0][2], C[1][1], C[1][2], C[2][2]
    w, dots = _best_plane_formula(xx, xy, xz, yy, yz, zz)
    nn2 = sum(t * t for t in w)
    M = max(abs(float(c)) for p in nb for c in p)
    S = max(float(mp.sqrt(sum((p[i] - m[i]) ** 2 for i in range(3)))) for p in P)
    dC = 0.0 if _plane_cov_exact(nb) else 4 * (k + 2) * U * M * S
    if nn2 == 0:
        n = [mp.mpf(0)] * 3
        d = mp.mpf(0)
    else:
        r = mp.sqrt(mpf(nn2))
        n = [mpf(t) / r for t in w]
        d = -sum(n[i] * mpf(m[i]) for i in range(3))
    dist = [sum(n[i] * mpf(p[i]) for i in range(3)) + d for p in P]
    # the normal's sensitivity to the covariance error (FP64 re-evaluation of the same formula, perturbed entry by entry)
    n0 = _unit(w)
    B_n = 64 * U
    if dC > 0:
        base = [float(t) for t in (xx, xy, xz, yy, yz, zz)]
        tot = 0.0
        for j in range(6):
            worst = 0.0
            for sgn in (-1.0, 1.0):
                pc = list(base)
                pc[j] += sgn * dC
                wp, _ = _best_plane_formula(*pc)
                worst = max(worst, float(np.abs(_unit(wp) - n0).max()))
            tot += worst
        B_n += 2 * tot
    if nn2 == 0 and dC == 0:
        B_n = 0.0                                     # every FP64 step is exact: the device must return the zero plane
    margin = max(dist) - mp.mpf(thres)
    B_dist = 2 * B_n * S + 16 * U * M
    verdict = bool(margin <= 0)
    decided = bool(abs(margin) > B_dist) and B_n < 0.5
    out.update(n=np.array([float(t) for t in n]), d=float(d), dist=dist, margin=margin, B_n=B_n, B_dist=B_dist,
               B_d=B_n * M + 8 * U * M, verdict=verdict, decided=decided, zero=(nn2 == 0), dots=dots, M=M, S=S, cov=C)
    return out


def sphere_exact(q, nb, thres=SPHERE_THRES):
    """Sphere test: nb is the nearest neighbour or None.  Valid iff found and the exact squared distance <= thres."""
    if nb is None:
        return dict(kind="sphere", verdict=False, decided=True, counted=True)
    d2 = sum((fr(q[i]) - fr(nb[i])) ** 2 for i in range(3))
    margin = mpf(d2) - mp.mpf(thres)
    dist = float(mp.sqrt(mpf(d2)))
    B = 8 * U * float(d2) + 4 * dist * U * max(max(abs(float(c)) for c in q), max(abs(float(c)) for c in nb))
    # the device's sequence: three differences, then fma(dz, dz, fma(dy, dy, dx * dx)); exact on these inputs => B = 0
    d = [float(q[i]) - float(nb[i]) for i in range(3)]
    ops = [(d[i], fr(q[i]) - fr(nb[i])) for i in range(3)]
    t = d[0] * d[0]
    ops.append((t, fr(d[0]) ** 2))
    for i in (1, 2):
        ex = fr(d[i]) ** 2 + fr(t)
        t = float(ex)                                 # one rounding, as the fma
        ops.append((t, ex))
    if _fp_exact(ops):
        B = 0.0
    decided = bool(abs(margin) > B or B == 0)
    return dict(kind="sphere", d2=d2, margin=margin, B=B, verdict=bool(margin <= 0), decided=decided)


# ----------------------------------------------------------------------------------------------------------------------
# SE(3): closed-form Rodrigues, the left Jacobian and their inverses (Sophus semantics: se3.cuh, ref so3.hpp / se3.hpp)
def _hat(w):
    return mp.matrix([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])


def _vec(a):
    return mp.matrix([mpf(fr(t)) for t in a])


def so3_exp_quat(om):
    """Unit quaternion (w, x, y, z) of exp(hat(om)), exact closed form."""
    th = mp.sqrt(sum(t * t for t in om))
    if th == 0:
        return [mp.mpf(1), mp.mpf(0), mp.mpf(0), mp.mpf(0)]
    s = mp.sin(th / 2) / th
    return [mp.cos(th / 2), s * om[0], s * om[1], s * om[2]]


def quat_rot(q):
    w, x, y, z = q
    return mp.matrix([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def left_jacobian(om):
    th = mp.sqrt(sum(t * t for t in om))
    W = _hat(om)
    if th == 0:
        return mp.eye(3)
    return mp.eye(3) + (1 - mp.cos(th)) / th ** 2 * W + (th - mp.sin(th)) / th ** 3 * (W * W)


def se3_exp(a):
    """exp of (upsilon, omega) with Sophus's semantics, in mpmath: returns (quaternion, R, t).  Below the Taylor switch
    (theta < 1e-10) Sophus uses V = R; the exact left Jacobian is used here and the difference is part of the bound."""
    om = [mpf(fr(t)) for t in a[3:]]
    q = so3_exp_quat(om)
    R = quat_rot(q)
    t = left_jacobian(om) * _vec(a[:3])
    return q, R, t


def exp_bounds(a):
    th = float(np.linalg.norm(np.asarray(a[3:], dtype=np.float64)))
    un = float(np.linalg.norm(np.asarray(a[:3], dtype=np.float64)))
    Bt = 64 * U * max(un, 1e-300) * (1 + th)
    if th < LIE_EPS:
        Bt += th * un
    return 64 * U, Bt


def quat_from_matrix(T):
    """Eigen's Quaternion(Matrix3) (Shoemake) on the exact doubles of a 4x4 (row-major numpy) matrix.  The trace test is
    the FP64 sum the device forms ((m00 + m11) + m22, no FMA possible); the diagonal comparisons are exact."""
    m = [[mpf(fr(T[i][j])) for j in range(3)] for i in range(3)]
    tr = (float(T[0][0]) + float(T[1][1])) + float(T[2][2])
    if tr > 0.0:
        s = mp.sqrt(m[0][0] + m[1][1] + m[2][2] + 1)
        w = s / 2
        s = mp.mpf("0.5") / s
        return [w, (m[2][1] - m[1][2]) * s, (m[0][2] - m[2][0]) * s, (m[1][0] - m[0][1]) * s], -1
    i = 0
    if float(T[1][1]) > float(T[0][0]):
        i = 1
    if float(T[2][2]) > float(T[i][i]):
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    s = mp.sqrt(m[i][i] - m[j][j] - m[k][k] + 1)
    v = [None] * 3
    v[i] = s / 2
    s = mp.mpf("0.5") / s
    w = (m[k][j] - m[j][k]) * s
    v[j] = (m[j][i] + m[i][j]) * s
    v[k] = (m[k][i] + m[i][k]) * s
    return [w, v[0], v[1], v[2]], i


def so3_log_quat(q):
    """Sophus's logAndTheta on an (exact) quaternion: atan form, +-pi / n when |w| < 1e-10 (sign from w > 0)."""
    w, x, y, z = q
    n2 = x * x + y * y + z * z
    if n2 < mp.mpf(LIE_EPS) ** 2:
        k = 2 / w - mp.mpf(2) / 3 * n2 / w ** 3
        th = 2 * n2 / w
    else:
        n = mp.sqrt(n2)
        if abs(w) < mp.mpf(LIE_EPS):
            k = (mp.pi if w > 0 else -mp.pi) / n
        else:
            k = 2 * mp.atan(n / w) / n
        th = k * n
    return [k * x, k * y, k * z], th


def left_jacobian_inv(om):
    th = mp.sqrt(sum(t * t for t in om))
    W = _hat(om)
    if th == 0:
        return mp.eye(3)
    c = (1 - th * mp.sin(th) / (2 * (1 - mp.cos(th)))) / th ** 2
    return mp.eye(3) - W / 2 + c * (W * W)


def se3_log_quat(q, t):
    om, th = so3_log_quat(q)
    # the exact rotation angle of om (|om|), used for V^-1; Sophus's V^-1 depends on theta only through om
    ups = left_jacobian_inv(om) * t
    return [ups[i] for i in range(3)] + om, th


def se3_log(T):
    """log of a 4x4 (row-major numpy) matrix with the device's semantics, exact on its doubles.  Returns (xi, theta, w,
    branch) with branch -1 for the trace branch of the quaternion extraction."""
    q, br = quat_from_matrix(T)
    t = mp.matrix([mpf(fr(T[i][3])) for i in range(3)])
    xi, th = se3_log_quat(q, t)
    return xi, th, q[0], br


def log_bounds(xi, th, w, tnorm):
    amp = 1 + 1 / max(float(mp.pi - abs(th)), 1e-3)
    Bw = 64 * U * amp + (2 * abs(float(w)) if abs(w) < LIE_EPS else 0.0)
    Bu = 256 * U * max(tnorm, 1.0) * amp + (2 * abs(float(w)) * tnorm if abs(w) < LIE_EPS else 0.0)
    return Bw, Bu


def se3_plus(x, d):
    """log(exp(d) * exp(x)) (ref: registration.cpp:162-173): quaternion product, translation a.t + R_a b.t."""
    qa, Ra, ta = se3_exp(d)
    qb, Rb, tb = se3_exp(x)
    w = qa[0] * qb[0] - qa[1] * qb[1] - qa[2] * qb[2] - qa[3] * qb[3]
    xx = qa[0] * qb[1] + qa[1] * qb[0] + qa[2] * qb[3] - qa[3] * qb[2]
    y = qa[0] * qb[2] + qa[2] * qb[0] + qa[3] * qb[1] - qa[1] * qb[3]
    z = qa[0] * qb[3] + qa[3] * qb[0] + qa[1] * qb[2] - qa[2] * qb[1]
    t = ta + Ra * tb
    xi, th = se3_log_quat([w, xx, y, z], t)
    return xi, th, w


def plus_bound(x, d, th, w):
    amp = 1 + 1 / max(float(mp.pi - abs(th)), 1e-3)
    B = 1024 * U * (1 + float(np.linalg.norm(x[:3])) + float(np.linalg.norm(d[:3]))) * amp
    thx, thd = float(np.linalg.norm(x[3:])), float(np.linalg.norm(d[3:]))
    for th_, un in ((thx, float(np.linalg.norm(x[:3]))), (thd, float(np.linalg.norm(d[:3])))):
        if th_ < LIE_EPS:
            B += th_ * un
    if abs(w) < LIE_EPS:
        B += 2 * abs(float(w)) * (1 + float(np.linalg.norm(x[:3])) + float(np.linalg.norm(d[:3])))
    return B


def ortho_error(R):
    """max |R R^T - I| over the 9 entries, exact on the doubles."""
    m = [[fr(R[i][j]) for j in range(3)] for i in range(3)]
    return max(abs(sum(m[i][k] * m[j][k] for k in range(3)) - (1 if i == j else 0)) for i in range(3) for j in range(3))
