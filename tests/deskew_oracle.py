"""CPU restatement of deskewing (include/tloam_b200.h, "Deskewing"; libtloam_b200_deskew.so), literal and in FP64:

    t_end = max of the finite t_i;  xi = log(last^-1 . curr);  s_i = (t_i - t_end) / P;  p'_i = exp(s_i . xi) . p_i

with the SE(3) exp / log of se3.cuh (Sophus' formulas: half-angle quaternion with its Taylor branch below theta = 1e-10,
translation through the left Jacobian).  s_i = 0 for a non-finite t_i or when no time is finite, and a row whose s_i . xi
is all zero is copied as it is.  test_deskew.py pins exp against scipy.linalg.expm of the 4 x 4 twist."""
import numpy as np

EPS = 1e-10                                                    # Sophus' kEpsilon (se3.cuh kLieEps)


def quat_to_rot(w, x, y, z):
    """rotation matrices (..., 3, 3) of unit quaternions, in se3.cuh's expression"""
    x2, y2, z2 = x + x, y + y, z + z
    wx, wy, wz, xx, xy, xz, yy, yz, zz = x2 * w, y2 * w, z2 * w, x2 * x, y2 * x, z2 * x, y2 * y, z2 * y, z2 * z
    return np.stack([np.stack([1.0 - (yy + zz), xy - wz, xz + wy], -1),
                     np.stack([xy + wz, 1.0 - (xx + zz), yz - wx], -1),
                     np.stack([xz - wy, yz + wx, 1.0 - (xx + yy)], -1)], -2)


def se3_exp(a):
    """a (..., 6) = (upsilon, omega) -> (R (..., 3, 3), t (..., 3))"""
    a = np.asarray(a, dtype=np.float64)
    u, om = a[..., :3], a[..., 3:]
    th2 = np.sum(om * om, axis=-1)
    small = th2 < EPS * EPS
    theta = np.where(small, 0.0, np.sqrt(th2))
    safe = np.where(small, 1.0, theta)
    kim = np.where(small, 0.5 - th2 / 48.0 + th2 * th2 / 3840.0, np.sin(0.5 * safe) / safe)
    kre = np.where(small, 1.0 - th2 / 8.0 + th2 * th2 / 384.0, np.cos(0.5 * safe))
    R = quat_to_rot(kre, kim * om[..., 0], kim * om[..., 1], kim * om[..., 2])
    # V = I + c1 W + c2 W^2 (theta >= eps), V = R below (Sophus)
    s = 2.0 * kim * safe * kre
    th2s = np.where(small, 1.0, th2)
    c1 = 2.0 * (kim * safe) ** 2 / th2s
    c2 = (safe - s) / (th2s * safe)
    w = np.cross(om, u)
    v = np.cross(om, w)
    t_big = u + c1[..., None] * w + c2[..., None] * v
    t_small = np.einsum("...ij,...j->...i", R, u)
    return R, np.where(small[..., None], t_small, t_big)


def matrix_to_quat(T):
    """Eigen's Quaternion(Matrix3) (Shoemake, branch on the trace) of a 4 x 4 rigid matrix -> (w, x, y, z)"""
    R = T[:3, :3]
    tr = np.trace(R)
    if tr > 0.0:
        s = np.sqrt(tr + 1.0)
        w, s = 0.5 * s, 0.5 / s
        return w, (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s
    i = 0
    if R[1, 1] > R[0, 0]:
        i = 1
    if R[2, 2] > R[i, i]:
        i = 2
    j, k = (i + 1) % 3, (i + 2) % 3
    s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
    v = [0.0, 0.0, 0.0]
    v[i], s = 0.5 * s, 0.5 / s
    w = (R[k, j] - R[j, k]) * s
    v[j] = (R[j, i] + R[i, j]) * s
    v[k] = (R[k, i] + R[i, k]) * s
    return w, v[0], v[1], v[2]


def se3_log(T):
    """4 x 4 rigid matrix -> (upsilon, omega)"""
    w, x, y, z = matrix_to_quat(T)
    n2 = x * x + y * y + z * z
    if n2 < EPS * EPS:
        k = 2.0 / w - (2.0 / 3.0) * n2 / (w * w * w)
        theta = 2.0 * n2 / w
    else:
        n = np.sqrt(n2)
        k = (np.pi if w > 0.0 else -np.pi) / n if abs(w) < EPS else 2.0 * np.arctan(n / w) / n
        theta = k * n
    om = np.array([k * x, k * y, k * z])
    c = 1.0 / 12.0 if abs(theta) < EPS else (1.0 - 0.5 * theta * w / np.sqrt(n2)) / (theta * theta)
    t = T[:3, 3]
    wv = np.cross(om, t)
    return np.concatenate([t - 0.5 * wv + c * np.cross(om, wv), om])


def increment(last, curr):
    """xi = log(last^-1 . curr): the constant-velocity increment of the pose history"""
    Rl, tl = last[:3, :3], last[:3, 3]
    step = np.eye(4)
    step[:3, :3] = Rl.T @ curr[:3, :3]
    step[:3, 3] = Rl.T @ (curr[:3, 3] - tl)
    return se3_log(step)


def t_end(times):
    """the largest finite time, or None"""
    t = np.asarray(times, dtype=np.float64)
    fin = np.isfinite(t)
    return float(t[fin].max()) if fin.any() else None


def deskew(xyz, times, period, last, curr):
    """the corrected scan (n x 3) of the raw scan xyz with per-row times over the frame period"""
    xyz = np.asarray(xyz, dtype=np.float64)
    t = np.asarray(times, dtype=np.float64)
    xi = increment(np.asarray(last, dtype=np.float64), np.asarray(curr, dtype=np.float64))
    te = t_end(t)
    with np.errstate(invalid="ignore"):
        s = np.where(np.isfinite(t), t - te, 0.0) / period if te is not None else np.zeros(len(t))
    v = s[:, None] * xi[None, :]
    moves = (v != 0.0).any(axis=1)
    out = xyz.copy()
    if moves.any():
        R, tt = se3_exp(v[moves])
        with np.errstate(invalid="ignore", over="ignore"):
            out[moves] = np.einsum("nij,nj->ni", R, xyz[moves]) + tt
    return out
