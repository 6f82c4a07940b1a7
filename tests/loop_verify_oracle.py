"""CPU restatement of loop verification (include/tloam_b200.h, "Loop verification"; libtloam_b200_loopv.so), step by step
in FP64:

    keyframe = VoxelDownSample(voxel) of the scan's finite rows at pose I (the global map's per-frame block)
    pass at T = (R, t):  p = R q + t for every q in Q;  match = the nearest m in M by d2 (lowest index on a tie);
                         inlier iff d2 <= r * r
    step:                e = p - m, J = [I, -[p]x];  H = sum J^T J, g = sum J^T e;  delta = -H^-1 g (LDL^T);
                         T <- exp(delta) . T
    radius:              after a step with |upsilon| < eps_t and |omega| < eps_r: converged at r == fine, else
                         r <- max(r / 2, fine)
    result:              one more pass at the final T with r = fine: inliers, rmse, fitness = mean d2 over all of Q

p and d2 are rounded exactly as the device rounds them (numpy does not contract a * b + c), so the first pass -- both sides
start from the same T -- is bit-identical.  Later T differ from the device's in the last bits (the reduction order and
exp's sin / cos), which the GPU tests bound at 1e-9.  exp is deskew_oracle.se3_exp (Sophus' formulas, pinned to expm)."""
import numpy as np

import global_map_oracle as gmo
from deskew_oracle import se3_exp

CONVERGED, ITERATION_LIMIT, FEW_INLIERS, SINGULAR, EMPTY = range(5)


def config(**overrides):
    """tloam_b200_loop_verify_default_config, with overrides"""
    c = dict(voxel=0.5, corr_dist_coarse=4.0, corr_dist_fine=1.0, max_iterations=40, eps_translation=1e-4, eps_rotation=1e-5,
             max_fitness=1.0)
    c.update(overrides)
    return c


def keyframe(oracle, scan, voxel):
    """the keyframe of a scan (n x 3, NaN / Inf rows allowed): the global map's frame block at pose I"""
    return gmo.frame_block(oracle, gmo.transform(scan, np.eye(4)), voxel)


def transform(Q, R, t):
    """p = R q + t, each component ((R[r,0] qx + R[r,1] qy) + R[r,2] qz) + t[r], every operation rounded"""
    Q = np.asarray(Q, dtype=np.float64).reshape(-1, 3)
    x, y, z = Q[:, 0], Q[:, 1], Q[:, 2]
    return np.column_stack([((R[r, 0] * x + R[r, 1] * y) + R[r, 2] * z) + t[r] for r in range(3)])


def nearest(P, M, chunk=512):
    """(index, d2) of the nearest row of M for every row of P: d2 = ((px - mx)^2 + (py - my)^2) + (pz - mz)^2, the lowest
    index on a tie (argmin takes the first minimum); an exhaustive search"""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    idx = np.zeros(len(P), dtype=np.int64)
    d2 = np.zeros(len(P))
    for a in range(0, len(P), chunk):
        p = P[a:a + chunk]
        dx = p[:, None, 0] - M[None, :, 0]
        dy = p[:, None, 1] - M[None, :, 1]
        dz = p[:, None, 2] - M[None, :, 2]
        d = (dx * dx + dy * dy) + dz * dz
        j = np.argmin(d, axis=1)
        idx[a:a + chunk] = j
        d2[a:a + chunk] = d[np.arange(len(p)), j]
    return idx, d2


def jacobian(P):
    """(n, 3, 6): J = [I, -[p]x] of the left perturbation exp(delta) . p"""
    J = np.zeros((len(P), 3, 6))
    J[:, [0, 1, 2], [0, 1, 2]] = 1.0
    px, py, pz = P[:, 0], P[:, 1], P[:, 2]
    J[:, 0, 4], J[:, 0, 5] = pz, -py
    J[:, 1, 3], J[:, 1, 5] = -pz, px
    J[:, 2, 3], J[:, 2, 4] = py, -px
    return J


def normal_equations(P, E):
    """H = sum J^T J, g = sum J^T e over the rows of P with residuals E"""
    J = jacobian(P)
    return np.einsum("nki,nkj->ij", J, J), np.einsum("nki,nk->i", J, E)


def ldlt_solve(H, b):
    """y with H y = b by LDL^T (ldlt6.cuh's order of operations); None when a pivot is not positive and finite or y is not
    finite"""
    L, d = np.eye(6), np.zeros(6)
    for j in range(6):
        d[j] = H[j, j] - sum(L[j, k] * L[j, k] * d[k] for k in range(j))
        if not (d[j] > 0.0 and np.isfinite(d[j])):
            return None
        for i in range(j + 1, 6):
            L[i, j] = (H[j, i] - sum(L[i, k] * L[j, k] * d[k] for k in range(j))) / d[j]
    z = np.zeros(6)
    for i in range(6):
        z[i] = b[i] - sum(L[i, k] * z[k] for k in range(i))
    y = np.zeros(6)
    for i in range(5, -1, -1):
        y[i] = z[i] / d[i] - sum(L[k, i] * y[k] for k in range(i + 1, 6))
    return y if np.isfinite(y).all() else None


def gauss_newton_step(P, Mm):
    """delta = -H^-1 g for the pairs (P, Mm); None when the solve fails"""
    H, g = normal_equations(P, P - Mm)
    y = ldlt_solve(H, g)
    return None if y is None else -y


def apply(delta, R, t):
    """exp(delta) . (R, t)"""
    Re, te = se3_exp(delta)
    return Re @ R, Re @ t + te


def run(Q, M, guess, cfg):
    """the verification of keyframe Q against keyframe M from guess (4 x 4): a dict with T, iterations, termination, inliers,
    rmse, fitness, accepted and passes (pass k = (index, d2) at the k-th iterate of T; the last one at the final T)"""
    Q = np.asarray(Q, dtype=np.float64).reshape(-1, 3)
    M = np.asarray(M, dtype=np.float64).reshape(-1, 3)
    guess = np.asarray(guess, dtype=np.float64)
    R, t = guess[:3, :3].copy(), guess[:3, 3].copy()
    out = dict(T=guess.copy(), iterations=0, termination=EMPTY, inliers=0, rmse=0.0, fitness=np.inf, accepted=False, passes=[])
    if len(Q) == 0 or len(M) == 0:
        return out
    fine = cfg["corr_dist_fine"]
    r, it, term, passes = cfg["corr_dist_coarse"], 0, ITERATION_LIMIT, []
    while True:
        P = transform(Q, R, t)
        idx, d2 = nearest(P, M)
        passes.append((idx, d2))
        inl = d2 <= r * r
        if inl.sum() < 6:
            term = FEW_INLIERS
            break
        delta = gauss_newton_step(P[inl], M[idx[inl]])
        if delta is None:
            term = SINGULAR
            break
        R, t = apply(delta, R, t)
        it += 1
        if np.sqrt(np.sum(delta[:3] ** 2)) < cfg["eps_translation"] and np.sqrt(np.sum(delta[3:] ** 2)) < cfg["eps_rotation"]:
            if r == fine:
                term = CONVERGED
                break
            r = max(r * 0.5, fine)
        if it >= cfg["max_iterations"]:
            break
    if term in (CONVERGED, ITERATION_LIMIT):                       # a stop without a step already searched at this T
        idx, d2 = nearest(transform(Q, R, t), M)
        passes.append((idx, d2))
    idx, d2 = passes[-1]
    inl = d2 <= fine * fine
    n = int(inl.sum())
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    fitness = float(np.mean(d2))
    out.update(T=T, iterations=it, termination=term, inliers=n, rmse=float(np.sqrt(np.sum(d2[inl]) / n)) if n else 0.0,
               fitness=fitness, accepted=term == CONVERGED and fitness <= cfg["max_fitness"], passes=passes)
    return out


def relative_error(T, T_ref):
    """(|dt| m, d_theta rad) of T^-1 . T_ref"""
    d = np.linalg.inv(T) @ T_ref
    return float(np.linalg.norm(d[:3, 3])), float(np.arccos(np.clip((np.trace(d[:3, :3]) - 1.0) / 2.0, -1.0, 1.0)))
