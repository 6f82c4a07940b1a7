"""CPU restatement of the pose graph (include/tloam_b200.h, "Pose graph"; libtloam_b200_pg.so) in FP64:

    edges:    odometry (k - 1, k), Z = O_{k-1}^-1 O_k, Omega_odom;  loop (candidate, query), Z = T_cand_query, Omega_loop
    residual: r = log(Z^-1 T_i^-1 T_j) (se3.cuh's Sophus log, (upsilon, omega));  cost = sum r^T Omega r
    step:     T_k <- exp(delta_k) T_k, node 0 fixed;  J_j = Ad(T_j^-1), J_i = -J_j;  H delta = b = -sum J^T Omega r
    solve:    H = M + B^T Omega_loop B (M the chain), by a scipy sparse direct solve of H (optimize's default), or by
              Woodbury as the device solves it: Y = M^-1 B^T and u = M^-1 b by a sparse LU of M, S = Omega_loop^-1 + B Y
              by a dense Cholesky, delta = u - Y S^-1 B u
    stop:     a step below both eps converges (applied); else a cost not <= the current one reverts it (COST_INCREASED);
              else accepted, up to max_iterations;  every run starts from the odometry poses

H is ill-conditioned on KITTI-sized graphs (a 4 540-block chain with sigmas 20x apart).  The sparse direct solve of H is at
its backward-error floor there (iterative refinement moves its first step's cost by 3e-9 relative on seq 00), while the
Woodbury form with a sparse LU of M loses up to 2e-2 of the first step's cost, so the GPU tests compare against the direct
solve; the device's block LDL^T of the chain and fixed-order reductions keep it within 2e-7 of it.  exp / log are
deskew_oracle's (Sophus' formulas)."""
import numpy as np
import scipy.linalg
import scipy.sparse as sp
import scipy.sparse.linalg as spl

from deskew_oracle import se3_exp, se3_log

CONVERGED, ITERATION_LIMIT, COST_INCREASED, SINGULAR, NO_LOOPS = range(5)


def config(**overrides):
    """tloam_b200_pose_graph_default_config, with overrides"""
    c = dict(sigma_odom_translation=0.02, sigma_odom_rotation=0.001, sigma_loop_translation=0.3, sigma_loop_rotation=0.002,
             max_iterations=20, eps_translation=1e-4, eps_rotation=1e-6)
    c.update(overrides)
    return c


def weights(cfg):
    """the diagonals of Omega_odom and Omega_loop"""
    wo = np.array([1.0 / cfg["sigma_odom_translation"] ** 2] * 3 + [1.0 / cfg["sigma_odom_rotation"] ** 2] * 3)
    wl = np.array([1.0 / cfg["sigma_loop_translation"] ** 2] * 3 + [1.0 / cfg["sigma_loop_rotation"] ** 2] * 3)
    return wo, wl


def inv_mul(A, B):
    """A^-1 B of rigid 4 x 4 matrices: R_A^T R_B, R_A^T (t_B - t_A)"""
    C = np.eye(4)
    C[:3, :3] = A[:3, :3].T @ B[:3, :3]
    C[:3, 3] = A[:3, :3].T @ (B[:3, 3] - A[:3, 3])
    return C


def exp4(xi):
    R, t = se3_exp(np.asarray(xi, dtype=np.float64))
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T


def hat(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def ad_inv(T):
    """Ad(T^-1) = [[R, [t]x R], [0, R]] with R = R_T^T, t = -R_T^T t_T"""
    R = T[:3, :3].T
    t = -R @ T[:3, 3]
    A = np.zeros((6, 6))
    A[:3, :3], A[:3, 3:], A[3:, 3:] = R, hat(t) @ R, R
    return A


def residual(Ti, Tj, Z):
    """r = log(Z^-1 T_i^-1 T_j)"""
    return se3_log(inv_mul(Z, inv_mul(Ti, Tj)))


def edges(O, loops):
    """[(i, j, Z, kind)]: the odometry chain, then the loop edges (kind 0: odometry, 1: loop)"""
    return [(k - 1, k, inv_mul(O[k - 1], O[k]), 0) for k in range(1, len(O))] + [(i, j, Z, 1) for i, j, Z in loops]


def linearize(T, E, cfg):
    """per edge (r, A = Ad(T_j^-1)) and the cost sum r^T Omega r"""
    w = weights(cfg)
    rs, As, cost = [], [], 0.0
    for i, j, Z, kind in E:
        r = residual(T[i], T[j], Z)
        rs.append(r)
        As.append(ad_inv(T[j]))
        cost += float(np.sum(w[kind] * r * r))
    return rs, As, cost


def _blocks(N, E, rs, As, cfg):
    """the chain M (sparse, nodes 1..N-1), B (6 L x 6 (N - 1), sparse), b = -g"""
    w = weights(cfg)
    n = 6 * (N - 1)
    g = np.zeros(6 * N)
    rows, cols, vals = [], [], []
    brows, bcols, bvals = [], [], []
    nl = 0
    for (i, j, Z, kind), r, A in zip(E, rs, As):
        q = A.T @ (w[kind] * r)
        g[6 * j:6 * j + 6] += q
        g[6 * i:6 * i + 6] -= q
        if kind == 0:
            P = A.T @ (w[0][:, None] * A)
            for a, sa in ((i, 1.0), (j, -1.0)):
                for c, sc in ((i, 1.0), (j, -1.0)):
                    if a and c:
                        ii, jj = np.meshgrid(np.arange(6) + 6 * (a - 1), np.arange(6) + 6 * (c - 1), indexing="ij")
                        rows.append(ii.ravel()); cols.append(jj.ravel()); vals.append((sa * sc * P).ravel())
        else:
            for node, sgn in ((i, -1.0), (j, 1.0)):
                if node:
                    ii, jj = np.meshgrid(np.arange(6) + 6 * nl, np.arange(6) + 6 * (node - 1), indexing="ij")
                    brows.append(ii.ravel()); bcols.append(jj.ravel()); bvals.append((sgn * A).ravel())
            nl += 1
    M = sp.csc_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))
    if nl and brows:
        B = sp.csr_matrix((np.concatenate(bvals), (np.concatenate(brows), np.concatenate(bcols))), shape=(6 * nl, n))
    else:
        B = sp.csr_matrix((6 * nl, n))
    return M, B, -g[6:]


def solve_woodbury(N, E, rs, As, cfg):
    """delta (6 (N - 1)) by Woodbury; None when the Cholesky of S fails"""
    _, wl = weights(cfg)
    M, B, b = _blocks(N, E, rs, As, cfg)
    lu = spl.splu(M)
    Y = lu.solve(np.ascontiguousarray(B.T.toarray()))
    u = lu.solve(b)
    L = B.shape[0] // 6
    S = np.diag(np.tile(1.0 / wl, L)) + B @ Y
    try:
        f = scipy.linalg.cho_factor(S, lower=True)
    except np.linalg.LinAlgError:
        return None
    return u - Y @ scipy.linalg.cho_solve(f, B @ u)


def solve_dense(N, E, rs, As, cfg):
    """delta by np.linalg.solve of the assembled H (for checks on small graphs)"""
    _, wl = weights(cfg)
    M, B, b = _blocks(N, E, rs, As, cfg)
    L = B.shape[0] // 6
    H = M.toarray() + B.T.toarray() @ np.diag(np.tile(wl, L)) @ B.toarray()
    return np.linalg.solve(H, b)


def solve_sparse(N, E, rs, As, cfg):
    """delta by a scipy sparse direct solve of the assembled H"""
    _, wl = weights(cfg)
    M, B, b = _blocks(N, E, rs, As, cfg)
    L = B.shape[0] // 6
    H = (M + B.T @ sp.diags(np.tile(wl, L)) @ B).tocsc()
    return spl.spsolve(H, b)


def optimize(O, loops, cfg, solve=solve_sparse):
    """O: N odometry poses (4 x 4); loops: [(candidate, query, Z)].  A dict with T (N x 4 x 4), iterations, termination,
    costs (the cost at the odometry poses, then after every accepted step), initial_cost, final_cost, step_translation,
    step_rotation"""
    O = [np.asarray(x, dtype=np.float64) for x in O]
    N = len(O)
    out = dict(T=np.array(O), iterations=0, termination=NO_LOOPS, costs=[], initial_cost=0.0, final_cost=0.0,
               step_translation=0.0, step_rotation=0.0)
    if not loops:
        return out
    E = edges(O, loops)
    T = [x.copy() for x in O]
    rs, As, cost = linearize(T, E, cfg)
    costs = [cost]
    it, term, st, sr = 0, ITERATION_LIMIT, 0.0, 0.0
    while True:
        d = solve(N, E, rs, As, cfg)
        if d is None:
            term = SINGULAR
            break
        d = d.reshape(N - 1, 6)
        Tn = [T[0]] + [exp4(d[k - 1]) @ T[k] for k in range(1, N)]
        st, sr = float(np.abs(d[:, :3]).max()), float(np.abs(d[:, 3:]).max())
        rn, An, cn = linearize(Tn, E, cfg)
        small = st < cfg["eps_translation"] and sr < cfg["eps_rotation"]
        if not small and not cn <= cost:
            term = COST_INCREASED
            break
        T, rs, As, cost = Tn, rn, An, cn
        costs.append(cost)
        it += 1
        if small:
            term = CONVERGED
            break
        if it >= cfg["max_iterations"]:
            break
    out.update(T=np.array(T), iterations=it, termination=term, costs=costs, initial_cost=costs[0], final_cost=cost,
               step_translation=st, step_rotation=sr)
    return out


def relative_error(T, T_ref):
    """(|dt| m, d_theta rad) of T^-1 . T_ref; the angle by atan2 of sin and cos, which, unlike arccos of the trace, resolves
    angles below 1e-8 rad"""
    d = inv_mul(T, T_ref)
    R = d[:3, :3]
    s = 0.5 * np.linalg.norm([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    return float(np.linalg.norm(d[:3, 3])), float(np.arctan2(s, (np.trace(R) - 1.0) / 2.0))
