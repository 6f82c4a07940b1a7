"""CPU restatement of the robust pose graph (include/tloam_b200.h, "Robust pose graph"; libtloam_b200_pgr.so with the
weighted stages of libtloam_b200_pg.so) in FP64, on top of pose_graph_oracle:

    residual: rho_l = r_l^T Omega_loop r_l of loop edge l, unweighted
    weights:  loop edge l's r and A = Ad(T_j^-1) scaled by sqrt(w_l), as k_pg_linearize stores them, so pose_graph_oracle's
              _blocks / solve_sparse assemble H = M + B^T (W Omega_loop) B and g = sum w A^T Omega r unchanged, and the
              cost is sum_odom r^T Omega r + sum_loop w_l r^T Omega r
    TLS:      T-LOAM's updateWeight with c2 = chi2_threshold (ref: src/models/registration/registration.cpp:858-876), with
              w = 1 at rho = 0
    schedule: stage 0 = pose_graph_oracle.optimize from the odometry poses; max rho <= c2 stops (ALL_INLIERS); else
              mu_0 = c2 / (2 max rho - c2), then per outer step the weights at the current poses, a stage of up to
              inner_iterations steps from them, mu <- gnc_factor mu; an all-0/1 update is followed by a last stage of up to
              max_iterations steps (CONVERGED); max_outer_iterations outer steps stop it (OUTER_LIMIT)

With every weight 1, the scaling is by exactly 1.0, so stage 0 is pose_graph_oracle.optimize bit for bit."""
import numpy as np

import pose_graph_oracle as pgo

CONVERGED, OUTER_LIMIT, ALL_INLIERS, SINGULAR, NO_LOOPS = range(5)


def config(**overrides):
    """tloam_b200_pose_graph_robust_default_config, with overrides"""
    c = dict(chi2_threshold=16.81, gnc_factor=1.4, inner_iterations=2, max_outer_iterations=100)
    c.update(overrides)
    return c


def residuals(T, loops, cfg):
    """rho_l = r_l^T Omega_loop r_l at the poses T"""
    _, wl = pgo.weights(cfg)
    return np.array([float(np.sum(wl * r * r)) for r in (pgo.residual(T[i], T[j], Z) for i, j, Z in loops)])


def tls(rho, mu, c2):
    """the TLS weights at mu: 0 at rho >= th1 = (mu + 1) / mu c2, 1 at rho <= th2 = mu / (mu + 1) c2 and at rho = 0,
    sqrt(c2 mu (mu + 1) / rho) - mu between"""
    rho = np.asarray(rho, dtype=np.float64)
    th1, th2 = (mu + 1.0) / mu * c2, mu / (mu + 1.0) * c2
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        mid = np.sqrt(c2 * mu * (mu + 1.0) / rho) - mu
    w = np.where(rho >= th1, 0.0, np.where(rho <= th2, 1.0, mid))
    w[rho == 0.0] = 1.0
    return w


def linearize(T, E, cfg, lw):
    """pose_graph_oracle.linearize with loop edge l's r and A scaled by sqrt(lw[l])"""
    w = pgo.weights(cfg)
    rs, As, cost, l = [], [], 0.0, 0
    for i, j, Z, kind in E:
        r, A = pgo.residual(T[i], T[j], Z), pgo.ad_inv(T[j])
        if kind:
            s = np.sqrt(lw[l])
            A, r, l = A * s, r * s, l + 1
        rs.append(r)
        As.append(A)
        cost += float(np.sum(w[kind] * r * r))
    return rs, As, cost


def stage(E, T0, lw, cfg, max_iterations, solve=pgo.solve_sparse):
    """up to max_iterations weighted Gauss-Newton steps from T0 under pose_graph_oracle.optimize's rules"""
    N = len(T0)
    T = [x.copy() for x in T0]
    rs, As, cost = linearize(T, E, cfg, lw)
    costs = [cost]
    it, term, st, sr = 0, pgo.ITERATION_LIMIT, 0.0, 0.0
    while True:
        d = solve(N, E, rs, As, cfg)
        if d is None:
            term = pgo.SINGULAR
            break
        d = d.reshape(N - 1, 6)
        Tn = [T[0]] + [pgo.exp4(d[k - 1]) @ T[k] for k in range(1, N)]
        st, sr = float(np.abs(d[:, :3]).max()), float(np.abs(d[:, 3:]).max())
        rn, An, cn = linearize(Tn, E, cfg, lw)
        small = st < cfg["eps_translation"] and sr < cfg["eps_rotation"]
        if not small and not cn <= cost:
            term = pgo.COST_INCREASED
            break
        T, rs, As, cost = Tn, rn, An, cn
        costs.append(cost)
        it += 1
        if small:
            term = pgo.CONVERGED
            break
        if it >= max_iterations:
            break
    return dict(T=T, iterations=it, termination=term, costs=costs, initial_cost=costs[0], final_cost=cost,
                step_translation=st, step_rotation=sr)


def optimize_robust(O, loops, cfg, rcfg, solve=pgo.solve_sparse):
    """O: N odometry poses; loops: [(candidate, query, Z)]; cfg: pose_graph_oracle.config; rcfg: config.  A dict with T,
    iterations (over every stage), termination (the last stage's), initial_cost (stage 0's), final_cost (the last stage's,
    weighted), step_translation, step_rotation, outer_iterations, gnc_termination, mu_final, inliers, rejected, weights,
    and stages: per stage (weights, its result)"""
    O = [np.asarray(x, dtype=np.float64) for x in O]
    L = len(loops)
    out = dict(T=np.array(O), iterations=0, termination=pgo.NO_LOOPS, initial_cost=0.0, final_cost=0.0,
               step_translation=0.0, step_rotation=0.0, outer_iterations=0, gnc_termination=NO_LOOPS, mu_final=0.0,
               inliers=0, rejected=0, weights=np.ones(L), stages=[])
    if not loops:
        return out
    E = pgo.edges(O, loops)
    c2 = rcfg["chi2_threshold"]
    w = np.ones(L)
    st = stage(E, O, w, cfg, cfg["max_iterations"], solve)
    stages = [(w, st)]
    iters, gnc, outer, mu, inl, rej = st["iterations"], None, 0, 0.0, L, 0
    if st["termination"] == pgo.SINGULAR:
        gnc = SINGULAR
    else:
        rho = residuals(st["T"], loops, cfg)
        mx = max(0.0, float(rho.max()))
        if mx <= c2:
            gnc = ALL_INLIERS
        else:
            mu = c2 / (2.0 * mx - c2)
            if mu <= 0.0:
                mu = 1e-10
    mu_final = 0.0
    while gnc is None:
        w = tls(rho, mu, c2)
        outer += 1
        mu_final, inl, rej = mu, int(np.sum(w == 1.0)), int(np.sum(w == 0.0))
        if inl + rej == L:
            st = stage(E, st["T"], w, cfg, cfg["max_iterations"], solve)
            stages.append((w, st))
            iters += st["iterations"]
            gnc = SINGULAR if st["termination"] == pgo.SINGULAR else CONVERGED
            break
        st = stage(E, st["T"], w, cfg, rcfg["inner_iterations"], solve)
        stages.append((w, st))
        iters += st["iterations"]
        if st["termination"] == pgo.SINGULAR:
            gnc = SINGULAR
        elif outer >= rcfg["max_outer_iterations"]:
            gnc = OUTER_LIMIT
        else:
            rho = residuals(st["T"], loops, cfg)
            mu = rcfg["gnc_factor"] * mu
    out.update(T=np.array(st["T"]), iterations=iters, termination=st["termination"], initial_cost=stages[0][1]["initial_cost"],
               final_cost=st["final_cost"], step_translation=st["step_translation"], step_rotation=st["step_rotation"],
               outer_iterations=outer, gnc_termination=gnc, mu_final=mu_final, inliers=inl, rejected=rej, weights=w,
               stages=stages)
    return out
