"""numpy restatement of the loop-corrected global map (include/tloam_b200.h "Loop-corrected global map"; k_gmc_* in
tloam_b200/csrc/map_correct.cu), bit for bit.

Poses are 4 x 4 float64 arrays (A[r, c]).  Every product and sum below is one numpy float64 operation, rounded on its own,
in the order the header states; nothing is fused, so the device's __dmul_rn / __dadd_rn / __dsub_rn give the same bits."""
import numpy as np

EYE = np.eye(4)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def _dot3(a0, b0, a1, b1, a2, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def compose(A, B):
    """A B of rigid poses: R_A R_B, R_A t_B + t_A; bottom row (0, 0, 0, 1)"""
    C = np.zeros((4, 4))
    for r in range(3):
        for c in range(3):
            C[r, c] = _dot3(A[r, 0], B[0, c], A[r, 1], B[1, c], A[r, 2], B[2, c])
        C[r, 3] = _dot3(A[r, 0], B[0, 3], A[r, 1], B[1, 3], A[r, 2], B[2, 3]) + A[r, 3]
    C[3, 3] = 1.0
    return C


def mul_inv(A, B):
    """A B^-1 in tloam_b200_pose_graph_correction's order: R = R_A R_B^T, t = t_A - R t_B"""
    C = np.zeros((4, 4))
    for r in range(3):
        for c in range(3):
            C[r, c] = _dot3(A[r, 0], B[c, 0], A[r, 1], B[c, 1], A[r, 2], B[c, 2])
    for r in range(3):
        C[r, 3] = A[r, 3] - _dot3(C[r, 0], B[0, 3], C[r, 1], B[1, 3], C[r, 2], B[2, 3])
    C[3, 3] = 1.0
    return C


def apply(C, O):
    """C O, or O itself when C is the identity bit for bit"""
    return np.array(O, dtype=np.float64) if same_bits(C, EYE) else compose(C, O)


def correction(T_opt, O_nodes):
    """the map -> odom correction: Delta of the last node the optimisation covered (T_opt: its n_opt poses), I without one"""
    return mul_inv(T_opt[-1], O_nodes[len(T_opt) - 1]) if len(T_opt) else EYE.copy()


def delta(k, T_opt, O_nodes):
    if k < 0:
        return EYE.copy()
    if k < len(T_opt):
        return mul_inv(T_opt[k], O_nodes[k])
    return correction(T_opt, O_nodes)


def transform_points(M, p):
    """x' = ((M00 x + M01 y) + M02 z) + M03 per row of p (n x 3)"""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    return np.stack([((M[r, 0] * x + M[r, 1] * y) + M[r, 2] * z) + M[r, 3] for r in range(3)], axis=1)


def correct(points, offsets, O, P, nodes, T_opt, O_nodes):
    """tloam_b200_global_map_correct: returns (points, P) after the call and the map -> odom correction M it stores.
    points (n x 3), offsets (frames + 1), O / P (frames x 4 x 4) the frame tables, nodes (frames), T_opt the last
    optimisation's poses (empty: none, or NO_LOOPS), O_nodes every node's odometry pose"""
    points = np.array(points, dtype=np.float64)
    P = np.array(P, dtype=np.float64)
    for f, k in enumerate(nodes):
        C = apply(delta(int(k), T_opt, O_nodes), O[f])
        if same_bits(C, P[f]):
            continue
        a, b = int(offsets[f]), int(offsets[f + 1])
        points[a:b] = transform_points(mul_inv(C, P[f]), points[a:b])
        P[f] = C
    return points, P, correction(T_opt, O_nodes)


def append_pose(M, O_f):
    """P_f of a tracked append: M O_f (a copy when M is I bit for bit)"""
    return apply(M, O_f)
