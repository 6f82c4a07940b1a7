"""numpy restatement of the occupancy grid of the global map (include/tloam_b200.h "Occupancy grid"; k_occ_* in
tloam_b200/csrc/occupancy.cu), bit for bit.

Every product, sum, quotient and square root below is one numpy float64 operation, rounded on its own, in the order the
header states; nothing is fused, so the device's __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn give the same
bits.  The sector rule is map_dynamic_oracle's column rule (Scan Context's sector rule).

Two forms: the vectorised one the GPU tests use, and a literal per-row / per-cell transcription the CPU tests pin it to.
Poses are 4 x 4 float64 arrays (A[r, c])."""
import math

import numpy as np

import map_dynamic_oracle as mdo
import scan_context_oracle as sco

DEFAULT = dict(resolution=0.1, n_cols=1024, z_lo=-1.2, z_hi=0.5, min_range=3.0, max_range=30.0, free_margin=0.1)
MAX_CELLS = 1 << 28


def config(**overrides):
    c = dict(DEFAULT)
    c.update(overrides)
    return c


def window(cfg):
    """W = (max_range + max(|z_lo|, |z_hi|)) + resolution"""
    return (cfg["max_range"] + max(abs(cfg["z_lo"]), abs(cfg["z_hi"]))) + cfg["resolution"]


# ---- vectorised ------------------------------------------------------------------------------------------------------
def _rho(x, y):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.sqrt(x * x + y * y)


def scan2d(scan, cfg, D=None):
    """(obstacles (n_cols, 3), floors (n_cols,)) of one append's sensor-frame rows; NaN where absent"""
    D = sco.boundaries(cfg["n_cols"]) if D is None else D
    p = np.asarray(scan, dtype=np.float64).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    rho = _rho(x, y)
    used = np.isfinite(p).all(axis=1) & (rho >= cfg["min_range"]) & (rho <= cfg["max_range"])
    j = mdo.columns(np.where(used, x, 0.0), np.where(used, y, 0.0), D, cfg["n_cols"])
    n = cfg["n_cols"]
    obst = np.full((n, 3), np.nan)
    floor = np.full(n, np.nan)
    band = used & (z >= cfg["z_lo"]) & (z <= cfg["z_hi"])
    idx = np.nonzero(band)[0]
    if len(idx):
        order = np.lexsort((idx, rho[idx], j[idx]))                # by sector, then rho, then row index
        idx = idx[order]
        first = np.ones(len(idx), dtype=bool)
        first[1:] = j[idx][1:] != j[idx][:-1]
        obst[j[idx[first]]] = p[idx[first]]
    low = used & (z < cfg["z_lo"])
    if low.any():
        fl = np.full(n, -np.inf)
        np.maximum.at(fl, j[low], rho[low])
        floor = np.where(np.isfinite(fl), fl, np.nan)
    return obst, floor


def extents(obst, floor):
    """e_j of every sector: the obstacle's rho, else the floor's rho, else NaN"""
    return np.where(np.isnan(obst[:, 0]), floor, _rho(obst[:, 0], obst[:, 1]))


def grid_extent(poses, cfg):
    """(origin_x, origin_y, width, height), or None past 2^28 cells or with a non-finite extent"""
    if len(poses) == 0:
        return 0.0, 0.0, 0, 0
    W, r = window(cfg), cfg["resolution"]
    t = np.array([P[:2, 3] for P in poses])
    lo, hi = t.min(axis=0), t.max(axis=0)
    ox, oy = r * math.floor((lo[0] - W) / r), r * math.floor((lo[1] - W) / r)
    fw, fh = math.floor(((hi[0] + W) - ox) / r) + 1, math.floor(((hi[1] + W) - oy) / r) + 1
    if fw * fh > MAX_CELLS:
        return None
    return ox, oy, int(fw), int(fh)


def free_counts(obst, floor, P, cfg, ox, oy, width, height, D=None, out=None):
    """adds one frame's free counts to out ((height, width) uint32, a new one when None) and returns it"""
    D = sco.boundaries(cfg["n_cols"]) if D is None else D
    W, r = window(cfg), cfg["resolution"]
    out = np.zeros((height, width), dtype=np.uint32) if out is None else out
    tx, ty = P[0, 3], P[1, 3]
    i0 = max(int(math.floor(((tx - W) - ox) / r)) - 1, 0)
    j0 = max(int(math.floor(((ty - W) - oy) / r)) - 1, 0)
    nw = int(math.ceil(2.0 * W / r)) + 3
    i = np.arange(i0, min(i0 + nw + 1, width))
    jy = np.arange(j0, min(j0 + nw + 1, height))
    cx = ox + (i.astype(np.float64) + 0.5) * r
    cy = oy + (jy.astype(np.float64) + 0.5) * r
    d0 = np.broadcast_to((cx - tx)[None, :], (len(jy), len(i)))
    d1 = np.broadcast_to((cy - ty)[:, None], (len(jy), len(i)))
    inside = (np.abs(d0) <= W) & (np.abs(d1) <= W)
    q0 = P[0, 0] * d0 + P[1, 0] * d1                               # q_r = R(0, r) d0 + R(1, r) d1
    q1 = P[0, 1] * d0 + P[1, 1] * d1
    rho = _rho(q0, q1)
    e = extents(obst, floor)[mdo.columns(q0.ravel(), q1.ravel(), D, cfg["n_cols"]).reshape(q0.shape)]
    with np.errstate(invalid="ignore"):
        f = inside & (rho >= cfg["min_range"]) & (rho + cfg["free_margin"] <= e)
    if len(i) and len(jy):
        out[jy[0]:jy[-1] + 1, i[0]:i[-1] + 1] += f.astype(np.uint32)
    return out


def world_xy(P, o):
    """x' = ((P00 x + P01 y) + P02 z) + P03, likewise y"""
    x, y, z = o[:, 0], o[:, 1], o[:, 2]
    return (((P[0, 0] * x + P[0, 1] * y) + P[0, 2] * z) + P[0, 3], ((P[1, 0] * x + P[1, 1] * y) + P[1, 2] * z) + P[1, 3])


def hit_counts(obst, P, cfg, ox, oy, width, height, out=None):
    """adds one frame's hits to out ((height, width) uint32, a new one when None); returns it and the frame's dropped
    count"""
    out = np.zeros((height, width), dtype=np.uint32) if out is None else out
    o = obst[~np.isnan(obst[:, 0])]
    if not len(o):
        return out, 0
    wx, wy = world_xy(P, o)
    r = cfg["resolution"]
    fx, fy = np.floor((wx - ox) / r), np.floor((wy - oy) / r)
    ok = (fx >= 0) & (fy >= 0) & (fx < width) & (fy < height)
    np.add.at(out, (fy[ok].astype(np.int64), fx[ok].astype(np.int64)), 1)
    return out, int((~ok).sum())


def values(occ, free):
    """-1 if n = 0, else (100 occ + n / 2) / n"""
    o, n = occ.astype(np.int64), occ.astype(np.int64) + free.astype(np.int64)
    return np.where(n == 0, -1, (100 * o + n // 2) // np.maximum(n, 1)).astype(np.int8)


def build(scans, poses, cfg):
    """scans: [(obstacles, floors)] per frame, poses: the build poses.  dict(origin, width, height, occupied, free, cells,
    dropped), or None for VOXEL_RANGE"""
    ext = grid_extent(poses, cfg)
    if ext is None:
        return None
    ox, oy, w, h = ext
    D = sco.boundaries(cfg["n_cols"])
    occ, free = np.zeros((h, w), dtype=np.uint32), np.zeros((h, w), dtype=np.uint32)
    dropped = 0
    for (ob, fl), P in zip(scans, poses):
        free_counts(ob, fl, P, cfg, ox, oy, w, h, D, free)
        dropped += hit_counts(ob, P, cfg, ox, oy, w, h, occ)[1]
    return dict(origin=(ox, oy), width=w, height=h, occupied=occ, free=free, cells=values(occ, free), dropped=dropped)


# ---- literal ---------------------------------------------------------------------------------------------------------
def sector_linear(x, y, D, n_cols):
    n_up = (n_cols - 1) // 2
    upper = y > 0 or (y == 0 and x >= 0)
    ks = range(0, n_up) if upper else range(n_up, n_cols - 1)
    return (0 if upper else n_up) + sum(1 for k in ks if float(D[k, 0]) * y - float(D[k, 1]) * x > 0)


def scan2d_literal(scan, cfg):
    D = sco.boundaries(cfg["n_cols"])
    n = cfg["n_cols"]
    best = [None] * n                                              # (rho, row index)
    floor = [None] * n
    for i, (x, y, z) in enumerate(np.asarray(scan, dtype=np.float64).reshape(-1, 3).tolist()):
        if not (math.isfinite(x) and math.isfinite(y) and math.isfinite(z)):
            continue
        rho = math.sqrt(x * x + y * y)
        if not (cfg["min_range"] <= rho <= cfg["max_range"]):
            continue
        j = sector_linear(x, y, D, n)
        if cfg["z_lo"] <= z <= cfg["z_hi"]:
            if best[j] is None or rho < best[j][0]:
                best[j] = (rho, i)
        elif z < cfg["z_lo"]:
            floor[j] = rho if floor[j] is None else max(floor[j], rho)
    rows = np.asarray(scan, dtype=np.float64).reshape(-1, 3)
    obst = np.array([rows[b[1]] if b else [np.nan] * 3 for b in best]).reshape(n, 3)
    return obst, np.array([np.nan if f is None else f for f in floor])


def build_literal(scans, poses, cfg):
    ext = grid_extent(poses, cfg)
    if ext is None:
        return None
    ox, oy, w, h = ext
    D = sco.boundaries(cfg["n_cols"])
    W, r = window(cfg), cfg["resolution"]
    occ, free = np.zeros((h, w), dtype=np.uint32), np.zeros((h, w), dtype=np.uint32)
    dropped = 0
    for (ob, fl), P in zip(scans, poses):
        e = []
        for j in range(cfg["n_cols"]):
            x, y = float(ob[j, 0]), float(ob[j, 1])
            e.append(float(fl[j]) if math.isnan(x) else math.sqrt(x * x + y * y))
        tx, ty = float(P[0, 3]), float(P[1, 3])
        for jy in range(h):
            cy = oy + (float(jy) + 0.5) * r
            d1 = cy - ty
            if not abs(d1) <= W:
                continue
            for i in range(w):
                cx = ox + (float(i) + 0.5) * r
                d0 = cx - tx
                if not abs(d0) <= W:
                    continue
                q0 = float(P[0, 0]) * d0 + float(P[1, 0]) * d1
                q1 = float(P[0, 1]) * d0 + float(P[1, 1]) * d1
                rho = math.sqrt(q0 * q0 + q1 * q1)
                if rho < cfg["min_range"]:
                    continue
                ej = e[sector_linear(q0, q1, D, cfg["n_cols"])]
                if not math.isnan(ej) and rho + cfg["free_margin"] <= ej:
                    free[jy, i] += 1
        for j in range(cfg["n_cols"]):
            x, y, z = (float(v) for v in ob[j])
            if math.isnan(x):
                continue
            wx = ((float(P[0, 0]) * x + float(P[0, 1]) * y) + float(P[0, 2]) * z) + float(P[0, 3])
            wy = ((float(P[1, 0]) * x + float(P[1, 1]) * y) + float(P[1, 2]) * z) + float(P[1, 3])
            fx, fy = math.floor((wx - ox) / r), math.floor((wy - oy) / r)
            if 0 <= fx < w and 0 <= fy < h:
                occ[fy, fx] += 1
            else:
                dropped += 1
    cells = np.full((h, w), -1, dtype=np.int8)
    for jy in range(h):
        for i in range(w):
            n = int(occ[jy, i]) + int(free[jy, i])
            if n:
                cells[jy, i] = (100 * int(occ[jy, i]) + n // 2) // n
    return dict(origin=(ox, oy), width=w, height=h, occupied=occ, free=free, cells=cells, dropped=dropped)
