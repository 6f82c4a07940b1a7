"""numpy restatement of the distance field and costmap of an occupancy grid (include/tloam_b200.h "Distance field and
costmap"; k_dist_* in tloam_b200/csrc/distance.cu), bit for bit.

The squared distance is exact integer arithmetic.  It is computed here by another route than the device's envelope: per
column the distance to the nearest cell of the other class from running maxima and minima of row indices, then per row
min over k of g_k^2 + (i - k)^2 by offsets d = 1, 2, ... until d^2 passes every cell's best.  The CPU tests pin it to a
brute force over all cell pairs and to scipy.ndimage.distance_transform_edt.

sd, the costs and the query are float64 operations, each rounded on its own in the header's order; the cost table uses
math.sqrt / math.exp, the libm the C++ library's std::sqrt / std::exp call.  Grids are (height, width) arrays, row j along
y and column i along x."""
import math

import numpy as np

OBSTACLE = 65                 # map_saver's classes: >= 65 obstacle, 0 .. 25 free, anything else unknown
FREE = 25
INF = 0xFFFFFFFF
DEFAULT = dict(inscribed_radius=0.9, inflation_radius=3.0, cost_scaling_factor=3.0)
_BIG = 1 << 62


def config(**overrides):
    c = dict(DEFAULT)
    c.update(overrides)
    return c


def obstacles(grid):
    return np.asarray(grid).astype(np.int16) >= OBSTACLE


def _column_distance(src):
    """(H, W) int64: per column, the row distance to the nearest True cell of src (_BIG when the column has none)"""
    H = src.shape[0]
    j = np.arange(H, dtype=np.int64)[:, None]
    above = np.maximum.accumulate(np.where(src, j, -1), axis=0)
    below = np.minimum.accumulate(np.where(src, j, _BIG)[::-1], axis=0)[::-1]
    return np.minimum(np.where(above >= 0, j - above, _BIG), np.where(below < _BIG, below - j, _BIG))


def _row_min(G):
    """(H, W) int64: min over k of G[:, k] + (i - k)^2 (G = _BIG: no site), by growing offsets"""
    W = G.shape[1]
    best = G.copy()
    for d in range(1, W):
        fin = best < _BIG
        if fin.all() and d * d >= int(best.max()):
            break
        dd = d * d
        np.minimum(best[:, d:], G[:, :-d] + dd, out=best[:, d:])
        np.minimum(best[:, :-d], G[:, d:] + dd, out=best[:, :-d])
    return best


def squared(grid):
    """sq (H, W) uint32: min di^2 + dj^2 to the nearest cell of the other class (obstacle against non-obstacle); INF when
    there is none"""
    ob = obstacles(grid)
    out = np.full(ob.shape, INF, dtype=np.uint32)
    if ob.size == 0:
        return out
    for src, at in ((ob, ~ob), (~ob, ob)):
        g = _column_distance(src)
        G = np.where(g < _BIG, g * g, _BIG)
        best = _row_min(G)
        sel = at & (best < _BIG)
        out[sel] = best[sel].astype(np.uint32)
    return out


def brute(grid):
    """sq by a brute force over every pair of cells, int64"""
    ob = obstacles(grid)
    H, W = ob.shape
    jj, ii = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    jj, ii, o = jj.ravel(), ii.ravel(), ob.ravel()
    out = np.full(H * W, INF, dtype=np.int64)
    for c in range(H * W):
        other = o != o[c]
        if other.any():
            out[c] = int(((jj[other] - jj[c]) ** 2 + (ii[other] - ii[c]) ** 2).min())
    return out.reshape(H, W)


def signed(sq, grid, resolution):
    """sd (H, W) float32: (float)(sqrt((double)sq) * resolution), negated at obstacle cells, +-inf at INF"""
    d = (np.sqrt(sq.astype(np.float64)) * resolution).astype(np.float32)
    d[sq == INF] = np.float32(np.inf)
    return np.where(obstacles(grid), -d, d)


def cell_radius(cfg, resolution):
    """R_c = (unsigned) ceil(inflation_radius / resolution)"""
    return int(math.ceil(cfg["inflation_radius"] / resolution))


def cost_table(cfg, resolution):
    """c by sq for sq = 0 .. R_c^2 (the library's table)"""
    r2 = cell_radius(cfg, resolution) ** 2
    t = np.zeros(r2 + 1, dtype=np.uint8)
    t[0] = 254
    for s in range(1, r2 + 1):
        dist = math.sqrt(float(s))
        if dist * resolution <= cfg["inscribed_radius"]:
            t[s] = 253
        else:
            t[s] = int(252.0 * math.exp(-cfg["cost_scaling_factor"] * (dist * resolution - cfg["inscribed_radius"])))
    return t


def compute_cost_literal(distance, resolution, inscribed_radius, weight):
    """costmap_2d's InflationLayer::computeCost, transcribed"""
    cost = 0
    if distance == 0:
        cost = 254
    elif distance * resolution <= inscribed_radius:
        cost = 253
    else:
        euclidean_distance = distance * resolution
        factor = math.exp(-1.0 * weight * (euclidean_distance - inscribed_radius))
        cost = int((253 - 1) * factor)
    return cost


def costs(sq, grid, cfg, resolution):
    """(H, W) uint8: 254 at obstacles; c (0 past R_c^2) at free cells; 253 or 255 at unknown cells"""
    v = np.asarray(grid).astype(np.int16)
    t = cost_table(cfg, resolution)
    r2 = len(t) - 1
    s = sq.astype(np.int64)
    c = np.where(s <= r2, t[np.minimum(s, r2)], 0).astype(np.uint8)
    free = (v >= 0) & (v <= FREE)
    out = np.where(free, c, np.where(c == 253, 253, 255)).astype(np.uint8)
    out[v >= OBSTACLE] = 254
    return out


def publisher_table():
    """costmap_2d's Costmap2DPublisher cost_translation_table_, transcribed"""
    t = [0] * 256
    t[0] = 0
    t[253] = 99
    t[254] = 100
    t[255] = -1
    for i in range(1, 253):
        t[i] = 1 + (97 * (i - 1)) // 251
    return t


def values(c):
    return np.asarray(publisher_table(), dtype=np.int8)[np.asarray(c, dtype=np.uint8)]


def field(grid, origin, resolution, cfg=None):
    """every output of one build of a host grid"""
    cfg = config() if cfg is None else cfg
    g = np.asarray(grid, dtype=np.int8)
    sq = squared(g)
    c = costs(sq, g, cfg, resolution)
    return dict(sq=sq, signed=signed(sq, g, resolution), costs=c, values=values(c), obstacles=int(obstacles(g).sum()),
                origin=(float(origin[0]), float(origin[1])), resolution=float(resolution))


def query(sd, origin, resolution, xy):
    """(distance (n,), gradient (n, 2)): the bilinear interpolation of sd at the cell centres, NaN where invalid or when sd
    holds an infinite value"""
    p = np.asarray(xy, dtype=np.float64).reshape(-1, 2)
    n = len(p)
    H, W = sd.shape
    d, g = np.full(n, np.nan), np.full((n, 2), np.nan)
    if W < 2 or H < 2 or not np.isfinite(sd).all():
        return d, g
    with np.errstate(invalid="ignore"):
        u = (p[:, 0] - origin[0]) / resolution - 0.5
        v = (p[:, 1] - origin[1]) / resolution - 0.5
        ok = (u >= 0.0) & (u <= W - 1.0) & (v >= 0.0) & (v <= H - 1.0)
    u, v = u[ok], v[ok]
    i = np.minimum(np.floor(u), W - 2).astype(np.int64)
    j = np.minimum(np.floor(v), H - 2).astype(np.int64)
    a, b = u - i, v - j
    s = sd.astype(np.float64)
    s00, s10, s01, s11 = s[j, i], s[j, i + 1], s[j + 1, i], s[j + 1, i + 1]
    ia, ib = 1.0 - a, 1.0 - b
    d[ok] = ib * (ia * s00 + a * s10) + b * (ia * s01 + a * s11)
    g[ok, 0] = (ib * (s10 - s00) + b * (s11 - s01)) / resolution
    g[ok, 1] = (ia * (s01 - s00) + a * (s11 - s10)) / resolution
    return d, g
