"""numpy restatement of dynamic-point removal for the global map (include/tloam_b200.h "Dynamic-point removal"; k_gmd_* in
tloam_b200/csrc/map_dynamic.cu), bit for bit.

Every product, sum, quotient and square root below is one numpy float64 operation, rounded on its own, in the order the
header states; nothing is fused, so the device's __dmul_rn / __dadd_rn / __dsub_rn / __ddiv_rn / __dsqrt_rn give the same
bits.  The column rule is scan_context_oracle's sector rule.

Two forms: the vectorised one the GPU tests use, and a literal per-row / per-pixel / per-point transcription the CPU tests
pin it to.  Poses are 4 x 4 float64 arrays (A[r, c])."""
import math

import numpy as np

import scan_context_oracle as sco

DEFAULT = dict(n_rows=64, fov_up=2.0, fov_down=-24.9, n_cols=1024, window_rows=1, window_cols=2, margin_abs=1.0,
               margin_rel=0.02, min_range=3.0, max_range=60.0, min_through=3)


def config(**overrides):
    c = dict(DEFAULT)
    c.update(overrides)
    return c


def row_bounds(cfg):
    """b_k = sin(lo + k (hi - lo) / n_rows), k = 0 .. n_rows, lo / hi the field of view in radians, by the C library"""
    lo, hi = cfg["fov_down"] * (math.pi / 180.0), cfg["fov_up"] * (math.pi / 180.0)
    n = cfg["n_rows"]
    return np.array([math.sin(lo + k * (hi - lo) / n) for k in range(n + 1)])


def col_bounds(cfg):
    return sco.boundaries(cfg["n_cols"])


# ---- vectorised ------------------------------------------------------------------------------------------------------
def _range(x, y, z):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.sqrt((x * x + y * y) + z * z)


def columns(x, y, D, n_cols):
    """the sector of every (x, y): binary search over the monotone sign sequence of each half-plane"""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    n_up = (n_cols - 1) // 2
    upper = (y > 0) | ((y == 0) & (x >= 0))
    base = np.where(upper, 0, n_up)                    # boundaries k = base + 1 .. base + len
    size = np.where(upper, n_up, n_cols - 1 - n_up)
    lo = np.zeros(x.shape, dtype=np.int64)
    hi = size.astype(np.int64)
    while True:
        act = lo < hi
        if not act.any():
            break
        mid = (lo + hi + 1) // 2
        k = np.where(act, base + mid, 1)              # boundary index k (1-based), a dummy where inactive
        c, s = D[k - 1, 0], D[k - 1, 1]
        with np.errstate(invalid="ignore"):
            t = (c * y - s * x) > 0
        lo = np.where(act & t, mid, lo)
        hi = np.where(act & ~t, mid - 1, hi)
    return base + lo


def columns_linear(x, y, D, n_cols):
    """the linear count of scan_context_oracle.rings_sectors (chunked)"""
    x, y = np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64)
    n_up = (n_cols - 1) // 2
    out = np.zeros(x.shape, dtype=np.int64)
    for a in range(0, len(x), 4096):
        xx, yy = x[a:a + 4096], y[a:a + 4096]
        cross = D[None, :, 0] * yy[:, None] - D[None, :, 1] * xx[:, None]
        upper = (yy > 0) | ((yy == 0) & (xx >= 0))
        out[a:a + 4096] = np.where(upper, (cross[:, :n_up] > 0).sum(axis=1), n_up + (cross[:, n_up:] > 0).sum(axis=1))
    return out


def rows(s, b):
    """(image row, inside) of every s = z / r: outside iff s < b_0 or s > b_n; else the count of k in 1 .. n - 1 with
    s > b_k, by binary search (b is non-decreasing)"""
    n = len(b) - 1
    inside = (s >= b[0]) & (s <= b[n])
    lo = np.zeros(s.shape, dtype=np.int64)
    hi = np.full(s.shape, n - 1, dtype=np.int64)
    while True:
        act = inside & (lo < hi)
        if not act.any():
            break
        mid = (lo + hi + 1) // 2
        t = s > b[np.where(act, mid, 1)]
        lo = np.where(act & t, mid, lo)
        hi = np.where(act & ~t, mid - 1, hi)
    return lo, inside


def pixels(p, cfg, b=None, D=None):
    """(pixel index, r, valid) of every row of p (n x 3)"""
    b = row_bounds(cfg) if b is None else b
    D = col_bounds(cfg) if D is None else D
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r = _range(x, y, z)
    ok = (r >= cfg["min_range"]) & (r <= cfg["max_range"])
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(ok, z / np.where(ok, r, 1.0), 0.0)
    row, inside = rows(s, b)
    col = columns(np.where(ok, x, 0.0), np.where(ok, y, 0.0), D, cfg["n_cols"])
    valid = ok & inside
    return np.where(valid, row * cfg["n_cols"] + col, 0), r, valid


def range_image(scan, cfg, b=None, D=None):
    """(n_rows * n_cols,) the minimum r per pixel, +inf = empty"""
    pix, r, valid = pixels(scan, cfg, b, D)
    img = np.full(cfg["n_rows"] * cfg["n_cols"], np.inf)
    np.minimum.at(img, pix[valid], r[valid])
    return img


def window_image(img, cfg):
    """the window minimum per pixel, NaN = unknown (an empty pixel in the window)"""
    R, S, wr, wc = cfg["n_rows"], cfg["n_cols"], cfg["window_rows"], cfg["window_cols"]
    a = img.reshape(R, S)
    w = np.full((R, S), np.inf)
    unknown = np.zeros((R, S), dtype=bool)
    for dr in range(-wr, wr + 1):
        lo, hi = max(0, -dr), min(R, R - dr)          # rows i with 0 <= i + dr < R
        if lo >= hi:
            continue
        for dc in range(-wc, wc + 1):
            v = np.roll(a[lo + dr:hi + dr], -dc, axis=1)  # v[i, j] = a[i + dr, (j + dc) mod S]
            unknown[lo:hi] |= np.isinf(v)
            w[lo:hi] = np.minimum(w[lo:hi], v)
    return np.where(unknown, np.nan, w).reshape(-1)


def to_sensor(points, pose):
    """q_r = (R(0, r) d0 + R(1, r) d1) + R(2, r) d2, d = m - t"""
    m = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    A = np.asarray(pose, dtype=np.float64)
    d0, d1, d2 = m[:, 0] - A[0, 3], m[:, 1] - A[1, 3], m[:, 2] - A[2, 3]
    return np.stack([(A[0, r] * d0 + A[1, r] * d1) + A[2, r] * d2 for r in range(3)], axis=1)


def vote(points, scan, pose, cfg):
    """the (through, hits) increments (uint32 0 / 1) one append with `scan` (sensor frame) at `pose` gives the rows of
    `points` (the map before the append)"""
    b, D = row_bounds(cfg), col_bounds(cfg)
    img = range_image(scan, cfg, b, D)
    win = window_image(img, cfg)
    q = to_sensor(points, pose)
    pix, r, valid = pixels(q, cfg, b, D)
    wm, c = win[pix], img[pix]
    mg = np.maximum(cfg["margin_abs"], cfg["margin_rel"] * r)
    with np.errstate(invalid="ignore"):
        through = valid & (wm > r + mg)
        hits = valid & np.isfinite(c) & (np.abs(c - r) <= mg)
    return through.astype(np.uint32), hits.astype(np.uint32)


class Votes:
    """the counters of a map that grows by appends: append(map_rows_before, scan, pose) votes on the rows present, then
    grow(n) adds n rows at (0, 0)"""

    def __init__(self, cfg):
        self.cfg = cfg
        self.through = np.zeros(0, dtype=np.uint32)
        self.hits = np.zeros(0, dtype=np.uint32)

    def append(self, map_before, scan, pose, new_rows):
        n = len(self.through)
        assert len(map_before) == n
        if n:
            t, h = vote(map_before, scan, pose, self.cfg)
            self.through = self.through + t
            self.hits = self.hits + h
        self.through = np.concatenate([self.through, np.zeros(new_rows, dtype=np.uint32)])
        self.hits = np.concatenate([self.hits, np.zeros(new_rows, dtype=np.uint32)])


def dynamic(through, hits, cfg):
    through, hits = np.asarray(through), np.asarray(hits)
    return (through >= cfg["min_through"]) & (through > hits)


def static_map(points, intensity, through, hits, cfg):
    keep = ~dynamic(through, hits, cfg)
    return np.asarray(points)[keep], (None if intensity is None else np.asarray(intensity)[keep])


# ---- literal transcription ---------------------------------------------------------------------------------------------
def _column_literal(x, y, D, n_cols):
    n_up = (n_cols - 1) // 2
    if y > 0 or (y == 0 and x >= 0):
        col, ks = 0, range(1, n_up + 1)
    else:
        col, ks = n_up, range(n_up + 1, n_cols)
    for k in ks:
        c, s = float(D[k - 1, 0]), float(D[k - 1, 1])
        if c * y - s * x > 0:
            col += 1
    return col


def _pixel_literal(x, y, z, cfg, b, D):
    r = math.sqrt((x * x + y * y) + z * z) if all(math.isfinite(v) for v in (x, y, z)) else math.nan
    if not (cfg["min_range"] <= r <= cfg["max_range"]):
        return None, r
    s = z / r
    n = cfg["n_rows"]
    if s < b[0] or s > b[n]:
        return None, r
    row = sum(1 for k in range(1, n) if s > float(b[k]))
    return row * cfg["n_cols"] + _column_literal(x, y, D, cfg["n_cols"]), r


def vote_literal(points, scan, pose, cfg):
    b, D = row_bounds(cfg), col_bounds(cfg)
    R, S, wr, wc = cfg["n_rows"], cfg["n_cols"], cfg["window_rows"], cfg["window_cols"]
    img = [math.inf] * (R * S)
    for x, y, z in np.asarray(scan, dtype=np.float64).reshape(-1, 3).tolist():
        pix, r = _pixel_literal(x, y, z, cfg, b, D)
        if pix is not None and r < img[pix]:
            img[pix] = r
    win = [math.nan] * (R * S)
    for i in range(R):
        for j in range(S):
            m, known = math.inf, True
            for ii in range(max(0, i - wr), min(R - 1, i + wr) + 1):
                for dj in range(-wc, wc + 1):
                    v = img[ii * S + (j + dj) % S]
                    known &= v != math.inf
                    m = min(m, v)
            win[i * S + j] = m if known else math.nan
    A = np.asarray(pose, dtype=np.float64)
    through, hits = [], []
    for mx, my, mz in np.asarray(points, dtype=np.float64).reshape(-1, 3).tolist():
        d = (mx - float(A[0, 3]), my - float(A[1, 3]), mz - float(A[2, 3]))
        q = [(float(A[0, r]) * d[0] + float(A[1, r]) * d[1]) + float(A[2, r]) * d[2] for r in range(3)]
        pix, r = _pixel_literal(q[0], q[1], q[2], cfg, b, D)
        t = h = 0
        if pix is not None:
            mg = max(cfg["margin_abs"], cfg["margin_rel"] * r)
            w, c = win[pix], img[pix]
            t = int(not math.isnan(w) and w > r + mg)
            h = int(c != math.inf and abs(c - r) <= mg)
        through.append(t)
        hits.append(h)
    return np.array(through, dtype=np.uint32), np.array(hits, dtype=np.uint32), np.array(img), np.array(win)
