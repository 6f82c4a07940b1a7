"""The terrain map (include/tloam_b200.h "Terrain") restated in numpy bit for bit, and a literal per-cell transcription of
it for small grids.

Every FP64 operation is rounded on its own, as numpy does it; extrema are taken on the ordered 64-bit encodings of the
doubles, so -0.0 orders below +0.0 and every extremum is order-independent; the plane fit's sums run over the window's
offsets dj outer, di inner, both ascending."""
import math

import numpy as np

MAX_CELLS = 1 << 28
SIGN = np.uint64(1 << 63)
ALL = np.uint64(0xFFFFFFFFFFFFFFFF)


def config(**overrides):
    """tloam_b200_terrain_default_config (max_slope in radians)"""
    c = dict(resolution=0.2, clearance=2.0, ground_radius=1.6, step_radius=0.3, slope_radius=0.4, max_step=0.10,
             max_slope=math.radians(15.0), max_roughness=0.10, min_points=1, min_fit=6, static_only=0,
             combine_occupancy=0)
    c.update(overrides)
    return c


def radius_cells(radius, resolution):
    """(unsigned) ceil(radius / resolution)"""
    return int(math.ceil(radius / resolution))


def enc(z):
    """the ordered encoding: a < b as doubles (with -0.0 < +0.0) iff enc(a) < enc(b)"""
    u = np.ascontiguousarray(z, dtype=np.float64).view(np.uint64)
    return np.where(u & SIGN != 0, ~u, u | SIGN)


def dec(k):
    k = np.asarray(k, dtype=np.uint64)
    return np.where(k & SIGN != 0, k & ~SIGN, ~k).view(np.float64)


def geometry(rows, resolution):
    """(origin_x, origin_y, width, height) of the finite rows, (0, 0, 0, 0) without any; None past 2^28 cells"""
    fin = rows[np.isfinite(rows).all(axis=1)]
    if len(fin) == 0:
        return 0.0, 0.0, 0, 0
    r = resolution
    lo = [dec(enc(fin[:, d]).min()) for d in range(2)]        # on the encodings: -0.0 orders below +0.0
    hi = [dec(enc(fin[:, d]).max()) for d in range(2)]
    ox, oy = r * float(np.floor(float(lo[0]) / r)), r * float(np.floor(float(lo[1]) / r))   # keeps -0.0
    fw, fh = math.floor((float(hi[0]) - ox) / r) + 1.0, math.floor((float(hi[1]) - oy) / r) + 1.0
    if not (fw <= MAX_CELLS and fh <= MAX_CELLS and fw * fh <= MAX_CELLS):
        return None
    return ox, oy, int(fw), int(fh)


def _window_extreme(keys, r, fill, op):
    """op (np.maximum / np.minimum) of keys over the (2r + 1)^2 window of every cell, clipped to the grid: a separable
    filter, each axis over the clipped range"""
    h, w = keys.shape
    out = keys.copy()
    for axis, size in ((1, w), (0, h)):
        src, acc = out, out.copy()
        for d in range(1, min(r, size - 1) + 1):
            sh = np.full_like(src, fill)
            if axis == 1:
                sh[:, :w - d] = src[:, d:]
                acc = op(acc, sh)
                sh = np.full_like(src, fill)
                sh[:, d:] = src[:, :w - d]
            else:
                sh[:h - d] = src[d:]
                acc = op(acc, sh)
                sh = np.full_like(src, fill)
                sh[d:] = src[:h - d]
            acc = op(acc, sh)
        out = acc
    return out


def _shift(a, di, dj, fill):
    """b[j, i] = a[j + dj, i + di], fill outside"""
    h, w = a.shape
    b = np.full_like(a, fill)
    ys, yd = (slice(dj, h), slice(0, h - dj)) if dj >= 0 else (slice(0, h + dj), slice(-dj, h))
    xs, xd = (slice(di, w), slice(0, w - di)) if di >= 0 else (slice(0, w + di), slice(-di, w))
    if h - abs(dj) > 0 and w - abs(di) > 0:
        b[yd, xd] = a[ys, xs]
    return b


def classify(step, slope, rough, known, cfg, tan_max_slope):
    """100 lethal, 0 traversable, -1 not known; a NaN comparison is false"""
    with np.errstate(invalid="ignore"):
        lethal = (step > cfg["max_step"]) | (slope > tan_max_slope) | (rough > cfg["max_roughness"])
    return np.where(known, np.where(lethal, 100, 0), -1).astype(np.int8)


def combine(t, o):
    """the terrain value t with the occupancy value o, cell by cell"""
    t, o = np.asarray(t, dtype=np.int64), np.asarray(o, dtype=np.int64)
    return np.where((t == 100) | (o >= 65), 100, np.where((t == 0) | ((o >= 0) & (o <= 25)), 0, -1)).astype(np.int8)


def build(rows, cfg, grid=None, occupancy=None):
    """the terrain of rows (n, 3) FP64.  grid: (origin_x, origin_y, resolution, width, height) of the occupancy build
    (combine_occupancy) with occupancy its values, or None (the rows' own extent at cfg's resolution).  Returns a dict of
    every layer and count, or None (VOXEL_RANGE)."""
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 3)
    if grid is None:
        res = cfg["resolution"]
        g = geometry(rows, res)
        if g is None:
            return None
        ox, oy, w, h = g
    else:
        ox, oy, res, w, h = grid
    rg, rs, rp = (radius_cells(cfg[k], res) for k in ("ground_radius", "step_radius", "slope_radius"))
    fin = np.isfinite(rows).all(axis=1)
    with np.errstate(invalid="ignore", over="ignore"):
        fi = np.floor((rows[:, 0] - ox) / res)
        fj = np.floor((rows[:, 1] - oy) / res)
    inside = fin & (fi >= 0) & (fi < w) & (fj >= 0) & (fj < h)
    P = rows[inside]
    cell = fj[inside].astype(np.int64) * w + fi[inside].astype(np.int64)
    n = w * h
    lo = np.zeros(n, dtype=np.uint64)                 # complemented ordered encodings of the least z (0: no row)
    np.maximum.at(lo, cell, ~enc(P[:, 2]))
    cnt = np.bincount(cell, minlength=n).astype(np.uint32)
    gkey = _window_extreme(lo.reshape(h, w), rg, np.uint64(0), np.maximum).ravel()
    G = np.where(gkey == 0, np.inf, dec(~gkey))
    thr = G[cell] + cfg["clearance"]
    ground = P[:, 2] <= thr
    ekey = np.zeros(n, dtype=np.uint64)
    np.maximum.at(ekey, cell[ground], enc(P[ground, 2]))
    m = np.bincount(cell[ground], minlength=n).astype(np.uint32)
    known = m >= cfg["min_points"]
    e = np.where(m > 0, dec(ekey), np.nan)
    K = np.where(known, ekey, np.uint64(0)).reshape(h, w)
    kmax = _window_extreme(K, rs, np.uint64(0), np.maximum).ravel()
    kmin = _window_extreme(np.where(known, ekey, ALL).reshape(h, w), rs, ALL, np.minimum).ravel()
    with np.errstate(invalid="ignore"):
        step = np.where(known, dec(kmax) - dec(kmin), np.nan)
    slope, rough = plane_fit(np.where(known, e, np.nan).reshape(h, w), rp, cfg["min_fit"], res)
    slope, rough = slope.ravel(), rough.ravel()
    tan = math.tan(cfg["max_slope"])
    tv = classify(step, slope, rough, known, cfg, tan)
    values = tv if occupancy is None else combine(tv, np.asarray(occupancy).ravel())
    shape = (h, w)
    return dict(origin=(ox, oy), resolution=res, width=w, height=h, radii=(rg, rs, rp),
                rows=len(rows), used=int(inside.sum()), skipped=int((~fin).sum()), dropped=int((fin & ~inside).sum()),
                overhang=int((~ground).sum()), known=int(known.sum()), lethal=int((tv == 100).sum()),
                combined=occupancy is not None,
                values=values.reshape(shape), ground=G.reshape(shape), elevation=e.reshape(shape),
                step=step.reshape(shape), slope=slope.reshape(shape), roughness=rough.reshape(shape),
                points=m.reshape(shape), count=cnt.reshape(shape), low=np.where(lo == 0, np.nan, dec(~lo)).reshape(shape))


def _cofactors(N, Su, Sv, Suu, Suv, Svv):
    """the exact integer cofactors and determinant of [[Suu, Suv, Su], [Suv, Svv, Sv], [Su, Sv, N]]"""
    C11 = Svv * N - Sv * Sv
    C12 = Sv * Su - Suv * N
    C13 = Suv * Sv - Svv * Su
    C22 = Suu * N - Su * Su
    C23 = Suv * Su - Suu * Sv
    C33 = Suu * Svv - Suv * Suv
    D = Suu * C11 + Suv * C12 + Su * C13
    return C11, C12, C13, C22, C23, C33, D


def plane_fit(E, rp, min_fit, res):
    """(slope, roughness) of every cell of E (height, width), NaN at unknown cells: the plane w = a u + b v + d over the
    known cells of the clipped (2 rp + 1)^2 window, u, v the cell offsets and w = E[k] - E[c]"""
    known = ~np.isnan(E)
    z = np.zeros(E.shape, dtype=np.int64)
    N, Su, Sv, Suu, Suv, Svv = z.copy(), z.copy(), z.copy(), z.copy(), z.copy(), z.copy()
    Sw, Suw, Svw = np.zeros(E.shape), np.zeros(E.shape), np.zeros(E.shape)
    offs = [(di, dj) for dj in range(-rp, rp + 1) for di in range(-rp, rp + 1)]
    for di, dj in offs:
        En = _shift(E, di, dj, np.nan)
        k = known & ~np.isnan(En)
        w = En - E
        N += k
        Su += k * di
        Sv += k * dj
        Suu += k * di * di
        Suv += k * di * dj
        Svv += k * dj * dj
        Sw = np.where(k, Sw + w, Sw)
        Suw = np.where(k, Suw + np.float64(di) * w, Suw)
        Svw = np.where(k, Svw + np.float64(dj) * w, Svw)
    C11, C12, C13, C22, C23, C33, D = (c.astype(np.float64) for c in _cofactors(N, Su, Sv, Suu, Suv, Svv))
    ok = known & (N >= min_fit) & (D != 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        a = ((C11 * Suw + C12 * Svw) + C13 * Sw) / D
        b = ((C12 * Suw + C22 * Svw) + C23 * Sw) / D
        d = ((C13 * Suw + C23 * Svw) + C33 * Sw) / D
        slope = np.sqrt(a * a + b * b) / res
        rough = np.zeros(E.shape)
        for di, dj in offs:
            En = _shift(E, di, dj, np.nan)
            k = ok & ~np.isnan(En)
            r = np.abs((En - E) - ((a * np.float64(di) + b * np.float64(dj)) + d))
            rough = np.where(k, np.maximum(rough, r), rough)
    return np.where(ok, slope, np.nan), np.where(ok, rough, np.nan)


# ---- the literal transcription ---------------------------------------------------------------------------------------
def _key(z):
    return int(enc(np.array([z]))[0])


def build_literal(rows, cfg, grid=None, occupancy=None):
    """the definition cell by cell in Python floats (each operation rounded on its own), for small grids"""
    rows = [tuple(float(v) for v in r) for r in np.asarray(rows, dtype=np.float64).reshape(-1, 3)]
    if grid is None:
        res = cfg["resolution"]
        fin = [r for r in rows if all(math.isfinite(v) for v in r)]
        if not fin:
            ox = oy = 0.0
            w = h = 0
        else:
            ox = res * float(np.floor(min((r[0] for r in fin), key=_key) / res))
            oy = res * float(np.floor(min((r[1] for r in fin), key=_key) / res))
            w = int(math.floor((max((r[0] for r in fin), key=_key) - ox) / res)) + 1
            h = int(math.floor((max((r[1] for r in fin), key=_key) - oy) / res)) + 1
    else:
        ox, oy, res, w, h = grid
    rg, rs, rp = (int(math.ceil(cfg[k] / res)) for k in ("ground_radius", "step_radius", "slope_radius"))
    cells = {}
    skipped = dropped = 0
    for r in rows:
        if not all(math.isfinite(v) for v in r):
            skipped += 1
            continue
        i, j = math.floor((r[0] - ox) / res), math.floor((r[1] - oy) / res)
        if not (0 <= i < w and 0 <= j < h):
            dropped += 1
            continue
        cells.setdefault((i, j), []).append(r[2])

    def window(i, j, rad):
        for jj in range(max(0, j - rad), min(h - 1, j + rad) + 1):
            for ii in range(max(0, i - rad), min(w - 1, i + rad) + 1):
                yield ii, jj

    def least(zs):
        return min(zs, key=_key)

    def most(zs):
        return max(zs, key=_key)

    zlo = {c: least(zs) for c, zs in cells.items()}
    G, E, M = {}, {}, {}
    overhang = 0
    for j in range(h):
        for i in range(w):
            ws = [zlo[c] for c in window(i, j, rg) if c in zlo]
            G[i, j] = least(ws) if ws else math.inf
    for (i, j), zs in cells.items():
        thr = G[i, j] + cfg["clearance"]
        g = [z for z in zs if z <= thr]
        overhang += len(zs) - len(g)
        M[i, j] = len(g)
        if g:
            E[i, j] = most(g)
    known = {c for c, v in M.items() if v >= cfg["min_points"]}
    tan = math.tan(cfg["max_slope"])
    out = {k: np.full((h, w), np.nan) for k in ("ground", "elevation", "step", "slope", "roughness")}
    values = np.full((h, w), -1, dtype=np.int8)
    points = np.zeros((h, w), dtype=np.uint32)
    lethal_n = 0
    for j in range(h):
        for i in range(w):
            out["ground"][j, i] = G[i, j]
            points[j, i] = M.get((i, j), 0)
            if (i, j) in E:
                out["elevation"][j, i] = E[i, j]
            if (i, j) not in known:
                continue
            ks = [E[c] for c in window(i, j, rs) if c in known]
            step = most(ks) - least(ks)
            fit = [(ii - i, jj - j, E[ii, jj] - E[i, j]) for ii, jj in window(i, j, rp) if (ii, jj) in known]
            N = len(fit)
            Su, Sv = sum(u for u, _, _ in fit), sum(v for _, v, _ in fit)
            Suu, Suv, Svv = (sum(u * u for u, _, _ in fit), sum(u * v for u, v, _ in fit), sum(v * v for _, v, _ in fit))
            Sw = Suw = Svw = 0.0
            for u, v, wv in fit:
                Sw = Sw + wv
                Suw = Suw + float(u) * wv
                Svw = Svw + float(v) * wv
            C11, C12, C13, C22, C23, C33, D = (float(c) for c in _cofactors(N, Su, Sv, Suu, Suv, Svv))
            slope = rough = math.nan
            if N >= cfg["min_fit"] and D != 0.0:
                a = ((C11 * Suw + C12 * Svw) + C13 * Sw) / D
                b = ((C12 * Suw + C22 * Svw) + C23 * Sw) / D
                d = ((C13 * Suw + C23 * Svw) + C33 * Sw) / D
                slope = math.sqrt(a * a + b * b) / res
                rough = 0.0
                for u, v, wv in fit:
                    rough = max(rough, abs(wv - ((a * float(u) + b * float(v)) + d)))
            out["step"][j, i], out["slope"][j, i], out["roughness"][j, i] = step, slope, rough
            lethal = step > cfg["max_step"] or slope > tan or rough > cfg["max_roughness"]
            values[j, i] = 100 if lethal else 0
            lethal_n += lethal
    if occupancy is not None:
        occ = np.asarray(occupancy).reshape(h, w)
        for j in range(h):
            for i in range(w):
                t, o = int(values[j, i]), int(occ[j, i])
                values[j, i] = 100 if (t == 100 or o >= 65) else (0 if (t == 0 or 0 <= o <= 25) else -1)
    return dict(origin=(ox, oy), width=w, height=h, skipped=skipped, dropped=dropped, overhang=overhang,
                used=sum(len(v) for v in cells.values()), known=len(known), lethal=lethal_n, values=values,
                points=points, **out)
