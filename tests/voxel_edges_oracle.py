"""Exact restatement of the device's voxel down-sample (k_vox_min -> k_vox_accum -> k_vox_emit / sorted emission) for the
edge tests of tests/test_voxel_edges.py.  It shares no FP64 code with the kernels or with the CPU oracle.

Membership.  The device computes, per axis, mb = min - voxel * 0.5 over the kept rows (finite, inside the crop box), then
idx = floor((p - mb) / voxel).  `membership` does the same with numpy's IEEE FP64 operations, which are the device's
(voxel * 0.5 is exact, so a contracted mb is the same double), so the indices are bit-exact.  `fraction_indices` spells
out every rounding with fractions.Fraction (each float() of a Fraction is one correctly rounded operation) as an
independent check of that claim; it also says which rows the rounding of the quotient alone puts in their voxel.

Error bound of the device's averages against the exact mean mu = (1/c) sum p_i of a voxel's c rows.  With B the voxel's
base mb + idx * voxel as the device rounds it:
  - each row adds q_i = llrint((p_i - B) * 2^40).  p_i - B is exact by Sterbenz (B <= p_i <= 2B for B > 0, mirrored for
    B < 0) except in voxels that straddle 0, where its rounding is below 2^-53 voxel; the quantisation is at most 2^-41;
  - sum q_i is an exact integer (below 2^63: see HEADROOM_M); its conversion to FP64 and the quotient by c are each
    rounded, below 2^-53 voxel each;
  - the final add B + m is rounded, half an ulp of the result.
mu = B + (1/c) sum (p_i - B) holds for any B, so
    |out - mu| <= 2^-41 + 3 * 2^-53 voxel + ulp(max |p|) / 2,
which `device_bound` pads to 2^-41 + 2^-51 voxel + 1.5 ulp(max |p|).  The SASS of k_vox_accum and of vox_average both
compute mb + idx * voxel with one DFMA, so the base the average adds back is the base the offsets were taken from; were
only one of them contracted, the two bases could differ by an ulp of B (`extra_ulp`).

The CPU oracle (oracle_voxel_down_sample) sums the rows in input order from 0 in FP64, then divides by c.  Its error is
at most gamma_{c-1} sum |p_i| / c + ulp(mu) / 2 <= (c + 1) 2^-53 max |p| (`oracle_bound`).

Scenes.  `scenes()` returns seeded cases (dicts with p, voxel and optionally lo / hi, the inclusive crop box) grouped by
name; `coverage` counts what each case exercises so that the tests can assert minimums on it.
"""
import math
from fractions import Fraction

import numpy as np

KEY_BITS = 21                     # per axis of the device's packed voxel key
HEADROOM_M = 2.0 ** 23            # a voxel's count * voxel must stay below this (2^63 / 2^40)
RANK_MAX = 32768                  # the sorted emission's rank sort takes lists up to this many voxels


# ---------------------------------------------------------------------------------------------------------------------
# restatement
# ---------------------------------------------------------------------------------------------------------------------
def kept_rows(p, lo=None, hi=None):
    """rows the device keeps: every coordinate finite and inside the inclusive box (lo / hi None: no box)"""
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    with np.errstate(invalid="ignore"):
        keep = np.isfinite(p).all(1)
        if lo is not None:
            keep &= (p >= np.asarray(lo)).all(1) & (p <= np.asarray(hi)).all(1)
    return keep


def membership(p, voxel, lo=None, hi=None):
    """(keep mask, idx (kept rows x 3) int64, mb (3,)) with the device's FP64 operations"""
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    keep = kept_rows(p, lo, hi)
    q = p[keep]
    if q.shape[0] == 0:
        return keep, np.zeros((0, 3), dtype=np.int64), np.zeros(3)
    mb = q.min(0) - voxel * 0.5
    idx = np.floor((q - mb) / voxel).astype(np.int64)
    return keep, idx, mb


def fraction_indices(values, mn, voxel):
    """for the distinct values of one axis: the index with each rounding spelled out, and whether the exact quotient
    would have put the row in another voxel.  Returns (idx, rounding_decides) as arrays over `values`."""
    v = Fraction(voxel)
    mb = float(Fraction(mn) - v / 2)                      # one rounding: min - voxel * 0.5 (voxel * 0.5 is exact)
    mbf = Fraction(mb)
    idx = np.empty(len(values), dtype=np.int64)
    dec = np.zeros(len(values), dtype=bool)
    for i, x in enumerate(values):
        diff = Fraction(x) - mbf
        d = float(diff)                                   # p - mb, rounded
        qt = float(Fraction(d) / v)                       # / voxel, rounded
        idx[i] = math.floor(qt)
        dec[i] = math.floor(diff / v) != idx[i]
    return idx, dec


def voxel_groups(idx):
    """(unique keys ascending (ix, iy, iz), inverse, counts)"""
    keys, inv, cnt = np.unique(idx, axis=0, return_inverse=True, return_counts=True)
    return keys, inv.reshape(-1), cnt


def exact_means(q, inv, nvox):
    """exact per-voxel means as Fractions (nvox x 3 lists)"""
    order = np.argsort(inv, kind="stable")
    bounds = np.searchsorted(inv[order], np.arange(nvox + 1))
    out = []
    for k in range(nvox):
        rows = q[order[bounds[k]:bounds[k + 1]]]
        c = rows.shape[0]
        out.append([_exact_sum(rows[:, d]) / c for d in range(3)])
    return out


def _exact_sum(col):
    """exact sum of FP64 values: repeated values are multiplied, not added one by one"""
    vals, cnt = np.unique(col, return_counts=True)
    return sum((Fraction(float(v)) * int(c) for v, c in zip(vals, cnt)), Fraction(0))


def reference(p, voxel, lo=None, hi=None):
    """the restatement of one case: keys ascending, counts, exact means (Fractions), per-voxel max |p|"""
    p = np.asarray(p, dtype=np.float64).reshape(-1, 3)
    keep, idx, mb = membership(p, voxel, lo, hi)
    q = p[keep]
    keys, inv, cnt = voxel_groups(idx)
    means = exact_means(q, inv, keys.shape[0])
    big = np.zeros(keys.shape[0])
    if q.shape[0]:
        np.maximum.at(big, inv, np.abs(q).max(1))
    return dict(keys=keys, inv=inv, counts=cnt, means=means, maxabs=big, mb=mb, idx=idx, kept=q)


def ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float64)))


def device_bound(voxel, maxabs, extra_ulp=0):
    """the device's bound against the exact mean, per voxel (see the module docstring)"""
    u = ulp(maxabs)
    return 2.0 ** -41 + 2.0 ** -51 * voxel + (1.5 + extra_ulp) * u


def oracle_bound(counts, maxabs):
    """the CPU oracle's running-sum bound against the exact mean, per voxel"""
    return (np.asarray(counts, dtype=np.float64) + 1.0) * 2.0 ** -53 * np.asarray(maxabs) * (1.0 + 1e-9) + 1e-300


def errors(got, means):
    """|got - exact mean| per voxel (max over the axes), as floats; got: (nvox x 3) in the order of means"""
    got = np.asarray(got, dtype=np.float64).reshape(-1, 3)
    return np.array([max(abs(float(Fraction(float(got[k, d])) - means[k][d])) for d in range(3)) for k in range(len(means))])


def keyable(idx):
    return idx.shape[0] == 0 or int(idx.max()) < (1 << KEY_BITS)


def coverage(case):
    """what a case exercises: rows on a face, within 2 ulp of one, decided by the quotient's rounding alone; the largest
    index, voxel count and count * voxel; the dropped rows"""
    p = np.asarray(case["p"], dtype=np.float64).reshape(-1, 3)
    voxel = case["voxel"]
    keep, idx, mb = membership(p, voxel, case.get("lo"), case.get("hi"))
    q = p[keep]
    cov = dict(rows=int(p.shape[0]), dropped=int((~keep).sum()), on_face=0, near_face=0, rounding_decides=0, max_index=-1,
               max_count=0, voxels=0, max_load_m=0.0, maxabs=float(np.abs(q).max()) if q.shape[0] else 0.0)
    if q.shape[0] == 0:
        return cov
    cov["max_index"] = int(idx.max())
    _, _, cnt = voxel_groups(idx)
    cov["voxels"], cov["max_count"] = int(cnt.size), int(cnt.max())
    cov["max_load_m"] = float(cnt.max()) * voxel
    with np.errstate(invalid="ignore"):
        quot = (q - mb) / voxel
    near = np.zeros(q.shape[0], dtype=bool)
    face = np.zeros(q.shape[0], dtype=bool)
    for d in range(3):
        k = np.round(quot[:, d])
        face |= quot[:, d] == k
        # a face in coordinates: mb + k * voxel, the row within 2 ulp of it
        x = mb[d] + k * voxel
        near |= np.abs(q[:, d] - x) <= 2 * ulp(q[:, d])
    cov["on_face"], cov["near_face"] = int(face.sum()), int(near.sum())
    dec = 0
    for d in range(3):
        vals, inv = np.unique(q[:, d], return_inverse=True)
        _, dv = fraction_indices(vals.tolist(), float(vals[0]), voxel)
        dec += int(dv[inv.reshape(-1)].sum())
    cov["rounding_decides"] = dec
    return cov


# ---------------------------------------------------------------------------------------------------------------------
# scenes
# ---------------------------------------------------------------------------------------------------------------------
def _quot(x, mb, voxel):
    return math.floor((x - mb) / voxel)


def _boundary(mb, voxel, k):
    """the first double whose rounded quotient (x - mb) / voxel reaches k"""
    x = mb + k * voxel
    while _quot(x, mb, voxel) >= k:
        x = math.nextafter(x, -math.inf)
    while _quot(x, mb, voxel) < k:
        x = math.nextafter(x, math.inf)
    return x


def _face_values(anchor, voxel, kmax, exact):
    """values of one axis around the faces 1..kmax of a cloud whose min is `anchor`: for dyadic voxels the faces
    themselves and 1 or 2 ulp either side, otherwise the last value below each face and the first at or above it (found
    with nextafter), and their neighbours"""
    mb = anchor - voxel * 0.5
    out = [anchor]
    for k in range(1, kmax + 1):
        x = mb + k * voxel if exact else _boundary(mb, voxel, k)
        lo1 = math.nextafter(x, -math.inf)
        out += [math.nextafter(lo1, -math.inf), lo1, x, math.nextafter(x, math.inf), math.nextafter(math.nextafter(x, math.inf), math.inf)]
    return np.array([v for v in out if v >= anchor])


def _face_cloud(rng, anchor, voxel, exact, n=3000, kmax=6):
    vals = [_face_values(anchor[d], voxel, kmax, exact) for d in range(3)]
    p = np.stack([rng.choice(vals[d], n) for d in range(3)], 1)
    p = np.concatenate([np.array([anchor], dtype=np.float64), p])       # the min of every axis
    return p


def scene_faces_dyadic(rng):
    return [dict(p=_face_cloud(rng, (a, a, a), v, True), voxel=v) for v in (0.25, 0.5, 1.0) for a in (0.0, 3.0)]


def scene_faces_rounded(rng):
    return [dict(p=_face_cloud(rng, (a, 0.7 * a, 0.0), v, False), voxel=v) for v in (0.1, 0.3, 0.45) for a in (0.0, 1.7)]


def scene_far(rng):
    cases = []
    for t in (1e3, -1e3, 1e4, -1e4, 1e5, -1e5):
        for v, exact in ((0.25, True), (0.3, False)):
            cases.append(dict(p=_face_cloud(rng, (t, -0.5 * t, 0.25 * t), v, exact, n=2000), voxel=v))
    for v in (0.25, 0.3, 1.0):                               # clusters straddling 0: voxels that hold both signs
        p = rng.uniform(-2.3, 2.1, (4000, 3))
        p[:200] = rng.choice([-0.0, 0.0, 5e-324, -5e-324, 1e-300, -1e-17, 1e-17], (200, 3))
        cases.append(dict(p=p, voxel=v))
    return cases


def _crowd(rng, c, base, voxel, tie=False):
    """c rows inside the voxel whose lowest corner row is `base` (the cloud's min), offsets from the voxel's base just
    under a multiple of 2^-40 (truncation instead of llrint would lose almost 2^-40 per row)"""
    mb = base - voxel * 0.5                                 # the voxel's base (index 0)
    k = rng.integers(int(0.5 * voxel * 2 ** 40) + 8, int(voxel * 2 ** 40) - 8, (c, 3)).astype(np.float64)
    u = np.spacing(base + voxel)
    p = mb + k * 2.0 ** -40 - u                             # exact: k 2^-40 and mb are multiples of u
    if tie:
        p[c // 2:] = p[0]
    p[0] = [base, base, base]
    return p


def scene_crowded(rng):
    cases = []
    for c in (1, 2, 1000, 100000):
        cases.append(dict(p=_crowd(rng, c, 5.0, 0.25), voxel=0.25))
    cases.append(dict(p=np.full((100000, 3), 1.2345678901234567), voxel=0.5))       # identical rows: the mean is the row
    cases.append(dict(p=_crowd(rng, 1000, 5.0, 0.25, tie=True), voxel=0.25))
    cases.append(dict(p=_crowd(rng, 1000, -37.0, 1.0), voxel=1.0))
    return cases


def _count_cloud(rng, nvox, voxel=0.5, per=1):
    """a cloud of exactly nvox occupied voxels (anchor row at the origin is voxel (0, 0, 0))"""
    box = (64, 64, 16) if nvox <= 65535 else (128, 64, 16)
    flat = rng.choice(box[0] * box[1] * box[2] - 1, nvox - 1, replace=False) + 1
    idx = np.stack(np.unravel_index(flat, box), 1)
    idx = np.concatenate([np.zeros((1, 3), dtype=np.int64), idx])
    idx = np.repeat(idx, per, axis=0)
    p = idx * voxel + rng.uniform(0.0, 0.4 * voxel, idx.shape)
    p[0] = 0.0
    return rng.permutation(p)


def scene_counts(rng):
    return [dict(p=_count_cloud(rng, n), voxel=0.5, nvox=n) for n in (1, 255, 256, 257, 16383, 16384, 16385, 32767, 32768, 32769)]


def scene_key_range(rng):
    """largest index 2^21 - 1 (the last keyable) and 2^21 (the first that is not), on each axis"""
    cases = []
    v = 0.25
    for d in range(3):
        for top in ((1 << KEY_BITS) - 1, 1 << KEY_BITS):
            p = rng.uniform(0.0, 2.0, (300, 3))
            p[0] = 0.0
            far = np.zeros(3)
            far[d] = top * v + 0.1                               # index floor((x + v/2) / v) = top
            p[1] = far
            p[2] = far + [0.01, 0.0, 0.0] if d else far + [0.0, 0.01, 0.0]
            cases.append(dict(p=p, voxel=v, top=top, axis=d))
    cases.append(dict(p=np.array([[0.0, 0.0, 0.0], [524288.0, 0.0, 0.0]]), voxel=0.25, top=1 << KEY_BITS, axis=0))
    return cases


def scene_headroom(rng):
    """count * voxel just below 2^23 m (64 m voxel, 2^17 - 1 rows at the top of the voxel) and at the limit"""
    v = 64.0
    cases = []
    for c in ((1 << 17) - 1, 1 << 17, (1 << 17) + 1):
        p = 64.0 - 2.0 ** -30 - rng.uniform(0.0, 2.0 ** -20, (c, 3))        # voxel 0 = [0, 64): offsets just under 64 m
        p[0] = 32.0                                                          # the min: base 32 - 64 / 2 = 0
        cases.append(dict(p=p, voxel=v, load=c * v))
    return cases


def scene_nonfinite(rng):
    p = rng.uniform(-3.0, 3.0, (5000, 3))
    bad = rng.choice(5000, 600, replace=False)
    vals = np.array([np.nan, np.inf, -np.inf])
    for j, i in enumerate(bad):
        p[i, j % 3] = vals[(j // 3) % 3]
    p[bad[:30]] = -1e9                                       # finite rows far below: not dropped
    p[bad[:30], 1] = -np.inf
    return [dict(p=p, voxel=v) for v in (0.25, 0.3)]


def scene_crop(rng):
    """frames cropped to c +- L: rows exactly at c - L and c + L on each face, one ulp outside, and rows outside the box
    below the cropped min"""
    cases = []
    for c, L, v in (((0.0, 0.0, 0.0), 10.0, 0.3), ((123.456, -77.7, 3.25), 25.0, 0.45), ((1e4 + 0.1, 2e3, -5.0), 40.0, 0.25)):
        c = np.array(c)
        lo, hi = c - L, c + L
        p = c + rng.uniform(-L, L, (4000, 3))
        k = 0
        for d in range(3):
            for edge, out in ((lo[d], -math.inf), (hi[d], math.inf)):
                for x in (edge, math.nextafter(edge, out)):
                    p[k:k + 20, d] = x
                    k += 20
        p[k:k + 50] = lo - rng.uniform(0.5, 30.0, (50, 3))   # outside, below the cropped min
        cases.append(dict(p=p, voxel=v, lo=lo, hi=hi, centre=c, L=L))
    return cases


SCENES = dict(faces_dyadic=scene_faces_dyadic, faces_rounded=scene_faces_rounded, far=scene_far, crowded=scene_crowded,
              counts=scene_counts, key_range=scene_key_range, headroom=scene_headroom, nonfinite=scene_nonfinite,
              crop=scene_crop)


def scene(name, seed=2024):
    return SCENES[name](np.random.default_rng([seed, list(SCENES).index(name)]))
