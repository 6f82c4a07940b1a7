"""CPU restatement of loop closure (include/tloam_b200.h "Loop closure", kernels in tloam_b200/csrc/scan_context.cu):
Scan Context descriptors and the exhaustive search, every operation rounded as the device rounds it, so that descriptors and
distances are compared bit for bit.  numpy's elementwise + - * / and sqrt are correctly rounded and never fused; every sum
below is an explicit loop in the definition's order (never np.sum, which sums pairwise).

Two forms: the vectorised one the GPU tests use, and a literal per-row / per-column transcription the CPU tests pin it to."""
import math
import struct

import numpy as np

DEFAULT = dict(lidar_height=2.0, n_ring=20, n_sector=60, max_radius=80.0, exclude_recent=50, dist_threshold=0.13)
_TOP = np.uint64(0x8000000000000000)


def config(**overrides):
    c = dict(DEFAULT)
    c.update(overrides)
    return c


def boundaries(n_sector):
    """(n_sector - 1, 2): (cos, sin) of 2 pi k / n_sector, k = 1 .., by the C library (math.cos / math.sin call libm, as the
    library's host code does)"""
    d = np.zeros((max(n_sector - 1, 0), 2))
    for k in range(1, n_sector):
        t = 2.0 * math.pi * k / n_sector
        d[k - 1] = (math.cos(t), math.sin(t))
    return d


# ---- vectorised ------------------------------------------------------------------------------------------------------
def _enc(v):
    u = np.ascontiguousarray(v, dtype=np.float64).view(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | _TOP)


def _dec(e):
    return np.where(e >> np.uint64(63), e & ~_TOP, ~e).view(np.float64)


def rings_sectors(xyz, cfg):
    """(kept rows' values z + lidar_height, ring, sector) of a scan"""
    p = np.asarray(xyz, dtype=np.float64).reshape(-1, 3)
    p = p[np.isfinite(p).all(axis=1)]
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r = np.sqrt(x * x + y * y)
    keep = r <= cfg["max_radius"]
    x, y, z, r = x[keep], y[keep], z[keep], r[keep]
    R, S = cfg["n_ring"], cfg["n_sector"]
    ring = np.clip(np.ceil(r / cfg["max_radius"] * R), 1, R).astype(np.int64) - 1
    D = boundaries(S)
    n_up = (S - 1) // 2
    cross = D[None, :, 0] * y[:, None] - D[None, :, 1] * x[:, None]
    upper = (y > 0) | ((y == 0) & (x >= 0))
    sector = np.where(upper, (cross[:, :n_up] > 0).sum(axis=1), n_up + (cross[:, n_up:] > 0).sum(axis=1))
    return z + cfg["lidar_height"], ring, sector


def descriptor(xyz, cfg):
    """(bins (n_ring, n_sector), ring key (n_ring,), column norms (n_sector,))"""
    R, S = cfg["n_ring"], cfg["n_sector"]
    v, ring, sector = rings_sectors(xyz, cfg)
    e = np.zeros(R * S, dtype=np.uint64)
    np.maximum.at(e, ring * S + sector, _enc(v))                   # the exact maximum, -0.0 < +0.0 as on the device
    bins = np.where(e == 0, 0.0, _dec(e)).reshape(R, S)
    acc = np.zeros(R)
    for s in range(S):
        acc = acc + bins[:, s]
    key = acc / float(S)
    acc = np.zeros(S)
    for r in range(R):
        acc = acc + bins[r] * bins[r]
    return bins, key, np.sqrt(acc)


def distances(query, cands):
    """(M, n_sector): the distance of query (a descriptor) to each candidate descriptor at every shift"""
    A, _, na = query
    R, S = A.shape
    if not cands:
        return np.zeros((0, S))
    B = np.stack([c[0] for c in cands])
    nb = np.stack([c[2] for c in cands])
    col = (np.arange(S)[None, :] - np.arange(S)[:, None]) % S     # [s, c]: the candidate's column that meets c
    nbs = nb[:, col]                                              # (M, S, S)
    valid = (na[None, None, :] != 0) & (nbs != 0)
    dot = np.zeros(nbs.shape)
    for r in range(R):
        dot = dot + A[r][None, None, :] * B[:, r, :][:, col]
    with np.errstate(divide="ignore", invalid="ignore"):
        cos = dot / (na[None, None, :] * nbs)
    total = np.zeros(nbs.shape[:2])
    count = np.zeros(nbs.shape[:2])
    for c in range(S):
        total = np.where(valid[..., c], total + cos[..., c], total)
        count = count + valid[..., c]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(count > 0, 1.0 - total / count, 1.0)


def yaw_of(shift, n_sector):
    k = n_sector - shift if 2 * shift >= n_sector else -shift
    return k * (2.0 * math.pi / n_sector)


def query(descs, i, exclude_recent, chunk=256):
    """frame i's result over frames j <= i - exclude_recent: (candidate, shift, distance, table (M, n_sector))"""
    M = i - exclude_recent + 1 if i >= exclude_recent else 0
    if M <= 0:
        return -1, 0, math.inf, np.zeros((0, descs[i][0].shape[1]))
    table = np.concatenate([distances(descs[i], descs[a:min(a + chunk, M)]) for a in range(0, M, chunk)])
    k = int(np.argmin(table))                                     # the first minimum: smallest j, then smallest s
    j, s = divmod(k, table.shape[1])
    return j, s, float(table[j, s]), table


# ---- literal transcription ---------------------------------------------------------------------------------------------
def _key(v):
    u = struct.unpack("<Q", struct.pack("<d", v))[0]
    return (~u & 0xFFFFFFFFFFFFFFFF) if u >> 63 else u | (1 << 63)


def descriptor_literal(xyz, cfg):
    R, S, h, maxr = cfg["n_ring"], cfg["n_sector"], cfg["lidar_height"], cfg["max_radius"]
    D = boundaries(S)
    n_up = (S - 1) // 2
    best = [[None] * S for _ in range(R)]
    for x, y, z in np.asarray(xyz, dtype=np.float64).reshape(-1, 3).tolist():
        if not (math.isfinite(x) and math.isfinite(y) and math.isfinite(z)):
            continue
        r = math.sqrt(x * x + y * y)
        if r > maxr:
            continue
        ring = min(max(math.ceil(r / maxr * R), 1), R) - 1
        if y > 0 or (y == 0 and x >= 0):
            sector, ks = 0, range(1, n_up + 1)
        else:
            sector, ks = n_up, range(n_up + 1, S)
        for k in ks:
            c, s = D[k - 1]
            if float(c) * y - float(s) * x > 0:
                sector += 1
        v = z + h
        if best[ring][sector] is None or _key(v) > _key(best[ring][sector]):
            best[ring][sector] = v
    bins = np.array([[0.0 if b is None else b for b in row] for row in best])
    key = np.zeros(R)
    for r in range(R):
        acc = 0.0
        for s in range(S):
            acc += float(bins[r, s])
        key[r] = acc / S
    norms = np.zeros(S)
    for c in range(S):
        acc = 0.0
        for r in range(R):
            acc += float(bins[r, c]) * float(bins[r, c])
        norms[c] = math.sqrt(acc)
    return bins, key, norms


def distance_literal(a, b, shift):
    (A, _, na), (B, _, nb) = a, b
    R, S = A.shape
    total, count = 0.0, 0
    for c in range(S):
        cb = (c - shift) % S
        if na[c] != 0 and nb[cb] != 0:
            dot = 0.0
            for r in range(R):
                dot += float(A[r, c]) * float(B[r, cb])
            total += dot / (float(na[c]) * float(nb[cb]))
            count += 1
    return 1.0 - total / count if count else 1.0
