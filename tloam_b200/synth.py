"""Deterministic synthetic Velodyne-64-shaped scenes for the TLS registration path (SURVEY.md 8(d)).

The world is an infinite, lattice-anchored "city": a ground plane at z = -1.73 (sensor height,
ref: config/mapping/segmentation.yaml:4), building blocks with vertical walls (planar features), vertical
poles (edge features, direction |z| > 0.85, ref: config/mapping/lidar_odometry.yaml:27) and compact blobs
(sphere features).  Every surface sample is a jittered lattice node whose jitter is a hash of its integer
node id, so the world is a pure function of (seed, position): consecutive frames of a stream see the same
map.  Scan features are *independent* samples of the same surfaces (different hash stream), moved into the
sensor frame with T_gt^-1, plus Gaussian noise and gross outliers.

Cloud order everywhere: (edge, sphere, planar, ground), as at the C ABI (ref: registration.cpp:233-236).
"""
from dataclasses import dataclass, field
import os

import numpy as np

CLOUDS = ("edge", "sphere", "planar", "ground")
GROUND_Z = -1.73

# lattice spacings (m): chosen so that >= 5 map neighbours exist inside each search radius
# (ref: config/mapping/lidar_odometry.yaml:7,9 use 0.3 / 0.45 voxels for the submaps)
SP_GROUND = 0.33
SP_WALL = 0.30
SP_POLE = 0.25
POLE_PITCH = 4.0
POLE_HEIGHT = 10.0
BLOCK_PITCH = 40.0
BLOB_PITCH = 8.0
BLOB_POINTS = 32


@dataclass
class SceneConfig:
    seed: int = 20260924
    n_map: tuple = (100_000, 20_000, 210_000, 170_000)      # edge, sphere, planar, ground (M = 500k)
    n_feat: tuple = (8_000, 1_600, 16_800, 13_600)           # F = 40k
    scan_noise: float = 0.01          # = noise_bound
    outlier_frac: float = 0.10
    outlier_mag: float = 0.30
    map_noise: float = 0.01
    feat_range_frac: float = 0.80     # features are drawn inside this fraction of the map half-extent


def scaled(scale, **kw):
    """BASELINE sizes scaled by `scale` in point count (area scales, density stays)."""
    base = SceneConfig()
    return SceneConfig(n_map=tuple(max(64, int(n * scale)) for n in base.n_map),
                       n_feat=tuple(max(32, int(n * scale)) for n in base.n_feat), **kw)


# ------------------------------------------------------------------------------------------------
# hashing: splitmix64 over uint64 arrays -> uniform [0,1)
# ------------------------------------------------------------------------------------------------
_M1 = np.uint64(0xBF58476D1CE4E5B9)
_M2 = np.uint64(0x94D049BB133111EB)
_G = np.uint64(0x9E3779B97F4A7C15)


def _mix(x):
    with np.errstate(over="ignore"):
        x = (x + _G).astype(np.uint64)
        x = (x ^ (x >> np.uint64(30))) * _M1
        x = (x ^ (x >> np.uint64(27))) * _M2
        return x ^ (x >> np.uint64(31))


def _key(*parts):
    """Combine integer arrays / scalars into one uint64 hash key."""
    h = np.uint64(0x243F6A8885A308D3)
    for p in parts:
        with np.errstate(over="ignore"):
            h = _mix(np.asarray(h, dtype=np.uint64) ^ (np.asarray(p).astype(np.int64).astype(np.uint64) * _G))
    return h


def _u01(key, stream):
    with np.errstate(over="ignore"):
        h = _mix(key ^ (np.asarray(stream, dtype=np.uint64) * _M1))
    return (h >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))


def _gauss(key, stream):
    u1 = np.maximum(_u01(key, stream), 1e-300)
    u2 = _u01(key, stream + 1)
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def _irange(lo, hi, pitch):
    return np.arange(int(np.floor(lo / pitch)) - 1, int(np.ceil(hi / pitch)) + 2, dtype=np.int64)


# ------------------------------------------------------------------------------------------------
# surface samplers: return (N,3) world points whose xy lie in the square |x-cx|,|y-cy| <= L
# `stream` selects the jitter stream: 0 = map, 1 = scan features.
# ------------------------------------------------------------------------------------------------
def _ground(seed, cx, cy, L, stream, noise):
    ix = _irange(cx - L, cx + L, SP_GROUND)
    iy = _irange(cy - L, cy + L, SP_GROUND)
    gx, gy = np.meshgrid(ix, iy, indexing="ij")
    gx = gx.ravel()
    gy = gy.ravel()
    k = _key(seed, 11, stream, gx, gy)
    x = (gx + 0.9 * (_u01(k, 1) - 0.5)) * SP_GROUND
    y = (gy + 0.9 * (_u01(k, 2) - 0.5)) * SP_GROUND
    z = GROUND_Z + noise * _gauss(k, 3)
    return np.stack([x, y, z], axis=1)


def _walls(seed, cx, cy, L, stream, noise):
    bx = _irange(cx - L, cx + L, BLOCK_PITCH)
    by = _irange(cy - L, cy + L, BLOCK_PITCH)
    out = []
    for ibx in bx:
        for iby in by:
            kb = _key(seed, 23, int(ibx), int(iby))
            ccx = (ibx + 0.5 + 0.2 * (float(_u01(kb, 1)) - 0.5)) * BLOCK_PITCH
            ccy = (iby + 0.5 + 0.2 * (float(_u01(kb, 2)) - 0.5)) * BLOCK_PITCH
            hx = 8.0 + 6.0 * float(_u01(kb, 3))
            hy = 8.0 + 6.0 * float(_u01(kb, 4))
            H = 6.0 + 6.0 * float(_u01(kb, 5))
            yaw = 0.12 * (float(_u01(kb, 6)) - 0.5)          # small block rotation: normals keep |n_z| = 0
            c, s = np.cos(yaw), np.sin(yaw)
            iz = np.arange(0, int(np.floor((H - GROUND_Z) / SP_WALL)), dtype=np.int64)
            for face in range(4):
                half = hx if face < 2 else hy               # half-length along the face
                off = hy if face < 2 else hx                # distance of the face from the centre
                sign = 1.0 if face % 2 == 0 else -1.0
                iu = np.arange(int(np.floor(-half / SP_WALL)), int(np.ceil(half / SP_WALL)) + 1, dtype=np.int64)
                gu, gz = np.meshgrid(iu, iz, indexing="ij")
                gu = gu.ravel()
                gz = gz.ravel()
                k = _key(seed, 29, stream, int(ibx), int(iby), face, gu, gz)
                u = (gu + 0.9 * (_u01(k, 1) - 0.5)) * SP_WALL
                z = GROUND_Z + (gz + 0.5 + 0.9 * (_u01(k, 2) - 0.5)) * SP_WALL
                d = sign * off + noise * _gauss(k, 3)       # along the face normal
                keep = np.abs(u) <= half
                u, z, d = u[keep], z[keep], d[keep]
                if face < 2:
                    lx, ly = u, d                           # normal = +-y
                else:
                    lx, ly = d, u                           # normal = +-x
                x = ccx + c * lx - s * ly
                y = ccy + s * lx + c * ly
                out.append(np.stack([x, y, z], axis=1))
    pts = np.concatenate(out, axis=0) if out else np.zeros((0, 3))
    keep = (np.abs(pts[:, 0] - cx) <= L) & (np.abs(pts[:, 1] - cy) <= L)
    return pts[keep]


def _poles(seed, cx, cy, L, stream, noise):
    ix = _irange(cx - L, cx + L, POLE_PITCH)
    iy = _irange(cy - L, cy + L, POLE_PITCH)
    gx, gy = np.meshgrid(ix, iy, indexing="ij")
    gx = gx.ravel()
    gy = gy.ravel()
    kp = _key(seed, 37, gx, gy)
    px = (gx + 0.5 + 0.6 * (_u01(kp, 1) - 0.5)) * POLE_PITCH
    py = (gy + 0.5 + 0.6 * (_u01(kp, 2) - 0.5)) * POLE_PITCH
    keep = (np.abs(px - cx) <= L) & (np.abs(py - cy) <= L)
    gx, gy, px, py = gx[keep], gy[keep], px[keep], py[keep]
    nz = int(POLE_HEIGHT / SP_POLE)
    iz = np.arange(nz, dtype=np.int64)
    GX = np.repeat(gx, nz)
    GY = np.repeat(gy, nz)
    IZ = np.tile(iz, gx.size)
    k = _key(seed, 41, stream, GX, GY, IZ)
    z = GROUND_Z + (IZ + 0.5 + 0.9 * (_u01(k, 1) - 0.5)) * SP_POLE
    x = np.repeat(px, nz) + noise * _gauss(k, 2)
    y = np.repeat(py, nz) + noise * _gauss(k, 4)
    return np.stack([x, y, z], axis=1)


def _blobs(seed, cx, cy, L, stream, noise):
    ix = _irange(cx - L, cx + L, BLOB_PITCH)
    iy = _irange(cy - L, cy + L, BLOB_PITCH)
    gx, gy = np.meshgrid(ix, iy, indexing="ij")
    gx = gx.ravel()
    gy = gy.ravel()
    kb = _key(seed, 53, gx, gy)
    bx = (gx + 0.5 + 0.7 * (_u01(kb, 1) - 0.5)) * BLOB_PITCH
    by = (gy + 0.5 + 0.7 * (_u01(kb, 2) - 0.5)) * BLOB_PITCH
    bz = GROUND_Z + 0.5 + 2.5 * _u01(kb, 3)
    br = 0.25 + 0.25 * _u01(kb, 4)
    keep = (np.abs(bx - cx) <= L) & (np.abs(by - cy) <= L)
    gx, gy, bx, by, bz, br = gx[keep], gy[keep], bx[keep], by[keep], bz[keep], br[keep]
    n = BLOB_POINTS
    GX = np.repeat(gx, n)
    GY = np.repeat(gy, n)
    J = np.tile(np.arange(n, dtype=np.int64), gx.size)
    k = _key(seed, 59, stream, GX, GY, J)
    # quasi-uniform directions on the sphere (Fibonacci) + jitter
    zc = 1.0 - 2.0 * (J + 0.5) / n + 0.02 * (_u01(k, 1) - 0.5)
    zc = np.clip(zc, -1.0, 1.0)
    phi = J * 2.399963229728653 + 0.3 * (_u01(k, 2) - 0.5)
    rxy = np.sqrt(1.0 - zc * zc)
    r = np.repeat(br, n) + noise * _gauss(k, 3)
    x = np.repeat(bx, n) + r * rxy * np.cos(phi)
    y = np.repeat(by, n) + r * rxy * np.sin(phi)
    z = np.repeat(bz, n) + r * zc
    return np.stack([x, y, z], axis=1)


_SAMPLERS = (_poles, _blobs, _walls, _ground)                       # edge, sphere, planar, ground
# nominal map density (points per m^2 of ground area) used to size the generation window
_DENSITY = (POLE_HEIGHT / SP_POLE / POLE_PITCH ** 2, BLOB_POINTS / BLOB_PITCH ** 2, 5.0, 1.0 / SP_GROUND ** 2)


def _half_extent(n, cloud):
    return 0.5 * np.sqrt(n / _DENSITY[cloud])


def _trim_nearest(pts, cx, cy, n):
    if pts.shape[0] <= n:
        return pts
    d = np.maximum(np.abs(pts[:, 0] - cx), np.abs(pts[:, 1] - cy))
    idx = np.argpartition(d, n - 1)[:n]
    idx.sort()                                                       # keep lattice order (deterministic)
    return pts[idx]


def se3_exp(a):
    """Plain numpy SE(3) exponential (upsilon, omega) -> 4x4; generator-side only."""
    a = np.asarray(a, dtype=np.float64)
    ups, om = a[:3], a[3:]
    th = np.linalg.norm(om)
    O = np.array([[0, -om[2], om[1]], [om[2], 0, -om[0]], [-om[1], om[0], 0]])
    if th < 1e-12:
        R = np.eye(3) + O
        V = np.eye(3) + 0.5 * O
    else:
        R = np.eye(3) + np.sin(th) / th * O + (1 - np.cos(th)) / th ** 2 * O @ O
        V = np.eye(3) + (1 - np.cos(th)) / th ** 2 * O + (th - np.sin(th)) / th ** 3 * O @ O
    T = np.eye(4)
    T[:3, :3] = R
    T[:3, 3] = V @ ups
    return T


def make_map(cfg, T_gt):
    """The four local-map clouds (world frame) around the pose T_gt. Returns list of (n_c,3) float64."""
    cx, cy = float(T_gt[0, 3]), float(T_gt[1, 3])
    clouds = []
    for c in range(4):
        L = _half_extent(cfg.n_map[c], c)
        pts = _SAMPLERS[c](cfg.seed, cx, cy, 1.25 * L + 2.0, 0, cfg.map_noise)
        clouds.append(np.ascontiguousarray(_trim_nearest(pts, cx, cy, cfg.n_map[c])))
    return clouds


def make_scan(cfg, T_gt, frame_id=0):
    """The four scan-feature clouds in the SENSOR frame for ground-truth pose T_gt."""
    cx, cy = float(T_gt[0, 3]), float(T_gt[1, 3])
    Tinv = np.linalg.inv(T_gt)
    rng = np.random.Generator(np.random.MT19937(cfg.seed + 7919 * (frame_id + 1)))
    clouds = []
    for c in range(4):
        L = cfg.feat_range_frac * _half_extent(cfg.n_map[c], c)
        pts = _SAMPLERS[c](cfg.seed, cx, cy, L, 1, 0.0)
        n = min(cfg.n_feat[c], pts.shape[0])
        sel = np.sort(rng.choice(pts.shape[0], size=n, replace=False))
        pts = pts[sel]
        pts = pts @ Tinv[:3, :3].T + Tinv[:3, 3]
        if cfg.scan_noise > 0:
            pts = pts + rng.normal(0.0, cfg.scan_noise, size=pts.shape)
        if cfg.outlier_frac > 0:
            m = rng.random(n) < cfg.outlier_frac
            pts[m] += rng.uniform(-cfg.outlier_mag, cfg.outlier_mag, size=(int(m.sum()), 3))
        clouds.append(np.ascontiguousarray(pts))
    return clouds


# config 1 (SURVEY.md 8(d)): fixed ground truth and prediction
CONFIG1_GT = (0.8, 0.02, 0.01, 0.001, -0.002, 0.015)
CONFIG1_PERTURB = (0.05, -0.03, 0.01, 0.004, -0.003, 0.006)


def config1(cfg=None):
    cfg = cfg or SceneConfig(seed=20260924 + 1000 * 1)
    T_gt = se3_exp(CONFIG1_GT)
    predict = T_gt @ se3_exp(CONFIG1_PERTURB)
    return dict(cfg=cfg, T_gt=T_gt, predict=predict, map=make_map(cfg, T_gt), scan=make_scan(cfg, T_gt, 0))


def config3(n_feat=500_000, n_map=2_000_000, seed=20260924 + 3000, noise=0.01, outlier_frac=0.10):
    """BASELINE config 3 (SURVEY.md 8(d)): dense indoor scan, planar-only residuals (factor_num = 2: the planar and
    ground builders, ref: registration.hpp:144-148), room 20 x 30 x 4 m.  ground cloud = floor, planar cloud = walls +
    ceiling, each half of the points; the edge / sphere clouds only carry the 16 dummy points the >= 10-point
    rule needs.  Surfaces are sampled uniformly at random (no lattice), spacing ~0.03 m at the full size."""
    rng = np.random.Generator(np.random.MT19937(seed))
    LX, LY, LZ = 20.0, 30.0, 4.0

    def floor(n):
        return np.stack([rng.uniform(0, LX, n), rng.uniform(0, LY, n), np.zeros(n)], axis=1)

    def shell(n):                                  # 4 walls + ceiling, area-proportional
        areas = np.array([LX * LZ, LX * LZ, LY * LZ, LY * LZ, LX * LY])
        which = rng.choice(5, size=n, p=areas / areas.sum())
        u, v = rng.uniform(0, 1, n), rng.uniform(0, 1, n)
        pts = np.zeros((n, 3))
        for k in range(5):
            m = which == k
            if k == 0:
                pts[m] = np.stack([u[m] * LX, np.zeros(m.sum()), v[m] * LZ], axis=1)
            elif k == 1:
                pts[m] = np.stack([u[m] * LX, np.full(m.sum(), LY), v[m] * LZ], axis=1)
            elif k == 2:
                pts[m] = np.stack([np.zeros(m.sum()), u[m] * LY, v[m] * LZ], axis=1)
            elif k == 3:
                pts[m] = np.stack([np.full(m.sum(), LX), u[m] * LY, v[m] * LZ], axis=1)
            else:
                pts[m] = np.stack([u[m] * LX, v[m] * LY, np.full(m.sum(), LZ)], axis=1)
        return pts

    T_gt = se3_exp([9.0, 14.0, 1.5, 0.01, -0.015, 0.6])
    predict = T_gt @ se3_exp([0.04, -0.03, 0.02, 0.004, -0.003, 0.006])
    dummy = np.array([[LX / 2, LY / 2, 1.0]]) + rng.normal(0, 0.05, (16, 3))
    mp = [dummy.copy(), dummy.copy(), shell(n_map // 2) + rng.normal(0, 0.003, (n_map // 2, 3)),
          floor(n_map - n_map // 2) + rng.normal(0, 0.003, (n_map - n_map // 2, 3))]
    Tinv = np.linalg.inv(T_gt)

    def to_scan(p):
        q = p @ Tinv[:3, :3].T + Tinv[:3, 3] + rng.normal(0, noise, p.shape)
        m = rng.random(len(q)) < outlier_frac
        q[m] += rng.uniform(-0.3, 0.3, (int(m.sum()), 3))
        return np.ascontiguousarray(q)

    scan = [to_scan(dummy), to_scan(dummy), to_scan(shell(n_feat // 2)), to_scan(floor(n_feat - n_feat // 2))]
    return dict(T_gt=T_gt, predict=predict, map=mp, scan=scan, factor_num=2)


def load_motion(seq="00"):
    here = os.path.dirname(os.path.abspath(__file__))
    path = os.path.join(here, "..", "tests", "golden", f"motion_seq{seq}.npy")
    return np.load(path).astype(np.float64)


@dataclass
class Stream:
    """KITTI-seq-shaped synthetic stream (config 2/4): ground-truth poses follow the relative motions of the
    reference's published trajectory (tests/golden/motion_seq*.npy, derived from doc/tloam_*.txt)."""
    cfg: SceneConfig = field(default_factory=SceneConfig)
    seq: str = "00"
    start: int = 0

    def __post_init__(self):
        self.motion = load_motion(self.seq)
        self.T = np.eye(4)
        for k in range(self.start):
            self.T = self.T @ se3_exp(self.motion[k % len(self.motion)])
        self.k = self.start

    def frame(self):
        """Returns dict(T_gt, map, scan, frame_id) for the current pose and advances the stream."""
        out = dict(T_gt=self.T.copy(), frame_id=self.k, map=make_map(self.cfg, self.T),
                   scan=make_scan(self.cfg, self.T, self.k))
        self.T = self.T @ se3_exp(self.motion[self.k % len(self.motion)])
        self.k += 1
        return out


def general_cloud(n=50_000, seed=20260924 + 4242, noise=0.004):
    """Synthetic "general" (non-ground, segmented) cloud for the PCA feature extraction, SENSOR frame, about n points:
    vertical wall patches (planar features), horizontal slabs (flat but not vertical), Gaussian blobs (sphere
    features), thin poles and isolated clutter (dropped by min_neigh).  Point spacing on the surfaces is 3-6 cm, so
    that a 0.2 m neighbourhood holds more than K = 20 points near the patch centres and fewer at their borders
    (ref for the consumer: src/models/feature_extraction/feature_extract.cpp:47-122)."""
    rng = np.random.Generator(np.random.MT19937(seed))
    parts = []

    def patch(count, origin, eu, ev, su, sv):
        uv = rng.random((count, 2)) * [su, sv]
        return origin + uv[:, :1] * eu + uv[:, 1:] * ev

    n_wall, n_slab, n_blob, n_pole = int(0.55 * n), int(0.15 * n), int(0.15 * n), int(0.10 * n)
    walls = max(4, n_wall // 3000)
    for w in range(walls):
        ang = rng.uniform(0, np.pi)
        eu = np.array([np.cos(ang), np.sin(ang), 0.0])
        org = np.array([rng.uniform(-40, 40), rng.uniform(-40, 40), rng.uniform(-1.5, 0.0)])
        parts.append(patch(n_wall // walls, org, eu, np.array([0.0, 0.0, 1.0]), 3.0, 1.8))
    slabs = max(2, n_slab // 3000)
    for s in range(slabs):
        org = np.array([rng.uniform(-40, 40), rng.uniform(-40, 40), rng.uniform(0.5, 2.5)])
        parts.append(patch(n_slab // slabs, org, np.array([1.0, 0.0, 0.0]), np.array([0.0, 1.0, 0.0]), 2.5, 2.0))
    blobs = max(8, n_blob // 150)
    for b in range(blobs):
        c = np.array([rng.uniform(-40, 40), rng.uniform(-40, 40), rng.uniform(-1.0, 2.0)])
        parts.append(c + rng.normal(0.0, 0.07, (n_blob // blobs, 3)))
    poles = max(4, n_pole // 400)
    for p in range(poles):
        c = np.array([rng.uniform(-40, 40), rng.uniform(-40, 40), -1.5])
        th, z = rng.uniform(0, 2 * np.pi, n_pole // poles), rng.uniform(0, 3.0, n_pole // poles)
        parts.append(c + np.c_[0.05 * np.cos(th), 0.05 * np.sin(th), z])
    pts = np.vstack(parts)
    pts = pts + rng.normal(0.0, noise, pts.shape)
    clutter = np.c_[rng.uniform(-45, 45, (max(n - pts.shape[0], 0), 2)), rng.uniform(-1.5, 3.0, max(n - pts.shape[0], 0))]
    pts = np.vstack([pts, clutter])
    return np.ascontiguousarray(pts[rng.permutation(pts.shape[0])])


def _street_hits(d, rng, lane_half_width):
    """Ray parameter of the first return of every unit direction d (inf: none) in the street scene: a ground plane at
    z = -1.73, two street-canyon walls y = +-lane_half_width (6 m high) and a few boxes."""
    t = np.full(len(d), np.inf)
    # ground
    with np.errstate(divide="ignore", invalid="ignore"):
        tg = np.where(d[:, 2] < -1e-6, -1.73 / d[:, 2], np.inf)
    t = np.minimum(t, tg)
    # walls y = +-lane_half_width, 6 m high
    for yw in (lane_half_width, -lane_half_width):
        with np.errstate(divide="ignore", invalid="ignore"):
            tw = np.where(d[:, 1] * yw > 1e-9, yw / d[:, 1], np.inf)
        z = tw * d[:, 2]
        t = np.minimum(t, np.where((z < 4.3) & (z > -1.73), tw, np.inf))
    # boxes (cars): axis-aligned, slab test
    for _ in range(12):
        c = np.array([rng.uniform(-40, 40), rng.uniform(-6, 6), -1.73 + 0.75])
        if abs(c[0]) < 4 and abs(c[1]) < 3:
            continue
        h = np.array([2.2, 0.9, 0.75])
        with np.errstate(divide="ignore", invalid="ignore"):
            t1, t2 = (c - h) / d, (c + h) / d
        tn, tf = np.nanmax(np.minimum(t1, t2), axis=1), np.nanmin(np.maximum(t1, t2), axis=1)
        t = np.minimum(t, np.where((tn <= tf) & (tn > 0), tn, np.inf))
    return t


def raw_scan(seed=20260924 + 5151, n_az=1875, noise=0.01, lane_half_width=8.0, drop=0.03):
    """A raw HDL-64E-shaped scan in the sensor frame, in the point ORDER the reference's beam estimate assumes
    (ref: src/models/segmentation/segmentation.cpp:341-384): beam after beam, every beam sweeping the azimuth from +x
    counter-clockwise through the four quadrants; elevation angles -24.9 deg + 0.4 deg per beam with the 1.7 deg gap
    after beam 31 (:194-196).  64 x 1875 = 120 000 rays are cast against a ground plane (z = -1.73 with gentle
    undulation), two street-canyon walls and a few boxes; rays without a return within 120 m are dropped."""
    rng = np.random.Generator(np.random.MT19937(seed))
    elev = np.array([-24.9 + 0.4 * i + (1.7 if i >= 31 else 0.0) for i in range(64)]) * np.pi / 180.0
    az = (np.arange(n_az) + 0.5) * (2 * np.pi / n_az)
    el, a = np.meshgrid(elev, az, indexing="ij")
    d = np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.sin(el)], axis=-1).reshape(-1, 3)
    t = _street_hits(d, rng, lane_half_width)
    keep = np.isfinite(t) & (t < 120.0) & (t > 3.0) & (rng.random(len(t)) >= drop)
    p = d[keep] * t[keep, None]
    p[:, 2] += 0.03 * np.sin(0.15 * p[:, 0]) * np.cos(0.11 * p[:, 1])           # gentle ground undulation
    return np.ascontiguousarray(p + rng.normal(0, noise, p.shape))


def vlp16_raw_scan(seed=20260924 + 6161, clockwise=True, start_azimuth=np.pi / 2, columns=1800, noise=0.01, lane_half_width=8.0,
                   drop=0.03, nonfinite=0.0, near=0.0):
    """A raw VLP-16-shaped scan of the street scene of raw_scan, in the driver's order: azimuth column after column, the 16
    lasers (-15 deg ... +15 deg in 2 deg steps) within a column.  The sweep starts at start_azimuth (rad, from +x) and turns
    clockwise seen from above (decreasing atan2, like the sensor) or counter-clockwise.  Rays without a return within
    120 m are dropped, as is a random fraction `drop`.  For the raw path: a fraction `nonfinite` of the rays becomes a NaN
    row (every third of them a +-Inf row instead), a fraction `near` becomes a return at 0.5-3 m (the vehicle body); both
    keep their place in the order.  About 29k points with the defaults."""
    rng = np.random.Generator(np.random.MT19937(seed))
    elev = np.radians(-15.0 + 2.0 * np.arange(16))
    step = 2 * np.pi / columns
    az = start_azimuth + (-1.0 if clockwise else 1.0) * (np.arange(columns) + 0.5) * step
    a, el = np.meshgrid(az, elev, indexing="ij")                                # column-major: lasers within a column
    d = np.stack([np.cos(el) * np.cos(a), np.cos(el) * np.sin(a), np.sin(el)], axis=-1).reshape(-1, 3)
    t = _street_hits(d, rng, lane_half_width)
    hit = np.isfinite(t) & (t < 120.0) & (rng.random(len(t)) >= drop)
    u = rng.random(len(t))
    bad = u < nonfinite
    close = (u >= nonfinite) & (u < nonfinite + near)
    t = np.where(close, 0.5 + 2.5 * rng.random(len(t)), t)
    keep = hit | bad | close
    p = d * np.where(np.isfinite(t), t, 0.0)[:, None]
    p[:, 2] += np.where(close, 0.0, 0.03 * np.sin(0.15 * p[:, 0]) * np.cos(0.11 * p[:, 1]))
    p = p + rng.normal(0, noise, p.shape)
    which = rng.integers(0, 3, len(t))
    p[bad & (which != 2), (which[bad & (which != 2)] % 3)] = np.nan
    p[bad & (which == 2), 0] = np.inf * np.sign(rng.random(int(np.sum(bad & (which == 2)))) - 0.5)
    return np.ascontiguousarray(p[keep])
