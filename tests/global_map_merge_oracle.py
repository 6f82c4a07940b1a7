"""numpy restatement of the merged global map (include/tloam_b200.h "Merged global map"; k_gmm_* in libtloam_b200_gmm.so):
VoxelDownSample of the whole map (ref: src/open3d/PointCloud2.cpp:358-403) with the voxels in ascending (ix, iy, iz).

- mb = min - voxel * 0.5 per axis, index floor((p - mb) / voxel), every operation rounded on its own (numpy's elementwise
  float64 operations are)
- refused (VoxelRangeError) when the max row's (max - mb) / voxel reaches 2^21 on an axis, or a row is not finite
- key ix << (by + bz) | iy << bz | iz with the bits of each axis' largest index; a stable argsort keeps each voxel's rows
  in row order
- the sums are sequential per voxel (+0.0, then += row by row): vectorised across voxels by looping over the position
  within the voxel, the voxels ordered by count so that the live ones are a prefix; then / count

`merge_literal` is the reference's loop transcribed (a dict of running sums, then sorted by key)."""
import math

import numpy as np

KEY_BITS = 21


class VoxelRangeError(Exception):
    pass


def _bounds(p, voxel):
    if not np.isfinite(p).all():
        raise VoxelRangeError("a row is not finite")
    mb = p.min(axis=0) - voxel * 0.5
    ref = (p.max(axis=0) - mb) / voxel
    if not (ref < float(1 << KEY_BITS)).all():
        raise VoxelRangeError("voxel_size is too small")
    return mb, ref


def keys(points, voxel):
    """(key per row, index per row (n, 3)) of the definition"""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    mb, ref = _bounds(p, voxel)
    idx = np.floor((p - mb) / voxel).astype(np.int64)
    bits = [int(t).bit_length() for t in np.floor(ref).astype(np.int64)]
    key = (idx[:, 0] << (bits[1] + bits[2])) | (idx[:, 1] << bits[2]) | idx[:, 2]
    return key, idx


def merge(points, voxel, intensity=None):
    """(xyz (n_vox, 3), intensity (n_vox,) or None) of VoxelDownSample(voxel), voxels in ascending (ix, iy, iz)"""
    p = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    inten = None if intensity is None else np.asarray(intensity, dtype=np.float64).reshape(-1)
    if len(p) == 0:
        return np.zeros((0, 3)), (None if inten is None else np.zeros(0))
    key, _ = keys(p, voxel)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    head = np.ones(len(ks), dtype=bool)
    head[1:] = ks[1:] != ks[:-1]
    start = np.nonzero(head)[0]
    count = np.diff(np.append(start, len(ks)))
    vals = p[order] if inten is None else np.column_stack([p[order], inten[order]])
    by_count = np.argsort(-count, kind="stable")                   # the voxels live at step k are a prefix
    cs, ss = count[by_count], start[by_count]
    sums = np.zeros((len(count), vals.shape[1]))
    live = len(cs)
    for k in range(int(cs[0])):
        while live and cs[live - 1] <= k:
            live -= 1
        sums[:live] = sums[:live] + vals[ss[:live] + k]
    out = np.empty_like(sums)
    out[by_count] = sums / cs.astype(np.float64)[:, None]
    return out[:, :3].copy(), (None if inten is None else out[:, 3].copy())


def merge_literal(points, voxel, intensity=None):
    """PointCloud2::VoxelDownSample's loop (:379-399) in Python floats, with the key-range rule above; sorted by index"""
    pts = [tuple(float(v) for v in row) for row in np.asarray(points, dtype=np.float64).reshape(-1, 3)]
    if not pts:
        return np.zeros((0, 3)), (None if intensity is None else np.zeros(0))
    for row in pts:
        if not all(math.isfinite(v) for v in row):
            raise VoxelRangeError("a row is not finite")
    half = voxel * 0.5
    mb = [min(r[d] for r in pts) - half for d in range(3)]
    for d in range(3):
        if not ((max(r[d] for r in pts) - mb[d]) / voxel < float(1 << KEY_BITS)):
            raise VoxelRangeError("voxel_size is too small")
    acc = {}
    for i, row in enumerate(pts):
        vi = tuple(int(math.floor((row[d] - mb[d]) / voxel)) for d in range(3))
        a = acc.setdefault(vi, [0, 0.0, 0.0, 0.0, 0.0])
        a[1] += row[0]
        a[2] += row[1]
        a[3] += row[2]
        if intensity is not None:
            a[4] += float(intensity[i])
        a[0] += 1
    xyz, inten = [], []
    for vi in sorted(acc):
        n, sx, sy, sz, si = acc[vi]
        xyz.append([sx / float(n), sy / float(n), sz / float(n)])
        inten.append(si / float(n))
    return np.array(xyz), (None if intensity is None else np.array(inten))
