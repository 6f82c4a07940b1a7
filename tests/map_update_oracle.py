"""numpy restatement of updating a prior map (include/tloam_b200.h "Updating a prior map"; k_mu_* in libtloam_b200_mapu.so
and k_gmd_* in libtloam_b200_gmd.so), bit for bit.

    votes:    map_dynamic_oracle.vote of the scan at T, on the prior rows, then on the additions of the earlier adds
    novelty:  p = T q by the localization's final pass (loop_verify_oracle.transform); new iff no prior row within
              novel_radius, by localize_oracle's grid (the cells it visits hold every row within the radius)
    build:    the prior rows not removed (map_dynamic_oracle.dynamic), then global_map_merge_oracle.merge of the additions
              not removed, the voxels kept that hold rows of at least min_frames distinct adds"""
import numpy as np

import global_map_merge_oracle as gmo
import localize_oracle as lo
import loop_verify_oracle as lvo
import loop_verify_submap_oracle as lso
import map_dynamic_oracle as mdo


def config(image=None, **overrides):
    """tloam_b200_map_update_default_config, with overrides (image: overrides of the range image's)"""
    c = dict(image=mdo.config(**(image or {})), novel_radius=0.5, voxel=0.5, min_frames=3)
    c.update(overrides)
    return c


def apply(T, Q):
    T = np.asarray(T, dtype=np.float64)
    return lvo.transform(Q, T[:3, :3], T[:3, 3])


def novel(g, P, r):
    """per row of P: no row of the grid's map has d2 <= r * r"""
    P = np.asarray(P, dtype=np.float64).reshape(-1, 3)
    near = np.zeros(len(P), dtype=bool)
    if len(P) and len(g["M"]):
        q, pos = lo.pairs(g, P, r)
        near[q[lso._d2(P[q], g["sxyz"][pos]) <= r * r]] = True
    return ~near


def distinct_frames(frames, start):
    """per voxel (rows frames[start[j]:start[j + 1]], non-decreasing): 1 + the number of increases"""
    frames = np.asarray(frames)
    inc = np.ones(len(frames), dtype=np.int64)
    inc[1:] = frames[1:] > frames[:-1]
    inc[start[:-1]] = 1
    return np.add.reduceat(inc, start[:-1]) if len(frames) else np.zeros(0, dtype=np.int64)


class Update:
    """the state of one prior map: add(scan, query, T) after each accepted localization, build() for the cloud"""

    def __init__(self, prior, cfg, cell=1.0):
        self.prior = np.asarray(prior, dtype=np.float64).reshape(-1, 3)
        self.cfg = cfg
        self.g = lo.grid(self.prior, cell)
        self.prior_through = np.zeros(len(self.prior), dtype=np.uint32)
        self.prior_hits = np.zeros(len(self.prior), dtype=np.uint32)
        self.xyz = np.zeros((0, 3))
        self.frame = np.zeros(0, dtype=np.uint32)
        self.through = np.zeros(0, dtype=np.uint32)
        self.hits = np.zeros(0, dtype=np.uint32)
        self.frames = 0

    def add(self, scan, query, T):
        """the scan rows (sensor frame) vote at T, then the new rows of the query (sensor frame) are appended"""
        img = self.cfg["image"]
        if len(self.prior):
            t, h = mdo.vote(self.prior, scan, T, img)
            self.prior_through, self.prior_hits = self.prior_through + t, self.prior_hits + h
        if len(self.xyz):
            t, h = mdo.vote(self.xyz, scan, T, img)
            self.through, self.hits = self.through + t, self.hits + h
        P = apply(T, query)
        new = novel(self.g, P, self.cfg["novel_radius"])
        k = int(new.sum())
        self.xyz = np.vstack([self.xyz, P[new]])
        self.frame = np.concatenate([self.frame, np.full(k, self.frames, dtype=np.uint32)])
        self.through = np.concatenate([self.through, np.zeros(k, dtype=np.uint32)])
        self.hits = np.concatenate([self.hits, np.zeros(k, dtype=np.uint32)])
        self.frames += 1
        return k

    def build(self):
        """(xyz, counts): the prior rows not removed in row order, then the supported voxels in ascending key order;
        raises global_map_merge_oracle.VoxelRangeError past 2^21 voxels"""
        img = self.cfg["image"]
        kept_prior = ~mdo.dynamic(self.prior_through, self.prior_hits, img)
        keep = ~mdo.dynamic(self.through, self.hits, img)
        A, F = self.xyz[keep], self.frame[keep]
        vox, support = np.zeros((0, 3)), np.zeros(0, dtype=np.int64)
        if len(A):
            key, _ = gmo.keys(A, self.cfg["voxel"])
            order = np.argsort(key, kind="stable")
            ks = key[order]
            heads = np.r_[True, ks[1:] != ks[:-1]]
            start = np.r_[np.flatnonzero(heads), len(ks)]
            vox, _ = gmo.merge(A, self.cfg["voxel"])
            support = distinct_frames(F[order], start)
        sup = support >= self.cfg["min_frames"]
        out = np.vstack([self.prior[kept_prior], vox[sup]])
        counts = dict(n_prior=len(self.prior), n_prior_removed=int((~kept_prior).sum()), n_additions=len(self.xyz),
                      n_additions_removed=int((~keep).sum()), n_voxels=len(vox), n_voxels_kept=int(sup.sum()),
                      n_total=len(out))
        return out, counts
