"""FrontEnd::processCloud (ref: src/front_end/front_end.cpp:181-199) and the selections of the first-frame branch / updateSubmap
(:285-305, :201-267) restated on the CPU oracle (oracle/pyoracle.py): VoxelDownSample of the ground and edge clouds,
extractPlanarSphere of the general cloud, SelectByIndex of the planar and sphere features.

Two points are fixed here that the reference leaves open or states oddly:
- VoxelDownSample emits voxels in std::unordered_map order (implementation-defined); the oracle emits them in ascending voxel
  index (ix, iy, iz), and so must the device for the scan features (the registration caps take them in index order).
- the reference's sphere lists hold ranks 0..n-1, not point indices (feature_extract.cpp:183-188, SURVEY Q12); SelectByIndex
  takes them literally, so the sphere feature is the general cloud's first n_sphere_scan points."""
import numpy as np


def voxel_indices(pts, voxel, min_bound):
    """the integer voxel index (ix, iy, iz) of every point of `pts` for a down-sample of a cloud whose minimum is min_bound
    (ref: src/open3d/PointCloud2.cpp:367, :381-383)"""
    mb = np.asarray(min_bound, dtype=np.float64) - voxel * 0.5
    return np.floor((np.asarray(pts, dtype=np.float64).reshape(-1, 3) - mb) / voxel).astype(np.int64)


def packed_keys(idx):
    """ix << 42 | iy << 21 | iz: numeric order = lexicographic order of non-negative indices below 2**21"""
    idx = np.asarray(idx, dtype=np.int64)
    return (idx[:, 0] << 42) | (idx[:, 1] << 21) | idx[:, 2]


def selections(oracle, general, **feature):
    """extractPlanarSphere + SelectByIndex: dict(planar, sphere, planar_sub, sphere_sub) of the general cloud"""
    general = np.ascontiguousarray(general, dtype=np.float64).reshape(-1, 3)
    if len(general) == 0:                       # calculatePCAInfo fails on an empty cloud: nothing selected (:49-54, :140)
        e = np.zeros((0, 3))
        return dict(planar=e, sphere=e, planar_sub=e, sphere_sub=e)
    p_scan, p_sub, s_scan, s_sub, _ = oracle.extract_planar_sphere(general, **feature)
    return dict(planar=general[p_scan], sphere=general[s_scan], planar_sub=general[p_sub], sphere_sub=general[s_sub])


def process_cloud(oracle, ground, edge, general, ground_down_sample=0.3, edge_down_sample=0.1, **feature):
    """the source of one frame: dict(edge, sphere, planar, ground) + the frame's submap selections (planar_sub, sphere_sub)"""
    out = selections(oracle, general, **feature)
    out["ground"] = oracle.voxel_down_sample(ground, ground_down_sample)
    out["edge"] = oracle.voxel_down_sample(edge, edge_down_sample)
    return out


def source(frame):
    """ABI cloud order: edge, sphere, planar, ground"""
    return [frame["edge"], frame["sphere"], frame["planar"], frame["ground"]]
