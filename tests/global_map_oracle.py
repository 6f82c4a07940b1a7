"""The global map of FrontEnd (ref: src/front_end/front_end.cpp:269-274, with mapping_flag set) restated on the CPU oracle:

    curr_map = raw.Transform(pose)                 # in place (PointCloud2.cpp:71-75)
    global_map += curr_map->VoxelDownSample(1.0)   # this frame only (:358-403), then operator+= (:96-132)

Fixed here where the reference leaves it open:
- non-finite rows are left out before the down-sample (the reference feeds them to GetMinBound and int(floor(NaN)));
- each frame's voxels come out in ascending voxel index (ix, iy, iz) (the oracle's VoxelDownSample order), frames in call
  order, so the map is deterministic;
- the first frame never reaches updateSubmap (:285-305 returns first): the loop appends from frame 1 on."""
import numpy as np


def transform(raw, pose):
    """T.p of every row (non-finite rows stay non-finite)"""
    raw = np.asarray(raw, dtype=np.float64).reshape(-1, 3)
    pose = np.asarray(pose, dtype=np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        return raw @ pose[:3, :3].T + pose[:3, 3]


def frame_block(oracle, registered, voxel=1.0):
    """VoxelDownSample(voxel) of the finite rows of one registered scan, ascending voxel key"""
    reg = np.asarray(registered, dtype=np.float64).reshape(-1, 3)
    fin = np.ascontiguousarray(reg[np.isfinite(reg).all(axis=1)])
    if len(fin) == 0:
        return np.zeros((0, 3))
    return oracle.voxel_down_sample(fin, voxel)


def global_map(oracle, registered_scans, voxel=1.0):
    """concatenation of the per-frame blocks: (map, offsets) with frame f = map[offsets[f]:offsets[f + 1]]"""
    blocks = [frame_block(oracle, r, voxel) for r in registered_scans]
    offsets = np.concatenate([[0], np.cumsum([len(b) for b in blocks], dtype=np.int64)])
    return (np.concatenate(blocks) if blocks else np.zeros((0, 3))), offsets


def front_end_map(oracle, raws, poses, voxel=1.0):
    """FrontEnd's loop: frame 0 seeds the submap and returns, frames 1.. are transformed by their pose and appended"""
    return global_map(oracle, [transform(r, p) for r, p in zip(raws[1:], poses[1:])], voxel)
