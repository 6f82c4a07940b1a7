"""The intensity channel of FrontEnd's global map (the reference's map is XYZI) restated literally on the CPU:

    curr_map = raw.Transform(pose)                 # intensity_ untouched (PointCloud2.cpp:71-75)
    global_map += curr_map->VoxelDownSample(1.0)   # per voxel: AccumulatedPoint (:253-286, :379-397), then operator+= (:96-132)

- AccumulatedPoint starts from intensity_ = 0.0 and adds cloud.intensity_[i] for the voxel's rows in ascending row order i
  (no NaN check), GetAverageIntensity = intensity_ / double(num_of_points_): a sequential FP64 sum from +0.0, / count.
- The down-sampled cloud has intensity iff the input HasIntensity(); operator+= ignores an empty cloud and otherwise keeps
  the map's channel iff (map empty || map has it) && the cloud has it.
- As in global_map_oracle.py, non-finite xyz rows are left out of the map, so their intensity is left out with them, and
  a frame's voxels come out in ascending voxel index (ix, iy, iz)."""
import numpy as np


def voxel_ranks(registered, voxel=1.0):
    """(rank per row of its voxel among the frame's voxels in ascending (ix, iy, iz), -1 for a non-finite row; voxel count)"""
    reg = np.asarray(registered, dtype=np.float64).reshape(-1, 3)
    fin = np.isfinite(reg).all(axis=1)
    ranks = np.full(len(reg), -1, dtype=np.int64)
    if not fin.any():
        return ranks, 0
    mb = reg[fin].min(axis=0) - voxel * 0.5                       # voxel_min_bound (:367)
    with np.errstate(invalid="ignore"):
        idx = np.floor((reg - mb) / voxel)                        # :381
    keys = sorted({tuple(int(v) for v in idx[i]) for i in range(len(reg)) if fin[i]})
    rank_of = {k: j for j, k in enumerate(keys)}
    for i in range(len(reg)):
        if fin[i]:
            ranks[i] = rank_of[tuple(int(v) for v in idx[i])]
    return ranks, len(keys)


def frame_intensity(registered, intensity, voxel=1.0):
    """the frame block's intensity, one value per voxel in emission order: the literal AccumulatedPoint loop"""
    ranks, nv = voxel_ranks(registered, voxel)
    inten = [float(v) for v in np.asarray(intensity, dtype=np.float64).reshape(-1)]
    acc = [0.0] * nv                                              # intensity_(0.0)
    num = [0] * nv
    for i, j in enumerate(ranks):                                 # ascending row order
        if j < 0:
            continue
        acc[j] = acc[j] + inten[i]
        num[j] += 1
    return np.array([acc[j] / float(num[j]) for j in range(nv)], dtype=np.float64)


class MapChannel:
    """points_ / intensity_ sizes of the map under PointCloud2::operator+= (only the sizes decide HasIntensity)"""

    def __init__(self):
        self.points = 0
        self.intensity = 0

    def has_intensity(self):                                      # PointCloud2.hpp:108-110
        return self.intensity != 0 and self.intensity == self.points

    def add(self, n_points, with_intensity):
        """+= a down-sampled frame of n_points points, with intensity iff the frame's raw cloud had it"""
        if n_points == 0:                                         # cloud.IsEmpty(): return early
            return self
        if (self.points == 0 or self.has_intensity()) and with_intensity:
            self.intensity = self.points + n_points                 # intensity_.resize(new_vert_num)
        else:
            self.intensity = 0                                    # intensity_.clear()
        self.points += n_points
        return self

    def reset(self):
        self.points = self.intensity = 0
        return self
