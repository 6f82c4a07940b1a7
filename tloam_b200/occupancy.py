"""Saving an occupancy grid for map_server: the P5 PGM and YAML pair ROS 1's map_saver writes."""
import os

import numpy as np

OCCUPIED_THRESH = 65          # map_saver: a value >= 65 is written black (0)
FREE_THRESH = 25              # and 0 .. 25 white (254); anything else, unknown (-1) included, grey (205)


def save_occupancy_map(stem, grid, origin, resolution):
    """writes stem.pgm and stem.yaml with ROS 1 map_saver's encoding; grid is (height, width) int8 in
    nav_msgs/OccupancyGrid's values with row 0 at the origin's y, and origin the (x, y) of the corner of cell (0, 0).
    Row 0 of the image is the grid's last row (the largest y), as map_server expects."""
    g = np.asarray(grid)
    if g.ndim != 2:
        raise ValueError("save_occupancy_map: grid must be (height, width)")
    v = g.astype(np.int16)
    img = np.full(v.shape, 205, dtype=np.uint8)
    img[(v >= 0) & (v <= FREE_THRESH)] = 254
    img[v >= OCCUPIED_THRESH] = 0
    h, w = img.shape
    with open(stem + ".pgm", "wb") as f:
        f.write(f"P5\n# CREATOR: tloam_b200.save_occupancy_map {resolution:.3f} m/pix\n{w} {h}\n255\n".encode())
        f.write(np.ascontiguousarray(img[::-1]).tobytes())
    with open(stem + ".yaml", "w") as f:
        f.write(f"image: {os.path.basename(stem)}.pgm\nresolution: {resolution:.6f}\n"
                f"origin: [{origin[0]:.6f}, {origin[1]:.6f}, 0.000000]\nnegate: 0\noccupied_thresh: 0.65\n"
                f"free_thresh: 0.196\n\n")
