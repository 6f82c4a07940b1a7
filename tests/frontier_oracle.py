"""numpy restatement of the frontier search (include/tloam_b200.h "Frontiers"; k_fr_* in tloam_b200/csrc/frontier.cu and
the host's cost and order in tloam_b200.cu), bit for bit.

Components are found by a vectorised union-find (hook each root under the least root it shares an edge with, then
compress) over the 8-neighbour edges of the frontier cells; every root is then its component's least linear index, as on
the device.  The CPU tests pin it to scipy.ndimage.label and to a literal explore_lite-style breadth-first search.  Every
FP64 expression is a numpy elementwise operation, each rounded on its own, in the header's order.  Grids are (height,
width) arrays, row j along y and column i along x; cells are (i, j)."""
from collections import deque

import numpy as np

INF = np.uint64(0xFFFFFFFFFFFFFFFF)
NONE = np.uint32(0xFFFFFFFF)
DEFAULT = dict(free_max=252, min_frontier_size=0.5, potential_scale=3.0, gain_scale=1.0)
BACK = ((-1, 0), (-1, -1), (0, -1), (1, -1))               # W, NW, N, NE: one direction of every 8-edge
FIELDS = ("id", "size", "sum_i", "sum_j", "min_i", "min_j", "max_i", "max_j", "centroid_x", "centroid_y", "approach_i",
          "approach_j", "approach_x", "approach_y", "approach_potential", "status", "distance", "cost")


def config(**overrides):
    c = dict(DEFAULT)
    c.update(overrides)
    return c


def config_valid(free_max, min_frontier_size, potential_scale, gain_scale):
    ok = [np.isfinite(v) and v >= 0.0 for v in (min_frontier_size, potential_scale, gain_scale)]
    return 0 <= free_max <= 252 and all(ok)


def frontier_cells(costs, free_max=252):
    """code 255 with a 4-neighbour inside the grid of code <= free_max"""
    c = np.asarray(costs)
    free = c <= free_max
    nb = np.zeros(c.shape, dtype=bool)
    nb[:, 1:] |= free[:, :-1]
    nb[:, :-1] |= free[:, 1:]
    nb[1:, :] |= free[:-1, :]
    nb[:-1, :] |= free[1:, :]
    return (c == 255) & nb


def components(F):
    """labels (H, W) uint32: the id of each frontier cell's 8-connected component, ids ascending with the component's
    least linear index; NONE elsewhere.  Returns (labels, count)."""
    F = np.asarray(F, dtype=bool)
    H, W = F.shape
    idx = np.flatnonzero(F.ravel())
    labels = np.full(H * W, NONE, dtype=np.uint32)
    if len(idx) == 0:
        return labels.reshape(H, W), 0
    pos = np.full(H * W, -1, dtype=np.int64)
    pos[idx] = np.arange(len(idx))
    jj, ii = np.divmod(idx, W)
    a, b = [], []
    for di, dj in BACK:
        ui, uj = ii + di, jj + dj
        ok = (ui >= 0) & (ui < W) & (uj >= 0)
        u = uj[ok] * W + ui[ok]
        nb = pos[u]
        a.append(np.flatnonzero(ok)[nb >= 0])
        b.append(nb[nb >= 0])
    a, b = np.concatenate(a), np.concatenate(b)
    parent = np.arange(len(idx))
    while True:
        while True:                                          # compress: every entry its root
            q = parent[parent]
            if np.array_equal(q, parent):
                break
            parent = q
        ra, rb = parent[a], parent[b]
        d = ra != rb
        if not d.any():
            break
        np.minimum.at(parent, np.maximum(ra[d], rb[d]), np.minimum(ra[d], rb[d]))
    roots, ids = np.unique(parent, return_inverse=True)      # positions ascend with the cells, so roots ascend too
    labels[idx] = ids.astype(np.uint32)
    return labels.reshape(H, W), len(roots)


def bfs_components(F):
    """a literal explore_lite-style search: scan the cells in index order and grow an unlabelled frontier cell's
    component by breadth-first search over its 8 neighbours"""
    F = np.asarray(F, dtype=bool)
    H, W = F.shape
    labels = np.full((H, W), NONE, dtype=np.uint32)
    k = 0
    for j in range(H):
        for i in range(W):
            if not F[j, i] or labels[j, i] != NONE:
                continue
            labels[j, i] = k
            q = deque([(i, j)])
            while q:
                ci, cj = q.popleft()
                for dj in (-1, 0, 1):
                    for di in (-1, 0, 1):
                        ni, nj = ci + di, cj + dj
                        if 0 <= ni < W and 0 <= nj < H and F[nj, ni] and labels[nj, ni] == NONE:
                            labels[nj, ni] = k
                            q.append((ni, nj))
            k += 1
    return labels, k


def search(costs, P, origin, resolution, neutral_cost=50, free_max=252, min_frontier_size=0.5, potential_scale=3.0,
           gain_scale=1.0):
    """the whole search: dict(labels, components, cells (frontier cells), frontiers (a dict of arrays over FIELDS, the kept
    ones in rank order), offsets (kept + 1) and ij (the kept frontiers' cells in rank order, each ascending))"""
    c = np.asarray(costs)
    P = np.asarray(P, dtype=np.uint64)
    H, W = c.shape
    F = frontier_cells(c, free_max)
    labels, nf = components(F)
    lab = labels.ravel()
    idx = np.flatnonzero(lab != NONE)                       # ascending
    ids = lab[idx].astype(np.int64)
    order = np.argsort(ids, kind="stable")                  # by id, each frontier's cells ascending
    cells = idx[order]
    n = np.bincount(ids, minlength=nf).astype(np.int64)
    start = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    cj, ci = np.divmod(cells, W)
    fr = {}
    if nf:
        heads = start[:-1]
        fr["sum_i"] = np.add.reduceat(ci, heads).astype(np.uint64)
        fr["sum_j"] = np.add.reduceat(cj, heads).astype(np.uint64)
        fr["min_i"], fr["max_i"] = np.minimum.reduceat(ci, heads), np.maximum.reduceat(ci, heads)
        fr["min_j"], fr["max_j"] = np.minimum.reduceat(cj, heads), np.maximum.reduceat(cj, heads)
        # the approach cell: the least (P, index) over the free 4-neighbours of the frontier's cells
        cid, cp, cu = [], [], []
        fid = np.repeat(np.arange(nf), n)
        for di, dj in ((1, 0), (-1, 0), (0, 1), (0, -1)):
            ui, uj = ci + di, cj + dj
            ok = (ui >= 0) & (ui < W) & (uj >= 0) & (uj < H)
            u = uj[ok] * W + ui[ok]
            free = c.ravel()[u] <= free_max
            cid.append(fid[ok][free])
            cu.append(u[free])
            cp.append(P.ravel()[u[free]])
        cid, cp, cu = np.concatenate(cid), np.concatenate(cp), np.concatenate(cu)
        o = np.lexsort((cu, cp, cid))
        first = np.unique(cid[o], return_index=True)[1]
        assert len(first) == nf
        au, ap = cu[o][first], cp[o][first]
    else:
        for k in ("sum_i", "sum_j", "min_i", "max_i", "min_j", "max_j"):
            fr[k] = np.zeros(0, dtype=np.int64)
        au, ap = np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.uint64)
    fr["id"] = np.arange(nf)
    fr["size"] = n
    nd = n.astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        fr["centroid_x"] = origin[0] + (fr["sum_i"].astype(np.float64) / nd + 0.5) * resolution
        fr["centroid_y"] = origin[1] + (fr["sum_j"].astype(np.float64) / nd + 0.5) * resolution
    fr["approach_j"], fr["approach_i"] = np.divmod(au.astype(np.int64), W)
    fr["approach_x"] = origin[0] + (fr["approach_i"].astype(np.float64) + 0.5) * resolution
    fr["approach_y"] = origin[1] + (fr["approach_j"].astype(np.float64) + 0.5) * resolution
    fr["approach_potential"] = ap
    reach = ap != INF
    fr["status"] = np.where(reach, 0, 1)
    size_m = nd * resolution
    dist = (ap.astype(np.float64) / (70.0 * float(neutral_cost))) * resolution
    fr["distance"] = np.where(reach, dist, np.inf)
    fr["cost"] = np.where(reach, potential_scale * dist - gain_scale * size_m, np.inf)
    kept = size_m >= min_frontier_size
    r = np.flatnonzero(kept & reach)
    r = r[np.lexsort((r, fr["cost"][r]))]
    rank = np.concatenate([r, np.flatnonzero(kept & ~reach)]).astype(np.int64)
    frontiers = {k: np.asarray(fr[k])[rank] for k in FIELDS}
    offsets = np.concatenate([[0], np.cumsum(n[rank])]).astype(np.int64)
    sel = np.repeat(start[rank] - offsets[:-1], n[rank]) + np.arange(offsets[-1])
    sj, si = np.divmod(cells[sel], W)
    ij = np.column_stack([si, sj]).astype(np.int32)
    return dict(labels=labels, components=nf, cells=len(idx), frontiers=frontiers, offsets=offsets, ij=ij,
                reachable=int((frontiers["status"] == 0).sum()))


def centres(cells, origin, resolution):
    """xy of cells (m, 2): origin + (i + 0.5) resolution, each operation rounded on its own"""
    c = np.asarray(cells, dtype=np.float64).reshape(-1, 2)
    return np.column_stack([origin[0] + (c[:, 0] + 0.5) * resolution, origin[1] + (c[:, 1] + 0.5) * resolution])
