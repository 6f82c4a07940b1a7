"""CPU restatement of relocalization in a prior map (include/tloam_b200.h, "Relocalization in a prior map"; k_rl_* in
libtloam_b200_reloc.so), built on scan_context_oracle and localize_oracle:

    search:   every place's distance at every shift (scan_context_oracle.distances); per place the first minimum over
              ascending shifts, the minimum by (distance, shift)
    top-K:    the places with distance < max_distance by (distance, place), the first top_k
    guess:    G = P_j . Rz(yaw_s), cos / sin of direction (-s) mod n_sector from the sector boundary table, the products
              in the prediction's order, t_G = t_P
    runs:     localize_oracle.run from each G
    select:   the accepted run minimal by (fitness, rank), else the minimal run; ambiguous against every other accepted run"""
import math

import numpy as np

import localize_oracle as lo
import loop_verify_submap_oracle as lso
import scan_context_oracle as sco


def config(**overrides):
    """tloam_b200_relocalize_default_config, with overrides"""
    d = sco.DEFAULT
    c = dict(lidar_height=d["lidar_height"], n_ring=d["n_ring"], n_sector=d["n_sector"], max_radius=d["max_radius"], top_k=8,
             max_distance=0.4, distinct_translation=2.0, distinct_rotation=math.radians(10.0), ambiguity_ratio=1.5)
    c.update(overrides)
    return c


def split(slot, R, S):
    """a descriptor slot as scan_context_oracle's (bins, ring key, norms)"""
    slot = np.asarray(slot, dtype=np.float64)
    return slot[:R * S].reshape(R, S), slot[R * S:R * S + R], slot[R * S + R:]


def pack(desc):
    """scan_context_oracle's (bins, ring key, norms) as one slot"""
    return np.concatenate([desc[0].ravel(), desc[1], desc[2]])


def place_search(query, places, chunk=256):
    """per place its best (distance, shift): the first minimum over ascending shifts"""
    S = query[0].shape[1]
    if not places:
        return np.zeros(0), np.zeros(0, dtype=np.int64)
    table = np.concatenate([sco.distances(query, places[a:a + chunk]) for a in range(0, len(places), chunk)])
    shift = np.argmin(table, axis=1)
    return table[np.arange(len(places)), shift], shift.astype(np.int64)


def top_k(dist, k, max_distance):
    """the first k places with distance < max_distance by (distance, place)"""
    idx = np.flatnonzero(dist < max_distance)
    order = idx[np.lexsort((idx, dist[idx]))]
    return order[:k]


def guess(P, shift, n_sector):
    """G = P . Rz(yaw_s) in the header's order"""
    m = (-int(shift)) % n_sector
    c, s = (1.0, 0.0) if m == 0 else tuple(sco.boundaries(n_sector)[m - 1])
    Rz = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
    P = np.asarray(P, dtype=np.float64)
    G = np.eye(4)
    for r in range(3):
        for j in range(3):
            G[r, j] = lso._dot3(P[r, 0], Rz[0, j], P[r, 1], Rz[1, j], P[r, 2], Rz[2, j])
        G[r, 3] = P[r, 3]
    return G


def select(runs, cfg):
    """(winner, ambiguous, accepted) over the runs in rank order"""
    if not runs:
        return -1, False, False
    acc = [k for k, r in enumerate(runs) if r["accepted"]]
    pool = acc if acc else range(len(runs))
    w = min(pool, key=lambda k: (runs[k]["fitness"], k))
    if not runs[w]["accepted"]:
        return w, False, False
    Tw = runs[w]["T"]
    bound = cfg["ambiguity_ratio"] * runs[w]["fitness"]
    cos_r = math.cos(cfg["distinct_rotation"])
    amb = False
    for k in acc:
        if k == w or not runs[k]["fitness"] <= bound:
            continue
        Tk = runs[k]["T"]
        dt = math.sqrt(lso._d2(Tk[None, :3, 3], Tw[None, :3, 3])[0])
        tr = 0.0
        for i in range(3):
            for j in range(3):
                tr = tr + Tw[i, j] * Tk[i, j]
        c = min(max((tr - 1.0) * 0.5, -1.0), 1.0)
        if dt > cfg["distinct_translation"] or c < cos_r:
            amb = True
    return w, amb, not amb


def relocalize(scan, Q, places, poses, g, nrm, valid, cfg, lcfg, O_now=None):
    """the relocalization of a raw scan (its down-sample Q) against places (descriptor tuples) at poses, over the map's
    index g: dict(query, distance, shift, top, guesses, runs, winner, ambiguous, accepted, T_map_odom)"""
    q = sco.descriptor(scan, cfg)
    dist, shift = place_search(q, places)
    top = top_k(dist, cfg["top_k"], cfg["max_distance"])
    guesses = [guess(poses[j], shift[j], cfg["n_sector"]) for j in top]
    runs = [lo.run(Q, g, nrm, valid, G, lcfg) for G in guesses]
    w, amb, ok = select(runs, cfg)
    O = np.eye(4) if O_now is None else np.asarray(O_now, dtype=np.float64)
    return dict(query=q, distance=dist, shift=shift, top=top, guesses=guesses, runs=runs, winner=w, ambiguous=amb,
                accepted=ok, T_map_odom=lo.map_odom(runs[w]["T"], O) if w >= 0 else None)
