"""CPU restatement (test infrastructure, not product) of the two steps of the segmentation nodelet that the VLP-16 / raw-scan
path adds to the existing oracle (oracle/pyoracle.py, used unchanged):

  estimateRingsAndTimes2, VLP_16 lambda   ref: src/models/segmentation/segmentation.cpp:386-429
  RemoveClosedNonFinitePoints             ref: :472-499 (called at :48 with near_dis, remove_nan = remove_infinite = true)

Both are transcribed statement by statement in Python: float arithmetic is IEEE double without contraction, and
math.atan2 / math.sqrt are the C library's, so the values are the ones a libm build of the reference computes.
Quirks kept literally:
  * the channel is beamId + correctTime, a real number: beamId = (int)(pitch + |initAngle| + 0.1) / verticalRes is an int
    divided by a double; correctTime is NOT clamped before the half pass (it can exceed 1);
  * the half pass starts at the first point with prevOri < 0 < ori, prevOri = 0.0 before point 0; prevOri then takes the
    MODIFIED ori = pi - ori >= 0, so it fires at most once; there is no -atan2 as in LOAM;
  * a point survives the removal iff no coordinate is NaN / Inf and pt.norm() >= dis_th * dis_th -- a norm against a
    SQUARED threshold (near_dis 3.0 removes every point closer than 9 m); norm = sqrt((x x + y y) + z z).
groundRemove's index lists, regions, threshold and planes do not depend on the channel: they are pyoracle.ground_extract's
(its HDL-64E beam loop only feeds the `beam` output).  With sensorModel 16, verticalRes 2.0, initAngle -15.0 the oracle's
initSections yields one bound and its getSection reads a missing bound as the last section (DESIGN.md §4d).
"""
import math

import numpy as np


def vlp16_channel(pts, init_angle=-15.0, vertical_res=2.0, stats=None):
    """The VLP_16 lambda line by line.  stats (dict, optional) receives half_pass (index of the first half-pass point or
    None) and clamped (how many correctTimes were clamped to 0.99999)."""
    pts = np.asarray(pts, dtype=np.float64).reshape(-1, 3).tolist()
    n = len(pts)
    if n == 0:
        return np.zeros(0)
    start = math.atan2(pts[0][1], pts[0][0])                         # :391-392
    end = math.atan2(pts[n - 1][1], pts[n - 1][0])
    if end - start > 3 * math.pi:                                    # :394-397
        end -= 2 * math.pi
    elif end - start < math.pi:
        end += 2 * math.pi
    scan_ori = end - start                                           # :399
    ang_bot = math.fabs(init_angle) + 0.1                            # :401
    prev, half, half_pass, first, clamped, out = 0.0, 0.0, False, None, 0, []
    for i, (x, y, z) in enumerate(pts):
        pitch = math.atan2(z, math.sqrt(x * x + y * y)) * 180.0 / math.pi     # :407
        beam_id = int(pitch + ang_bot) / vertical_res                # :408 (static_cast<int> truncates toward zero)
        ori = math.atan2(y, x)                                       # :410
        t = math.fabs(ori - start) / scan_ori
        if prev < 0.0 and ori > 0.0:                                 # :413-416
            half_pass = True
            half = math.fabs(prev - start)
            first = i
        if half_pass:                                                # :418-423
            ori = math.pi - ori
            t = (ori + half) / scan_ori
            if t > 1.0:
                t = 0.99999
                clamped += 1
        out.append(beam_id + t)                                      # :425-426
        prev = ori                                                   # :428
    if stats is not None:
        stats.update(half_pass=first, clamped=clamped)
    return np.array(out)


def remove_closed_nonfinite(pts, dis_th):
    """RemoveClosedNonFinitePoints(cloud, dis_th, true, true) line by line: indices of the kept points, in input order."""
    keep = []
    for i, (x, y, z) in enumerate(np.asarray(pts, dtype=np.float64).reshape(-1, 3).tolist()):
        is_nan = math.isnan(x) or math.isnan(y) or math.isnan(z)
        is_inf = math.isinf(x) or math.isinf(y) or math.isinf(z)
        if not is_nan and not is_inf and math.sqrt((x * x + y * y) + z * z) >= dis_th * dis_th:
            keep.append(i)
    return np.array(keep, dtype=np.uintp)


def ground_remove(oracle, pts, **overrides):
    """groundRemove (ref: :738-770) with the channel the reference leaves in the intensity channel: dict(ground, object,
    intensity, region, height_threshold, planes); None for a sensor_model other than 64 / 16 (the `default:` branch)."""
    cfg = oracle.ground_config(**overrides)
    if cfg.sensor_model not in (64, 16):
        return None
    ge = oracle.ground_extract(pts, **overrides)
    if cfg.sensor_model == 16:
        ge["intensity"] = vlp16_channel(pts, cfg.init_angle, cfg.vertical_res)
    else:
        ge["intensity"] = ge["beam"].astype(np.float64)              # :376
    del ge["beam"]
    return ge


def raw_chain(oracle, raw, near_dis=3.0, ring_min_num=131, channel=None, ground=None, dcvc=None):
    """spinOnce :48-66 -- RemoveClosedNonFinitePoints -> groundRemove -> DCVC -> extractEdgePoint -- with index lists into
    the raw scan.  ground: groundRemove configuration overrides (default: the VLP-16 settings); channel: per raw point,
    replaces the restated channel in the edge step."""
    g = dict(sensor_model=16, vertical_res=2.0, init_angle=-15.0) if ground is None else ground
    keep = remove_closed_nonfinite(raw, near_dis)
    scan = np.ascontiguousarray(np.asarray(raw)[keep])
    ge = ground_remove(oracle, scan, **g)
    ch = ge["intensity"] if channel is None else np.asarray(channel)[keep]
    obj = np.ascontiguousarray(scan[ge["object"]])
    seg = oracle.dcvc(obj, **(dcvc or {}))
    sp = ge["object"][seg["segmented"]]
    ee = oracle.extract_edge(np.ascontiguousarray(scan[sp]), ch[sp], sensor_model=g.get("sensor_model", 64), ring_min_num=ring_min_num)
    return dict(keep=keep, ground=keep[ge["ground"]], edge=keep[sp[ee["edge"]]], general=keep[sp[ee["non_edge"]]], sizes=seg["sizes"],
                boxes=seg["boxes"], intensity=ge["intensity"])
