"""Every entry point of the device's voxel down-sample against the exact restatement of tests/voxel_edges_oracle.py, at voxel
faces, far from the origin, in crowded voxels, at the voxel counts where the sorted emission changes method, at the key's
range limit and at the fixed-point sums' headroom.

CPU: the restatement's FP64 membership equals the one with every rounding spelled out in Fractions; the CPU oracle's
membership equals the restatement's on every scene (it keys with 64-bit integers, so the key-range scene too) and its
averages stay within its running-sum bound of the exact mean; the scenes cover what they claim.
GPU: membership exact and averages within the derived bound (voxel_down_sample, process_cloud in ascending key order,
submap_init / submap_update with the crop box, the global map with its intensity, loop keyframes, the localize query),
clouds whose extent reaches 2^21 voxels or whose rows could overflow the sums refused with VOXEL_RANGE, bit-identical
repeats."""
import numpy as np
import pytest

import voxel_edges_oracle as vo

K21 = 1 << vo.KEY_BITS


def cases(name):
    return vo.scene(name)


def kept(case):
    return case["p"][vo.kept_rows(case["p"], case.get("lo"), case.get("hi"))]


def check_sorted(got, case, where):
    """got: the device's voxels in ascending key order; returns the largest error in units of the bound"""
    ref = vo.reference(case["p"], case["voxel"], case.get("lo"), case.get("hi"))
    got = np.asarray(got).reshape(-1, 3)
    assert got.shape[0] == ref["keys"].shape[0], (where, got.shape[0], ref["keys"].shape[0])
    err = vo.errors(got, ref["means"])
    bound = vo.device_bound(case["voxel"], ref["maxabs"])
    worst = int(np.argmax(err / bound)) if len(err) else 0
    assert (err <= bound).all(), (where, worst, ref["keys"][worst], err[worst], bound[worst])
    return float((err / bound).max()) if len(err) else 0.0


def check_unordered(got, case, where):
    """got: the device's voxels in any order, matched one to one to the restatement's voxels by their exact means (voxels
    on either side of a face can have means closer than the bound: each output takes the nearest mean still free)"""
    from scipy.spatial import cKDTree
    ref = vo.reference(case["p"], case["voxel"], case.get("lo"), case.get("hi"))
    got = np.asarray(got).reshape(-1, 3)
    assert got.shape[0] == ref["keys"].shape[0], (where, got.shape[0], ref["keys"].shape[0])
    approx = np.array([[float(m) for m in row] for row in ref["means"]]).reshape(-1, 3)
    k = min(8, got.shape[0])
    d, j = cKDTree(approx).query(got, k=k)
    d, j = d.reshape(got.shape[0], k), j.reshape(got.shape[0], k)
    slot = np.full(got.shape[0], -1)
    free = np.ones(got.shape[0], dtype=bool)
    for i in np.argsort(d[:, 0], kind="stable"):
        c = [jj for jj in j[i] if free[jj]]
        assert c, (where, i)
        slot[i] = c[0]
        free[c[0]] = False
    order = np.argsort(slot)
    return check_sorted(got[order], case, where)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["faces_dyadic", "faces_rounded", "far", "key_range", "nonfinite", "crop"])
def test_restatement_membership_is_the_fraction_membership(name):
    for case in cases(name):
        keep, idx, mb = vo.membership(case["p"], case["voxel"], case.get("lo"), case.get("hi"))
        q = case["p"][keep]
        for d in range(3):
            vals, inv = np.unique(q[:, d], return_inverse=True)
            fi, _ = vo.fraction_indices(vals.tolist(), float(vals[0]), case["voxel"])
            assert np.array_equal(fi[inv.reshape(-1)], idx[:, d]), (name, d)
            assert mb[d] == float(vals[0]) - case["voxel"] * 0.5


def test_restatement_means_are_exact():
    from fractions import Fraction
    p = np.array([[0.1, 0.2, 0.3], [0.1 + 2 ** -50, 0.2, 0.3], [0.15, 0.2, 0.3]])
    ref = vo.reference(p, 1.0)
    assert len(ref["means"]) == 1
    assert ref["means"][0][0] == (Fraction(0.1) * 2 + Fraction(2 ** -50) + Fraction(0.15)) / 3
    # a truncating sum would be off by almost 2^-40 per row in the crowded scene: the bound is below that
    case = cases("crowded")[2]
    assert vo.device_bound(case["voxel"], np.abs(case["p"]).max()) < 0.6 * 2 ** -40


MIN_COVERAGE = {
    "faces_dyadic": dict(on_face=5000, near_face=15000, rounding_decides=100),
    "faces_rounded": dict(near_face=15000, rounding_decides=1000),
    "far": dict(near_face=10000),
    "crowded": dict(max_count=100000),
    "counts": dict(voxels=148225),
    "key_range": dict(),
    "headroom": dict(max_count=(1 << 17) + 1),
    "nonfinite": dict(dropped=1200),
    "crop": dict(dropped=510),
}


@pytest.mark.parametrize("name", sorted(vo.SCENES))
def test_scene_coverage(name):
    covs = [vo.coverage(c) for c in cases(name)]
    for k, want in MIN_COVERAGE[name].items():
        have = max(c[k] for c in covs) if k.startswith("max") else sum(c[k] for c in covs)
        assert have >= want, (name, k, have, want)
    if name == "counts":
        assert sorted(c["voxels"] for c in covs) == [1, 255, 256, 257, 16383, 16384, 16385, 32767, 32768, 32769]
    if name == "key_range":
        tops = sorted(c["max_index"] for c in covs)
        assert tops.count(K21 - 1) == 3 and tops.count(K21) == 4
    if name == "headroom":
        loads = sorted(c["max_load_m"] for c in covs)
        assert loads[0] < vo.HEADROOM_M <= loads[1]
    if name == "crop":
        for c in cases(name):                    # rows exactly on every face of the box, and one ulp outside each
            p, lo, hi = c["p"], c["lo"], c["hi"]
            for d in range(3):
                assert (p[:, d] == lo[d]).sum() >= 20 and (p[:, d] == hi[d]).sum() >= 20
                assert (p[:, d] == np.nextafter(lo[d], -np.inf)).sum() >= 20
            assert (p < lo).all(1).sum() >= 50 and vo.membership(p, c["voxel"])[2][0] < vo.membership(p, c["voxel"], lo, hi)[2][0]


@pytest.mark.parametrize("name", sorted(vo.SCENES))
def test_oracle_membership_and_running_sum_bound(oracle, name):
    """the CPU oracle (finite rows: it is not defined on others) against the restatement, voxel for voxel in key order"""
    for case in cases(name):
        if name == "headroom" and case["p"].shape[0] > (1 << 17):
            continue                                           # same rows, one more: nothing new for the oracle
        q = kept(case)
        got = oracle.voxel_down_sample(q, case["voxel"])
        ref = vo.reference(q, case["voxel"])
        assert got.shape[0] == ref["keys"].shape[0], name
        err = vo.errors(got, ref["means"])
        assert (err <= vo.oracle_bound(ref["counts"], ref["maxabs"])).all(), name


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _reg():
    import tloam_b200
    return tloam_b200.LocalRegistration()


def _status(fn, *a, **k):
    import tloam_b200
    try:
        fn(*a, **k)
    except tloam_b200.RegistrationError as e:
        return e.status
    return 0


GPU_SCENES = ["faces_dyadic", "faces_rounded", "far", "crowded", "counts", "nonfinite", "crop"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_SCENES)
def test_gpu_voxel_down_sample_is_exact_membership_within_the_bound(name):
    r = _reg()
    worst = 0.0
    for case in cases(name):
        p = case["p"] if "lo" not in case else kept(case)       # no crop box on this entry point
        c = dict(case, p=p)
        c.pop("lo", None), c.pop("hi", None)
        worst = max(worst, check_unordered(r.voxel_down_sample(p, case["voxel"]), c, name))
    print(f"\nvoxel_down_sample {name}: largest error {worst:.3f} of the bound")
    r.close()


@pytest.mark.gpu
def test_gpu_voxel_down_sample_key_range_and_headroom():
    from tloam_b200 import _lib
    r = _reg()
    for case in cases("key_range"):
        if case["top"] < K21:
            check_unordered(r.voxel_down_sample(case["p"], case["voxel"]), case, ("key", case["axis"]))
        else:                                                   # would alias index 2^21 onto 0: refused
            assert _status(r.voxel_down_sample, case["p"], case["voxel"]) == _lib.ERR_VOXEL_RANGE, case["axis"]
    for case in cases("headroom"):
        if case["load"] < vo.HEADROOM_M:
            worst = check_unordered(r.voxel_down_sample(case["p"], case["voxel"]), case, "headroom")
            print(f"\nvoxel_down_sample headroom: largest error {worst:.3f} of the bound")
        else:
            assert _status(r.voxel_down_sample, case["p"], case["voxel"]) == _lib.ERR_VOXEL_RANGE, case["load"]
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["counts", "faces_dyadic", "faces_rounded", "far", "crowded", "nonfinite"])
def test_gpu_process_cloud_emits_ascending_keys_row_for_row(name):
    r = _reg()
    worst = 0.0
    for case in cases(name):
        p, v = case["p"], case["voxel"]
        n = r.process_cloud(p, p[::-1].copy(), np.zeros((0, 3)), ground_down_sample=v, edge_down_sample=v)
        worst = max(worst, check_sorted(r.source_cloud(3), case, (name, "ground")))
        worst = max(worst, check_sorted(r.source_cloud(0), dict(case, p=p[::-1].copy()), (name, "edge")))
        assert n[1] == n[2] == 0
    print(f"\nprocess_cloud {name}: largest error {worst:.3f} of the bound")
    r.close()


@pytest.mark.gpu
def test_gpu_process_cloud_and_submap_init_key_range():
    from tloam_b200 import _lib
    r = _reg()
    small = np.random.default_rng(1).uniform(0, 1, (50, 3))
    for case in cases("key_range"):
        p, v = case["p"], case["voxel"]
        run = lambda: r.process_cloud(p, small, np.zeros((0, 3)), ground_down_sample=v, edge_down_sample=0.3)   # noqa: E731
        init = lambda: r.submap_init(small, p, small, small, ground_down_sample=v)                             # noqa: E731
        if case["top"] < K21:
            run()
            check_sorted(r.source_cloud(3), case, ("process_cloud", case["axis"]))
            init()
            check_unordered(r.submap_cloud(3), case, ("submap_init", case["axis"]))
        else:
            assert _status(run) == _lib.ERR_VOXEL_RANGE and _status(init) == _lib.ERR_VOXEL_RANGE, case["axis"]
    head = cases("headroom")
    assert _status(r.process_cloud, head[1]["p"], small, np.zeros((0, 3)), ground_down_sample=64.0) == _lib.ERR_VOXEL_RANGE
    assert _status(r.submap_init, small, head[2]["p"], small, small, ground_down_sample=64.0) == _lib.ERR_VOXEL_RANGE
    # a crop box of 2 L / voxel + 1 >= 2^21 voxels could key past the range in a later update: refused up front
    L = (K21 - 1) * 0.3 / 2                                     # 2 L / 0.3 + 1 = 2^21 up to rounding
    assert _status(r.submap_init, small, small, small, small, edge_crop_box_length=L * (1 + 1e-12)) == _lib.ERR_INVALID_ARG
    assert _status(r.submap_init, small, small, small, small, ground_crop_box_length=L * 1.5 * (1 + 1e-12)) == _lib.ERR_INVALID_ARG   # voxel 0.45
    r.submap_init(small, small, small, small, edge_crop_box_length=L * (1 - 1e-9))
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["crop", "faces_dyadic", "faces_rounded"])
def test_gpu_submap_init_and_update_match_the_restatement_and_the_oracle(oracle, name):
    """the scene's rows become the source's edge and ground features, appended with a translation-only pose to an empty
    map and cropped to pose.t +- L: the map clouds against the restatement (box included) and the oracle's Submap"""
    r = _reg()
    for case in cases(name):
        v = case["voxel"]
        c = case.get("centre", np.zeros(3))
        L = case.get("L", 1e3)
        cfg = dict(edge_down_sample_submap=v, ground_down_sample_submap=v, edge_crop_box_length=L, ground_crop_box_length=L,
                   ground_down_sample=v)
        pose = np.eye(4)
        pose[:3, 3] = c
        sensor = case["p"] - c
        world = sensor + c                                      # the transform both sides compute (identity rotation)
        ex = dict(case, p=world, lo=c - L, hi=c + L)
        empty = np.zeros((0, 3))
        r.submap_init(empty, sensor, empty, empty, **cfg)
        check_unordered(r.submap_cloud(3), dict(case, p=sensor, lo=None, hi=None), (name, "init"))
        r.submap_init(empty, empty, empty, empty, **cfg)
        tiny = np.random.default_rng(2).uniform(0, 1, (12, 3))
        r.set_input_source([sensor, tiny, tiny, sensor])
        r.submap_update(pose, tiny)
        sm = oracle.Submap(**cfg)
        sm.init(empty, empty, empty, empty)
        sm.update(pose, sensor, sensor, tiny, tiny)
        for cloud in (0, 3):
            got = r.submap_cloud(cloud)
            check_unordered(got, ex, (name, "update", cloud))
            want = sm.cloud(cloud)
            assert want.shape == got.shape, (name, cloud)
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["key_range", "faces_dyadic", "faces_rounded"])
def test_gpu_global_map_append_blocks_and_intensity(name):
    """each appended frame (pose I) is its voxels in ascending key order within the bound; the intensity of a voxel is the
    average over exactly its xyz rows; the key range's first unkeyable index is refused with VOXEL_RANGE"""
    from fractions import Fraction
    import tloam_b200
    from tloam_b200 import _lib
    for case in cases(name):
        r = _reg()
        p, v = case["p"], case["voxel"]
        r.enable_global_map(voxel=v)
        inten = np.random.default_rng(7).integers(0, 256, p.shape[0]).astype(np.float64)
        r.global_map_append(p, np.eye(4), intensity=inten)
        if case.get("top", 0) >= K21:
            with pytest.raises(tloam_b200.RegistrationError) as e:
                r.global_map_size()
            assert e.value.status == _lib.ERR_VOXEL_RANGE
            assert r.global_map_size() == (0, 0)
            r.close()
            continue
        got = r.global_map()
        check_sorted(got, case, (name, "global map"))
        assert r.global_map_has_intensity()                     # k_gmi_rank found every row's voxel (its bug flag is clear)
        ref = vo.reference(p, v)
        gi = r.global_map_intensity()
        for k in range(len(gi)):
            rows = inten[ref["inv"] == k]
            want = Fraction(int(rows.sum())) / len(rows)
            assert abs(Fraction(float(gi[k])) - want) <= Fraction(abs(float(want))) * Fraction(2 ** -52), (name, k)
        r.close()


@pytest.mark.gpu
def test_gpu_loop_keyframe_and_localize_query_at_the_key_range():
    import tloam_b200
    from tloam_b200 import _lib
    for case in cases("key_range"):
        p, v = case["p"], case["voxel"]
        r = _reg()
        r.loop_enable(exclude_recent=0)
        r.loop_verify_enable(voxel=v)
        r.loop_add(p)
        kf = r.loop_keyframe(0)
        r.localize_enable(voxel=v)
        r.localize_set_map(np.random.default_rng(3).uniform(-20, 20, (4000, 3)))
        if case["top"] < K21:
            check_sorted(kf, case, ("keyframe", case["axis"]))
            r.localize(p, np.eye(4))
            check_sorted(r.localize_query(), case, ("localize", case["axis"]))
        else:
            assert len(kf) == 0, case["axis"]                  # refused: an empty slot
            with pytest.raises(tloam_b200.RegistrationError) as e:
                r.localize(p, np.eye(4))
            assert e.value.status == _lib.ERR_VOXEL_RANGE
        r.close()


@pytest.mark.gpu
def test_gpu_repeats_are_bit_identical():
    r = _reg()
    for name in ("crowded", "faces_rounded"):
        for case in cases(name)[:3]:
            a = r.voxel_down_sample(case["p"], case["voxel"])
            b = r.voxel_down_sample(case["p"], case["voxel"])
            key = lambda x: x[np.lexsort((x[:, 2], x[:, 1], x[:, 0]))]     # noqa: E731  (the unsorted emission's order varies)
            assert np.array_equal(key(a), key(b))
            r.process_cloud(case["p"], case["p"], np.zeros((0, 3)), ground_down_sample=case["voxel"], edge_down_sample=case["voxel"])
            g1 = r.source_cloud(3)
            r.process_cloud(case["p"], case["p"], np.zeros((0, 3)), ground_down_sample=case["voxel"], edge_down_sample=case["voxel"])
            assert np.array_equal(g1, r.source_cloud(3))
    r.close()
