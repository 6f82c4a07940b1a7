"""Host-side mirror of the reference's registration interface, over the C-ABI CUDA library.

`LocalRegistration` mirrors tloam::LocalRegistration / RegistrationInterface
(ref: include/tloam/models/registration/registration_interface.hpp:40-48,
      include/tloam/models/registration/registration.hpp:142-165): same method names
(snake_case), same argument meaning, status codes instead of aborts.  It is a thin ctypes shell:
all arithmetic happens in libtloam_b200.so on the GPU.  There is no CPU path.
"""
import ctypes as C
import dataclasses
import math

import numpy as np

from . import _lib

CLOUDS = ("edge", "sphere", "planar", "ground")  # ABI order (ref: registration.cpp:233-236)


class RegistrationError(RuntimeError):
    def __init__(self, status, where, detail=""):
        self.status = status
        msg = _lib.load().tloam_b200_status_string(status).decode()
        super().__init__(f"{where}: {msg} (status {status}) {detail}")


def default_config(**overrides):
    """The "TLS:" block defaults (ref: config/mapping/lidar_odometry.yaml:23-39)."""
    cfg = _lib.TlsConfig()
    _lib.load().tloam_b200_default_config(C.byref(cfg))
    for k, v in overrides.items():
        if k == "reinit_dir":
            for i in range(3):
                cfg.reinit_dir[i] = float(v[i])
        else:
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
    return cfg


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


_F32 = np.dtype("<f4")


def packed_scan(arr):
    """The tloam_packed_scan descriptor of a raw scan in the sensor's own float32 layout, for the *_packed calls (one upload,
    unpacked on the device).  arr is one of
      - a numpy structured array (a PointCloud2's records: np.frombuffer(msg.data, dtype)) with little-endian float32 fields
        x, y, z and optionally intensity, any itemsize and offsets;
      - a float32 (n, 4) array (a KITTI .bin scan: np.fromfile(path, "<f4").reshape(-1, 4)), intensity in column 3;
      - a float32 (n, 3) array, no intensity.
    It must be C-contiguous; anything else raises ValueError.  The descriptor keeps a reference to arr."""
    if not isinstance(arr, np.ndarray) or not arr.flags.c_contiguous:
        raise ValueError("packed_scan: a C-contiguous numpy array is required")
    fields = arr.dtype.fields
    if fields is not None:
        off = {}
        for name in ("x", "y", "z", "intensity"):
            if name not in fields:
                if name == "intensity":
                    continue
                raise ValueError(f"packed_scan: the records have no field {name!r}")
            dt, o = fields[name][:2]
            if dt != _F32:
                raise ValueError(f"packed_scan: field {name!r} is {dt.str}, not little-endian float32")
            off[name] = o
        d = _lib.PackedScan(arr.ctypes.data, arr.size, arr.dtype.itemsize, off["x"], off["y"], off["z"], off.get("intensity", -1))
    elif arr.dtype == _F32 and arr.ndim == 2 and arr.shape[1] in (3, 4):
        d = _lib.PackedScan(arr.ctypes.data, arr.shape[0], 4 * arr.shape[1], 0, 4, 8, 12 if arr.shape[1] == 4 else -1)
    else:
        raise ValueError(f"packed_scan: {arr.dtype.str} array of shape {arr.shape} is neither structured records nor float32 "
                         "(n, 3) / (n, 4)")
    d._keep = arr
    return d


def _packed(scan):
    return scan if isinstance(scan, _lib.PackedScan) else packed_scan(scan)


# the per-point time fields drivers publish: name -> (PointField datatype, numpy dtype, unit to seconds)
_TIME_FIELDS = (("time", 7, np.dtype("<f4"), 1.0),          # velodyne_pointcloud XYZIRT: float32 s from the sweep's start
                ("t", 6, np.dtype("<u4"), 1e-9),            # Ouster: uint32 ns
                ("timestamp", 8, np.dtype("<f8"), 1.0))     # Hesai: float64 s


def packed_time(arr):
    """The tloam_packed_time descriptor of the per-point time field of a structured array (the records packed_scan
    describes), for the timed packed calls: the first of `time` (little-endian float32, s), `t` (little-endian uint32, ns)
    and `timestamp` (little-endian float64, s) the records have, which must have that type.  Anything else raises
    ValueError."""
    fields = getattr(getattr(arr, "dtype", None), "fields", None)
    if not isinstance(arr, np.ndarray) or fields is None:
        raise ValueError("packed_time: a numpy structured array is required")
    for name, datatype, dt, unit in _TIME_FIELDS:
        if name in fields:
            fdt, off = fields[name][:2]
            if fdt != dt:
                raise ValueError(f"packed_time: field {name!r} is {fdt.str}, not {dt.str}")
            return _lib.PackedTime(off, datatype, unit)
    raise ValueError("packed_time: the records have no field 'time', 't' or 'timestamp'")


@dataclasses.dataclass(frozen=True)
class LoopResult:
    """tloam_loop_result: query = the newest added frame; candidate = its best earlier frame (-1: none eligible), found at
    column shift `shift` with Scan Context distance `distance`; yaw (rad): p_candidate ~ Rz(yaw) . p_query."""
    query: int
    candidate: int
    shift: int
    yaw: float
    distance: float
    is_loop: bool


@dataclasses.dataclass(frozen=True)
class LoopVerifyResult:
    """tloam_loop_verify_result: T (4 x 4) = T_cand_query, p_candidate ~ T . p_query; termination is one of
    LoopVerifyResult.CONVERGED .. EMPTY; accepted = converged and fitness <= max_fitness."""
    query: int
    candidate: int
    T: np.ndarray
    fitness: float
    rmse: float
    inliers: int
    n_query_points: int
    n_candidate_points: int
    iterations: int
    termination: int
    accepted: bool
    CONVERGED, ITERATION_LIMIT, FEW_INLIERS, SINGULAR, EMPTY = range(5)


@dataclasses.dataclass(frozen=True)
class LocalizeResult:
    """tloam_localize_result: T (4 x 4) = map <- sensor, T_map_odom = T . O_now^-1, guess = the G the run started from;
    termination is one of LoopVerifyResult.CONVERGED .. EMPTY; accepted = converged and fitness <= max_fitness."""
    T: np.ndarray
    T_map_odom: np.ndarray
    guess: np.ndarray
    iterations: int
    termination: int
    accepted: bool
    inliers: int
    rmse: float
    fitness: float
    n_query_points: int
    n_map_points: int


@dataclasses.dataclass(frozen=True)
class GlobalRegistrationResult:
    """tloam_global_registration_result: T (4 x 4) = target <- source (from global_register_loop: T_cand_query, a guess
    for loop_verify); termination is one of GlobalRegistrationResult.CONVERGED .. EMPTY; accepted = inliers >= min_inliers
    and fitness >= min_fitness."""
    T: np.ndarray
    n_source_points: int
    n_target_points: int
    n_source_features: int
    n_target_features: int
    n_correspondences: int
    n_valid_hypotheses: int
    best_hypothesis: int
    best_inliers: int
    inliers: int
    inlier_rmse: float
    fitness: float
    refine_iterations: int
    termination: int
    accepted: bool
    CONVERGED, ITERATION_LIMIT, FEW_INLIERS, FEW_CORRESPONDENCES, NO_HYPOTHESIS, EMPTY = range(6)


@dataclasses.dataclass(frozen=True)
class RelocalizeResult:
    """tloam_relocalize_result: result = the winner's LocalizeResult; place / shift / distance its candidate (place -1
    without hypotheses); winner = its rank; accepted = the winner is accepted and no distinct hypothesis fits about as
    well (ambiguous)."""
    result: LocalizeResult
    place: int
    shift: int
    distance: float
    n_hypotheses: int
    winner: int
    ambiguous: bool
    accepted: bool


@dataclasses.dataclass(frozen=True)
class MapUpdateAddResult:
    """tloam_map_update_add_result: used = the last localization was accepted and voted; frame = this add's frame number
    (-1 when not used); the scan rows that voted and the query rows tested for novelty."""
    used: bool
    frame: int
    n_scan_points: int
    n_query_points: int


@dataclasses.dataclass(frozen=True)
class MapUpdateResult:
    """tloam_map_update_result: the counts of a build; n_total = kept prior rows + supported voxels."""
    n_prior: int
    n_prior_removed: int
    n_additions: int
    n_additions_removed: int
    n_voxels: int
    n_voxels_kept: int
    n_total: int


@dataclasses.dataclass(frozen=True)
class DistanceField:
    """a built distance field (include/tloam_b200.h "Distance field and costmap"), each (height, width) in the grid's
    layout: signed = sd (float32, m, negative at obstacle cells, +-inf without a cell of the other class), sq (uint32,
    the squared distance in cells), costs (uint8, costmap_2d's codes), values (int8, Costmap2DPublisher's values); origin
    = (x, y) of the corner of cell (0, 0); obstacles = the obstacle cells."""
    signed: np.ndarray
    sq: np.ndarray
    costs: np.ndarray
    values: np.ndarray
    origin: tuple
    resolution: float
    obstacles: int


@dataclasses.dataclass(frozen=True)
class PlanField:
    """a built plan (include/tloam_b200.h "Path planning"): potential (height, width) uint64, the least cost of a path
    from each cell to the goal (0xFFFFFFFFFFFFFFFF: impassable or cut off), in the grid's layout; origin = (x, y) of the
    corner of cell (0, 0); goal = its cell (i, j); reachable = the cells with a finite potential; rounds and tiles = the
    relaxation rounds that had work and the tiles they relaxed."""
    potential: np.ndarray
    origin: tuple
    resolution: float
    goal: tuple
    reachable: int
    rounds: int
    tiles: int


@dataclasses.dataclass(frozen=True)
class PlanPath:
    """one start's path down the last plan: cells (m, 2) int32 (i, j) from the start to the goal, xy (m, 2) their centres
    in m, cost = the start's potential, status 0 reached, 1 start not finite or outside the grid, 2 start impassable, 3
    goal unreachable (no cells, cost 0xFFFFFFFFFFFFFFFF unless the status is 0)."""
    cells: np.ndarray
    xy: np.ndarray
    cost: int
    status: int


@dataclasses.dataclass(frozen=True)
class Frontier:
    """one kept frontier of a search (include/tloam_b200.h "Frontiers"), in rank order: id = its number before the filter
    (ascending least cell index), size = cells, sums = (Si, Sj) of its cells' i and j, bbox = (min_i, min_j, max_i,
    max_j), centroid = (x, y) m, approach = the approach cell (i, j), approach_xy its centre, approach_potential = the
    plan's P there, status 0 reachable or 1 unreachable, distance = m of free-cell path and cost (+inf when unreachable),
    cells (size, 2) int32 (i, j) ascending by linear index and xy (size, 2) their centres."""
    id: int
    size: int
    sums: tuple
    bbox: tuple
    centroid: tuple
    approach: tuple
    approach_xy: tuple
    approach_potential: int
    status: int
    distance: float
    cost: float
    cells: np.ndarray
    xy: np.ndarray


@dataclasses.dataclass(frozen=True)
class TerrainMap:
    """a built terrain map (include/tloam_b200.h "Terrain"), each layer (height, width) in the grid's layout: values (int8:
    100 lethal, 0 traversable, -1 not known; combined with the occupancy grid's when combined), ground G (+inf without a
    row in its window), elevation e (NaN without a ground-side row), step, slope (m per m) and roughness (NaN where not
    known or not defined), points m (ground-side rows); origin = (x, y) of the corner of cell (0, 0); radii = (rg, rs, rp)
    in cells; info = tloam_terrain_info's counts."""
    values: np.ndarray
    ground: np.ndarray
    elevation: np.ndarray
    step: np.ndarray
    slope: np.ndarray
    roughness: np.ndarray
    points: np.ndarray
    origin: tuple
    resolution: float
    radii: tuple
    combined: bool
    info: dict


@dataclasses.dataclass(frozen=True)
class OccupancyGrid:
    """a built occupancy grid (include/tloam_b200.h "Occupancy grid"): cells (height, width) int8 in nav_msgs/OccupancyGrid's
    values (-1 unknown, 0 .. 100), row j along y and column i along x, with the counts it came from (uint32 each); origin
    = (x, y) of the corner of cell (0, 0); dropped = the hits outside the grid; cell_tests = the window cells the free
    pass visited."""
    cells: np.ndarray
    occupied: np.ndarray
    free: np.ndarray
    origin: tuple
    resolution: float
    frames: int
    dropped: int
    cell_tests: int


@dataclasses.dataclass(frozen=True)
class PoseGraphResult:
    """tloam_pose_graph_result: termination is one of PoseGraphResult.CONVERGED .. NO_LOOPS; the costs are sum r^T Omega r
    at the odometry poses and at the returned poses; step_* are the last step's largest |upsilon| / |omega| component."""
    nodes: int
    loop_edges: int
    iterations: int
    termination: int
    initial_cost: float
    final_cost: float
    step_translation: float
    step_rotation: float
    CONVERGED, ITERATION_LIMIT, COST_INCREASED, SINGULAR, NO_LOOPS = range(5)


@dataclasses.dataclass(frozen=True)
class PoseGraphRobustResult:
    """tloam_pose_graph_robust_result: pg is the PoseGraphResult of the whole run (iterations over every stage, the last
    stage's termination, weighted costs); gnc_termination is one of PoseGraphRobustResult.CONVERGED .. NO_LOOPS; inliers
    and rejected count the loop edges with weight exactly 1 and exactly 0; mu_final is the mu of the last weight update."""
    pg: PoseGraphResult
    outer_iterations: int
    gnc_termination: int
    mu_final: float
    inliers: int
    rejected: int
    CONVERGED, OUTER_LIMIT, ALL_INLIERS, SINGULAR, NO_LOOPS = range(5)


def rz(yaw):
    """the 4 x 4 rotation about z by yaw (rad); the C library's cos / sin, as the C++ shim's verifyLoop"""
    c, s = math.cos(yaw), math.sin(yaw)
    T = np.eye(4)
    T[:2, :2] = [[c, -s], [s, c]]
    return T


class Frame:
    """Mirror of tloam::Frame (ref: registration_interface.hpp:19-38): the four feature clouds, (n,3) float64.
    scan_cloud is accepted and ignored, as in the reference (registration.cpp:232-239)."""

    def __init__(self, edge_feature, sphere_feature, planar_feature, ground_feature, scan_cloud=None):
        self.edge_feature = edge_feature
        self.sphere_feature = sphere_feature
        self.planar_feature = planar_feature
        self.ground_feature = ground_feature
        self.scan_cloud = scan_cloud

    def clouds(self):
        return [self.edge_feature, self.sphere_feature, self.planar_feature, self.ground_feature]


class LocalRegistration:
    def __init__(self, config=None, device=0, stream=None, _borrowed=None, **overrides):
        self._L = _lib.load()
        self.cfg = config if config is not None else default_config(**overrides)
        self._owned = _borrowed is None
        if _borrowed is None:
            h = C.c_void_p()
            rc = self._L.tloam_b200_create(C.byref(self.cfg), int(device), C.c_void_p(stream or 0), C.byref(h))
            if rc != _lib.OK:
                raise RegistrationError(rc, "tloam_b200_create")
        else:
            h = C.c_void_p(_borrowed)     # a sequence of a BatchRegistration: the batch owns the handle
        self._h = h
        self._keep = []
        self.n_source = [0, 0, 0, 0]

    def close(self):
        if getattr(self, "_h", None):
            if self._owned:
                self._L.tloam_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, where):
        if rc != _lib.OK:
            detail = self._L.tloam_b200_last_error(self._h).decode() if rc == _lib.ERR_CUDA else ""
            raise RegistrationError(rc, where, detail)

    # ---- RegistrationInterface ----
    @staticmethod
    def _host_args(frame):
        clouds = frame.clouds() if isinstance(frame, Frame) else list(frame)
        arrs = [_f64(c).reshape(-1, 3) for c in clouds]
        ptrs = (C.POINTER(C.c_double) * 4)(*[_dp(a) for a in arrs])
        ns = (C.c_size_t * 4)(*[a.shape[0] for a in arrs])
        return arrs, ptrs, ns

    def set_input_source(self, frame):
        arrs, ptrs, ns = self._host_args(frame)
        self._check(self._L.tloam_b200_set_source(self._h, ptrs, ns), "set_input_source")
        self.n_source = [a.shape[0] for a in arrs]
        self._keep_source_host = arrs         # pipelined mode (set_async_inputs): the upload may still be reading them
        return True

    def set_input_target(self, frame):
        arrs, ptrs, ns = self._host_args(frame)
        self._check(self._L.tloam_b200_set_target(self._h, ptrs, ns), "set_input_target")
        return True

    @staticmethod
    def _device_args(tensors):
        ptrs = (C.c_void_p * 4)(*[int(t.data_ptr()) for t in tensors])
        ns = (C.c_size_t * 4)(*[int(t.shape[0]) for t in tensors])
        return ptrs, ns

    def _order_after_producer(self, tensors, producer_stream):
        """The tensors are read IN PLACE by kernels on the handle's stream: order that stream behind the stream that
        produced them (default: torch's current stream on the tensors' device) -- a device-side wait, the host does not
        block -- and tell torch's caching allocator that another stream uses the memory."""
        if producer_stream is None:
            import torch
            producer_stream = torch.cuda.current_stream(tensors[0].device).cuda_stream
        self._check(self._L.tloam_b200_wait_stream(self._h, C.c_void_p(int(producer_stream))), "wait_stream")

    def set_input_source_device(self, tensors, producer_stream=None):
        """tensors: 4 CUDA float64 (n,3) contiguous torch tensors on this handle's device."""
        ptrs, ns = self._device_args(tensors)
        self._order_after_producer(tensors, producer_stream)
        self._check(self._L.tloam_b200_set_source_device(self._h, ptrs, ns), "set_input_source_device")
        self.n_source = [int(t.shape[0]) for t in tensors]
        self._keep_source = list(tensors)     # read in place by kernels still in flight: keep them alive until replaced
        return True

    def set_input_target_device(self, tensors, producer_stream=None):
        ptrs, ns = self._device_args(tensors)
        self._order_after_producer(tensors, producer_stream)
        self._check(self._L.tloam_b200_set_target_device(self._h, ptrs, ns), "set_input_target_device")
        self._keep_target = list(tensors)     # idem
        return True

    def scan_matching(self, predict_pose, want_stats=False):
        """predict_pose: 4x4 numpy (row-major view of the Isometry3d). Returns result 4x4 [, Stats]."""
        p = _f64(np.asarray(predict_pose).T).reshape(16)
        out = np.zeros(16)
        st = _lib.Stats() if want_stats else None
        rc = self._L.tloam_b200_scan_match(self._h, _dp(p), _dp(out), C.byref(st) if st is not None else None)
        self._check(rc, "scan_matching")
        T = out.reshape(4, 4).T.copy()
        return (T, st) if want_stats else T

    def scan_matching_predicted(self, want_stats=False):
        """(f)-3: scanMatching with the constant-velocity prediction of FrontEnd::updateLidarOdometry
        (ref: front_end.cpp:329-330) computed on the device from the two last results."""
        out = np.zeros(16)
        st = _lib.Stats() if want_stats else None
        rc = self._L.tloam_b200_scan_match_predicted(self._h, _dp(out), C.byref(st) if st is not None else None)
        self._check(rc, "scan_matching_predicted")
        T = out.reshape(4, 4).T.copy()
        return (T, st) if want_stats else T

    def set_pose_history(self, last_pose, curr_pose):
        a = _f64(np.asarray(last_pose).T).reshape(16)
        b = _f64(np.asarray(curr_pose).T).reshape(16)
        self._check(self._L.tloam_b200_set_pose_history(self._h, _dp(a), _dp(b)), "set_pose_history")

    def scan_matching_async(self, predict_pose):
        p = _f64(np.asarray(predict_pose).T).reshape(16)
        self._check(self._L.tloam_b200_scan_match_async(self._h, _dp(p)), "scan_matching_async")

    def get_result(self, want_stats=False):
        out = np.zeros(16)
        st = _lib.Stats() if want_stats else None
        rc = self._L.tloam_b200_get_result(self._h, _dp(out), C.byref(st) if st is not None else None)
        self._check(rc, "get_result")
        T = out.reshape(4, 4).T.copy()
        return (T, st) if want_stats else T

    def get_fitness_score(self):
        a, b = C.c_double(0), C.c_double(0)
        self._check(self._L.tloam_b200_fitness(self._h, C.byref(a), C.byref(b)), "get_fitness_score")
        return a.value, b.value

    def get_transform(self):
        out = np.zeros(16)
        self._check(self._L.tloam_b200_get_transform(self._h, _dp(out)), "get_transform")
        return out.reshape(4, 4).T.copy()

    def get_pose_increment(self):
        out = np.zeros(16)
        self._check(self._L.tloam_b200_get_pose_increment(self._h, _dp(out)), "get_pose_increment")
        return out.reshape(4, 4).T.copy()

    def dense_check_counters(self):
        out = (C.c_uint * 16)()
        self._check(self._L.tloam_b200_dense_check_counters(self._h, out), "dense_check_counters")
        return [int(v) for v in out]

    def synchronize(self):
        self._check(self._L.tloam_b200_synchronize(self._h), "synchronize")

    def launch_count(self):
        return int(self._L.tloam_b200_launch_count(self._h))

    def set_profiling(self, on):
        self._check(self._L.tloam_b200_set_profiling(self._h, 1 if on else 0), "set_profiling")

    def get_profile(self):
        """dict kernel-class -> (launches, total_ms), from CUDA events around every launch."""
        p = _lib.Profile()
        self._check(self._L.tloam_b200_get_profile(self._h, C.byref(p)), "get_profile")
        out = {k: (int(p.launches[i]), float(p.total_ms[i])) for i, k in enumerate(_lib.KERNEL_CLASSES)}
        self.last_dbg = [int(v) for v in p.dbg]
        return out

    # ---- device-side submap maintenance ((f)-1, mirrors FrontEnd::updateSubmap) ----
    def submap_init(self, edge, ground_raw, planar_sub, sphere_sub, **cfg_overrides):
        cfg = _lib.SubmapConfig()
        self._L.tloam_b200_submap_default_config(C.byref(cfg))
        for k, v in cfg_overrides.items():
            setattr(cfg, k, v)
        a = [_f64(x).reshape(-1, 3) for x in (edge, ground_raw, planar_sub, sphere_sub)]
        self._check(self._L.tloam_b200_submap_init(self._h, C.byref(cfg), _dp(a[0]), a[0].shape[0], _dp(a[1]), a[1].shape[0],
                                                   _dp(a[2]), a[2].shape[0], _dp(a[3]), a[3].shape[0]), "submap_init")

    def submap_update(self, pose, planar_sub, sphere_sub=None):
        p = _f64(np.asarray(pose).T).reshape(16)
        a = _f64(planar_sub).reshape(-1, 3)
        b = _f64(sphere_sub if sphere_sub is not None else np.zeros((0, 3))).reshape(-1, 3)
        self._check(self._L.tloam_b200_submap_update(self._h, _dp(p), _dp(a), a.shape[0], _dp(b), b.shape[0]), "submap_update")

    def submap_update_chained(self, planar_sub):
        """FrontEnd::updateSubmap with the pose of the frame that was just enqueued, read on the device."""
        a = _f64(planar_sub).reshape(-1, 3)
        self._keep_planar = a
        self._check(self._L.tloam_b200_submap_update_chained(self._h, _dp(a), a.shape[0]), "submap_update_chained")

    def set_async_inputs(self, on):
        self._check(self._L.tloam_b200_set_async_inputs(self._h, 1 if on else 0), "set_async_inputs")

    def set_frame_fitness(self, on):
        self._check(self._L.tloam_b200_set_frame_fitness(self._h, 1 if on else 0), "set_frame_fitness")

    def get_frame_fitness(self):
        a, b = C.c_double(0), C.c_double(0)
        self._check(self._L.tloam_b200_get_frame_fitness(self._h, C.byref(a), C.byref(b)), "get_frame_fitness")
        return a.value, b.value

    def scan_matching_predicted_async(self):
        self._check(self._L.tloam_b200_scan_match_predicted_async(self._h), "scan_matching_predicted_async")

    def submap_cloud(self, cloud):
        n = (C.c_size_t * 4)()
        self._check(self._L.tloam_b200_submap_sizes(self._h, n), "submap_sizes")
        out = np.zeros((n[cloud], 3))
        self._check(self._L.tloam_b200_submap_download(self._h, cloud, _dp(out), n[cloud]), "submap_download")
        return out

    def voxel_down_sample(self, pts, voxel):
        a = _f64(pts).reshape(-1, 3)
        out = np.zeros_like(a)
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_voxel_down_sample(self._h, _dp(a), a.shape[0], float(voxel), _dp(out), C.byref(n)), "voxel_down_sample")
        return out[:n.value].copy()

    # ---- "next" row (f)-2: PCA feature extraction (ref: feature_extract.cpp:47-122, 133-197) ----
    def _feature_config(self, overrides):
        c = _lib.FeatureConfig()
        self._L.tloam_b200_feature_default_config(C.byref(c))
        for k, v in overrides.items():
            setattr(c, k, v)
        return c

    def extract_planar_sphere(self, general_cloud, **overrides):
        """featureExtract::extractPlanarSphere on the device.  Returns (planar_scan_index, planar_submap_index,
        sphere_scan_index, sphere_submap_index, sphere_candidates); the two sphere lists hold ranks (reference quirk),
        sphere_candidates the point indices those ranks refer to."""
        a = _f64(general_cloud).reshape(-1, 3)
        c = self._feature_config(overrides)
        n = a.shape[0]
        bufs = [np.zeros(max(n, 1), dtype=np.uintp) for _ in range(5)]
        cnt = [C.c_size_t(0) for _ in range(4)]
        szp = C.POINTER(C.c_size_t)
        self._check(self._L.tloam_b200_extract_planar_sphere(
            self._h, C.byref(c), _dp(a), n, bufs[0].ctypes.data_as(szp), C.byref(cnt[0]), bufs[1].ctypes.data_as(szp),
            C.byref(cnt[1]), bufs[2].ctypes.data_as(szp), C.byref(cnt[2]), bufs[3].ctypes.data_as(szp), C.byref(cnt[3]),
            bufs[4].ctypes.data_as(szp)), "extract_planar_sphere")
        return (bufs[0][:cnt[0].value].copy(), bufs[1][:cnt[1].value].copy(), bufs[2][:cnt[2].value].copy(),
                bufs[3][:cnt[3].value].copy(), bufs[4][:cnt[3].value].copy())

    def pca_info(self, general_cloud, **overrides):
        """featureExtract::calculatePCAInfo on the device: dict of cvr, flatness, sphericity, normal (n,3), num_sum, neigh (n,K)."""
        a = _f64(general_cloud).reshape(-1, 3)
        c = self._feature_config(overrides)
        n = a.shape[0]
        out = {"cvr": np.zeros(n), "flatness": np.zeros(n), "sphericity": np.zeros(n), "normal": np.zeros((n, 3)),
               "num_sum": np.zeros(n, dtype=np.int32), "neigh": np.full((n, c.K), -1, dtype=np.int32)}
        ip = C.POINTER(C.c_int)
        self._check(self._L.tloam_b200_pca_info(self._h, C.byref(c), _dp(a), n, _dp(out["cvr"]), _dp(out["flatness"]),
                                                _dp(out["sphericity"]), _dp(out["normal"]),
                                                out["num_sum"].ctypes.data_as(ip), out["neigh"].ctypes.data_as(ip)),
                    "pca_info")
        return out

    # ---- "next" row (f)-4, first part: ground extraction (ref: segmentation.cpp:738-770) ----
    def ground_extract(self, scan, **overrides):
        """Segmentation::groundRemove on the device.  Returns dict(ground, object, beam, region, height_threshold, planes)."""
        a = _f64(scan).reshape(-1, 3)
        n = a.shape[0]
        c = _lib.GroundConfig()
        self._L.tloam_b200_ground_default_config(C.byref(c))
        for k, v in overrides.items():
            setattr(c, k, v)
        g = np.zeros(max(n, 1), dtype=np.uintp)
        o = np.zeros(max(n, 1), dtype=np.uintp)
        ng, no = C.c_size_t(0), C.c_size_t(0)
        beam = np.zeros(max(n, 1), dtype=np.int32)
        region = np.zeros(max(n, 1), dtype=np.int32)
        thr = C.c_double(0)
        planes = np.zeros((12, 8, 4))
        szp, ip = C.POINTER(C.c_size_t), C.POINTER(C.c_int)
        self._check(self._L.tloam_b200_ground_extract(self._h, C.byref(c), _dp(a), n, g.ctypes.data_as(szp), C.byref(ng),
                                                      o.ctypes.data_as(szp), C.byref(no), beam.ctypes.data_as(ip),
                                                      region.ctypes.data_as(ip), C.byref(thr), _dp(planes)), "ground_extract")
        return dict(ground=g[:ng.value].copy(), object=o[:no.value].copy(), beam=beam[:n].copy(), region=region[:n].copy(),
                    height_threshold=thr.value, planes=planes)

    def ground_remove(self, scan, **overrides):
        """ground_extract with the reference's FP64 intensity channel (VLP-16: beamId + correctTime, sensor_model=16).
        Returns dict(ground, object, intensity, region, height_threshold, planes)."""
        a = _f64(scan).reshape(-1, 3)
        n = a.shape[0]
        c = _lib.GroundConfig()
        self._L.tloam_b200_ground_default_config(C.byref(c))
        for k, v in overrides.items():
            setattr(c, k, v)
        g = np.zeros(max(n, 1), dtype=np.uintp)
        o = np.zeros(max(n, 1), dtype=np.uintp)
        ng, no = C.c_size_t(0), C.c_size_t(0)
        inten = np.zeros(max(n, 1))
        region = np.zeros(max(n, 1), dtype=np.int32)
        thr = C.c_double(0)
        planes = np.zeros((12, 8, 4))
        szp, ip = C.POINTER(C.c_size_t), C.POINTER(C.c_int)
        self._check(self._L.tloam_b200_ground_remove(self._h, C.byref(c), _dp(a), n, g.ctypes.data_as(szp), C.byref(ng),
                                                     o.ctypes.data_as(szp), C.byref(no), _dp(inten), region.ctypes.data_as(ip),
                                                     C.byref(thr), _dp(planes)), "ground_remove")
        return dict(ground=g[:ng.value].copy(), object=o[:no.value].copy(), intensity=inten[:n].copy(), region=region[:n].copy(),
                    height_threshold=thr.value, planes=planes)

    # ---- "next" row (f)-4, second part: edge extraction (ref: segmentation.cpp:1144-1304) ----
    def extract_edge(self, points, intensity, sensor_model=64, ring_min_num=16):
        """Segmentation::extractEdgePoint on the device.  intensity holds the beam id of every point (as groundRemove leaves
        it).  Returns dict(edge, non_edge): index lists into the input in the reference's append order."""
        a = _f64(points).reshape(-1, 3)
        it = _f64(intensity).reshape(-1)
        n = a.shape[0]
        if it.shape[0] != n:
            raise ValueError("one intensity (beam id) per point")
        e = np.zeros(max(n, 1), dtype=np.uintp)
        o = np.zeros(max(n, 1), dtype=np.uintp)
        ne, no = C.c_size_t(0), C.c_size_t(0)
        szp = C.POINTER(C.c_size_t)
        self._check(self._L.tloam_b200_extract_edge(self._h, sensor_model, ring_min_num, _dp(a), _dp(it), n, e.ctypes.data_as(szp),
                                                    C.byref(ne), o.ctypes.data_as(szp), C.byref(no)), "extract_edge")
        return dict(edge=e[:ne.value].copy(), non_edge=o[:no.value].copy())

    # ---- "next" row (f)-4, third part: object segmentation = DCVC (ref: segmentation.cpp:772-1112) ----
    def object_segmentation(self, points, details=True, **overrides):
        """Segmentation::objectSegmentation on the device.  Returns dict(segmented, sizes, boxes[, root, cluster, voxel,
        polar, ext]): the segmented scan as indices (cluster after cluster), cluster sizes / boxes, and with `details` per
        point the smallest index of its DCVC class, its 1-based cluster number (0 = filtered), the reference's voxel index
        and the polar triple (four more downloads; the C++ shim does not ask for them)."""
        a = _f64(points).reshape(-1, 3)
        n = a.shape[0]
        c = _lib.DcvcConfig()
        self._L.tloam_b200_dcvc_default_config(C.byref(c))
        for k, v in overrides.items():
            setattr(c, k, v)
        m = max(n, 1)
        seg = np.zeros(m, dtype=np.uintp)
        sizes = np.zeros(m, dtype=np.int32)
        boxes = np.zeros((m, 6))
        nseg, ncl = C.c_size_t(0), C.c_int(0)
        szp, ip = C.POINTER(C.c_size_t), C.POINTER(C.c_int)
        if details:
            root, cluster, voxel = (np.zeros(m, dtype=np.int32) for _ in range(3))
            polar = np.zeros(3 * m + 4)
            extra = (root.ctypes.data_as(ip), cluster.ctypes.data_as(ip), voxel.ctypes.data_as(ip), _dp(polar))
        else:
            extra = (None, None, None, None)
        self._check(self._L.tloam_b200_object_segmentation(self._h, C.byref(c), _dp(a), n, seg.ctypes.data_as(szp), C.byref(nseg),
                                                           C.byref(ncl), sizes.ctypes.data_as(ip), _dp(boxes), *extra),
                    "object_segmentation")
        k = ncl.value
        out = dict(segmented=seg[:nseg.value].copy(), sizes=sizes[:k].copy(), boxes=boxes[:k].copy())
        if details:
            out.update(root=root[:n].copy(), cluster=cluster[:n].copy(), voxel=voxel[:n].copy(),
                       polar=polar[:3 * n].reshape(-1, 3).copy(), ext=polar[3 * n:3 * n + 4].copy())
        return out

    # ---- "next" row (f)-4: the three segmentation steps as one call (ref: segmentation.cpp:47-66) ----
    def segment_scan(self, scan, ring_min_num=131, ground=None, dcvc=None):
        """groundRemove -> objectSegmentation -> extractEdgePoint chained on the device (one upload, one download).  Returns
        dict(ground, edge, general, sizes, boxes, beam): index lists into `scan`, the cluster table, the beam estimate per point.  ground / dcvc: dicts of
        configuration overrides."""
        a = _f64(scan).reshape(-1, 3)
        n = a.shape[0]
        gc, dc = _lib.GroundConfig(), _lib.DcvcConfig()
        self._L.tloam_b200_ground_default_config(C.byref(gc))
        self._L.tloam_b200_dcvc_default_config(C.byref(dc))
        for k, v in (ground or {}).items():
            setattr(gc, k, v)
        for k, v in (dcvc or {}).items():
            setattr(dc, k, v)
        m = max(n, 1)
        g, e, o = (np.zeros(m, dtype=np.uintp) for _ in range(3))
        ng, ne, no = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        ncl = C.c_int(0)
        sizes = np.zeros(m, dtype=np.int32)
        beam = np.zeros(m, dtype=np.int32)
        boxes = np.zeros((m, 6))
        szp, ip = C.POINTER(C.c_size_t), C.POINTER(C.c_int)
        self._check(self._L.tloam_b200_segment_scan(self._h, C.byref(gc), C.byref(dc), ring_min_num, _dp(a), n, g.ctypes.data_as(szp), C.byref(ng),
                                                    e.ctypes.data_as(szp), C.byref(ne), o.ctypes.data_as(szp), C.byref(no), C.byref(ncl),
                                                    sizes.ctypes.data_as(ip), _dp(boxes), beam.ctypes.data_as(ip)), "segment_scan")
        k = ncl.value
        return dict(ground=g[:ng.value].copy(), edge=e[:ne.value].copy(), general=o[:no.value].copy(), sizes=sizes[:k].copy(),
                    boxes=boxes[:k].copy(), beam=beam[:n].copy())

    def _segmentation_configs(self, ground, dcvc):
        gc, dc = _lib.GroundConfig(), _lib.DcvcConfig()
        self._L.tloam_b200_ground_default_config(C.byref(gc))
        self._L.tloam_b200_dcvc_default_config(C.byref(dc))
        for k, v in (ground or {}).items():
            setattr(gc, k, v)
        for k, v in (dcvc or {}).items():
            setattr(dc, k, v)
        return gc, dc

    def segment_raw_scan(self, scan, near_dis=3.0, ring_min_num=131, ground=None, dcvc=None):
        """RemoveClosedNonFinitePoints(near_dis) -> groundRemove -> objectSegmentation -> extractEdgePoint on the device, the
        raw scan as the driver delivers it (NaN / Inf rows allowed; a point is kept iff its norm is >= near_dis**2, as in the
        reference).  Returns dict(ground, edge, general, sizes, boxes, intensity): index lists into the RAW scan, the cluster
        table, the FP64 channel per raw point (NaN where removed).  ground / dcvc: dicts of configuration overrides."""
        a = _f64(scan).reshape(-1, 3)
        return self._segment_raw("segment_raw_scan", (_dp(a), a.shape[0]), a.shape[0], near_dis, ring_min_num, ground, dcvc)

    def segment_raw_scan_packed(self, scan, near_dis=3.0, ring_min_num=131, ground=None, dcvc=None):
        """segment_raw_scan of a raw scan in the sensor's float32 layout (a packed_scan descriptor, or an array packed_scan
        accepts): one upload, unpacked on the device.  Its intensity field is not read; the result is segment_raw_scan's."""
        d = _packed(scan)
        return self._segment_raw("segment_raw_scan_packed", (C.byref(d),), d.n, near_dis, ring_min_num, ground, dcvc)

    def _segment_raw(self, fn, scan_args, n, near_dis, ring_min_num, ground, dcvc):
        gc, dc = self._segmentation_configs(ground, dcvc)
        m = max(n, 1)
        g, e, o = (np.zeros(m, dtype=np.uintp) for _ in range(3))
        ng, ne, no = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        ncl = C.c_int(0)
        sizes = np.zeros(m, dtype=np.int32)
        inten = np.zeros(m)
        boxes = np.zeros((m, 6))
        szp, ip = C.POINTER(C.c_size_t), C.POINTER(C.c_int)
        self._check(getattr(self._L, "tloam_b200_" + fn)(self._h, C.byref(gc), C.byref(dc), ring_min_num, float(near_dis), *scan_args,
                                                         g.ctypes.data_as(szp), C.byref(ng), e.ctypes.data_as(szp), C.byref(ne),
                                                         o.ctypes.data_as(szp), C.byref(no), C.byref(ncl), sizes.ctypes.data_as(ip),
                                                         _dp(boxes), _dp(inten)), fn)
        k = ncl.value
        return dict(ground=g[:ng.value].copy(), edge=e[:ne.value].copy(), general=o[:no.value].copy(), sizes=sizes[:k].copy(),
                    boxes=boxes[:k].copy(), intensity=inten[:n].copy())

    # ---- FrontEnd::processCloud on the device (ref: src/front_end/front_end.cpp:181-199) ----
    def _submap_config(self, overrides):
        cfg = _lib.SubmapConfig()
        self._L.tloam_b200_submap_default_config(C.byref(cfg))
        for k, v in overrides.items():
            setattr(cfg, k, v)
        return cfg

    def process_cloud(self, ground, edge, general, ground_down_sample=0.3, edge_down_sample=0.1, **feature):
        """VoxelDownSample(ground / edge), extractPlanarSphere(general) and the SelectByIndex gathers on the device; the four
        features become the source (as set_input_source would).  feature: tloam_feature_config overrides.  Returns the four
        source sizes (edge, sphere, planar, ground)."""
        a = [_f64(x).reshape(-1, 3) for x in (ground, edge, general)]
        c = self._feature_config(feature)
        ns = (C.c_size_t * 4)()
        self._check(self._L.tloam_b200_process_cloud(self._h, C.byref(c), float(ground_down_sample), float(edge_down_sample), _dp(a[0]),
                                                     a[0].shape[0], _dp(a[1]), a[1].shape[0], _dp(a[2]), a[2].shape[0], ns),
                    "process_cloud")
        self.n_source = [int(v) for v in ns]
        return list(self.n_source)

    def process_raw_scan(self, scan, near_dis=3.0, ring_min_num=131, ground=None, dcvc=None, feature=None, ground_down_sample=0.3,
                         edge_down_sample=0.1, time=None, frame_period=0.1):
        """segment_raw_scan -> process_cloud on the device with one upload of the raw scan and no index list going home.
        ground / dcvc / feature: dicts of configuration overrides.  Returns the four source sizes.
        time: one value per row (in the unit of frame_period) to deskew the scan with the pose history's constant-velocity
        increment (include/tloam_b200.h, Deskewing); None: the scan is taken as it is."""
        a = _f64(scan).reshape(-1, 3)
        if time is None:
            return self._process_raw("process_raw_scan", (_dp(a), a.shape[0]), a.shape[0], near_dis, ring_min_num, ground, dcvc,
                                     feature, ground_down_sample, edge_down_sample)
        t = _f64(time).reshape(-1)
        if t.shape[0] != a.shape[0]:
            raise ValueError(f"process_raw_scan: {t.shape[0]} times for {a.shape[0]} rows")
        return self._process_raw("process_raw_scan_timed", (_dp(a), _dp(t), a.shape[0], float(frame_period)), a.shape[0], near_dis,
                                 ring_min_num, ground, dcvc, feature, ground_down_sample, edge_down_sample)

    def process_raw_scan_packed(self, scan, near_dis=3.0, ring_min_num=131, ground=None, dcvc=None, feature=None, ground_down_sample=0.3,
                                edge_down_sample=0.1, deskew=False, frame_period=0.1):
        """process_raw_scan of a raw scan in the sensor's float32 layout (a packed_scan descriptor, or an array packed_scan
        accepts): one upload, unpacked on the device.  With an intensity field, global_map_append_frame() appends the frame
        with that intensity, read on the device.  deskew: correct the scan with the records' time field (packed_time) over
        frame_period seconds, read where the records were uploaded."""
        d = _packed(scan)
        if not deskew:
            return self._process_raw("process_raw_scan_packed", (C.byref(d),), d.n, near_dis, ring_min_num, ground, dcvc, feature,
                                     ground_down_sample, edge_down_sample)
        t = packed_time(getattr(d, "_keep", None))
        return self._process_raw("process_raw_scan_packed_timed", (C.byref(d), C.byref(t), float(frame_period)), d.n, near_dis,
                                 ring_min_num, ground, dcvc, feature, ground_down_sample, edge_down_sample)

    def _process_raw(self, fn, scan_args, n, near_dis, ring_min_num, ground, dcvc, feature, ground_down_sample, edge_down_sample):
        gc, dc = self._segmentation_configs(ground, dcvc)
        fc = self._feature_config(feature or {})
        ns = (C.c_size_t * 4)()
        self._check(getattr(self._L, "tloam_b200_" + fn)(self._h, C.byref(gc), C.byref(dc), ring_min_num, float(near_dis), C.byref(fc),
                                                         float(ground_down_sample), float(edge_down_sample), *scan_args, ns), fn)
        self.n_source = [int(v) for v in ns]
        self._raw_scan_rows = n                # global_map_append_frame(intensity=...) takes one value per row
        return list(self.n_source)

    def source_cloud(self, cloud):
        """the current source cloud `cloud` (0 edge, 1 sphere, 2 planar, 3 ground), sensor frame"""
        out = np.zeros((self.n_source[cloud], 3))
        self._check(self._L.tloam_b200_source_download(self._h, cloud, _dp(out), out.shape[0]), "source_download")
        return out

    def submap_init_frame(self, **cfg_overrides):
        """the first-frame seeding (ref: front_end.cpp:285-305) from the last processed frame"""
        cfg = self._submap_config(cfg_overrides)
        self._check(self._L.tloam_b200_submap_init_frame(self._h, C.byref(cfg)), "submap_init_frame")

    def submap_update_frame(self, pose):
        """submap_update with the last processed frame's planar-submap selection, read on the device"""
        p = _f64(np.asarray(pose).T).reshape(16)
        self._check(self._L.tloam_b200_submap_update_frame(self._h, _dp(p)), "submap_update_frame")

    def submap_update_frame_chained(self):
        """submap_update_chained with the last processed frame's planar-submap selection: no host input at all"""
        self._check(self._L.tloam_b200_submap_update_frame_chained(self._h), "submap_update_frame_chained")

    # ---- global map (FrontEnd::updateSubmap with mapping_flag, ref: src/front_end/front_end.cpp:269-274) ----
    def enable_global_map(self, voxel=1.0, initial_capacity=1 << 20):
        """start an empty map: every appended raw scan is transformed, VoxelDownSample(voxel)'d on its own and concatenated"""
        cfg = _lib.GlobalMapConfig(float(voxel), int(initial_capacity))
        self._check(self._L.tloam_b200_global_map_enable(self._h, C.byref(cfg)), "global_map_enable")
        self._global_map_voxel = float(voxel)                          # global_map_merged's default

    def reset_global_map(self):
        self._check(self._L.tloam_b200_global_map_reset(self._h), "global_map_reset")

    @staticmethod
    def _intensity(intensity, rows):
        v = _f64(intensity).reshape(-1)
        if v.shape[0] != rows:
            raise ValueError(f"intensity has {v.shape[0]} values for {rows} rows")
        return v

    def global_map_append(self, scan, pose=None, intensity=None):
        """append a host raw scan (NaN / Inf rows allowed) with `pose` (4x4), or with the pose of the frame just enqueued on
        this handle when pose is None (no host round trip).  intensity: one value per row (the reference's XYZI map: each
        voxel gets the average of its rows'), or None for a frame without intensity"""
        a = _f64(scan).reshape(-1, 3)
        p = None if pose is None else _f64(np.asarray(pose).T).reshape(16)
        if intensity is not None:
            v = self._intensity(intensity, a.shape[0])
            if p is None:
                rc = self._L.tloam_b200_global_map_append_intensity_chained(self._h, _dp(a), _dp(v), a.shape[0])
            else:
                rc = self._L.tloam_b200_global_map_append_intensity(self._h, _dp(p), _dp(a), _dp(v), a.shape[0])
        elif p is None:
            rc = self._L.tloam_b200_global_map_append_chained(self._h, _dp(a), a.shape[0])
        else:
            rc = self._L.tloam_b200_global_map_append(self._h, _dp(p), _dp(a), a.shape[0])
        self._check(rc, "global_map_append")

    def global_map_append_packed(self, scan, pose=None):
        """global_map_append of a host raw scan in the sensor's float32 layout (a packed_scan descriptor, or an array
        packed_scan accepts): one upload, unpacked on the device.  With an intensity field it is an intensity frame."""
        d = _packed(scan)
        if pose is None:
            rc = self._L.tloam_b200_global_map_append_packed_chained(self._h, C.byref(d))
        else:
            p = _f64(np.asarray(pose).T).reshape(16)
            rc = self._L.tloam_b200_global_map_append_packed(self._h, _dp(p), C.byref(d))
        self._check(rc, "global_map_append_packed")

    def global_map_append_frame(self, pose=None, intensity=None):
        """append the raw scan the last process_raw_scan uploaded (read on the device); pose None = chained.  intensity: one
        value per row of that scan, or None (after process_raw_scan_packed with an intensity field: that intensity)"""
        p = None if pose is None else _f64(np.asarray(pose).T).reshape(16)
        if intensity is not None:
            v = self._intensity(intensity, getattr(self, "_raw_scan_rows", 0))
            if p is None:
                rc = self._L.tloam_b200_global_map_append_frame_intensity_chained(self._h, _dp(v))
            else:
                rc = self._L.tloam_b200_global_map_append_frame_intensity(self._h, _dp(p), _dp(v))
        elif p is None:
            rc = self._L.tloam_b200_global_map_append_frame_chained(self._h)
        else:
            rc = self._L.tloam_b200_global_map_append_frame(self._h, _dp(p))
        self._check(rc, "global_map_append_frame")

    def global_map_has_intensity(self):
        """True if the map has an intensity channel (PointCloud2::HasIntensity); raises like global_map_size"""
        has = C.c_int(0)
        self._check(self._L.tloam_b200_global_map_has_intensity(self._h, C.byref(has)), "global_map_has_intensity")
        return bool(has.value)

    def global_map_intensity(self, first=0, count=None):
        """intensities of map points [first, first + count) (all from `first` when count is None), float64; raises
        RegistrationError(ERR_NOT_READY) when the map has no intensity channel"""
        if count is None:
            count = self.global_map_size()[0] - first
        out = np.zeros(max(count, 0))
        self._check(self._L.tloam_b200_global_map_intensity_download(self._h, int(first), int(count), _dp(out)),
                    "global_map_intensity_download")
        return out

    def global_map_size(self):
        """(points, frames) of the map; raises RegistrationError(ERR_VOXEL_RANGE) once after a refused frame"""
        n, f = C.c_size_t(0), C.c_size_t(0)
        self._check(self._L.tloam_b200_global_map_size(self._h, C.byref(n), C.byref(f)), "global_map_size")
        return n.value, f.value

    def global_map(self, first=0, count=None):
        """map points [first, first + count) (all from `first` when count is None), (count, 3) float64"""
        if count is None:
            count = self.global_map_size()[0] - first
        out = np.zeros((max(count, 0), 3))
        self._check(self._L.tloam_b200_global_map_download(self._h, int(first), int(count), _dp(out)), "global_map_download")
        return out

    def global_map_frames(self):
        """frame offsets: n_frames + 1 entries, frame f is map[offsets[f]:offsets[f + 1]]"""
        nf = self.global_map_size()[1]
        out = np.zeros(nf + 1, dtype=np.uint64)
        self._check(self._L.tloam_b200_global_map_frame_offsets(self._h, out.ctypes.data_as(C.POINTER(C.c_size_t)), nf + 1),
                    "global_map_frame_offsets")
        return out.astype(np.int64)

    def global_map_capacity(self):
        """(capacity in points, growths since enable_global_map)"""
        c, g = C.c_size_t(0), C.c_size_t(0)
        self._check(self._L.tloam_b200_global_map_capacity(self._h, C.byref(c), C.byref(g)), "global_map_capacity")
        return c.value, g.value

    def registered_scan(self):
        """T.p of every row of the last appended raw scan, raw order (non-finite rows stay non-finite)"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_registered_scan_download(self._h, None, 0, C.byref(n))
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "registered_scan_download")
        out = np.zeros((n.value, 3))
        self._check(self._L.tloam_b200_registered_scan_download(self._h, _dp(out), n.value, C.byref(n)), "registered_scan_download")
        return out

    # ---- loop closure (Scan Context descriptors, exact search; include/tloam_b200.h "Loop closure") ----
    def loop_enable(self, **overrides):
        """start an empty descriptor database; overrides: fields of tloam_loop_config (lidar_height, n_ring, n_sector,
        max_radius, exclude_recent, dist_threshold, initial_capacity_frames)"""
        cfg = _lib.LoopConfig()
        self._L.tloam_b200_loop_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_loop_enable(self._h, C.byref(cfg)), "loop_enable")
        self._loop_shape = (cfg.n_ring, cfg.n_sector)

    def loop_reset(self):
        self._check(self._L.tloam_b200_loop_reset(self._h), "loop_reset")

    def loop_add_frame(self):
        """add the raw scan the last process_raw_scan* uploaded (corrected when timed), read on the device, and enqueue its
        query; the result is read by loop_result"""
        self._check(self._L.tloam_b200_loop_add_frame(self._h), "loop_add_frame")

    def loop_add(self, scan):
        """the same for a host cloud (n x 3, NaN / Inf rows allowed)"""
        a = _f64(scan).reshape(-1, 3)
        self._check(self._L.tloam_b200_loop_add(self._h, _dp(a), a.shape[0]), "loop_add")

    def loop_result(self):
        """the newest add's LoopResult (waits for that add only)"""
        r = _lib.LoopResult()
        self._check(self._L.tloam_b200_loop_result(self._h, C.byref(r)), "loop_result")
        return LoopResult(r.query, r.candidate, r.shift, r.yaw, r.distance, bool(r.is_loop))

    def loop_size(self):
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_loop_size(self._h, C.byref(n)), "loop_size")
        return n.value

    def loop_descriptor(self, frame):
        """frame's (bins (n_ring, n_sector), ring key (n_ring,), column norms (n_sector,))"""
        R, S = self._loop_shape
        out = np.zeros(R * S + R + S)
        self._check(self._L.tloam_b200_loop_descriptor_download(self._h, int(frame), _dp(out)), "loop_descriptor_download")
        return out[:R * S].reshape(R, S), out[R * S:R * S + R], out[R * S + R:]

    # ---- loop verification (keyframes and a scan-to-scan ICP; include/tloam_b200.h "Loop verification") ----
    def loop_verify_enable(self, **overrides):
        """keep a keyframe of every later loop add (only while the database is empty); overrides: fields of
        tloam_loop_verify_config (voxel, corr_dist_coarse, corr_dist_fine, max_iterations, eps_translation, eps_rotation,
        max_fitness, initial_capacity_points)"""
        cfg = _lib.LoopVerifyConfig()
        self._L.tloam_b200_loop_verify_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_loop_verify_enable(self._h, C.byref(cfg)), "loop_verify_enable")

    def loop_keyframe(self, frame):
        """frame's keyframe (n x 3), sensor frame"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_loop_keyframe_download(self._h, int(frame), None, 0, C.byref(n))   # the size
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "loop_keyframe_download")
            return np.zeros((0, 3))
        out = np.zeros((n.value, 3))
        self._check(self._L.tloam_b200_loop_keyframe_download(self._h, int(frame), _dp(out), n.value, C.byref(n)),
                    "loop_keyframe_download")
        return out

    def loop_verify(self, query, candidate, guess=None, yaw=None):
        """align keyframe query to keyframe candidate from guess (4 x 4; default identity), or from Rz(yaw) (the loop
        result's yaw); returns a LoopVerifyResult"""
        if yaw is not None:
            if guess is not None:
                raise ValueError("loop_verify: give guess or yaw, not both")
            guess = rz(yaw)
        g = None if guess is None else np.asfortranarray(np.asarray(guess, dtype=np.float64).reshape(4, 4)).ravel(order="F").copy()
        r = _lib.LoopVerifyResult()
        self._check(self._L.tloam_b200_loop_verify(self._h, int(query), int(candidate), None if g is None else _dp(g), C.byref(r)),
                    "loop_verify")
        T = np.array(r.T[:]).reshape(4, 4, order="F")
        return LoopVerifyResult(r.query, r.candidate, T, r.fitness, r.rmse, r.inliers, r.n_query_points, r.n_candidate_points,
                                r.iterations, r.termination, bool(r.accepted))

    def loop_verify_matches(self, k):
        """the last loop_verify's matches at pass k (the k-th iterate of T; k = iterations: the final pass): per query
        keyframe point the candidate keyframe row (-1: none) and its d2"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_loop_verify_matches(self._h, int(k), None, None, 0, C.byref(n))    # the size
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "loop_verify_matches")
        idx, d2 = np.zeros(n.value, dtype=np.int32), np.zeros(n.value)
        self._check(self._L.tloam_b200_loop_verify_matches(self._h, int(k), idx.ctypes.data_as(C.POINTER(C.c_int)), _dp(d2), n.value,
                                                           C.byref(n)), "loop_verify_matches")
        return idx, d2

    # ---- loop verification against a submap (the keyframes around the candidate, point to plane; include/tloam_b200.h
    #      "Loop verification against a submap") ----
    def loop_verify_submap_enable(self, **overrides):
        """needs loop_verify_enable; overrides: fields of tloam_loop_verify_submap_config (half_window, normal_radius,
        min_normal_neighbours, max_planarity, corr_dist_coarse, corr_dist_fine, max_iterations, eps_translation,
        eps_rotation, max_fitness)"""
        cfg = _lib.LoopVerifySubmapConfig()
        self._L.tloam_b200_loop_verify_submap_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_loop_verify_submap_enable(self._h, C.byref(cfg)), "loop_verify_submap_enable")

    def loop_verify_submap(self, query, candidate, guess=None, yaw=None, poses=None):
        """align keyframe query to the submap around keyframe candidate from guess (4 x 4; default identity) or Rz(yaw).
        poses: the (hi - lo + 1) x 4 x 4 poses of the window's frames lo .. hi; None: the pose graph's nodes.  Returns a
        LoopVerifyResult"""
        if yaw is not None:
            if guess is not None:
                raise ValueError("loop_verify_submap: give guess or yaw, not both")
            guess = rz(yaw)
        g = None if guess is None else np.asfortranarray(np.asarray(guess, dtype=np.float64).reshape(4, 4)).ravel(order="F").copy()
        p = None if poses is None else np.ascontiguousarray(np.asarray(poses, dtype=np.float64).reshape(-1, 4, 4).transpose(0, 2, 1))
        r = _lib.LoopVerifyResult()
        self._check(self._L.tloam_b200_loop_verify_submap(self._h, int(query), int(candidate), None if g is None else _dp(g),
                                                          None if p is None else _dp(p), C.byref(r)), "loop_verify_submap")
        T = np.array(r.T[:]).reshape(4, 4, order="F")
        return LoopVerifyResult(r.query, r.candidate, T, r.fitness, r.rmse, r.inliers, r.n_query_points, r.n_candidate_points,
                                r.iterations, r.termination, bool(r.accepted))

    def loop_verify_submap_target(self):
        """the last loop_verify_submap's target: (xyz (n x 3), normal (n x 3), valid (n,) bool, neighbours (n,))"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_loop_verify_submap_target(self._h, None, None, None, None, 0, C.byref(n))   # the size
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "loop_verify_submap_target")
        xyz, nrm = np.zeros((n.value, 3)), np.zeros((n.value, 3))
        valid, cnt = np.zeros(n.value, dtype=np.uint8), np.zeros(n.value, dtype=np.int32)
        self._check(self._L.tloam_b200_loop_verify_submap_target(
            self._h, _dp(xyz), _dp(nrm), valid.ctypes.data_as(C.POINTER(C.c_ubyte)), cnt.ctypes.data_as(C.POINTER(C.c_int)),
            n.value, C.byref(n)), "loop_verify_submap_target")
        return xyz, nrm, valid.astype(bool), cnt

    def loop_verify_submap_matches(self, k):
        """the last loop_verify_submap's matches at pass k (k = iterations: the final pass): per query keyframe point the
        target row (-1: none) and its d2"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_loop_verify_submap_matches(self._h, int(k), None, None, 0, C.byref(n))    # the size
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "loop_verify_submap_matches")
        idx, d2 = np.zeros(n.value, dtype=np.int32), np.zeros(n.value)
        self._check(self._L.tloam_b200_loop_verify_submap_matches(self._h, int(k), idx.ctypes.data_as(C.POINTER(C.c_int)), _dp(d2),
                                                                  n.value, C.byref(n)), "loop_verify_submap_matches")
        return idx, d2

    # ---- pose graph (odometry and verified loop edges, Gauss-Newton; include/tloam_b200.h "Pose graph") ----
    def pose_graph_enable(self, **overrides):
        """start an empty pose graph; overrides: fields of tloam_pose_graph_config (sigma_odom_translation,
        sigma_odom_rotation, sigma_loop_translation, sigma_loop_rotation, max_iterations, eps_translation, eps_rotation,
        max_loop_edges, initial_capacity_nodes)"""
        cfg = _lib.PoseGraphConfig()
        self._L.tloam_b200_pose_graph_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_pose_graph_enable(self._h, C.byref(cfg)), "pose_graph_enable")

    def pose_graph_reset(self):
        self._check(self._L.tloam_b200_pose_graph_reset(self._h), "pose_graph_reset")

    def pose_graph_add_node(self, pose=None):
        """a node at pose (4 x 4), or, with None, at the device pose of the last enqueued frame (get_result's pose)"""
        if pose is None:
            self._check(self._L.tloam_b200_pose_graph_add_node_chained(self._h), "pose_graph_add_node_chained")
            return
        p = np.asfortranarray(np.asarray(pose, dtype=np.float64).reshape(4, 4)).ravel(order="F").copy()
        self._check(self._L.tloam_b200_pose_graph_add_node(self._h, _dp(p)), "pose_graph_add_node")

    def pose_graph_add_loop(self, v):
        """a loop edge from an accepted LoopVerifyResult (v.candidate, v.query, Z = v.T)"""
        r = _lib.LoopVerifyResult()
        r.query, r.candidate = int(v.query), int(v.candidate)
        r.T[:] = [float(x) for x in np.asarray(v.T, dtype=np.float64).reshape(4, 4).ravel(order="F")]
        r.fitness, r.rmse, r.inliers = float(v.fitness), float(v.rmse), int(v.inliers)
        r.n_query_points, r.n_candidate_points = int(v.n_query_points), int(v.n_candidate_points)
        r.iterations, r.termination, r.accepted = int(v.iterations), int(v.termination), int(bool(v.accepted))
        self._check(self._L.tloam_b200_pose_graph_add_loop(self._h, C.byref(r)), "pose_graph_add_loop")

    def pose_graph_size(self):
        """(nodes, loop edges)"""
        n, l = C.c_size_t(0), C.c_size_t(0)
        self._check(self._L.tloam_b200_pose_graph_size(self._h, C.byref(n), C.byref(l)), "pose_graph_size")
        return n.value, l.value

    def pose_graph_optimize(self):
        r = _lib.PoseGraphResult()
        self._check(self._L.tloam_b200_pose_graph_optimize(self._h, C.byref(r)), "pose_graph_optimize")
        return PoseGraphResult(r.nodes, r.loop_edges, r.iterations, r.termination, r.initial_cost, r.final_cost,
                               r.step_translation, r.step_rotation)

    def pose_graph_optimize_robust(self, **overrides):
        """GNC with a TLS cost over the loop edges (include/tloam_b200.h "Robust pose graph"); overrides: fields of
        tloam_pose_graph_robust_config (chi2_threshold, gnc_factor, inner_iterations, max_outer_iterations)"""
        cfg = _lib.PoseGraphRobustConfig()
        self._L.tloam_b200_pose_graph_robust_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        r = _lib.PoseGraphRobustResult()
        self._check(self._L.tloam_b200_pose_graph_optimize_robust(self._h, C.byref(cfg), C.byref(r)), "pose_graph_optimize_robust")
        p = r.pg
        return PoseGraphRobustResult(PoseGraphResult(p.nodes, p.loop_edges, p.iterations, p.termination, p.initial_cost,
                                                     p.final_cost, p.step_translation, p.step_rotation),
                                     r.outer_iterations, r.gnc_termination, r.mu_final, r.inliers, r.rejected)

    def pose_graph_loop_weights(self, first=0, count=None):
        """(count,): the last optimisation's loop-edge weights (1.0 after a plain one and for edges added after it)"""
        n = self.pose_graph_size()[1]
        if count is None:
            count = n - first
        if first < 0 or count < 0 or first + count > n:
            raise RegistrationError(_lib.ERR_INVALID_ARG, "pose_graph_loop_weights")
        out = np.zeros(count)
        self._check(self._L.tloam_b200_pose_graph_loop_weights(self._h, int(first), int(count), _dp(out)), "pose_graph_loop_weights")
        return out

    def pose_graph_poses(self, first=0, count=None):
        """(count, 4, 4): the last optimisation's poses, the odometry poses for nodes it did not cover"""
        n = self.pose_graph_size()[0]
        if count is None:
            count = n - first
        if first < 0 or count < 0 or first + count > n:
            raise RegistrationError(_lib.ERR_INVALID_ARG, "pose_graph_download")
        out = np.zeros(16 * count)
        self._check(self._L.tloam_b200_pose_graph_download(self._h, int(first), int(count), _dp(out)), "pose_graph_download")
        return out.reshape(count, 4, 4).transpose(0, 2, 1).copy()

    def pose_graph_correction(self):
        """T_opt(N - 1) . O_{N-1}^-1 of the last optimisation (map -> odom); identity before one"""
        out = np.zeros(16)
        self._check(self._L.tloam_b200_pose_graph_correction(self._h, _dp(out)), "pose_graph_correction")
        return out.reshape(4, 4).T.copy()

    # ---- loop-corrected global map (include/tloam_b200.h "Loop-corrected global map") ----
    def global_map_correction_enable(self):
        """record every later append's odometry and current pose (only on an empty map)"""
        self._check(self._L.tloam_b200_global_map_correction_enable(self._h), "global_map_correction_enable")

    def global_map_correct(self, nodes):
        """move every map frame f to Delta_{nodes[f]} O_f of the last pose-graph optimisation (nodes[f] = -1: leave it);
        len(nodes) must be the map's frame count"""
        n = np.ascontiguousarray(np.asarray(nodes, dtype=np.int64).reshape(-1))
        p = n.ctypes.data_as(C.POINTER(C.c_longlong)) if n.size else None
        self._check(self._L.tloam_b200_global_map_correct(self._h, p, n.size), "global_map_correct")

    def global_map_frame_poses(self, first=0, count=None):
        """(odometry poses, current poses) of map frames [first, first + count), each (count, 4, 4)"""
        if count is None:
            count = self.global_map_size()[1] - first
        if first < 0 or count < 0:
            raise RegistrationError(_lib.ERR_INVALID_ARG, "global_map_frame_poses")
        o, c = np.zeros(16 * count), np.zeros(16 * count)
        self._check(self._L.tloam_b200_global_map_frame_poses(self._h, int(first), int(count), _dp(o), _dp(c)),
                    "global_map_frame_poses")
        return tuple(x.reshape(count, 4, 4).transpose(0, 2, 1).copy() for x in (o, c))

    # ---- dynamic-point removal (include/tloam_b200.h "Dynamic-point removal") ----
    def global_map_dynamic_enable(self, **overrides):
        """free-space votes from every later append on the map rows before it (only on an empty map); overrides: fields of
        tloam_global_map_dynamic_config (n_rows, fov_up, fov_down, n_cols, window_rows, window_cols, margin_abs,
        margin_rel, min_range, max_range, min_through)"""
        cfg = _lib.GlobalMapDynamicConfig()
        self._L.tloam_b200_global_map_dynamic_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown dynamic-removal field {k!r}")
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_global_map_dynamic_enable(self._h, C.byref(cfg)), "global_map_dynamic_enable")

    def global_map_votes(self, first=0, count=None):
        """(through, hits) of map rows [first, first + count), uint32 each"""
        if count is None:
            count = self.global_map_size()[0] - first
        if first < 0 or count < 0:
            raise RegistrationError(_lib.ERR_INVALID_ARG, "global_map_votes_download")
        t, h = np.zeros(count, dtype=np.uint32), np.zeros(count, dtype=np.uint32)
        up = C.POINTER(C.c_uint)
        self._check(self._L.tloam_b200_global_map_votes_download(self._h, int(first), int(count), t.ctypes.data_as(up),
                                                                 h.ctypes.data_as(up)), "global_map_votes_download")
        return t, h

    def global_map_static(self):
        """(xyz (n, 3), intensity (n,) or None): the map rows not judged dynamic, in row order"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_global_map_static_download(self._h, None, None, 0, C.byref(n))
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "global_map_static_download")
        has = self.global_map_has_intensity()
        xyz = np.zeros((n.value, 3))
        inten = np.zeros(n.value) if has else None
        self._check(self._L.tloam_b200_global_map_static_download(self._h, _dp(xyz), _dp(inten) if has else None, n.value,
                                                                  C.byref(n)), "global_map_static_download")
        return xyz[:n.value], (inten[:n.value] if has else None)

    # ---- merged global map (include/tloam_b200.h "Merged global map") ----
    def global_map_merged(self, voxel=None, static=False):
        """(xyz (n, 3), intensity (n,) or None): the map (or with static=True its rows not judged dynamic) merged into one
        voxel grid, VoxelDownSample(voxel) of the whole map, voxels in ascending (ix, iy, iz).  voxel=None: the map's own"""
        v = getattr(self, "_global_map_voxel", 1.0) if voxel is None else float(voxel)
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_global_map_merge(self._h, v, 1 if static else 0, C.byref(n)), "global_map_merge")
        has = self.global_map_has_intensity()
        xyz = np.zeros((n.value, 3))
        inten = np.zeros(n.value) if has else None
        self._check(self._L.tloam_b200_global_map_merged_download(self._h, 0, n.value, _dp(xyz), _dp(inten) if has else None),
                    "global_map_merged_download")
        return xyz, inten

    # ---- localization in a prior map (include/tloam_b200.h "Localization in a prior map") ----
    def localize_enable(self, **overrides):
        """turn localization on and drop any loaded map; overrides: fields of tloam_localize_config (voxel, cell,
        normal_radius, min_normal_neighbours, max_planarity, corr_dist_coarse, corr_dist_fine, max_iterations,
        eps_translation, eps_rotation, max_fitness)"""
        cfg = _lib.LocalizeConfig()
        self._L.tloam_b200_localize_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_localize_enable(self._h, C.byref(cfg)), "localize_enable")

    def localize_set_map(self, xyz):
        """load a prior map (n x 3) and build its grid index and normals"""
        p = np.ascontiguousarray(np.asarray(xyz, dtype=np.float64).reshape(-1, 3))
        self._check(self._L.tloam_b200_localize_set_map(self._h, _dp(p) if len(p) else None, len(p)), "localize_set_map")

    def localize_set_map_merged(self):
        """load the last global_map_merged on the device as the prior map"""
        self._check(self._L.tloam_b200_localize_set_map_merged(self._h), "localize_set_map_merged")

    @staticmethod
    def _localize_out(r):
        f = lambda a: np.array(a[:]).reshape(4, 4, order="F")                                    # noqa: E731
        return LocalizeResult(f(r.T), f(r.T_map_odom), f(r.guess), r.iterations, r.termination, bool(r.accepted), r.inliers,
                              r.rmse, r.fitness, r.n_query_points, r.n_map_points)

    def localize_frame(self, guess=None):
        """localize the scan the last process_raw_scan left on the device, from guess (4 x 4, map <- sensor) or, with None,
        from the prediction L_prev . O_prev^-1 . O_now.  Returns a LocalizeResult"""
        g = None if guess is None else np.asarray(guess, dtype=np.float64).reshape(4, 4).ravel(order="F").copy()
        r = _lib.LocalizeResult()
        self._check(self._L.tloam_b200_localize_frame(self._h, None if g is None else _dp(g), C.byref(r)), "localize_frame")
        return self._localize_out(r)

    def localize(self, xyz, guess=None):
        """localize a host cloud (n x 3); as localize_frame"""
        p = np.ascontiguousarray(np.asarray(xyz, dtype=np.float64).reshape(-1, 3))
        g = None if guess is None else np.asarray(guess, dtype=np.float64).reshape(4, 4).ravel(order="F").copy()
        r = _lib.LocalizeResult()
        self._check(self._L.tloam_b200_localize(self._h, _dp(p) if len(p) else None, len(p), None if g is None else _dp(g),
                                                C.byref(r)), "localize")
        return self._localize_out(r)

    def localize_matches(self, k):
        """the last localization's matches at pass k (k = iterations: the final pass): per query row the map row (-1:
        none) and its d2"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_localize_matches(self._h, int(k), None, None, 0, C.byref(n))
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "localize_matches")
        idx, d2 = np.zeros(n.value, dtype=np.int32), np.zeros(n.value)
        self._check(self._L.tloam_b200_localize_matches(self._h, int(k), idx.ctypes.data_as(C.POINTER(C.c_int)), _dp(d2),
                                                        n.value, C.byref(n)), "localize_matches")
        return idx, d2

    def localize_query(self):
        """the last localization's query: the down-sampled scan (n x 3)"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_localize_query(self._h, None, 0, C.byref(n))
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "localize_query")
        xyz = np.zeros((n.value, 3))
        self._check(self._L.tloam_b200_localize_query(self._h, _dp(xyz), n.value, C.byref(n)), "localize_query")
        return xyz

    def localize_map_normals(self):
        """the loaded map's (normal (n x 3), valid (n,) bool, neighbours (n,))"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_localize_map_normals(self._h, None, None, None, 0, C.byref(n))
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "localize_map_normals")
        nrm, valid, cnt = np.zeros((n.value, 3)), np.zeros(n.value, dtype=np.uint8), np.zeros(n.value, dtype=np.int32)
        self._check(self._L.tloam_b200_localize_map_normals(self._h, _dp(nrm), valid.ctypes.data_as(C.POINTER(C.c_ubyte)),
                                                            cnt.ctypes.data_as(C.POINTER(C.c_int)), n.value, C.byref(n)),
                    "localize_map_normals")
        return nrm, valid.astype(bool), cnt

    def localize_cells(self, n_rows):
        """the loaded map's cell table: (sorted rows (n_rows,), cell keys (n_cells,), cell starts (n_cells + 1,))"""
        nc = C.c_size_t(0)
        rows, keys = np.zeros(n_rows, dtype=np.uint32), np.zeros(n_rows, dtype=np.uint64)
        starts = np.zeros(n_rows + 1, dtype=np.uint32)
        up = C.POINTER(C.c_uint)
        self._check(self._L.tloam_b200_localize_cells(self._h, rows.ctypes.data_as(up), keys.ctypes.data_as(C.POINTER(C.c_ulonglong)),
                                                      starts.ctypes.data_as(up), n_rows, C.byref(nc)), "localize_cells")
        return rows, keys[:nc.value], starts[:nc.value + 1]

    # ---- global registration (include/tloam_b200.h "Global registration") ----
    def global_registration_enable(self, **overrides):
        """turn global registration on; overrides: fields of tloam_global_registration_config (voxel, cell, normal_radius,
        min_normal_neighbours, feature_radius, max_correspondence_distance, n_hypotheses, seed, edge_similarity,
        min_triangle_area, max_refine_iterations, min_inliers, min_fitness)"""
        cfg = _lib.GlobalRegistrationConfig()
        self._L.tloam_b200_global_registration_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_global_registration_enable(self._h, C.byref(cfg)), "global_registration_enable")

    @staticmethod
    def _global_registration_out(r):
        return GlobalRegistrationResult(np.array(r.T[:]).reshape(4, 4, order="F"), r.n_source_points, r.n_target_points,
                                        r.n_source_features, r.n_target_features, r.n_correspondences, r.n_valid_hypotheses,
                                        r.best_hypothesis, r.best_inliers, r.inliers, r.inlier_rmse, r.fitness,
                                        r.refine_iterations, r.termination, bool(r.accepted))

    def global_register(self, source, target):
        """align host cloud source (n x 3) to host cloud target (m x 3) with no guess; returns a GlobalRegistrationResult"""
        p = np.ascontiguousarray(np.asarray(source, dtype=np.float64).reshape(-1, 3))
        q = np.ascontiguousarray(np.asarray(target, dtype=np.float64).reshape(-1, 3))
        r = _lib.GlobalRegistrationResult()
        self._check(self._L.tloam_b200_global_register(self._h, _dp(p) if len(p) else None, len(p), _dp(q) if len(q) else None,
                                                       len(q), C.byref(r)), "global_register")
        return self._global_registration_out(r)

    def global_register_loop(self, query, candidate):
        """align loop keyframe query to loop keyframe candidate with no guess: T = T_cand_query"""
        r = _lib.GlobalRegistrationResult()
        self._check(self._L.tloam_b200_global_register_loop(self._h, int(query), int(candidate), C.byref(r)),
                    "global_register_loop")
        return self._global_registration_out(r)

    def global_registration_side(self, side):
        """the last run's side (0 source, 1 target): dict of keypoints (n x 3), oriented normals (n x 3), valid (n,), SPFH
        counts (n x 33), features (n x 33) and has_feature (n,)"""
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_global_registration_side(self._h, int(side), None, None, None, None, None, None,
                                                                1 << 62, C.byref(n)), "global_registration_side")
        m = n.value
        out = dict(xyz=np.zeros((m, 3)), normal=np.zeros((m, 3)), valid=np.zeros(m, dtype=np.uint8),
                   spfh=np.zeros((m, 33), dtype=np.int32), feature=np.zeros((m, 33)), has_feature=np.zeros(m, dtype=np.uint8))
        ub, ip = C.POINTER(C.c_ubyte), C.POINTER(C.c_int)
        self._check(self._L.tloam_b200_global_registration_side(
            self._h, int(side), _dp(out["xyz"]), _dp(out["normal"]), out["valid"].ctypes.data_as(ub), out["spfh"].ctypes.data_as(ip),
            _dp(out["feature"]), out["has_feature"].ctypes.data_as(ub), m, C.byref(n)), "global_registration_side")
        out["valid"], out["has_feature"] = out["valid"].astype(bool), out["has_feature"].astype(bool)
        return out

    def global_registration_correspondences(self):
        """the last run's mutual pairs (n x 2: source row, target row) in source order"""
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_global_registration_correspondences(self._h, None, 1 << 62, C.byref(n)),
                    "global_registration_correspondences")
        out = np.zeros((n.value, 2), dtype=np.int32)
        self._check(self._L.tloam_b200_global_registration_correspondences(self._h, out.ctypes.data_as(C.POINTER(C.c_int)),
                                                                            n.value, C.byref(n)),
                    "global_registration_correspondences")
        return out

    def global_registration_hypotheses(self):
        """the last run's inliers per hypothesis (-1: rejected)"""
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_global_registration_hypotheses(self._h, None, 1 << 62, C.byref(n)),
                    "global_registration_hypotheses")
        out = np.zeros(n.value, dtype=np.int32)
        self._check(self._L.tloam_b200_global_registration_hypotheses(self._h, out.ctypes.data_as(C.POINTER(C.c_int)), n.value,
                                                                       C.byref(n)), "global_registration_hypotheses")
        return out

    # ---- relocalization in a prior map (include/tloam_b200.h "Relocalization in a prior map") ----
    def relocalize_enable(self, **overrides):
        """turn relocalization on (localization must be on) and drop the places; overrides: fields of
        tloam_relocalize_config (lidar_height, n_ring, n_sector, max_radius, top_k, max_distance, distinct_translation,
        distinct_rotation, ambiguity_ratio)"""
        cfg = _lib.RelocalizeConfig()
        self._L.tloam_b200_relocalize_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not hasattr(cfg, k):
                raise KeyError(k)
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_relocalize_enable(self._h, C.byref(cfg)), "relocalize_enable")
        self._reloc_slot = cfg.n_ring * cfg.n_sector + cfg.n_ring + cfg.n_sector

    def relocalize_set_places(self, descriptors, poses):
        """load the places: descriptor slots (n x slot, as loop_descriptors returns them) and poses (n x 4 x 4, map <- sensor)"""
        P = np.asarray(poses, dtype=np.float64).reshape(-1, 4, 4)
        p = np.ascontiguousarray(P.transpose(0, 2, 1))                            # column-major per pose
        n = len(P)
        d = np.ascontiguousarray(np.asarray(descriptors, dtype=np.float64))
        slot = getattr(self, "_reloc_slot", None)
        if slot is None:
            raise RuntimeError("relocalize_set_places: relocalize_enable first")
        if d.shape != (n, slot):
            raise ValueError(f"relocalize_set_places: descriptors of shape {d.shape}, want ({n}, {slot}) for {n} poses")
        self._check(self._L.tloam_b200_relocalize_set_places(self._h, _dp(d) if n else None, _dp(p) if n else None, n),
                    "relocalize_set_places")

    def relocalize_set_places_loop(self, poses):
        """load the places from the handle's own loop database, with one pose per loop frame (n x 4 x 4)"""
        P = np.asarray(poses, dtype=np.float64).reshape(-1, 4, 4)
        p = np.ascontiguousarray(P.transpose(0, 2, 1))
        self._check(self._L.tloam_b200_relocalize_set_places_loop(self._h, _dp(p) if len(P) else None, len(P)),
                    "relocalize_set_places_loop")

    def _relocalize_out(self, r):
        return RelocalizeResult(self._localize_out(r.result), r.place, r.shift, r.distance, r.n_hypotheses, r.winner,
                                bool(r.ambiguous), bool(r.accepted))

    def relocalize_frame(self):
        """relocalize the scan the last process_raw_scan left on the device; returns a RelocalizeResult"""
        r = _lib.RelocalizeResult()
        self._check(self._L.tloam_b200_relocalize_frame(self._h, C.byref(r)), "relocalize_frame")
        return self._relocalize_out(r)

    def relocalize(self, xyz):
        """relocalize a host cloud (n x 3); as relocalize_frame"""
        p = np.ascontiguousarray(np.asarray(xyz, dtype=np.float64).reshape(-1, 3))
        r = _lib.RelocalizeResult()
        self._check(self._L.tloam_b200_relocalize(self._h, _dp(p) if len(p) else None, len(p), C.byref(r)), "relocalize")
        return self._relocalize_out(r)

    def relocalize_hypotheses(self):
        """the last relocalization's hypotheses in rank order: [(place, shift, distance, LocalizeResult)]"""
        n = C.c_size_t(0)
        buf = (_lib.RelocalizeHypothesis * 64)()
        self._check(self._L.tloam_b200_relocalize_hypotheses(self._h, buf, 64, C.byref(n)), "relocalize_hypotheses")
        return [(buf[k].place, buf[k].shift, buf[k].distance, self._localize_out(buf[k].result)) for k in range(n.value)]

    def relocalize_matches(self, hypothesis, k):
        """hypothesis's matches at pass k, as localize_matches"""
        n = C.c_size_t(0)
        rc = self._L.tloam_b200_relocalize_matches(self._h, int(hypothesis), int(k), None, None, 0, C.byref(n))
        if rc != _lib.ERR_INVALID_ARG or n.value == 0:
            self._check(rc, "relocalize_matches")
        idx, d2 = np.zeros(n.value, dtype=np.int32), np.zeros(n.value)
        self._check(self._L.tloam_b200_relocalize_matches(self._h, int(hypothesis), int(k), idx.ctypes.data_as(C.POINTER(C.c_int)),
                                                          _dp(d2), n.value, C.byref(n)), "relocalize_matches")
        return idx, d2

    # ---- updating a prior map (include/tloam_b200.h "Updating a prior map") ----
    def map_update_enable(self, image=None, **overrides):
        """turn updating of the loaded prior map on (localization must be on) and empty its state; image: a dict of
        tloam_global_map_dynamic_config overrides for the votes' range image; overrides: novel_radius, voxel, min_frames"""
        cfg = _lib.MapUpdateConfig()
        self._L.tloam_b200_map_update_default_config(C.byref(cfg))
        for k, v in (image or {}).items():
            if not any(f[0] == k for f in cfg.image._fields_):
                raise TypeError(f"unknown image field {k!r}")
            setattr(cfg.image, k, v)
        for k, v in overrides.items():
            if k == "image" or not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown map-update field {k!r}")
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_map_update_enable(self._h, C.byref(cfg)), "map_update_enable")

    def map_update_add(self):
        """vote with the last localization's scan at its T and append its new query rows; a rejected localization gives
        used=False and changes nothing.  Returns a MapUpdateAddResult"""
        r = _lib.MapUpdateAddResult()
        self._check(self._L.tloam_b200_map_update_add(self._h, C.byref(r)), "map_update_add")
        return MapUpdateAddResult(bool(r.used), r.frame, r.n_scan_points, r.n_query_points)

    def map_update_build(self):
        """(xyz (n, 3), MapUpdateResult): the prior rows not removed, in row order, then the additions' voxels that enough
        adds support"""
        r = _lib.MapUpdateResult()
        self._check(self._L.tloam_b200_map_update_build(self._h, C.byref(r)), "map_update_build")
        xyz = np.zeros((r.n_total, 3))
        self._check(self._L.tloam_b200_map_update_download(self._h, 0, r.n_total, _dp(xyz)), "map_update_download")
        return xyz, MapUpdateResult(r.n_prior, r.n_prior_removed, r.n_additions, r.n_additions_removed, r.n_voxels,
                                    r.n_voxels_kept, r.n_total)

    def map_update_size(self):
        """(prior rows, addition rows, built rows)"""
        a, b, c = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        self._check(self._L.tloam_b200_map_update_size(self._h, C.byref(a), C.byref(b), C.byref(c)), "map_update_size")
        return a.value, b.value, c.value

    def map_update_votes(self, which):
        """(through, hits), uint32 each, of every prior row (which=0) or every addition (which=1)"""
        n = self.map_update_size()[1 if which else 0]
        t, h = np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint32)
        up = C.POINTER(C.c_uint)
        self._check(self._L.tloam_b200_map_update_votes(self._h, int(which), 0, n, t.ctypes.data_as(up), h.ctypes.data_as(up)),
                    "map_update_votes")
        return t, h

    def map_update_additions(self):
        """(xyz (n, 3), frame (n,) uint32) of every addition, in the order they were appended"""
        n = self.map_update_size()[1]
        xyz, f = np.zeros((n, 3)), np.zeros(n, dtype=np.uint32)
        self._check(self._L.tloam_b200_map_update_additions(self._h, 0, n, _dp(xyz), f.ctypes.data_as(C.POINTER(C.c_uint))),
                    "map_update_additions")
        return xyz, f

    # ---- occupancy grid (include/tloam_b200.h "Occupancy grid") ----
    def occupancy_enable(self, **overrides):
        """record a 2D scan per later append (only on an empty map); overrides: fields of tloam_occupancy_config
        (resolution, n_cols, z_lo, z_hi, min_range, max_range, free_margin)"""
        cfg = _lib.OccupancyConfig()
        self._L.tloam_b200_occupancy_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown occupancy field {k!r}")
            setattr(cfg, k, v)
        self._check(self._L.tloam_b200_occupancy_enable(self._h, C.byref(cfg)), "occupancy_enable")
        self._occupancy_cols = cfg.n_cols

    def occupancy_build(self):
        """rasterise every map frame at its current pose; returns an OccupancyGrid"""
        info = _lib.OccupancyInfo()
        self._check(self._L.tloam_b200_occupancy_build(self._h, C.byref(info)), "occupancy_build")
        shape = (info.height, info.width)
        cells = np.zeros(shape, dtype=np.int8)
        occ, free = np.zeros(shape, dtype=np.uint32), np.zeros(shape, dtype=np.uint32)
        up = C.POINTER(C.c_uint)
        self._check(self._L.tloam_b200_occupancy_download(self._h, cells.ctypes.data_as(C.POINTER(C.c_byte)),
                                                          occ.ctypes.data_as(up), free.ctypes.data_as(up), cells.size),
                    "occupancy_download")
        return OccupancyGrid(cells, occ, free, (info.origin_x, info.origin_y), info.resolution, info.frames, info.dropped,
                             info.cell_tests)

    def occupancy_scans(self, first=0, count=None):
        """(obstacles (count, n_cols, 3), floors (count, n_cols), poses (count, 4, 4)) of map frames [first, first + count):
        each sector's obstacle in the sensor frame and its floor range (NaN when absent), and the pose recorded at the
        append"""
        if count is None:
            count = self.global_map_size()[1] - first
        if first < 0 or count < 0:
            raise RegistrationError(_lib.ERR_INVALID_ARG, "occupancy_scans_download")
        n_cols = getattr(self, "_occupancy_cols", 0)
        scans, poses = np.zeros((count, n_cols, 4)), np.zeros((count, 16))
        self._check(self._L.tloam_b200_occupancy_scans_download(self._h, int(first), int(count), _dp(scans), _dp(poses)),
                    "occupancy_scans_download")
        return scans[:, :, :3].copy(), scans[:, :, 3].copy(), poses.reshape(count, 4, 4).transpose(0, 2, 1).copy()

    # ---- distance field and costmap (include/tloam_b200.h "Distance field and costmap") ----
    def distance_build(self, grid=None, origin=None, resolution=None, **overrides):
        """the distance field and costmap of the last occupancy_build (grid None), or of a host grid: (height, width) int8
        in nav_msgs/OccupancyGrid's values with its origin (x, y) and resolution; overrides: fields of
        tloam_distance_config (inscribed_radius, inflation_radius, cost_scaling_factor).  Returns a DistanceField."""
        def build(cfg, info):
            if grid is None:
                self._check(self._L.tloam_b200_distance_build(self._h, C.byref(cfg), C.byref(info)), "distance_build")
                return
            g = np.ascontiguousarray(grid, dtype=np.int8)
            if g.ndim != 2 or origin is None or resolution is None:
                raise RegistrationError(_lib.ERR_INVALID_ARG, "distance_build_grid")
            self._check(self._L.tloam_b200_distance_build_grid(
                self._h, C.byref(cfg), g.ctypes.data_as(C.POINTER(C.c_byte)), g.shape[1], g.shape[0], float(origin[0]),
                float(origin[1]), float(resolution), C.byref(info)), "distance_build_grid")
        return self._distance_field(build, overrides)

    def _distance_field(self, build, overrides):
        """the distance config with the overrides, build(cfg, info) (a checked C call), then the field's download"""
        cfg = _lib.DistanceConfig()
        self._L.tloam_b200_distance_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown distance field {k!r}")
            setattr(cfg, k, v)
        info = _lib.DistanceInfo()
        build(cfg, info)
        shape = (info.height, info.width)
        sd, sq = np.zeros(shape, dtype=np.float32), np.zeros(shape, dtype=np.uint32)
        costs, values = np.zeros(shape, dtype=np.uint8), np.zeros(shape, dtype=np.int8)
        self._check(self._L.tloam_b200_distance_download(
            self._h, sd.ctypes.data_as(C.POINTER(C.c_float)), sq.ctypes.data_as(C.POINTER(C.c_uint)),
            costs.ctypes.data_as(C.POINTER(C.c_ubyte)), values.ctypes.data_as(C.POINTER(C.c_byte)), sd.size),
            "distance_download")
        return DistanceField(sd, sq, costs, values, (info.origin_x, info.origin_y), info.resolution, info.obstacles)

    # ---- terrain (include/tloam_b200.h "Terrain") ----
    def terrain_build(self, cloud=None, **overrides):
        """the terrain map of the global map (cloud None) or of a host cloud (n, 3); overrides: fields of
        tloam_terrain_config (resolution, clearance, ground_radius, step_radius, slope_radius, max_step, max_slope in
        radians, max_roughness, min_points, min_fit, static_only, combine_occupancy).  Returns a TerrainMap."""
        cfg = _lib.TerrainConfig()
        self._L.tloam_b200_terrain_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown terrain field {k!r}")
            setattr(cfg, k, v)
        info = _lib.TerrainInfo()
        if cloud is None:
            self._check(self._L.tloam_b200_terrain_build(self._h, C.byref(cfg), C.byref(info)), "terrain_build")
        else:
            c = _f64(cloud).reshape(-1, 3)
            self._check(self._L.tloam_b200_terrain_build_cloud(self._h, C.byref(cfg), _dp(c), c.shape[0], C.byref(info)),
                        "terrain_build_cloud")
        shape = (info.height, info.width)
        values, points = np.zeros(shape, dtype=np.int8), np.zeros(shape, dtype=np.uint32)
        layers = [np.zeros(shape) for _ in range(5)]
        self._check(self._L.tloam_b200_terrain_download(self._h, values.ctypes.data_as(C.POINTER(C.c_byte)),
                                                        *[_dp(a) for a in layers], points.ctypes.data_as(C.POINTER(C.c_uint)),
                                                        values.size), "terrain_download")
        return TerrainMap(values, *layers, points, (info.origin_x, info.origin_y), info.resolution,
                          (info.ground_cells, info.step_cells, info.slope_cells), bool(info.combined),
                          {name: getattr(info, name) for name, _ in info._fields_})

    def distance_build_terrain(self, **overrides):
        """the distance field and costmap of the last terrain_build's values; overrides: fields of tloam_distance_config.
        Returns a DistanceField."""
        return self._distance_field(lambda cfg, info: self._check(self._L.tloam_b200_distance_build_terrain(
            self._h, C.byref(cfg), C.byref(info)), "distance_build_terrain"), overrides)

    def distance_query(self, xy):
        """(distance (n,), gradient (n, 2)) of the last distance_build at the points xy (n, 2): sd interpolated bilinearly
        between the cell centres, NaN outside them or on a field with an infinite value"""
        p = np.ascontiguousarray(xy, dtype=np.float64).reshape(-1, 2)
        d, g = np.zeros(len(p)), np.zeros((len(p), 2))
        self._check(self._L.tloam_b200_distance_query(self._h, _dp(p), len(p), _dp(d), _dp(g)), "distance_query")
        return d, g

    # ---- path planning (include/tloam_b200.h "Path planning") ----
    def plan_build(self, goal, **overrides):
        """the potential to the goal (x, y) on the last distance_build's costs; overrides: fields of tloam_plan_config
        (neutral_cost, cost_factor, allow_unknown).  Returns a PlanField."""
        cfg = _lib.PlanConfig()
        self._L.tloam_b200_plan_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown plan field {k!r}")
            setattr(cfg, k, v)
        info = _lib.PlanInfo()
        self._check(self._L.tloam_b200_plan_build(self._h, C.byref(cfg), float(goal[0]), float(goal[1]), C.byref(info)),
                    "plan_build")
        P = np.zeros((info.height, info.width), dtype=np.uint64)
        self._check(self._L.tloam_b200_plan_download(self._h, P.ctypes.data_as(C.POINTER(C.c_ulonglong)), P.size),
                    "plan_download")
        return PlanField(P, (info.origin_x, info.origin_y), info.resolution, (info.goal_i, info.goal_j), info.reachable,
                         info.rounds, info.tiles)

    def plan_paths(self, starts):
        """one PlanPath per start (n, 2) of xy, down the last plan_build"""
        p = np.ascontiguousarray(starts, dtype=np.float64).reshape(-1, 2)
        n = len(p)
        offsets = np.zeros(n + 1, dtype=np.uintp)
        statuses = np.zeros(n, dtype=np.int32)
        costs = np.zeros(n, dtype=np.uint64)
        self._check(self._L.tloam_b200_plan_paths(
            self._h, _dp(p), n, offsets.ctypes.data_as(C.POINTER(C.c_size_t)), statuses.ctypes.data_as(C.POINTER(C.c_int)),
            costs.ctypes.data_as(C.POINTER(C.c_ulonglong))), "plan_paths")
        m = int(offsets[-1])
        ij = np.zeros((m, 2), dtype=np.int32)
        xy = np.zeros((m, 2))
        self._check(self._L.tloam_b200_plan_path_cells(self._h, ij.ctypes.data_as(C.POINTER(C.c_int)), _dp(xy), m),
                    "plan_path_cells")
        return [PlanPath(ij[offsets[s]:offsets[s + 1]], xy[offsets[s]:offsets[s + 1]], int(costs[s]), int(statuses[s]))
                for s in range(n)]

    # ---- frontiers (include/tloam_b200.h "Frontiers") ----
    def frontier_search(self, **overrides):
        """the frontiers of the last distance_build, ranked by the last plan_build (build it with its goal at the robot);
        overrides: fields of tloam_frontier_config (free_max, min_frontier_size, potential_scale, gain_scale).  Returns
        (info, frontiers): info a dict of tloam_frontier_info's fields, frontiers the kept ones in rank order."""
        cfg = _lib.FrontierConfig()
        self._L.tloam_b200_frontier_default_config(C.byref(cfg))
        for k, v in overrides.items():
            if not any(f[0] == k for f in cfg._fields_):
                raise TypeError(f"unknown frontier field {k!r}")
            setattr(cfg, k, v)
        info = _lib.FrontierInfo()
        self._check(self._L.tloam_b200_frontier_search(self._h, C.byref(cfg), C.byref(info)), "frontier_search")
        recs = (_lib.FrontierRecord * max(info.kept, 1))()
        self._check(self._L.tloam_b200_frontier_download(self._h, recs, info.kept), "frontier_download")
        offsets = np.zeros(info.kept + 1, dtype=np.uintp)
        m = sum(recs[k].size for k in range(info.kept))
        ij = np.zeros((m, 2), dtype=np.int32)
        xy = np.zeros((m, 2))
        self._check(self._L.tloam_b200_frontier_cells(self._h, offsets.ctypes.data_as(C.POINTER(C.c_size_t)),
                                                      ij.ctypes.data_as(C.POINTER(C.c_int)), _dp(xy), m), "frontier_cells")
        out = []
        for k in range(info.kept):
            r = recs[k]
            a, b = int(offsets[k]), int(offsets[k + 1])
            out.append(Frontier(r.id, r.size, (r.sum_i, r.sum_j), (r.min_i, r.min_j, r.max_i, r.max_j),
                                (r.centroid_x, r.centroid_y), (r.approach_i, r.approach_j), (r.approach_x, r.approach_y),
                                r.approach_potential, r.status, r.distance, r.cost, ij[a:b], xy[a:b]))
        self._frontier_shape = (info.height, info.width)
        return {name: getattr(info, name) for name, _ in info._fields_}, out

    def frontier_labels(self):
        """the last frontier_search's label of every cell, (height, width) uint32: its frontier's id before the filter,
        0xFFFFFFFF elsewhere"""
        shape = getattr(self, "_frontier_shape", (0, 0))
        lab = np.zeros(shape, dtype=np.uint32)
        self._check(self._L.tloam_b200_frontier_labels(self._h, lab.ctypes.data_as(C.POINTER(C.c_uint)), lab.size),
                    "frontier_labels")
        return lab

    def localize_set_map_updated(self):
        """load the last map_update_build on the device as the prior map"""
        self._check(self._L.tloam_b200_localize_set_map_updated(self._h), "localize_set_map_updated")

    def loop_descriptors(self, first=0, count=None):
        """the descriptor slots of loop frames [first, first + count) in one copy (count None: to the last), count x slot:
        what relocalize_set_places takes"""
        R, S = self._loop_shape
        if count is None:
            count = self.loop_size() - first
        out = np.zeros((count, R * S + R + S))
        self._check(self._L.tloam_b200_loop_descriptors_download(self._h, int(first), int(count), _dp(out) if count else None),
                    "loop_descriptors_download")
        return out

    # ---- shared map (multi-GPU) ----
    def map_blob_size(self):
        n = C.c_size_t(0)
        self._check(self._L.tloam_b200_map_blob_size(self._h, C.byref(n)), "map_blob_size")
        return n.value

    def map_export(self, dev_ptr, nbytes):
        self._check(self._L.tloam_b200_map_export(self._h, C.c_void_p(dev_ptr), nbytes), "map_export")

    def map_import(self, dev_ptr, nbytes):
        self._check(self._L.tloam_b200_map_import(self._h, C.c_void_p(dev_ptr), nbytes), "map_import")

    def map_send_buffer(self):
        p, n = C.c_void_p(), C.c_size_t(0)
        self._check(self._L.tloam_b200_map_send_buffer(self._h, C.byref(p), C.byref(n)), "map_send_buffer")
        return p.value, n.value

    def map_recv_buffer(self, n_map):
        ns = (C.c_size_t * 4)(*[int(v) for v in n_map])
        p, n = C.c_void_p(), C.c_size_t(0)
        self._check(self._L.tloam_b200_map_recv_buffer(self._h, ns, C.byref(p), C.byref(n)), "map_recv_buffer")
        return p.value, n.value

    def map_adopt(self, producer_stream):
        self._check(self._L.tloam_b200_map_adopt(self._h, C.c_void_p(int(producer_stream))), "map_adopt")

    def signal_stream(self, consumer_stream):
        self._check(self._L.tloam_b200_signal_stream(self._h, C.c_void_p(int(consumer_stream))), "signal_stream")

    def map_origin(self):
        o = np.zeros(3)
        self._check(self._L.tloam_b200_get_map_origin(self._h, _dp(o)), "map_origin")
        return o

    # ---- piecewise (parity tests) ----
    def knn(self, cloud, queries, radius, k):
        q = _f64(queries).reshape(-1, 3)
        nq = q.shape[0]
        idx = np.full((nq, k), -1, dtype=np.int32)
        d2 = np.full((nq, k), np.inf)
        cnt = np.zeros(nq, dtype=np.int32)
        rc = self._L.tloam_b200_knn(self._h, cloud, _dp(q), nq, float(radius), int(k),
                                    idx.ctypes.data_as(C.POINTER(C.c_int)), _dp(d2),
                                    cnt.ctypes.data_as(C.POINTER(C.c_int)))
        self._check(rc, "knn")
        return idx, d2, cnt

    def build_factors(self, cloud, x):
        n = self.n_source[cloud]
        valid = np.zeros(n, dtype=np.int32)
        prim = np.zeros((n, 6))
        x = _f64(x)
        rc = self._L.tloam_b200_build_factors(self._h, cloud, _dp(x), valid.ctypes.data_as(C.POINTER(C.c_int)),
                                              _dp(prim), n)
        self._check(rc, "build_factors")
        return valid, prim

    def eval_point_to_point(self, x, p, q, w):
        x, p, q, w = _f64(x), _f64(p).reshape(-1, 3), _f64(q).reshape(-1, 3), _f64(w).reshape(-1)
        m = p.shape[0]
        r, J, c = np.zeros((m, 3)), np.zeros((m, 3, 6)), np.zeros(m)
        self._check(self._L.tloam_b200_eval_point_to_point(self._h, _dp(x), m, _dp(p), _dp(q), _dp(w), _dp(r), _dp(J), _dp(c)),
                    "eval_point_to_point")
        return r, J, c

    def eval_point_to_line(self, x, p, a, b, w):
        x, p, a, b, w = _f64(x), _f64(p).reshape(-1, 3), _f64(a).reshape(-1, 3), _f64(b).reshape(-1, 3), _f64(w).reshape(-1)
        m = p.shape[0]
        r, J, c = np.zeros((m, 3)), np.zeros((m, 3, 6)), np.zeros(m)
        self._check(self._L.tloam_b200_eval_point_to_line(self._h, _dp(x), m, _dp(p), _dp(a), _dp(b), _dp(w), _dp(r), _dp(J), _dp(c)),
                    "eval_point_to_line")
        return r, J, c

    def eval_point_to_plane(self, x, p, n, d, w):
        x, p, n, d, w = _f64(x), _f64(p).reshape(-1, 3), _f64(n).reshape(-1, 3), _f64(d).reshape(-1), _f64(w).reshape(-1)
        m = p.shape[0]
        r, J, c = np.zeros((m, 1)), np.zeros((m, 1, 6)), np.zeros(m)
        self._check(self._L.tloam_b200_eval_point_to_plane(self._h, _dp(x), m, _dp(p), _dp(n), _dp(d), _dp(w), _dp(r), _dp(J), _dp(c)),
                    "eval_point_to_plane")
        return r, J, c

    def se3_exp(self, a):
        a = _f64(a)
        T = np.zeros(16)
        self._check(self._L.tloam_b200_se3_exp(self._h, _dp(a), _dp(T)), "se3_exp")
        return T.reshape(4, 4).T.copy()

    def se3_log(self, T):
        t = _f64(np.asarray(T).T).reshape(16)
        a = np.zeros(6)
        self._check(self._L.tloam_b200_se3_log(self._h, _dp(t), _dp(a)), "se3_log")
        return a

    def min_on_boundary_2d(self, B, g, radius):
        B, g = _f64(B).reshape(4), _f64(g).reshape(2)
        y = np.zeros(2)
        self._check(self._L.tloam_b200_min_on_boundary_2d(self._h, _dp(B), _dp(g), float(radius), _dp(y)), "min_on_boundary_2d")
        return y

    def se3_plus(self, x, d):
        x, d = _f64(x), _f64(d)
        out = np.zeros(6)
        self._check(self._L.tloam_b200_se3_plus(self._h, _dp(x), _dp(d), _dp(out)), "se3_plus")
        return out


class BatchRegistration:
    """S independent sequences registered together (tloam_b200_batch_*): one launch sequence per batch frame.
    `self.seq[i]` is a LocalRegistration view of sequence i (set_input_*, submap_*, get_transform ... per sequence);
    scan_matching() steps all of them.  Per-sequence poses are bit-identical to the un-batched path."""

    def __init__(self, S, config=None, device=0, **overrides):
        self._L = _lib.load()
        self.cfg = config if config is not None else default_config(**overrides)
        self.S = int(S)
        b = C.c_void_p()
        rc = self._L.tloam_b200_batch_create(C.byref(self.cfg), int(device), self.S, C.byref(b))
        if rc != _lib.OK:
            raise RegistrationError(rc, "tloam_b200_batch_create")
        self._b = b
        self.seq = [LocalRegistration(config=self.cfg, _borrowed=self._L.tloam_b200_batch_handle(b, i)) for i in range(self.S)]
        self._keep = {}

    def close(self):
        if getattr(self, "_b", None):
            for r in self.seq:
                r.close()
            self._L.tloam_b200_batch_destroy(self._b)
            self._b = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, where):
        if rc != _lib.OK:
            raise RegistrationError(rc, where, self._L.tloam_b200_batch_last_error(self._b).decode())

    def pack_device(self, per_seq_tensors):
        """Marshal S x 4 CUDA tensors once (outside a timed loop); pass the result to set_input_*_device."""
        flat = [t for seq in per_seq_tensors for t in seq]
        assert len(flat) == 4 * self.S
        ptrs = (C.c_void_p * (4 * self.S))(*[int(t.data_ptr()) for t in flat])
        ns = (C.c_size_t * (4 * self.S))(*[int(t.shape[0]) for t in flat])
        return ptrs, ns, flat

    def pack_host(self, per_seq_clouds):
        flat = [_f64(c).reshape(-1, 3) for seq in per_seq_clouds for c in seq]
        assert len(flat) == 4 * self.S
        ptrs = (C.POINTER(C.c_double) * (4 * self.S))(*[_dp(a) for a in flat])
        ns = (C.c_size_t * (4 * self.S))(*[a.shape[0] for a in flat])
        return ptrs, ns, flat

    def _set(self, fn, packed, what):
        ptrs, ns, flat = packed
        self._check(fn(self._b, ptrs, ns), what)
        self._keep[what] = flat            # device inputs are read in place: keep them alive until replaced
        if what.startswith("source"):
            for i, r in enumerate(self.seq):
                r.n_source = [int(ns[4 * i + c]) for c in range(4)]

    def set_input_target_device(self, packed):
        self._set(self._L.tloam_b200_batch_set_target_device, packed, "target_device")

    def set_input_source_device(self, packed):
        self._set(self._L.tloam_b200_batch_set_source_device, packed, "source_device")

    def set_input_target(self, packed):
        self._set(self._L.tloam_b200_batch_set_target, packed, "target")

    def set_input_source(self, packed):
        self._set(self._L.tloam_b200_batch_set_source, packed, "source")

    def scan_matching(self, predicts=None):
        """predicts: (S,4,4) or None (device-side constant-velocity prediction).  Returns (S,4,4) poses, statuses."""
        out = np.zeros((self.S, 16))
        st = np.zeros(self.S, dtype=np.int32)
        p = None
        if predicts is not None:
            p = _f64(np.transpose(np.asarray(predicts).reshape(self.S, 4, 4), (0, 2, 1))).reshape(-1)
        rc = self._L.tloam_b200_batch_scan_match(self._b, _dp(p) if p is not None else None, _dp(out),
                                                 st.ctypes.data_as(C.POINTER(C.c_int)))
        self._check(rc, "batch_scan_matching")
        return np.transpose(out.reshape(self.S, 4, 4), (0, 2, 1)).copy(), st

    def scan_matching_async(self, predicts=None):
        """Enqueue only (several BatchRegistration objects can be in flight on one GPU: their serial solver tails then
        overlap with the others' parallel phases); fetch with get_results()."""
        p = None
        if predicts is not None:
            p = _f64(np.transpose(np.asarray(predicts).reshape(self.S, 4, 4), (0, 2, 1))).reshape(-1)
            self._keep["predicts"] = p
        self._check(self._L.tloam_b200_batch_scan_match_async(self._b, _dp(p) if p is not None else None), "batch_scan_matching_async")

    def get_results(self):
        out = np.zeros((self.S, 16))
        st = np.zeros(self.S, dtype=np.int32)
        rc = self._L.tloam_b200_batch_get_results(self._b, _dp(out), st.ctypes.data_as(C.POINTER(C.c_int)), None)
        self._check(rc, "batch_get_results")
        return np.transpose(out.reshape(self.S, 4, 4), (0, 2, 1)).copy(), st

    def launch_count(self):
        return int(self._L.tloam_b200_batch_launch_count(self._b))

    def set_profiling(self, on):
        self._check(self._L.tloam_b200_batch_set_profiling(self._b, 1 if on else 0), "batch_set_profiling")

    def get_profile(self):
        p = _lib.Profile()
        self._check(self._L.tloam_b200_batch_get_profile(self._b, C.byref(p)), "batch_get_profile")
        return {k: (int(p.launches[i]), float(p.total_ms[i])) for i, k in enumerate(_lib.KERNEL_CLASSES)}
