"""ctypes loader for libtloam_b200.so (the C-ABI CUDA library). Fails loudly: there is no CPU fallback."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# TLOAM_B200_LIB: alternative build of the same library (A/B experiments with -D variants); never a different backend
LIB_PATH = os.environ.get("TLOAM_B200_LIB") or os.path.join(HERE, "libtloam_b200.so")

MAX_OUTER = 16
MAX_INNER = 8

(OK, ERR_INVALID_ARG, ERR_TOO_FEW_POINTS, ERR_BAD_POSE, ERR_CUDA, ERR_NO_DEVICE, ERR_NOT_READY, ERR_NUMERIC, ERR_MAP_DENSITY,
 ERR_VOXEL_RANGE) = range(10)


class TlsConfig(C.Structure):
    """tloam_tls_config (include/tloam_b200.h) = the YAML "TLS:" block of the reference."""
    _fields_ = [
        ("k_corr", C.c_int), ("factor_num", C.c_int),
        ("edge_dist_thres", C.c_double), ("sphere_dist_thres", C.c_double),
        ("planar_dist_thres", C.c_double), ("ground_dist_thres", C.c_double),
        ("edge_dir_thres", C.c_double),
        ("edge_maxnum", C.c_int), ("sphere_maxnum", C.c_int), ("planar_maxnum", C.c_int), ("ground_maxnum", C.c_int),
        ("max_iterations", C.c_int),
        ("cost_threshold", C.c_double), ("gnc_factor", C.c_double), ("noise_bound", C.c_double),
        ("fitness_thres", C.c_double),
        ("ceres_max_num_iterations", C.c_int),
        ("reinit_dir", C.c_double * 3),
        ("initial_trust_region_radius", C.c_double),
    ]


class SubmapConfig(C.Structure):
    """tloam_submap_config (ref: config/mapping/lidar_odometry.yaml:6-17)."""
    _fields_ = [("ground_down_sample", C.c_double), ("ground_down_sample_submap", C.c_double),
                ("edge_down_sample_submap", C.c_double), ("planar_frame_size", C.c_int), ("sphere_frame_size", C.c_int),
                ("edge_crop_box_length", C.c_double), ("ground_crop_box_length", C.c_double)]


class GlobalMapConfig(C.Structure):
    """tloam_global_map_config (the reference's global map: front_end.cpp:269-274, VoxelDownSample(1.0))."""
    _fields_ = [("voxel", C.c_double), ("initial_capacity_points", C.c_size_t)]


class PackedScan(C.Structure):
    """tloam_packed_scan (include/tloam_b200.h): n little-endian records of point_step bytes with FLOAT32 x / y / z (and
    intensity, or intensity_offset -1) fields.  Build one with tloam_b200.packed_scan."""
    _fields_ = [("data", C.c_void_p), ("n", C.c_size_t), ("point_step", C.c_size_t), ("x_offset", C.c_int), ("y_offset", C.c_int),
                ("z_offset", C.c_int), ("intensity_offset", C.c_int)]


class PackedTime(C.Structure):
    """tloam_packed_time (include/tloam_b200.h): the time field of a tloam_packed_scan record (PointField datatype 6 UINT32,
    7 FLOAT32 or 8 FLOAT64, times unit).  Build one with tloam_b200.packed_time."""
    _fields_ = [("offset", C.c_int), ("datatype", C.c_int), ("unit", C.c_double)]


class LoopConfig(C.Structure):
    """tloam_loop_config (include/tloam_b200.h "Loop closure"): Scan Context's parameters and the database's first capacity."""
    _fields_ = [("lidar_height", C.c_double), ("n_ring", C.c_int), ("n_sector", C.c_int), ("max_radius", C.c_double),
                ("exclude_recent", C.c_int), ("dist_threshold", C.c_double), ("initial_capacity_frames", C.c_size_t)]


class LoopResult(C.Structure):
    """tloam_loop_result: the newest add's best earlier frame (candidate -1: none eligible)."""
    _fields_ = [("query", C.c_longlong), ("candidate", C.c_longlong), ("shift", C.c_int), ("is_loop", C.c_int),
                ("yaw", C.c_double), ("distance", C.c_double)]


class LoopVerifyConfig(C.Structure):
    """tloam_loop_verify_config (include/tloam_b200.h "Loop verification"): the keyframe voxel and the ICP's schedule."""
    _fields_ = [("voxel", C.c_double), ("corr_dist_coarse", C.c_double), ("corr_dist_fine", C.c_double),
                ("max_iterations", C.c_int), ("eps_translation", C.c_double), ("eps_rotation", C.c_double),
                ("max_fitness", C.c_double), ("initial_capacity_points", C.c_size_t)]


class LoopVerifySubmapConfig(C.Structure):
    """tloam_loop_verify_submap_config (include/tloam_b200.h "Loop verification against a submap")."""
    _fields_ = [("half_window", C.c_int), ("normal_radius", C.c_double), ("min_normal_neighbours", C.c_int),
                ("max_planarity", C.c_double), ("corr_dist_coarse", C.c_double), ("corr_dist_fine", C.c_double),
                ("max_iterations", C.c_int), ("eps_translation", C.c_double), ("eps_rotation", C.c_double),
                ("max_fitness", C.c_double)]


class GlobalMapDynamicConfig(C.Structure):
    """tloam_global_map_dynamic_config (include/tloam_b200.h "Dynamic-point removal")."""
    _fields_ = [("n_rows", C.c_int), ("fov_up", C.c_double), ("fov_down", C.c_double), ("n_cols", C.c_int),
                ("window_rows", C.c_int), ("window_cols", C.c_int), ("margin_abs", C.c_double), ("margin_rel", C.c_double),
                ("min_range", C.c_double), ("max_range", C.c_double), ("min_through", C.c_int)]


class LoopVerifyResult(C.Structure):
    """tloam_loop_verify_result: T_cand_query (column-major) and the ICP's verdict."""
    _fields_ = [("query", C.c_longlong), ("candidate", C.c_longlong), ("T", C.c_double * 16), ("fitness", C.c_double),
                ("rmse", C.c_double), ("inliers", C.c_longlong), ("n_query_points", C.c_longlong),
                ("n_candidate_points", C.c_longlong), ("iterations", C.c_int), ("termination", C.c_int), ("accepted", C.c_int)]


class LocalizeConfig(C.Structure):
    """tloam_localize_config (include/tloam_b200.h "Localization in a prior map")."""
    _fields_ = [("voxel", C.c_double), ("cell", C.c_double), ("normal_radius", C.c_double),
                ("min_normal_neighbours", C.c_int), ("max_planarity", C.c_double), ("corr_dist_coarse", C.c_double),
                ("corr_dist_fine", C.c_double), ("max_iterations", C.c_int), ("eps_translation", C.c_double),
                ("eps_rotation", C.c_double), ("max_fitness", C.c_double)]


class LocalizeResult(C.Structure):
    """tloam_localize_result: T (map <- sensor), T_map_odom and the guess (column-major), and the ICP's verdict."""
    _fields_ = [("T", C.c_double * 16), ("T_map_odom", C.c_double * 16), ("guess", C.c_double * 16),
                ("iterations", C.c_int), ("termination", C.c_int), ("accepted", C.c_int), ("inliers", C.c_longlong),
                ("rmse", C.c_double), ("fitness", C.c_double), ("n_query_points", C.c_longlong),
                ("n_map_points", C.c_longlong)]


class RelocalizeConfig(C.Structure):
    """tloam_relocalize_config (include/tloam_b200.h "Relocalization in a prior map")."""
    _fields_ = [("lidar_height", C.c_double), ("n_ring", C.c_int), ("n_sector", C.c_int), ("max_radius", C.c_double),
                ("top_k", C.c_int), ("max_distance", C.c_double), ("distinct_translation", C.c_double),
                ("distinct_rotation", C.c_double), ("ambiguity_ratio", C.c_double)]


class RelocalizeHypothesis(C.Structure):
    """tloam_relocalize_hypothesis: a candidate place, its shift and distance, and its run."""
    _fields_ = [("place", C.c_longlong), ("shift", C.c_int), ("distance", C.c_double), ("result", LocalizeResult)]


class RelocalizeResult(C.Structure):
    """tloam_relocalize_result: the winner's run, its place, and the selection."""
    _fields_ = [("result", LocalizeResult), ("place", C.c_longlong), ("shift", C.c_int), ("distance", C.c_double),
                ("n_hypotheses", C.c_int), ("winner", C.c_int), ("ambiguous", C.c_int), ("accepted", C.c_int)]


class MapUpdateConfig(C.Structure):
    """tloam_map_update_config (include/tloam_b200.h "Updating a prior map"): the votes' image and the additions' rules."""
    _fields_ = [("image", GlobalMapDynamicConfig), ("novel_radius", C.c_double), ("voxel", C.c_double), ("min_frames", C.c_int)]


class MapUpdateAddResult(C.Structure):
    """tloam_map_update_add_result: whether the add was used, its frame number and the rows it read."""
    _fields_ = [("used", C.c_int), ("frame", C.c_longlong), ("n_scan_points", C.c_longlong), ("n_query_points", C.c_longlong)]


class MapUpdateResult(C.Structure):
    """tloam_map_update_result: the counts of a build."""
    _fields_ = [("n_prior", C.c_longlong), ("n_prior_removed", C.c_longlong), ("n_additions", C.c_longlong),
                ("n_additions_removed", C.c_longlong), ("n_voxels", C.c_longlong), ("n_voxels_kept", C.c_longlong),
                ("n_total", C.c_longlong)]


class OccupancyConfig(C.Structure):
    """tloam_occupancy_config (include/tloam_b200.h "Occupancy grid")."""
    _fields_ = [("resolution", C.c_double), ("n_cols", C.c_int), ("z_lo", C.c_double), ("z_hi", C.c_double),
                ("min_range", C.c_double), ("max_range", C.c_double), ("free_margin", C.c_double)]


class OccupancyInfo(C.Structure):
    """tloam_occupancy_info: the grid's origin, resolution and size, the frames rasterised, the dropped hits and the window
    cells the free pass visited."""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("width", C.c_size_t),
                ("height", C.c_size_t), ("frames", C.c_size_t), ("dropped", C.c_ulonglong), ("cell_tests", C.c_ulonglong)]


class DistanceConfig(C.Structure):
    """tloam_distance_config (include/tloam_b200.h "Distance field and costmap")."""
    _fields_ = [("inscribed_radius", C.c_double), ("inflation_radius", C.c_double), ("cost_scaling_factor", C.c_double)]


class DistanceInfo(C.Structure):
    """tloam_distance_info: the field's origin, resolution and size, and its obstacle cells."""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("width", C.c_size_t),
                ("height", C.c_size_t), ("obstacles", C.c_size_t)]


class PlanConfig(C.Structure):
    """tloam_plan_config (include/tloam_b200.h "Path planning")."""
    _fields_ = [("neutral_cost", C.c_uint), ("cost_factor", C.c_uint), ("allow_unknown", C.c_int)]


class PlanInfo(C.Structure):
    """tloam_plan_info: the plan's origin, resolution and size, its goal cell, reachable cells, rounds and tiles."""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("width", C.c_size_t),
                ("height", C.c_size_t), ("goal_i", C.c_size_t), ("goal_j", C.c_size_t), ("reachable", C.c_size_t),
                ("rounds", C.c_ulonglong), ("tiles", C.c_ulonglong)]


class GlobalRegistrationConfig(C.Structure):
    """tloam_global_registration_config (include/tloam_b200.h "Global registration")."""
    _fields_ = [("voxel", C.c_double), ("cell", C.c_double), ("normal_radius", C.c_double), ("min_normal_neighbours", C.c_int),
                ("feature_radius", C.c_double), ("max_correspondence_distance", C.c_double), ("n_hypotheses", C.c_int),
                ("seed", C.c_ulonglong), ("edge_similarity", C.c_double), ("min_triangle_area", C.c_double),
                ("max_refine_iterations", C.c_int), ("min_inliers", C.c_int), ("min_fitness", C.c_double)]


class GlobalRegistrationResult(C.Structure):
    """tloam_global_registration_result: T (target <- source, column-major), the counts of each stage and the verdict."""
    _fields_ = [("T", C.c_double * 16), ("n_source_points", C.c_longlong), ("n_target_points", C.c_longlong),
                ("n_source_features", C.c_longlong), ("n_target_features", C.c_longlong), ("n_correspondences", C.c_longlong),
                ("n_valid_hypotheses", C.c_int), ("best_hypothesis", C.c_int), ("best_inliers", C.c_int), ("inliers", C.c_int),
                ("inlier_rmse", C.c_double), ("fitness", C.c_double), ("refine_iterations", C.c_int), ("termination", C.c_int),
                ("accepted", C.c_int)]


class FrontierConfig(C.Structure):
    """tloam_frontier_config (include/tloam_b200.h "Frontiers")."""
    _fields_ = [("free_max", C.c_uint), ("min_frontier_size", C.c_double), ("potential_scale", C.c_double),
                ("gain_scale", C.c_double)]


class FrontierRecord(C.Structure):
    """tloam_frontier: one kept frontier of a search."""
    _fields_ = [("id", C.c_uint), ("status", C.c_int), ("size", C.c_size_t), ("sum_i", C.c_ulonglong),
                ("sum_j", C.c_ulonglong), ("min_i", C.c_size_t), ("min_j", C.c_size_t), ("max_i", C.c_size_t),
                ("max_j", C.c_size_t), ("centroid_x", C.c_double), ("centroid_y", C.c_double),
                ("approach_i", C.c_size_t), ("approach_j", C.c_size_t), ("approach_x", C.c_double),
                ("approach_y", C.c_double), ("approach_potential", C.c_ulonglong), ("distance", C.c_double),
                ("cost", C.c_double)]


class FrontierInfo(C.Structure):
    """tloam_frontier_info: the grid, the plan's goal cell, the frontier cells, the frontiers before and after the filter
    and the kept reachable ones."""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("width", C.c_size_t),
                ("height", C.c_size_t), ("goal_i", C.c_size_t), ("goal_j", C.c_size_t), ("cells", C.c_size_t),
                ("components", C.c_size_t), ("kept", C.c_size_t), ("reachable", C.c_size_t)]


class TerrainConfig(C.Structure):
    """tloam_terrain_config (include/tloam_b200.h "Terrain"): the grid, the windows and the thresholds."""
    _fields_ = [("resolution", C.c_double), ("clearance", C.c_double), ("ground_radius", C.c_double),
                ("step_radius", C.c_double), ("slope_radius", C.c_double), ("max_step", C.c_double),
                ("max_slope", C.c_double), ("max_roughness", C.c_double), ("min_points", C.c_uint), ("min_fit", C.c_uint),
                ("static_only", C.c_int), ("combine_occupancy", C.c_int)]


class TerrainInfo(C.Structure):
    """tloam_terrain_info: the grid, the radii in cells, the rows' counts, the known and lethal cells"""
    _fields_ = [("origin_x", C.c_double), ("origin_y", C.c_double), ("resolution", C.c_double), ("width", C.c_size_t),
                ("height", C.c_size_t), ("ground_cells", C.c_uint), ("step_cells", C.c_uint), ("slope_cells", C.c_uint),
                ("rows", C.c_size_t), ("used", C.c_size_t), ("skipped", C.c_size_t), ("dropped", C.c_size_t),
                ("overhang", C.c_size_t), ("known", C.c_size_t), ("lethal", C.c_size_t), ("combined", C.c_int)]


class PoseGraphConfig(C.Structure):
    """tloam_pose_graph_config (include/tloam_b200.h "Pose graph"): the edges' sigmas and the Gauss-Newton schedule."""
    _fields_ = [("sigma_odom_translation", C.c_double), ("sigma_odom_rotation", C.c_double),
                ("sigma_loop_translation", C.c_double), ("sigma_loop_rotation", C.c_double), ("max_iterations", C.c_int),
                ("eps_translation", C.c_double), ("eps_rotation", C.c_double), ("max_loop_edges", C.c_size_t),
                ("initial_capacity_nodes", C.c_size_t)]


class PoseGraphResult(C.Structure):
    """tloam_pose_graph_result"""
    _fields_ = [("nodes", C.c_longlong), ("loop_edges", C.c_longlong), ("iterations", C.c_int), ("termination", C.c_int),
                ("initial_cost", C.c_double), ("final_cost", C.c_double), ("step_translation", C.c_double),
                ("step_rotation", C.c_double)]


class PoseGraphRobustConfig(C.Structure):
    """tloam_pose_graph_robust_config (include/tloam_b200.h "Robust pose graph"): the TLS threshold and the GNC schedule."""
    _fields_ = [("chi2_threshold", C.c_double), ("gnc_factor", C.c_double), ("inner_iterations", C.c_int),
                ("max_outer_iterations", C.c_int)]


class PoseGraphRobustResult(C.Structure):
    """tloam_pose_graph_robust_result"""
    _fields_ = [("pg", PoseGraphResult), ("outer_iterations", C.c_int), ("gnc_termination", C.c_int),
                ("mu_final", C.c_double), ("inliers", C.c_longlong), ("rejected", C.c_longlong)]


class InnerTrace(C.Structure):
    _fields_ = [
        ("x_candidate", C.c_double * 6), ("candidate_cost", C.c_double), ("model_cost_change", C.c_double),
        ("relative_decrease", C.c_double), ("step_norm_scaled", C.c_double), ("radius", C.c_double),
        ("accepted", C.c_int), ("used_gauss_newton", C.c_int),
    ]


class OuterTrace(C.Structure):
    _fields_ = [
        ("x_start", C.c_double * 6), ("x_end", C.c_double * 6),
        ("initial_cost", C.c_double), ("final_cost", C.c_double),
        ("H0", C.c_double * 36), ("g0", C.c_double * 6),
        ("mu", C.c_double), ("th1", C.c_double), ("th2", C.c_double),
        ("slot_sum", C.c_double * 4), ("n_factors", C.c_int * 4),
        ("n_inner", C.c_int), ("termination", C.c_int),
        ("inner", InnerTrace * MAX_INNER),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("n_outer", C.c_int), ("converged_early", C.c_int),
        ("x_init", C.c_double * 6), ("x_final", C.c_double * 6),
        ("gpu_launches", C.c_int), ("gpu_ms", C.c_float),
        ("outer", OuterTrace * MAX_OUTER),
    ]


KERNEL_CLASSES = ("map_bbox", "map_origin", "map_insert", "map_offsets", "map_scatter", "stage_source",
                  "begin_frame", "correspond", "eval_first", "eval", "submap", "feature", "first", "dense_bin", "dense", "fitness", "ground", "map_fine", "fine", "edge", "object")


class FeatureConfig(C.Structure):
    """tloam_feature_config (include/tloam_b200.h)."""
    _fields_ = [("radius", C.c_double), ("K", C.c_int), ("min_neigh", C.c_int), ("planar_num", C.c_int),
                ("sphere_num", C.c_int), ("cvr_scan", C.c_double), ("cvr_submap", C.c_double),
                ("planar_scan_thres", C.c_double), ("planar_submap_thres", C.c_double),
                ("planar_vertic_thres", C.c_double)]


class DcvcConfig(C.Structure):
    """tloam_dcvc_config (ref: config/mapping/segmentation.yaml DCVC + velodyne ranges)."""
    _fields_ = [("start_r", C.c_double), ("delta_r", C.c_double), ("delta_p", C.c_double), ("delta_a", C.c_double),
                ("min_seg", C.c_int), ("sensor_min_range", C.c_double), ("sensor_max_range", C.c_double),
                ("min_pitch_init", C.c_double), ("max_pitch_init", C.c_double), ("min_polar_init", C.c_double),
                ("max_polar_init", C.c_double)]


class GroundConfig(C.Structure):
    """tloam_ground_config (ref: config/mapping/segmentation.yaml)."""
    _fields_ = [("sensor_model", C.c_int), ("sensor_height", C.c_double), ("vertical_res", C.c_double), ("init_angle", C.c_double),
                ("sensor_min_range", C.c_double), ("sensor_max_range", C.c_double), ("quadrant", C.c_int), ("num_sec", C.c_int),
                ("plane_dis", C.c_double), ("max_iter", C.c_int), ("ground_seed_num", C.c_int)]


class Profile(C.Structure):
    _fields_ = [("launches", C.c_longlong * len(KERNEL_CLASSES)), ("total_ms", C.c_double * len(KERNEL_CLASSES)),
                ("dbg", C.c_ulonglong * 16)]


EXPORTS = [
    "tloam_b200_default_config", "tloam_b200_status_string", "tloam_b200_last_error", "tloam_b200_create",
    "tloam_b200_destroy", "tloam_b200_set_source", "tloam_b200_set_target", "tloam_b200_set_source_device",
    "tloam_b200_set_target_device", "tloam_b200_scan_match", "tloam_b200_scan_match_async", "tloam_b200_get_result",
    "tloam_b200_fitness", "tloam_b200_get_transform", "tloam_b200_get_pose_increment", "tloam_b200_synchronize",
    "tloam_b200_launch_count", "tloam_b200_map_blob_size", "tloam_b200_map_export", "tloam_b200_map_import",
    "tloam_b200_get_map_origin", "tloam_b200_knn", "tloam_b200_build_factors", "tloam_b200_eval_point_to_point",
    "tloam_b200_eval_point_to_line", "tloam_b200_eval_point_to_plane", "tloam_b200_se3_exp", "tloam_b200_se3_log",
    "tloam_b200_se3_plus", "tloam_b200_min_on_boundary_2d", "tloam_b200_host_alloc", "tloam_b200_host_free", "tloam_b200_set_profiling",
    "tloam_b200_get_profile", "tloam_b200_set_trace", "tloam_b200_submap_default_config", "tloam_b200_submap_init",
    "tloam_b200_submap_update", "tloam_b200_submap_sizes", "tloam_b200_submap_download", "tloam_b200_voxel_down_sample",
    "tloam_b200_scan_match_predicted_async", "tloam_b200_scan_match_predicted", "tloam_b200_set_pose_history",
    "tloam_b200_feature_default_config", "tloam_b200_extract_planar_sphere", "tloam_b200_pca_info",
    "tloam_b200_batch_create", "tloam_b200_batch_destroy", "tloam_b200_batch_size", "tloam_b200_batch_handle",
    "tloam_b200_batch_set_target", "tloam_b200_batch_set_source", "tloam_b200_batch_set_target_device",
    "tloam_b200_batch_set_source_device", "tloam_b200_batch_scan_match", "tloam_b200_batch_scan_match_async",
    "tloam_b200_batch_get_results", "tloam_b200_batch_launch_count", "tloam_b200_batch_last_error",
    "tloam_b200_batch_set_profiling", "tloam_b200_batch_get_profile",
    "tloam_b200_submap_update_chained", "tloam_b200_set_frame_fitness", "tloam_b200_get_frame_fitness",
    "tloam_b200_set_async_inputs", "tloam_b200_wait_stream", "tloam_b200_dense_check_counters",
    "tloam_b200_ground_default_config", "tloam_b200_ground_extract", "tloam_b200_extract_edge", "tloam_b200_dcvc_default_config", "tloam_b200_object_segmentation", "tloam_b200_segment_scan", "tloam_b200_ground_remove", "tloam_b200_segment_raw_scan", "tloam_b200_map_layout_bytes",
    "tloam_b200_map_send_buffer", "tloam_b200_map_recv_buffer", "tloam_b200_map_adopt", "tloam_b200_signal_stream",
    "tloam_b200_process_cloud", "tloam_b200_process_raw_scan", "tloam_b200_source_download", "tloam_b200_submap_init_frame",
    "tloam_b200_submap_update_frame", "tloam_b200_submap_update_frame_chained",
    "tloam_b200_global_map_default_config", "tloam_b200_global_map_enable", "tloam_b200_global_map_reset",
    "tloam_b200_global_map_append", "tloam_b200_global_map_append_chained", "tloam_b200_global_map_append_frame",
    "tloam_b200_global_map_append_frame_chained", "tloam_b200_global_map_size", "tloam_b200_global_map_download",
    "tloam_b200_global_map_frame_offsets", "tloam_b200_global_map_capacity", "tloam_b200_registered_scan_download",
    "tloam_b200_global_map_append_intensity", "tloam_b200_global_map_append_intensity_chained",
    "tloam_b200_global_map_append_frame_intensity", "tloam_b200_global_map_append_frame_intensity_chained",
    "tloam_b200_global_map_has_intensity", "tloam_b200_global_map_intensity_download",
    "tloam_b200_segment_raw_scan_packed", "tloam_b200_process_raw_scan_packed", "tloam_b200_global_map_append_packed",
    "tloam_b200_global_map_append_packed_chained",
    "tloam_b200_process_raw_scan_timed", "tloam_b200_process_raw_scan_packed_timed",
    "tloam_b200_loop_default_config", "tloam_b200_loop_enable", "tloam_b200_loop_reset", "tloam_b200_loop_add_frame",
    "tloam_b200_loop_add", "tloam_b200_loop_result", "tloam_b200_loop_size", "tloam_b200_loop_descriptor_download",
    "tloam_b200_loop_verify_default_config", "tloam_b200_loop_verify_enable", "tloam_b200_loop_keyframe_download",
    "tloam_b200_loop_verify", "tloam_b200_loop_verify_matches",
    "tloam_b200_pose_graph_default_config", "tloam_b200_pose_graph_enable", "tloam_b200_pose_graph_reset",
    "tloam_b200_pose_graph_add_node", "tloam_b200_pose_graph_add_node_chained", "tloam_b200_pose_graph_add_loop",
    "tloam_b200_pose_graph_size", "tloam_b200_pose_graph_optimize", "tloam_b200_pose_graph_download",
    "tloam_b200_pose_graph_correction", "tloam_b200_pose_graph_robust_default_config",
    "tloam_b200_pose_graph_optimize_robust", "tloam_b200_pose_graph_loop_weights",
    "tloam_b200_global_map_correction_enable", "tloam_b200_global_map_correct", "tloam_b200_global_map_frame_poses",
    "tloam_b200_loop_verify_submap_default_config", "tloam_b200_loop_verify_submap_enable", "tloam_b200_loop_verify_submap",
    "tloam_b200_loop_verify_submap_target", "tloam_b200_loop_verify_submap_matches",
    "tloam_b200_global_map_dynamic_default_config", "tloam_b200_global_map_dynamic_enable",
    "tloam_b200_global_map_votes_download", "tloam_b200_global_map_static_download",
    "tloam_b200_global_map_merge", "tloam_b200_global_map_merged_download",
    "tloam_b200_localize_default_config", "tloam_b200_localize_enable", "tloam_b200_localize_set_map",
    "tloam_b200_localize_set_map_merged", "tloam_b200_localize_frame", "tloam_b200_localize", "tloam_b200_localize_matches",
    "tloam_b200_localize_query", "tloam_b200_localize_map_normals", "tloam_b200_localize_cells",
    "tloam_b200_loop_descriptors_download", "tloam_b200_relocalize_default_config", "tloam_b200_relocalize_enable",
    "tloam_b200_relocalize_set_places", "tloam_b200_relocalize_set_places_loop", "tloam_b200_relocalize_frame",
    "tloam_b200_relocalize", "tloam_b200_relocalize_hypotheses", "tloam_b200_relocalize_matches",
    "tloam_b200_map_update_default_config", "tloam_b200_map_update_enable", "tloam_b200_map_update_add",
    "tloam_b200_map_update_build", "tloam_b200_map_update_size", "tloam_b200_map_update_download",
    "tloam_b200_map_update_votes", "tloam_b200_map_update_additions", "tloam_b200_localize_set_map_updated",
    "tloam_b200_occupancy_default_config", "tloam_b200_occupancy_enable", "tloam_b200_occupancy_build",
    "tloam_b200_occupancy_download", "tloam_b200_occupancy_scans_download",
    "tloam_b200_distance_default_config", "tloam_b200_distance_build", "tloam_b200_distance_build_grid",
    "tloam_b200_distance_download", "tloam_b200_distance_query",
    "tloam_b200_plan_default_config", "tloam_b200_plan_build", "tloam_b200_plan_download", "tloam_b200_plan_paths",
    "tloam_b200_plan_path_cells",
    "tloam_b200_frontier_default_config", "tloam_b200_frontier_search", "tloam_b200_frontier_download",
    "tloam_b200_frontier_cells", "tloam_b200_frontier_labels",
    "tloam_b200_terrain_default_config", "tloam_b200_terrain_build", "tloam_b200_terrain_build_cloud",
    "tloam_b200_terrain_download", "tloam_b200_distance_build_terrain",
    "tloam_b200_global_registration_default_config", "tloam_b200_global_registration_enable", "tloam_b200_global_register",
    "tloam_b200_global_register_loop", "tloam_b200_global_registration_side", "tloam_b200_global_registration_correspondences",
    "tloam_b200_global_registration_hypotheses",
]

_lib = None


def load():
    """Load the CUDA library. Raises if it has not been built (python -m tloam_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: build it with `python -m tloam_b200.build` "
                           "(there is no CPU fallback for the registration path)")
    L = C.CDLL(LIB_PATH)
    dp = C.POINTER(C.c_double)
    ip = C.POINTER(C.c_int)
    vp = C.c_void_p
    L.tloam_b200_default_config.argtypes = [C.POINTER(TlsConfig)]
    L.tloam_b200_default_config.restype = None
    L.tloam_b200_status_string.argtypes = [C.c_int]
    L.tloam_b200_status_string.restype = C.c_char_p
    L.tloam_b200_last_error.argtypes = [vp]
    L.tloam_b200_last_error.restype = C.c_char_p
    L.tloam_b200_create.argtypes = [C.POINTER(TlsConfig), C.c_int, vp, C.POINTER(vp)]
    L.tloam_b200_destroy.argtypes = [vp]
    for name in ("set_source", "set_target"):
        f = getattr(L, "tloam_b200_" + name)
        f.argtypes = [vp, C.POINTER(dp), C.POINTER(C.c_size_t)]
    for name in ("set_source_device", "set_target_device"):
        f = getattr(L, "tloam_b200_" + name)
        f.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.tloam_b200_scan_match.argtypes = [vp, dp, dp, C.POINTER(Stats)]
    L.tloam_b200_scan_match_async.argtypes = [vp, dp]
    L.tloam_b200_get_result.argtypes = [vp, dp, C.POINTER(Stats)]
    L.tloam_b200_scan_match_predicted_async.argtypes = [vp]
    L.tloam_b200_scan_match_predicted.argtypes = [vp, dp, C.POINTER(Stats)]
    L.tloam_b200_set_pose_history.argtypes = [vp, dp, dp]
    L.tloam_b200_fitness.argtypes = [vp, dp, dp]
    L.tloam_b200_get_transform.argtypes = [vp, dp]
    L.tloam_b200_get_pose_increment.argtypes = [vp, dp]
    L.tloam_b200_synchronize.argtypes = [vp]
    L.tloam_b200_launch_count.argtypes = [vp]
    L.tloam_b200_launch_count.restype = C.c_longlong
    L.tloam_b200_map_blob_size.argtypes = [vp, C.POINTER(C.c_size_t)]
    L.tloam_b200_map_export.argtypes = [vp, vp, C.c_size_t]
    L.tloam_b200_map_import.argtypes = [vp, vp, C.c_size_t]
    L.tloam_b200_get_map_origin.argtypes = [vp, dp]
    L.tloam_b200_knn.argtypes = [vp, C.c_int, dp, C.c_size_t, C.c_double, C.c_int, ip, dp, ip]
    L.tloam_b200_build_factors.argtypes = [vp, C.c_int, dp, ip, dp, C.c_size_t]
    L.tloam_b200_eval_point_to_point.argtypes = [vp, dp, C.c_size_t, dp, dp, dp, dp, dp, dp]
    L.tloam_b200_eval_point_to_line.argtypes = [vp, dp, C.c_size_t, dp, dp, dp, dp, dp, dp, dp]
    L.tloam_b200_eval_point_to_plane.argtypes = [vp, dp, C.c_size_t, dp, dp, dp, dp, dp, dp, dp]
    L.tloam_b200_se3_exp.argtypes = [vp, dp, dp]
    L.tloam_b200_se3_log.argtypes = [vp, dp, dp]
    L.tloam_b200_se3_plus.argtypes = [vp, dp, dp, dp]
    L.tloam_b200_min_on_boundary_2d.argtypes = [vp, dp, dp, C.c_double, dp]
    L.tloam_b200_host_alloc.argtypes = [C.POINTER(vp), C.c_size_t]
    L.tloam_b200_host_free.argtypes = [vp]
    L.tloam_b200_set_profiling.argtypes = [vp, C.c_int]
    L.tloam_b200_get_profile.argtypes = [vp, C.POINTER(Profile)]
    L.tloam_b200_set_trace.argtypes = [vp, C.c_int]
    L.tloam_b200_submap_default_config.argtypes = [C.POINTER(SubmapConfig)]
    L.tloam_b200_submap_default_config.restype = None
    L.tloam_b200_submap_init.argtypes = [vp, C.POINTER(SubmapConfig), dp, C.c_size_t, dp, C.c_size_t, dp, C.c_size_t, dp, C.c_size_t]
    L.tloam_b200_submap_update.argtypes = [vp, dp, dp, C.c_size_t, dp, C.c_size_t]
    L.tloam_b200_submap_sizes.argtypes = [vp, C.POINTER(C.c_size_t)]
    L.tloam_b200_submap_download.argtypes = [vp, C.c_int, dp, C.c_size_t]
    L.tloam_b200_voxel_down_sample.argtypes = [vp, dp, C.c_size_t, C.c_double, dp, C.POINTER(C.c_size_t)]
    szp = C.POINTER(C.c_size_t)
    L.tloam_b200_feature_default_config.argtypes = [C.POINTER(FeatureConfig)]
    L.tloam_b200_feature_default_config.restype = None
    L.tloam_b200_extract_planar_sphere.argtypes = [vp, C.POINTER(FeatureConfig), dp, C.c_size_t, szp, szp, szp, szp, szp,
                                                   szp, szp, szp, szp]
    L.tloam_b200_pca_info.argtypes = [vp, C.POINTER(FeatureConfig), dp, C.c_size_t, dp, dp, dp, dp,
                                      C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.tloam_b200_batch_create.argtypes = [C.POINTER(TlsConfig), C.c_int, C.c_int, C.POINTER(vp)]
    L.tloam_b200_batch_destroy.argtypes = [vp]
    L.tloam_b200_batch_size.argtypes = [vp]
    L.tloam_b200_batch_handle.argtypes = [vp, C.c_int]
    L.tloam_b200_batch_handle.restype = vp
    for name in ("set_target", "set_source"):
        getattr(L, "tloam_b200_batch_" + name).argtypes = [vp, C.POINTER(dp), szp]
        getattr(L, "tloam_b200_batch_" + name + "_device").argtypes = [vp, C.POINTER(vp), szp]
    L.tloam_b200_batch_scan_match.argtypes = [vp, dp, dp, ip]
    L.tloam_b200_batch_scan_match_async.argtypes = [vp, dp]
    L.tloam_b200_batch_get_results.argtypes = [vp, dp, ip, C.POINTER(C.c_float)]
    L.tloam_b200_batch_launch_count.argtypes = [vp]
    L.tloam_b200_batch_launch_count.restype = C.c_longlong
    L.tloam_b200_batch_last_error.argtypes = [vp]
    L.tloam_b200_batch_last_error.restype = C.c_char_p
    L.tloam_b200_batch_set_profiling.argtypes = [vp, C.c_int]
    L.tloam_b200_submap_update_chained.argtypes = [vp, dp, C.c_size_t]
    L.tloam_b200_set_frame_fitness.argtypes = [vp, C.c_int]
    L.tloam_b200_get_frame_fitness.argtypes = [vp, dp, dp]
    L.tloam_b200_set_async_inputs.argtypes = [vp, C.c_int]
    L.tloam_b200_wait_stream.argtypes = [vp, vp]
    L.tloam_b200_dense_check_counters.argtypes = [vp, C.POINTER(C.c_uint)]
    L.tloam_b200_map_layout_bytes.argtypes = [vp, szp, szp]
    L.tloam_b200_map_send_buffer.argtypes = [vp, C.POINTER(vp), szp]
    L.tloam_b200_map_recv_buffer.argtypes = [vp, szp, C.POINTER(vp), szp]
    L.tloam_b200_map_adopt.argtypes = [vp, vp]
    L.tloam_b200_signal_stream.argtypes = [vp, vp]
    L.tloam_b200_ground_default_config.argtypes = [C.POINTER(GroundConfig)]
    L.tloam_b200_ground_default_config.restype = None
    L.tloam_b200_ground_extract.argtypes = [vp, C.POINTER(GroundConfig), dp, C.c_size_t, szp, szp, szp, szp, ip, ip, dp, dp]
    L.tloam_b200_ground_remove.argtypes = [vp, C.POINTER(GroundConfig), dp, C.c_size_t, szp, szp, szp, szp, dp, ip, dp, dp]
    L.tloam_b200_extract_edge.argtypes = [vp, C.c_int, C.c_int, dp, dp, C.c_size_t, szp, szp, szp, szp]
    L.tloam_b200_dcvc_default_config.argtypes = [C.POINTER(DcvcConfig)]
    L.tloam_b200_dcvc_default_config.restype = None
    L.tloam_b200_object_segmentation.argtypes = [vp, C.POINTER(DcvcConfig), dp, C.c_size_t, szp, szp, ip, ip, dp, ip, ip, ip, dp]
    L.tloam_b200_segment_scan.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, dp, C.c_size_t, szp, szp, szp, szp, szp, szp,
                                          ip, ip, dp, ip]
    L.tloam_b200_segment_raw_scan.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, C.c_double, dp, C.c_size_t, szp, szp,
                                              szp, szp, szp, szp, ip, ip, dp, dp]
    L.tloam_b200_batch_get_profile.argtypes = [vp, C.POINTER(Profile)]
    L.tloam_b200_process_cloud.argtypes = [vp, C.POINTER(FeatureConfig), C.c_double, C.c_double, dp, C.c_size_t, dp, C.c_size_t, dp,
                                           C.c_size_t, szp]
    L.tloam_b200_process_raw_scan.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, C.c_double,
                                              C.POINTER(FeatureConfig), C.c_double, C.c_double, dp, C.c_size_t, szp]
    L.tloam_b200_source_download.argtypes = [vp, C.c_int, dp, C.c_size_t]
    L.tloam_b200_submap_init_frame.argtypes = [vp, C.POINTER(SubmapConfig)]
    L.tloam_b200_submap_update_frame.argtypes = [vp, dp]
    L.tloam_b200_submap_update_frame_chained.argtypes = [vp]
    L.tloam_b200_global_map_default_config.argtypes = [C.POINTER(GlobalMapConfig)]
    L.tloam_b200_global_map_default_config.restype = None
    L.tloam_b200_global_map_enable.argtypes = [vp, C.POINTER(GlobalMapConfig)]
    L.tloam_b200_global_map_reset.argtypes = [vp]
    L.tloam_b200_global_map_append.argtypes = [vp, dp, dp, C.c_size_t]
    L.tloam_b200_global_map_append_chained.argtypes = [vp, dp, C.c_size_t]
    L.tloam_b200_global_map_append_frame.argtypes = [vp, dp]
    L.tloam_b200_global_map_append_frame_chained.argtypes = [vp]
    L.tloam_b200_global_map_size.argtypes = [vp, szp, szp]
    L.tloam_b200_global_map_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp]
    L.tloam_b200_global_map_frame_offsets.argtypes = [vp, szp, C.c_size_t]
    L.tloam_b200_global_map_capacity.argtypes = [vp, szp, szp]
    L.tloam_b200_registered_scan_download.argtypes = [vp, dp, C.c_size_t, szp]
    L.tloam_b200_global_map_append_intensity.argtypes = [vp, dp, dp, dp, C.c_size_t]
    L.tloam_b200_global_map_append_intensity_chained.argtypes = [vp, dp, dp, C.c_size_t]
    L.tloam_b200_global_map_append_frame_intensity.argtypes = [vp, dp, dp]
    L.tloam_b200_global_map_append_frame_intensity_chained.argtypes = [vp, dp]
    L.tloam_b200_global_map_has_intensity.argtypes = [vp, C.POINTER(C.c_int)]
    L.tloam_b200_global_map_intensity_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp]
    pk = C.POINTER(PackedScan)
    L.tloam_b200_segment_raw_scan_packed.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, C.c_double, pk, szp,
                                                     szp, szp, szp, szp, szp, ip, ip, dp, dp]
    L.tloam_b200_process_raw_scan_packed.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, C.c_double,
                                                     C.POINTER(FeatureConfig), C.c_double, C.c_double, pk, szp]
    L.tloam_b200_global_map_append_packed.argtypes = [vp, dp, pk]
    L.tloam_b200_global_map_append_packed_chained.argtypes = [vp, pk]
    L.tloam_b200_process_raw_scan_timed.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, C.c_double,
                                                    C.POINTER(FeatureConfig), C.c_double, C.c_double, dp, dp, C.c_size_t, C.c_double,
                                                    szp]
    L.tloam_b200_process_raw_scan_packed_timed.argtypes = [vp, C.POINTER(GroundConfig), C.POINTER(DcvcConfig), C.c_int, C.c_double,
                                                           C.POINTER(FeatureConfig), C.c_double, C.c_double, pk,
                                                           C.POINTER(PackedTime), C.c_double, szp]
    L.tloam_b200_loop_default_config.argtypes = [C.POINTER(LoopConfig)]
    L.tloam_b200_loop_default_config.restype = None
    L.tloam_b200_loop_enable.argtypes = [vp, C.POINTER(LoopConfig)]
    L.tloam_b200_loop_reset.argtypes = [vp]
    L.tloam_b200_loop_add_frame.argtypes = [vp]
    L.tloam_b200_loop_add.argtypes = [vp, dp, C.c_size_t]
    L.tloam_b200_loop_result.argtypes = [vp, C.POINTER(LoopResult)]
    L.tloam_b200_loop_size.argtypes = [vp, szp]
    L.tloam_b200_loop_descriptor_download.argtypes = [vp, C.c_size_t, dp]
    L.tloam_b200_loop_verify_default_config.argtypes = [C.POINTER(LoopVerifyConfig)]
    L.tloam_b200_loop_verify_default_config.restype = None
    L.tloam_b200_loop_verify_enable.argtypes = [vp, C.POINTER(LoopVerifyConfig)]
    L.tloam_b200_loop_keyframe_download.argtypes = [vp, C.c_size_t, dp, C.c_size_t, szp]
    L.tloam_b200_loop_verify.argtypes = [vp, C.c_longlong, C.c_longlong, dp, C.POINTER(LoopVerifyResult)]
    L.tloam_b200_loop_verify_matches.argtypes = [vp, C.c_int, C.POINTER(C.c_int), dp, C.c_size_t, szp]
    L.tloam_b200_pose_graph_default_config.argtypes = [C.POINTER(PoseGraphConfig)]
    L.tloam_b200_pose_graph_default_config.restype = None
    L.tloam_b200_pose_graph_enable.argtypes = [vp, C.POINTER(PoseGraphConfig)]
    L.tloam_b200_pose_graph_reset.argtypes = [vp]
    L.tloam_b200_pose_graph_add_node.argtypes = [vp, dp]
    L.tloam_b200_pose_graph_add_node_chained.argtypes = [vp]
    L.tloam_b200_pose_graph_add_loop.argtypes = [vp, C.POINTER(LoopVerifyResult)]
    L.tloam_b200_pose_graph_size.argtypes = [vp, szp, szp]
    L.tloam_b200_pose_graph_optimize.argtypes = [vp, C.POINTER(PoseGraphResult)]
    L.tloam_b200_pose_graph_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp]
    L.tloam_b200_pose_graph_correction.argtypes = [vp, dp]
    L.tloam_b200_pose_graph_robust_default_config.argtypes = [C.POINTER(PoseGraphRobustConfig)]
    L.tloam_b200_pose_graph_robust_default_config.restype = None
    L.tloam_b200_pose_graph_optimize_robust.argtypes = [vp, C.POINTER(PoseGraphRobustConfig), C.POINTER(PoseGraphRobustResult)]
    L.tloam_b200_pose_graph_loop_weights.argtypes = [vp, C.c_size_t, C.c_size_t, dp]
    L.tloam_b200_global_map_correction_enable.argtypes = [vp]
    L.tloam_b200_global_map_correct.argtypes = [vp, C.POINTER(C.c_longlong), C.c_size_t]
    L.tloam_b200_global_map_frame_poses.argtypes = [vp, C.c_size_t, C.c_size_t, dp, dp]
    L.tloam_b200_loop_verify_submap_default_config.argtypes = [C.POINTER(LoopVerifySubmapConfig)]
    L.tloam_b200_loop_verify_submap_default_config.restype = None
    L.tloam_b200_loop_verify_submap_enable.argtypes = [vp, C.POINTER(LoopVerifySubmapConfig)]
    L.tloam_b200_loop_verify_submap.argtypes = [vp, C.c_longlong, C.c_longlong, dp, dp, C.POINTER(LoopVerifyResult)]
    L.tloam_b200_loop_verify_submap_target.argtypes = [vp, dp, dp, C.POINTER(C.c_ubyte), C.POINTER(C.c_int), C.c_size_t, szp]
    L.tloam_b200_loop_verify_submap_matches.argtypes = [vp, C.c_int, C.POINTER(C.c_int), dp, C.c_size_t, szp]
    L.tloam_b200_global_map_dynamic_default_config.argtypes = [C.POINTER(GlobalMapDynamicConfig)]
    L.tloam_b200_global_map_dynamic_default_config.restype = None
    L.tloam_b200_global_map_dynamic_enable.argtypes = [vp, C.POINTER(GlobalMapDynamicConfig)]
    up = C.POINTER(C.c_uint)
    L.tloam_b200_global_map_votes_download.argtypes = [vp, C.c_size_t, C.c_size_t, up, up]
    L.tloam_b200_global_map_static_download.argtypes = [vp, dp, dp, C.c_size_t, szp]
    L.tloam_b200_global_map_merge.argtypes = [vp, C.c_double, C.c_int, szp]
    L.tloam_b200_global_map_merged_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp, dp]
    L.tloam_b200_localize_default_config.argtypes = [C.POINTER(LocalizeConfig)]
    L.tloam_b200_localize_default_config.restype = None
    L.tloam_b200_localize_enable.argtypes = [vp, C.POINTER(LocalizeConfig)]
    L.tloam_b200_localize_set_map.argtypes = [vp, dp, C.c_size_t]
    L.tloam_b200_localize_set_map_merged.argtypes = [vp]
    L.tloam_b200_localize_frame.argtypes = [vp, dp, C.POINTER(LocalizeResult)]
    L.tloam_b200_localize.argtypes = [vp, dp, C.c_size_t, dp, C.POINTER(LocalizeResult)]
    L.tloam_b200_localize_matches.argtypes = [vp, C.c_int, C.POINTER(C.c_int), dp, C.c_size_t, szp]
    L.tloam_b200_localize_query.argtypes = [vp, dp, C.c_size_t, szp]
    L.tloam_b200_localize_map_normals.argtypes = [vp, dp, C.POINTER(C.c_ubyte), C.POINTER(C.c_int), C.c_size_t, szp]
    L.tloam_b200_localize_cells.argtypes = [vp, up, C.POINTER(C.c_ulonglong), up, C.c_size_t, szp]
    L.tloam_b200_loop_descriptors_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp]
    L.tloam_b200_relocalize_default_config.argtypes = [C.POINTER(RelocalizeConfig)]
    L.tloam_b200_relocalize_default_config.restype = None
    L.tloam_b200_relocalize_enable.argtypes = [vp, C.POINTER(RelocalizeConfig)]
    L.tloam_b200_relocalize_set_places.argtypes = [vp, dp, dp, C.c_size_t]
    L.tloam_b200_relocalize_set_places_loop.argtypes = [vp, dp, C.c_size_t]
    L.tloam_b200_relocalize_frame.argtypes = [vp, C.POINTER(RelocalizeResult)]
    L.tloam_b200_relocalize.argtypes = [vp, dp, C.c_size_t, C.POINTER(RelocalizeResult)]
    L.tloam_b200_relocalize_hypotheses.argtypes = [vp, C.POINTER(RelocalizeHypothesis), C.c_size_t, szp]
    L.tloam_b200_relocalize_matches.argtypes = [vp, C.c_int, C.c_int, C.POINTER(C.c_int), dp, C.c_size_t, szp]
    L.tloam_b200_map_update_default_config.argtypes = [C.POINTER(MapUpdateConfig)]
    L.tloam_b200_map_update_default_config.restype = None
    L.tloam_b200_map_update_enable.argtypes = [vp, C.POINTER(MapUpdateConfig)]
    L.tloam_b200_map_update_add.argtypes = [vp, C.POINTER(MapUpdateAddResult)]
    L.tloam_b200_map_update_build.argtypes = [vp, C.POINTER(MapUpdateResult)]
    L.tloam_b200_map_update_size.argtypes = [vp, szp, szp, szp]
    L.tloam_b200_map_update_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp]
    L.tloam_b200_map_update_votes.argtypes = [vp, C.c_int, C.c_size_t, C.c_size_t, up, up]
    L.tloam_b200_map_update_additions.argtypes = [vp, C.c_size_t, C.c_size_t, dp, up]
    L.tloam_b200_localize_set_map_updated.argtypes = [vp]
    L.tloam_b200_occupancy_default_config.argtypes = [C.POINTER(OccupancyConfig)]
    L.tloam_b200_occupancy_default_config.restype = None
    L.tloam_b200_occupancy_enable.argtypes = [vp, C.POINTER(OccupancyConfig)]
    L.tloam_b200_occupancy_build.argtypes = [vp, C.POINTER(OccupancyInfo)]
    L.tloam_b200_occupancy_download.argtypes = [vp, C.POINTER(C.c_byte), up, up, C.c_size_t]
    L.tloam_b200_occupancy_scans_download.argtypes = [vp, C.c_size_t, C.c_size_t, dp, dp]
    L.tloam_b200_distance_default_config.argtypes = [C.POINTER(DistanceConfig)]
    L.tloam_b200_distance_default_config.restype = None
    L.tloam_b200_distance_build.argtypes = [vp, C.POINTER(DistanceConfig), C.POINTER(DistanceInfo)]
    L.tloam_b200_distance_build_grid.argtypes = [vp, C.POINTER(DistanceConfig), C.POINTER(C.c_byte), C.c_size_t, C.c_size_t,
                                                 C.c_double, C.c_double, C.c_double, C.POINTER(DistanceInfo)]
    L.tloam_b200_distance_download.argtypes = [vp, C.POINTER(C.c_float), up, C.POINTER(C.c_ubyte), C.POINTER(C.c_byte),
                                               C.c_size_t]
    L.tloam_b200_distance_query.argtypes = [vp, dp, C.c_size_t, dp, dp]
    L.tloam_b200_plan_default_config.argtypes = [C.POINTER(PlanConfig)]
    L.tloam_b200_plan_default_config.restype = None
    L.tloam_b200_plan_build.argtypes = [vp, C.POINTER(PlanConfig), C.c_double, C.c_double, C.POINTER(PlanInfo)]
    L.tloam_b200_plan_download.argtypes = [vp, C.POINTER(C.c_ulonglong), C.c_size_t]
    L.tloam_b200_plan_paths.argtypes = [vp, dp, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int),
                                        C.POINTER(C.c_ulonglong)]
    L.tloam_b200_plan_path_cells.argtypes = [vp, C.POINTER(C.c_int), dp, C.c_size_t]
    L.tloam_b200_frontier_default_config.argtypes = [C.POINTER(FrontierConfig)]
    L.tloam_b200_frontier_default_config.restype = None
    L.tloam_b200_frontier_search.argtypes = [vp, C.POINTER(FrontierConfig), C.POINTER(FrontierInfo)]
    L.tloam_b200_frontier_download.argtypes = [vp, C.POINTER(FrontierRecord), C.c_size_t]
    L.tloam_b200_frontier_cells.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_int), dp, C.c_size_t]
    L.tloam_b200_frontier_labels.argtypes = [vp, C.POINTER(C.c_uint), C.c_size_t]
    L.tloam_b200_terrain_default_config.argtypes = [C.POINTER(TerrainConfig)]
    L.tloam_b200_terrain_default_config.restype = None
    L.tloam_b200_terrain_build.argtypes = [vp, C.POINTER(TerrainConfig), C.POINTER(TerrainInfo)]
    L.tloam_b200_terrain_build_cloud.argtypes = [vp, C.POINTER(TerrainConfig), dp, C.c_size_t, C.POINTER(TerrainInfo)]
    L.tloam_b200_terrain_download.argtypes = [vp, C.POINTER(C.c_byte), dp, dp, dp, dp, dp, C.POINTER(C.c_uint), C.c_size_t]
    L.tloam_b200_distance_build_terrain.argtypes = [vp, C.POINTER(DistanceConfig), C.POINTER(DistanceInfo)]
    L.tloam_b200_global_registration_default_config.argtypes = [C.POINTER(GlobalRegistrationConfig)]
    L.tloam_b200_global_registration_default_config.restype = None
    L.tloam_b200_global_registration_enable.argtypes = [vp, C.POINTER(GlobalRegistrationConfig)]
    L.tloam_b200_global_register.argtypes = [vp, dp, C.c_size_t, dp, C.c_size_t, C.POINTER(GlobalRegistrationResult)]
    L.tloam_b200_global_register_loop.argtypes = [vp, C.c_longlong, C.c_longlong, C.POINTER(GlobalRegistrationResult)]
    L.tloam_b200_global_registration_side.argtypes = [vp, C.c_int, dp, dp, C.POINTER(C.c_ubyte), ip, dp, C.POINTER(C.c_ubyte),
                                                      C.c_size_t, szp]
    L.tloam_b200_global_registration_correspondences.argtypes = [vp, ip, C.c_size_t, szp]
    L.tloam_b200_global_registration_hypotheses.argtypes = [vp, ip, C.c_size_t, szp]
    _lib = L
    return L
