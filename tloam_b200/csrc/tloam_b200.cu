// tloam_b200.cu -- kernels + C ABI of libtloam_b200.so (sm_90a). See include/tloam_b200.h for the boundary
// and registration.cuh for the execution model.  No CPU fallback exists anywhere in this file.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>
#include <functional>
#include <mutex>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "registration.cuh"
#include "solver.cuh"
#include "map_build.cuh"
#include "frame_kernels.cuh"
#include "dense_search.cuh"
#include "fine_search.cuh"
#include "submap.cuh"
#include "feature_extract.cuh"
#include "ground_extract.cuh"
#include "edge_extract.cuh"
#include "object_segment.cuh"
#include "host_stage.h"
#include "gmap_intensity.h"
#include "unpack_scan.h"
#include "deskew.h"
#include "scan_context.h"
#include "loop_verify.h"
#include "loop_verify_submap.h"
#include "pose_graph.h"
#include "pose_graph_robust.h"
#include "map_correct.h"
#include "map_dynamic.h"
#include "map_merge.h"
#include "localize.h"
#include "relocalize.h"
#include "map_update.h"
#include "occupancy.h"
#include "distance.h"
#include "plan.h"
#include "global_registration.h"
#include "frontier.h"
#include "terrain.h"



// =================================================================================================
// Host side: handle + C ABI
// =================================================================================================
using namespace tloam;

// bounds and count of a host cloud's finite rows, the rows the voxel kernels keep (vox_in_box drops a row with a
// non-finite coordinate); n == 0: none
struct VoxExtent { double lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0}; size_t n = 0; bool known = true; };

#define CU_TRY(expr)                                                                                   \
  do {                                                                                                 \
    cudaError_t e__ = (expr);                                                                          \
    if (e__ != cudaSuccess) {                                                                          \
      snprintf(h->last_error, sizeof(h->last_error), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
               __FILE__, __LINE__);                                                                    \
      return TLOAM_B200_ERR_CUDA;                                                                      \
    }                                                                                                  \
  } while (0)

struct tloam_b200_handle {
  tloam_tls_config cfg;
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  cudaStream_t copy_stream = nullptr;              // H2D of the map clouds, overlapped with the build (set_target)
  cudaEvent_t ev_copy[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  int last_uploaded = 0;
  cudaEvent_t ev_src = nullptr;                    // set_source: the H2D copies have landed
  cudaStream_t fit_stream = nullptr;               // per-frame getFitnessScore runs beside the registration (fork / join in the frame graph)
  cudaEvent_t ev_fit[2] = {nullptr, nullptr};
  char last_error[512] = {0};
  HostStage hstage;                                // pageable host inputs: chunked, multi-threaded staging through pinned slots
  // tloam_b200_segment_scan: the three segmentation stages chained on the device.  A stage that finds `active` reads its
  // input from dev_xyz / dev_intensity (no upload) and, instead of copying its index lists home, leaves the device
  // pointers and counts here for the gather kernel that feeds the next stage.
  struct SegChain {
    bool active = false;
    const double* dev_xyz = nullptr; const double* dev_intensity = nullptr;
    const unsigned* ground = nullptr; const unsigned* object = nullptr; const int* beam = nullptr; const double* intensity = nullptr;
    unsigned n_ground = 0, n_object = 0;
    const unsigned long long* seg = nullptr; unsigned n_seg = 0;
    const unsigned long long* edge = nullptr; const unsigned long long* non_edge = nullptr; unsigned n_edge = 0, n_non = 0;
  } seg;
  unsigned char* d_chain = nullptr; size_t cap_chain = 0;
  long long launches = 0;
  int launches_frame = 0;
  // source
  size_t n_src[4] = {0, 0, 0, 0};
  bool have_src = false, have_tgt = false, frame_pending = false;
  double* d_stage_src = nullptr; size_t cap_stage_src = 0;      // points (the CURRENT staging buffer: one of d_stage_buf[])
  // pipelined handles (set_async_inputs) upload scan k+1 on a stream of its own while frame k is still being registered:
  // two staging buffers alternate; a buffer is free again once its last reader (k_stage_source, or the submap update
  // that appends the staged edge / ground features) has run
  double* d_stage_buf[2] = {nullptr, nullptr}; size_t cap_stage_buf[2] = {0, 0};
  int stage_cur = 0;
  cudaStream_t src_stream = nullptr;
  cudaEvent_t ev_stage_free[2] = {nullptr, nullptr};
  bool stage_free_valid[2] = {false, false};
  double* d_feat = nullptr; size_t cap_pad = 0;                 // 3 + 2 + 6 arrays of cap_pad doubles
  unsigned char* d_flags = nullptr;                             // flags + active
  int* d_blk_count = nullptr; double* d_partial = nullptr; size_t cap_blocks = 0;
  unsigned* d_counter = nullptr;
  FrameState* d_state = nullptr; bool own_state = true;         // a batch owns the states of its handles (one array)
  tloam_b200_stats* d_stats = nullptr;
  // target
  size_t n_tgt[4] = {0, 0, 0, 0};
  double* d_stage_tgt = nullptr; size_t cap_stage_tgt = 0;
  unsigned* d_scratch = nullptr; size_t cap_scratch = 0;        // slot_of + rank_of
  unsigned char* d_blob = nullptr; size_t cap_blob = 0, blob_bytes = 0;
  // second blob: a map being RECEIVED (shared-map broadcast) while frames still register against the active one
  unsigned char* d_blob_in = nullptr; size_t cap_blob_in = 0, blob_in_bytes = 0; MapHeader hdr_in; bool blob_in_ready = false;
  MapHeader hdr;                                                // host copy of the layout (origin filled lazily)
  bool origin_known = false;
  // pinned host staging for results
  double* h_result = nullptr;                                   // 16 result + 2 (status, done)
  tloam_b200_stats* h_stats = nullptr;
  DeviceCtx ctx;
  int total_blocks = 0;
  // whole-frame CUDA graph (re-captured only when the device context changes)
  Predict* h_predict = nullptr; Predict* d_predict = nullptr;
  cudaGraphExec_t gexec = nullptr; DeviceCtx gctx; bool gvalid = false; int glaunches = 0; bool use_graph = true;
  bool use_fused = false;   // k_first (search + fit + first evaluation in one kernel): opt-in, TLOAM_B200_FUSE=1
  bool gfused = false;      // topology of the instantiated graph
  // optional per-kernel-class timing (CUDA events around every launch; off by default)
  bool profiling = false;
  bool traced_last = false;
  bool trace = false;                                           // record tloam_b200_stats traces
  std::vector<cudaEvent_t> ev_pool;
  struct Span { int cls; cudaEvent_t a, b; };
  std::vector<Span> spans;
  size_t ev_next = 0;
  tloam_b200_profile prof;
  unsigned long long* d_dbg = nullptr;
  // ---- device-resident submap ((f)-1) ----
  tloam_submap_config scfg;
  bool submap_ready = false;
  double* d_acc[2] = {nullptr, nullptr};   size_t cap_acc[2] = {0, 0}, n_acc[2] = {0, 0};     // edge, ground accumulators
  double* d_acc_tmp = nullptr;             size_t cap_acc_tmp = 0;
  // n_acc is the host's UPPER BOUND of each accumulator; the exact counts live on the device (no host round trip per
  // frame): d_cnt[0..3] unused, [4 + 2k + acc_cur[k]] = points in accumulator k, [8] scratch, [12] / [13] voxels of the
  // ground / edge feature of tloam_b200_process_cloud
  unsigned* d_cnt = nullptr;               int acc_cur[2] = {0, 0};
  unsigned long long cum_add[2] = {0, 0}, known_cum[2] = {0, 0};  size_t known_cnt[2] = {0, 0};
  struct CntProbe { cudaEvent_t ev = nullptr; unsigned* h_vals = nullptr; unsigned long long cum[2] = {0, 0}; bool pending = false; };
  CntProbe probes[4];                      int probe_next = 0;
  bool src_staged = false;                 // d_stage_src holds the current source (needed by submap_update)
  const double* src_ptr[4] = {nullptr, nullptr, nullptr, nullptr};   // where each source cloud is read (tloam_b200_source_download)
  // ---- FrontEnd::processCloud on the device (tloam_b200_process_cloud / _process_raw_scan): the last processed frame.
  //      d_frame = raw ground | raw edge | general | planar-submap selection (general[planar_submap_index]); the
  //      sphere-submap selection is the general cloud's first fr_ns_sub points (the reference's rank lists, SURVEY Q12) ----
  double* d_frame = nullptr;               size_t cap_frame = 0;
  size_t fr_ng = 0, fr_ne = 0, fr_nn = 0, fr_np_sub = 0, fr_ns_sub = 0;
  bool have_frame = false;
  VoxExtent fr_ground_ext;                 // a bound of the raw ground cloud's extent (submap_init_frame's key range check)
  // pipelined results (async_inputs): two pinned result slots + events, so that the host can stay one frame ahead
  cudaEvent_t ev_res[2] = {nullptr, nullptr};
  long long frames_enqueued = 0, frames_fetched = 0;
  bool frame_fitness = false, gfitness = false;   // k_fitness + reduce appended to every frame (graph topology flag)
  double last_fitness = 0.0, last_rmse = 0.0;
  bool async_inputs = false;               // tloam_b200_set_async_inputs: host buffers stay valid until the next sync
  // per-frame health metric (getFitnessScore) without allocation: block partials + the reduced pair in the state
  double* d_fit = nullptr;                 size_t cap_fit = 0;
  std::vector<double*> ring;               std::vector<size_t> ring_n, ring_cap;               // planar sliding window
  double* d_cat = nullptr;                 size_t cap_cat = 0, n_cat = 0;                       // concatenated planar window
  double* d_sphere0 = nullptr;             size_t n_sphere0 = 0; bool sphere_is_init = false;  // frame-0 sphere submap
  double* d_up = nullptr;                  size_t cap_up = 0;                                   // upload staging
  unsigned char* d_vox = nullptr;          size_t cap_vox = 0;                                  // voxel hash scratch
  // submap update: the ground accumulator is cropped / down-sampled on a stream of its own beside the edge accumulator
  // (own scratch and output buffer); the newest planar frame is uploaded on src_stream while the frame is registered
  unsigned char* d_vox1 = nullptr;         size_t cap_vox1 = 0;
  double* d_acc_tmp1 = nullptr;            size_t cap_acc_tmp1 = 0;
  double* d_up_planar = nullptr;           size_t cap_up_planar = 0;
  cudaStream_t sub_stream = nullptr;
  cudaEvent_t ev_sub[2] = {nullptr, nullptr};
  cudaEvent_t ev_planar_in = nullptr, ev_planar_free = nullptr, ev_planar_done = nullptr;
  bool planar_free_valid = false;
  // ---- PCA feature extraction ((f)-2): one arena, carved up per call ----
  unsigned char* d_fe = nullptr;           size_t cap_fe = 0;  bool fe_attr_set = false;
  double* d_pose = nullptr;
  unsigned char* d_ge = nullptr;           size_t cap_ge = 0;   // ground extraction ((f)-4) arena
  // ---- dense-map correspondence path (dense_search.cuh): query binning scratch + the search-path decision ----
  unsigned char* d_dense = nullptr;        size_t cap_dense = 0, dense_zero_bytes = 0;
  DenseArgs dargs, gdargs;                 // current / captured in the graph
  unsigned* h_mapstats = nullptr;          // pinned: occupied bricks per cloud of the newest map
  cudaEvent_t ev_stats = nullptr;          bool stats_pending = false, stats_known = false;
  unsigned nbricks[4] = {0, 0, 0, 0};
  int dense_mode = 0;                      // TLOAM_B200_DENSE: "auto" -> -1 (points per brick), unset -> 0 never, "1" always
  // two-level grid (fine_search.cuh): TLOAM_B200_FINE unset / "auto" -> -1 (by the density of the previous map),
  // "0" never, "1" always.  map_fine_mask: clouds of the ACTIVE map that were built with the second level
  int dense_kernel = 0, gdense_kernel = 0; // which kernel serves ctx.dense_mask: 1 = TMA-staged (dense_search.cuh), 2 = two-level grid
  int fine_mode = -1;
  int map_fine_mask = 0;
  float4* d_fine_tmp = nullptr;            size_t cap_fine_tmp = 0;
  bool dense_attr_set = false;
  bool fe_sort_attr_set = false, ge_attr_set = false, ee_attr_set = false, os_attr_set = false;   // per handle: function attributes are per device
  bool dense_check = false;                // TLOAM_B200_DENSE_CHECK=1: every dense query is re-searched by the plain path and compared
  int num_sms = 132;                       // H100 SXM; replaced by the device's count at create
  // ---- the raw scan of the last tloam_b200_process_raw_scan (in d_chain): valid while no segmentation / process call
  //      has run since, i.e. while seg_gen == raw_gen ----
  unsigned long long seg_gen = 0, raw_gen = ~0ull;
  const double* raw_scan = nullptr;        size_t raw_n = 0;
  const double* raw_int = nullptr;         // its intensity (in d_chain) when it came packed with an intensity field
  unsigned char* d_packed = nullptr;       size_t cap_packed = 0;                               // uploaded packed records
  // ---- global map (tloam_b200_global_map_*, submap.cuh): nothing is allocated or launched until it is enabled ----
  bool gmap_on = false;
  double gmap_voxel = 1.0;
  GMapState* d_gmap_st = nullptr;
  double* d_gmap_pose = nullptr;
  double* d_gmap = nullptr;                size_t cap_gmap = 0;                                 // map points
  unsigned long long* d_gmap_off = nullptr; size_t cap_gmap_off = 0;                            // frame table entries
  double* d_gmap_reg = nullptr;            size_t cap_gmap_reg = 0, gmap_reg_n = 0; bool gmap_reg_valid = false;
  double* d_gmap_fin = nullptr;            size_t cap_gmap_fin = 0;                             // finite rows (voxel input)
  // the host's upper bound of the map size = gmap_known (an exact count, read asynchronously) + the rows appended since
  // (gmap_cum - gmap_known_cum); gmap_calls bounds the frame count
  unsigned long long gmap_cum = 0, gmap_known_cum = 0, gmap_known = 0, gmap_calls = 0;
  size_t gmap_growths = 0;
  struct GMapProbe { cudaEvent_t ev = nullptr; unsigned long long* h_count = nullptr; unsigned long long cum = 0; bool pending = false; };
  GMapProbe gmap_probes[4];                int gmap_probe_next = 0;
  // ---- the map's pose tables (tloam_b200_global_map_correction*, libtloam_b200_gmc.so): O_f and P_f of every frame, with
  //      the capacity of the frame table; M, the pose later appends are expressed in (map <- odom), and whether it is I ----
  bool gmc_on = false;
  double* d_gmc_O = nullptr;               double* d_gmc_P = nullptr;   size_t cap_gmc = 0;
  double gmc_M[16];                        bool gmc_M_identity = true;
  unsigned char* d_gmc_scratch = nullptr;  size_t cap_gmc_scratch = 0;                         // node table, M_f, moved
  // ---- dynamic-point removal (tloam_b200_global_map_dynamic*, libtloam_b200_gmd.so): two counters per map row with the
  //      capacity of d_gmap (zero past the map's count), the range and window images, the row and column boundary tables ----
  bool gmd_on = false;
  tloam_global_map_dynamic_config gmd_cfg;
  unsigned* d_gmd_through = nullptr;       unsigned* d_gmd_hits = nullptr;   size_t cap_gmd = 0;
  unsigned long long* d_gmd_image = nullptr; double* d_gmd_window = nullptr; double* d_gmd_bounds = nullptr;
  size_t cap_gmd_image = 0, cap_gmd_bounds = 0;
  unsigned char* d_gmd_scratch = nullptr;  size_t cap_gmd_scratch = 0;                         // the static download
  // ---- the occupancy grid (tloam_b200_occupancy*, libtloam_b200_occ.so): a 2D scan and a pose per frame slot, with the
  //      capacity of the frame table; the sector boundaries; the last build's grid (occupied, free, values) ----
  bool occ_on = false;
  tloam_occupancy_config occ_cfg;
  double* d_occ_scans = nullptr;           double* d_occ_poses = nullptr;   size_t cap_occ = 0;
  double* d_occ_dirs = nullptr;            size_t cap_occ_dirs = 0;
  unsigned char* d_occ_grid = nullptr;     size_t cap_occ_grid = 0;                            // cells of the buffer
  unsigned char* d_occ_small = nullptr;    // the extent at 0, dropped at 64
  bool occ_built = false;                  tloam_occupancy_info occ_info;
  // ---- the distance field (tloam_b200_distance*, libtloam_b200_dist.so): the last build's cells (sq, sd, the column
  //      distance, the row pass's stacks, a host grid's copy, costs, values: 19 B each), the column pass's band records,
  //      the cost table and the query's points; allocated by the first call that needs them, grown only ----
  unsigned char* d_dist = nullptr;         size_t cap_dist = 0;                                // cells of the buffer
  unsigned* d_dist_bands = nullptr;        size_t cap_dist_bands = 0;
  unsigned char* d_dist_table = nullptr;   size_t cap_dist_table = 0;
  unsigned long long* d_dist_small = nullptr;                                                  // the obstacle count
  double* d_dist_q = nullptr;              size_t cap_dist_q = 0;                              // points: xy, distance, gradient
  bool dist_built = false;                 tloam_distance_info dist_info;
  unsigned long long dist_serial = 0;                                                          // successful builds
  // ---- the plan (tloam_b200_plan*, libtloam_b200_plan.so): the last build's cells (P 8, t 2: 10 B each), the tile
  //      stamps and the two worklists (12 B per tile), the worklists' state, the last paths' starts and outputs (24 B per
  //      start) and cells (8 B each); allocated by the first call that needs them, grown only ----
  unsigned char* d_plan = nullptr;         size_t cap_plan = 0;                                // cells of the buffer
  unsigned* d_plan_tiles = nullptr;        size_t cap_plan_tiles = 0;                          // stamps, then 2 lists
  tloam_plan_state* d_plan_state = nullptr;
  unsigned char* d_plan_q = nullptr;       size_t cap_plan_q = 0;                              // starts of the buffer
  int* d_plan_cells = nullptr;             size_t cap_plan_cells = 0;                          // path cells of the buffer
  bool plan_built = false;                 tloam_plan_info plan_info;
  bool plan_paths_kept = false;            size_t plan_path_total = 0;                         // cells of the last paths
  unsigned long long plan_serial = 0;      tloam_plan_config plan_cfg;                         // the field it was built on
  // ---- the frontiers (tloam_b200_frontier*, libtloam_b200_frontier.so): per cell the label (4 B), per tile a flag, the
  //      compaction's block counts and the state; per frontier cell the radix sort's keys and rows (24 B), its
  //      histograms and the heads (4 B); per frontier 64 B of statistics.  Allocated by the first search that needs
  //      them, grown only; the ranked frontiers on the host ----
  unsigned* d_fr_labels = nullptr;         size_t cap_fr_labels = 0;                           // cells of the buffer
  unsigned char* d_fr_tiles = nullptr;     size_t cap_fr_tiles = 0;
  unsigned char* d_fr_small = nullptr;                                                         // block counts, state
  unsigned char* d_fr_sort = nullptr;      size_t cap_fr_sort = 0;                             // frontier cells of it
  bool fr_kept = false;                    tloam_frontier_info fr_info;
  std::vector<tloam_frontier> fr_ranked;   unsigned fr_sorted = 0;                             // row buffer of the cells
  // ---- the terrain (tloam_b200_terrain*, libtloam_b200_terrain.so): the last build's cells (65 B each: four encodings,
  //      three layers, two counts, the value), the host cloud's rows (24 B each) and the state; allocated by the first
  //      build that needs them, grown only ----
  unsigned char* d_ter = nullptr;          size_t cap_ter = 0;                                 // cells of the buffer
  double* d_ter_cloud = nullptr;           size_t cap_ter_cloud = 0;                           // rows of the buffer
  tloam_ter_state* d_ter_state = nullptr;
  bool ter_built = false;                  tloam_terrain_info ter_info;
  // ---- the merged map (tloam_b200_global_map_merge*, libtloam_b200_gmm.so): the radix sort's scratch (24 B per map row)
  //      and the last merge's voxels (32 B each), allocated by the first merge and grown; the snapshot is dropped by
  //      enable / reset and by the next merge ----
  unsigned char* d_gmm_scratch = nullptr;  size_t cap_gmm_scratch = 0;
  double* d_gmm_out = nullptr;             size_t cap_gmm_out = 0;                             // n x 3 xyz, then n intensity
  bool gmm_valid = false;                  bool gmm_has = false;   size_t gmm_n = 0;
  // ---- the map's intensity channel (tloam_b200_global_map_*intensity*, libtloam_b200_gmi.so): allocated on the first
  //      intensity append; d_gmi_map has the capacity of d_gmap ----
  bool gmi_used = false;                   // an intensity frame was appended since enable / reset
  unsigned* d_gmi_st = nullptr;            // [0] the map has the channel, [1] a finite row found no voxel (sticky)
  double* d_gmi_map = nullptr;
  double* d_gmi_in = nullptr;              size_t cap_gmi_in = 0;                               // uploaded intensities
  void* d_gmi_scratch = nullptr;           size_t cap_gmi_scratch = 0;
  // ---- loop closure (tloam_b200_loop_*, libtloam_b200_loop.so): nothing is allocated or launched until it is enabled.
  //      loop_frames is exact (every add is one frame); the database grows x1.5 when full ----
  bool loop_on = false;
  tloam_loop_config loop_cfg;
  double* d_loop_db = nullptr;             size_t loop_cap = 0, loop_frames = 0, loop_growths = 0;   // descriptor slots
  double* d_loop_dirs = nullptr;           // sector boundary directions
  double* d_loop_in = nullptr;             size_t cap_loop_in = 0;                                   // host clouds (loop_add)
  tloam_sc_best* d_loop_best = nullptr;    // TLOAM_SC_MAX_BLOCKS block minima, then the result
  tloam_sc_best* h_loop_best = nullptr;    // pinned: the newest add's result, landed when ev_loop has
  cudaEvent_t ev_loop = nullptr;
  bool loop_has_result = false;            long long loop_query = -1;
  // ---- loop verification (tloam_b200_loop_verify*, libtloam_b200_loopv.so): a keyframe per loop frame, kept by the
  //      global map's ordered path in buffers of its own; nothing is allocated or launched until it is enabled.  The
  //      host's bound of the store size = lv_known (exact, read asynchronously) + the rows added since ----
  bool lv_on = false;
  tloam_loop_verify_config lv_cfg;
  GMapState* d_lv_st = nullptr;            // count = store points, frames = keyframes
  double* d_lv_pose = nullptr;             // identity
  double* d_lv_pts = nullptr;              size_t cap_lv = 0;                                   // keyframe points
  unsigned long long* d_lv_off = nullptr;  size_t cap_lv_off = 0;                               // keyframe f: [off[f], off[f + 1])
  double* d_lv_reg = nullptr;              size_t cap_lv_reg = 0;
  double* d_lv_fin = nullptr;              size_t cap_lv_fin = 0;
  unsigned long long lv_cum = 0, lv_known_cum = 0, lv_known = 0;
  size_t lv_growths = 0;
  GMapProbe lv_probes[4];                  int lv_probe_next = 0;
  tloam_lv_state* d_lv_state = nullptr;
  unsigned char* d_lv_scratch = nullptr;   size_t cap_lv_scratch = 0;                           // the verification's scratch
  bool lv_ran = false;                     int lv_passes = 0;   unsigned long long lv_nq = 0;   // the last verification
  const int* lv_match_index = nullptr;    const double* lv_match_d2 = nullptr;                 // its matches, pass-major
  // ---- loop verification against a submap (tloam_b200_loop_verify_submap*, libtloam_b200_loopvs.so): reads the keyframe
  //      store above and the pose graph's node store; its scratch is allocated by the first run and grown ----
  bool lvs_on = false;
  tloam_loop_verify_submap_config lvs_cfg;
  unsigned char* d_lvs_scratch = nullptr;  size_t cap_lvs_scratch = 0;
  bool lvs_ran = false;                    int lvs_passes = 0;   unsigned long long lvs_nq = 0, lvs_nm = 0;   // the last run
  tloam_lvs_args lvs_last;                 // its buffers (target, normals, matches)
  // ---- localization in a prior map (tloam_b200_localize*, libtloam_b200_loc.so): the map and its index (one buffer,
  //      grown by a load), the query's ordered down-sample and the run's scratch; nothing is allocated or launched until
  //      it is enabled ----
  bool loc_on = false;
  tloam_localize_config loc_cfg;
  unsigned char* d_loc_map = nullptr;      size_t cap_loc_map = 0;     // map, sorted map, rows, cells, normals
  unsigned char* d_loc_scratch = nullptr;  size_t cap_loc_scratch = 0; // the index build's radix sort
  bool loc_loaded = false;                 size_t loc_n = 0;           tloam_loc_index_args loc_index;
  GMapState* d_loc_qst = nullptr;
  double* d_loc_reg = nullptr;             size_t cap_loc_reg = 0;
  double* d_loc_fin = nullptr;             size_t cap_loc_fin = 0;
  double* d_loc_q = nullptr;               size_t cap_loc_q = 0;       // the query (ordered down-sample)
  double* d_loc_in = nullptr;              size_t cap_loc_in = 0;      // a host cloud
  unsigned char* d_loc_run = nullptr;      size_t cap_loc_run = 0;     // state, memory, partials, matches
  bool loc_have_prev = false;              // a localization since the load: the prediction has its memory
  bool loc_ran = false;                    int loc_passes = 0;  size_t loc_nq = 0;   tloam_loc_args loc_last;
  // what the last tloam_b200_localize* read, for tloam_b200_map_update_add: its serial number, the scan rows (the raw scan
  // or d_loc_in) with the generation they must still have, and the verdict
  unsigned long long loc_serial = 0;       const double* loc_src = nullptr;  size_t loc_src_n = 0;
  bool loc_src_raw = false;                unsigned long long loc_src_gen = 0, loc_in_gen = 0;  bool loc_accepted = false;
  // ---- updating a prior map (tloam_b200_map_update*, libtloam_b200_mapu.so and libtloam_b200_gmd.so): the prior rows'
  //      counters, the additions (xyz, frame, counters in one buffer), the range image and the built cloud; nothing is
  //      allocated or launched until it is enabled ----
  bool mu_on = false;                      tloam_map_update_config mu_cfg;
  bool mu_fresh = true;                    // the state is empty: the next add or build clears the counters
  unsigned long long mu_min_serial = 0, mu_added_serial = 0;  unsigned mu_frames = 0;
  size_t mu_known = 0, mu_pending = 0;     // the additions' count at the last read-back, and the query rows added since
  double* d_mu_tables = nullptr;           size_t cap_mu_tables = 0;
  unsigned long long* d_mu_image = nullptr; double* d_mu_window = nullptr;  size_t cap_mu_image = 0;
  unsigned* d_mu_prior = nullptr;          size_t cap_mu_prior = 0;   // through [0, cap), hits [cap, 2 cap)
  unsigned char* d_mu_add = nullptr;       size_t cap_mu_add = 0;     // xyz, frame, through, hits of cap rows each
  unsigned char* d_mu_small = nullptr;     // the pose at 0, counts at 128, the static part's block counts at 1024
  unsigned char* d_mu_q = nullptr;         size_t cap_mu_q = 0;       // per query row: the flag and T q
  std::vector<void*> mu_retired;           // buffers an add replaced, freed at the next point that synchronises anyway
  unsigned char* d_mu_build = nullptr;     size_t cap_mu_build = 0;
  double* d_mu_out = nullptr;              size_t cap_mu_out = 0;     bool mu_built = false;  size_t mu_built_n = 0;
  // ---- relocalization in a prior map (tloam_b200_relocalize*, libtloam_b200_reloc.so): the places (descriptor slots,
  //      poses, per-place best distance and shift in one buffer), the query's descriptor and down-sample, the batch ----
  bool rl_on = false;                      tloam_relocalize_config rl_cfg;
  double* d_rl_dirs = nullptr;             // sector boundary directions of rl_cfg.n_sector
  unsigned char* d_rl_places = nullptr;    size_t cap_rl_places = 0;  size_t rl_n = 0;  bool rl_loaded = false;
  unsigned char* d_rl_small = nullptr;     // the query's GMapState at 0, its descriptor slot at 256
  double* d_rl_q = nullptr;                size_t cap_rl_q = 0;
  unsigned char* d_rl_run = nullptr;       size_t cap_rl_run = 0;     // states, candidates, partials, matches
  bool rl_ran = false;                     size_t rl_nq = 0, rl_qn = 0;  tloam_rl_args rl_last;   // rl_qn: query rows
  std::vector<tloam_loc_state> rl_states;  tloam_rl_top rl_top;
  // ---- pose graph (tloam_b200_pose_graph*, libtloam_b200_pg.so): the node store on the device, the loop edges on the
  //      host until an optimisation uploads them; nothing is allocated or launched until it is enabled ----
  bool pg_on = false;
  tloam_pose_graph_config pg_cfg;
  double* d_pg_O = nullptr;                size_t cap_pg = 0;   size_t pg_nodes = 0;   size_t pg_growths = 0;
  std::vector<long long> pg_ij;            std::vector<double> pg_Z;                           // the loop edges
  unsigned char* d_pg_scratch = nullptr;   size_t cap_pg_scratch = 0;
  tloam_pg_state* d_pg_state = nullptr;
  const double* d_pg_T = nullptr;          size_t pg_opt_nodes = 0;                            // the last optimisation
  const double* d_pgr_w = nullptr;         size_t pgr_w_edges = 0;                             // its loop weights (robust)
  // ---- global registration (tloam_b200_global_register*, libtloam_b200_greg.so): per side the keypoints, their index,
  //      normals and features in one buffer; the host clouds' down-sample and the run's pairs, hypotheses and state;
  //      nothing is allocated or launched until it is enabled ----
  bool gr_on = false;                      tloam_global_registration_config gr_cfg;
  unsigned char* d_gr_side[2] = {nullptr, nullptr};  size_t cap_gr_side[2] = {0, 0};
  unsigned char* d_gr_scratch = nullptr;   size_t cap_gr_scratch = 0;  // an index build's radix sort
  unsigned char* d_gr_small = nullptr;     // the down-sample's GMapState at 0, the identity pose at 256
  double* d_gr_reg = nullptr;              size_t cap_gr_reg = 0;
  double* d_gr_fin = nullptr;              size_t cap_gr_fin = 0;
  double* d_gr_q = nullptr;                size_t cap_gr_q = 0;        // a host cloud's keypoints
  double* d_gr_in = nullptr;               size_t cap_gr_in = 0;       // a host cloud
  unsigned char* d_gr_run = nullptr;       size_t cap_gr_run = 0;      // state, pairs, hypotheses, inlier sets
  bool gr_ran = false;                     tloam_gr_args gr_last;      unsigned long long gr_nc = 0;  int gr_nh = 0;
};

// launch bookkeeping: counts the kernel and, in profiling mode, brackets it with events
struct LaunchScope {
  tloam_b200_handle* h; int cls; cudaEvent_t a = nullptr, b = nullptr;
  LaunchScope(tloam_b200_handle* hh, int c) : h(hh), cls(c) {
    h->launches++;
    if (h->profiling) {
      while (h->ev_pool.size() < h->ev_next + 2) { cudaEvent_t e; cudaEventCreate(&e); h->ev_pool.push_back(e); }
      a = h->ev_pool[h->ev_next++]; b = h->ev_pool[h->ev_next++];
      cudaEventRecord(a, h->stream);
    }
  }
  ~LaunchScope() {
    if (h->profiling) { cudaEventRecord(b, h->stream); h->spans.push_back({cls, a, b}); }
  }
};
#define TL_LAUNCH(cls, ...) do { LaunchScope ls__(h, cls); __VA_ARGS__; } while (0)

static size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

// per-sequence grids (the same function of the cloud sizes in single and batched mode => identical reduction trees)
static int eval_grid_of(int nb) {      // k_eval: grid-stride over the feature blocks, a whole number of clusters
  return ((nb < kEvalGridCap ? nb : kEvalGridCap) + kEvalCluster - 1) / kEvalCluster * kEvalCluster;
}
static int first_grid_of(int nb) {     // k_first: one block per 64 features, rounded up to the cluster size
  return (2 * nb + kEvalCluster - 1) / kEvalCluster * kEvalCluster;
}

extern "C" {

void tloam_b200_default_config(tloam_tls_config* c) {   // ref: config/mapping/lidar_odometry.yaml:23-39
  c->k_corr = 10; c->factor_num = 4;
  c->edge_dist_thres = 1.0; c->sphere_dist_thres = 0.5; c->planar_dist_thres = 0.5; c->ground_dist_thres = 0.5;
  c->edge_dir_thres = 0.85;
  c->edge_maxnum = 1200; c->sphere_maxnum = 200; c->planar_maxnum = 2500; c->ground_maxnum = 2000;
  c->max_iterations = 4; c->cost_threshold = 0.000000005; c->gnc_factor = 11.8; c->noise_bound = 0.01;
  c->fitness_thres = 0.02;
  c->ceres_max_num_iterations = 4;
  c->reinit_dir[0] = 1.0; c->reinit_dir[1] = 1.0; c->reinit_dir[2] = 1.0;
  c->initial_trust_region_radius = 1e4;
}

const char* tloam_b200_status_string(int s) {
  switch (s) {
    case TLOAM_B200_OK: return "ok";
    case TLOAM_B200_ERR_INVALID_ARG: return "invalid argument";
    case TLOAM_B200_ERR_TOO_FEW_POINTS: return "a cloud has fewer than 10 points";
    case TLOAM_B200_ERR_BAD_POSE: return "predicted pose is not a rigid transform";
    case TLOAM_B200_ERR_CUDA: return "CUDA error";
    case TLOAM_B200_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
    case TLOAM_B200_ERR_NOT_READY: return "source or target not set";
    case TLOAM_B200_ERR_NUMERIC: return "non-finite value in the solve";
    case TLOAM_B200_ERR_MAP_DENSITY: return "a map cell holds more than 65535 points";
    case TLOAM_B200_ERR_VOXEL_RANGE: return "a cloud spans 2^21 or more voxels on an axis (voxel size too small), or n * voxel >= 2^23 m";
    default: return "unknown status";
  }
}

static double radius_of(const tloam_tls_config& c, int cloud) {
  return cloud == 0 ? c.edge_dist_thres : cloud == 1 ? c.sphere_dist_thres : cloud == 2 ? c.planar_dist_thres : c.ground_dist_thres;
}

int tloam_b200_create(const tloam_tls_config* cfg, int device, void* stream, tloam_b200_handle** out) {
  if (!cfg || !out) return TLOAM_B200_ERR_INVALID_ARG;
  *out = nullptr;
  if (cfg->factor_num < 2 || cfg->factor_num > 4 || cfg->max_iterations < 1 ||
      cfg->max_iterations > TLOAM_B200_MAX_OUTER || cfg->ceres_max_num_iterations < 0 ||
      cfg->ceres_max_num_iterations > TLOAM_B200_MAX_INNER || !(cfg->initial_trust_region_radius > 0.0))
    return TLOAM_B200_ERR_INVALID_ARG;
  for (int c = 0; c < 4; ++c) if (!(radius_of(*cfg, c) > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device < 0 || device >= ndev) {
    cudaGetLastError();
    return TLOAM_B200_ERR_NO_DEVICE;
  }
  tloam_b200_handle* h = new (std::nothrow) tloam_b200_handle();
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  h->cfg = *cfg;
  h->device = device;
  auto fail = [&](int code) { tloam_b200_destroy(h); return code; };
  if (cudaSetDevice(device) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (stream) { h->stream = (cudaStream_t)stream; h->own_stream = false; }
  else {
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
    h->own_stream = true;
  }
  if (cudaEventCreate(&h->ev0) != cudaSuccess || cudaEventCreate(&h->ev1) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  for (int i = 0; i < 5; ++i)
    if (cudaEventCreateWithFlags(&h->ev_copy[i], cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaEventCreateWithFlags(&h->ev_src, cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaStreamCreateWithFlags(&h->fit_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaStreamCreateWithFlags(&h->src_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaStreamCreateWithFlags(&h->sub_stream, cudaStreamNonBlocking) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  for (int i = 0; i < 2; ++i)
    if (cudaEventCreateWithFlags(&h->ev_sub[i], cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaEventCreateWithFlags(&h->ev_planar_in, cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaEventCreateWithFlags(&h->ev_planar_free, cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaEventCreateWithFlags(&h->ev_planar_done, cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  for (int i = 0; i < 2; ++i)
    if (cudaEventCreateWithFlags(&h->ev_stage_free[i], cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  for (int i = 0; i < 2; ++i)
    if (cudaEventCreateWithFlags(&h->ev_fit[i], cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  for (int i = 0; i < 2; ++i)
    if (cudaEventCreateWithFlags(&h->ev_res[i], cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMalloc(&h->d_cnt, 32 * sizeof(unsigned)) != cudaSuccess || cudaMemset(h->d_cnt, 0, 32 * sizeof(unsigned)) != cudaSuccess)
    return fail(TLOAM_B200_ERR_CUDA);
  for (auto& pr : h->probes) {
    if (cudaEventCreateWithFlags(&pr.ev, cudaEventDisableTiming) != cudaSuccess || cudaMallocHost(&pr.h_vals, 2 * sizeof(unsigned)) != cudaSuccess)
      return fail(TLOAM_B200_ERR_CUDA);
  }
  if (cudaMalloc(&h->d_state, sizeof(FrameState)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMalloc(&h->d_stats, sizeof(tloam_b200_stats)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMalloc(&h->d_counter, 256) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMallocHost(&h->h_result, 64 * sizeof(double)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);   // [0..31] slot 0 + scratch, [32..63] slot 1
  if (cudaMallocHost(&h->h_stats, sizeof(tloam_b200_stats)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMallocHost(&h->h_predict, sizeof(Predict)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMalloc(&h->d_predict, sizeof(Predict)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  { const char* e = getenv("TLOAM_B200_NO_GRAPH"); h->use_graph = !(e && e[0] == '1'); }
  // the fused first evaluation (k_first) is opt-in: its evaluation spills and runs on half the lanes, which costs what
  // the saved launch gains (DESIGN.md section 4a)
  { const char* e = getenv("TLOAM_B200_FUSE"); h->use_fused = (e && e[0] == '1'); }
  { const char* e = getenv("TLOAM_B200_NO_FUSE"); if (e && e[0] == '1') h->use_fused = false; }
  { const char* e = getenv("TLOAM_B200_DENSE_CHECK"); h->dense_check = (e && e[0] == '1'); }
  // dense-map search path (dense_search.cuh): off unless asked for.  "1" = always for the K = 5 clouds, "auto" = by the
  // points-per-brick statistics of the map.  Measured on config 3 it is still SLOWER than the lane-pair search (4.1 vs
  // 3.0 ms per launch, DESIGN.md section 4): correct and TMA-staged, not yet a win.
  { const char* e = getenv("TLOAM_B200_DENSE"); h->dense_mode = 0; if (e && e[0] == '1') h->dense_mode = 1; else if (e && e[0] == 'a') h->dense_mode = -1; }
  { const char* e = getenv("TLOAM_B200_FINE"); h->fine_mode = -1; if (e && e[0] == '1') h->fine_mode = 1; else if (e && e[0] == '0') h->fine_mode = 0; }
  if (cudaMallocHost(&h->h_mapstats, 4 * sizeof(unsigned)) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaEventCreateWithFlags(&h->ev_stats, cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  { int v = 0; if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && v > 0) h->num_sms = v; }
  memset(&h->dargs, 0, sizeof(h->dargs)); memset(&h->gdargs, 0, sizeof(h->gdargs));
  if (kEvalCluster > 8) {                          // cluster sizes above 8 are "non-portable": opt in per kernel
    if (cudaFuncSetAttribute(k_eval<true, false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
        cudaFuncSetAttribute(k_eval<false, false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
        cudaFuncSetAttribute(k_eval<true, true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
        cudaFuncSetAttribute(k_eval<false, true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
        cudaFuncSetAttribute(k_first<false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
        cudaFuncSetAttribute(k_first<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess)
      return fail(TLOAM_B200_ERR_CUDA);
  }
  // identity curr/last pose (the reference leaves them uninitialised until the first scanMatching)
  FrameState init;
  memset(&init, 0, sizeof(init));
  for (int i = 0; i < 16; ++i) init.curr_pose[i] = init.last_pose[i] = init.result[i] = (i % 5 == 0) ? 1.0 : 0.0;
  init.frame_done = 1;
  if (cudaMemcpy(h->d_state, &init, sizeof(init), cudaMemcpyHostToDevice) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMemset(h->d_counter, 0, 256) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  memset(&h->ctx, 0, sizeof(h->ctx));
  memset(&h->hdr, 0, sizeof(h->hdr));
  *out = h;
  return TLOAM_B200_OK;
}

int tloam_b200_destroy(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  if (h->copy_stream) cudaStreamSynchronize(h->copy_stream);
  h->hstage.shutdown();
  cudaFree(h->d_stage_buf[0]); cudaFree(h->d_stage_buf[1]); cudaFree(h->d_feat); cudaFree(h->d_flags); cudaFree(h->d_blk_count);
  cudaFree(h->d_partial); cudaFree(h->d_counter); if (h->own_state) cudaFree(h->d_state); cudaFree(h->d_stats);
  cudaFree(h->d_stage_tgt); cudaFree(h->d_scratch); cudaFree(h->d_blob); cudaFree(h->d_blob_in); cudaFree(h->d_dbg);
  cudaFree(h->d_acc[0]); cudaFree(h->d_acc[1]); cudaFree(h->d_acc_tmp); cudaFree(h->d_cat); cudaFree(h->d_sphere0);
  cudaFree(h->d_cnt); cudaFree(h->d_fit); cudaFree(h->d_ge);
  for (auto& pr : h->probes) { if (pr.ev) cudaEventDestroy(pr.ev); if (pr.h_vals) cudaFreeHost(pr.h_vals); }
  cudaFree(h->d_up); cudaFree(h->d_vox); cudaFree(h->d_pose); cudaFree(h->d_fe);
  for (double* p : h->ring) cudaFree(p);
  if (h->h_result) cudaFreeHost(h->h_result);
  if (h->h_stats) cudaFreeHost(h->h_stats);
  if (h->h_predict) cudaFreeHost(h->h_predict);
  if (h->h_mapstats) cudaFreeHost(h->h_mapstats);
  if (h->ev_stats) cudaEventDestroy(h->ev_stats);
  cudaFree(h->d_dense);
  cudaFree(h->d_fine_tmp);
  cudaFree(h->d_predict);
  if (h->gexec) cudaGraphExecDestroy(h->gexec);
  for (cudaEvent_t e : h->ev_pool) cudaEventDestroy(e);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  for (int i = 0; i < 5; ++i) if (h->ev_copy[i]) cudaEventDestroy(h->ev_copy[i]);
  if (h->ev_src) cudaEventDestroy(h->ev_src);
  if (h->fit_stream) { cudaStreamSynchronize(h->fit_stream); cudaStreamDestroy(h->fit_stream); }
  if (h->src_stream) { cudaStreamSynchronize(h->src_stream); cudaStreamDestroy(h->src_stream); }
  if (h->sub_stream) { cudaStreamSynchronize(h->sub_stream); cudaStreamDestroy(h->sub_stream); }
  for (int i = 0; i < 2; ++i) if (h->ev_sub[i]) cudaEventDestroy(h->ev_sub[i]);
  if (h->ev_planar_in) cudaEventDestroy(h->ev_planar_in);
  if (h->ev_planar_free) cudaEventDestroy(h->ev_planar_free);
  if (h->ev_planar_done) cudaEventDestroy(h->ev_planar_done);
  cudaFree(h->d_vox1); cudaFree(h->d_acc_tmp1); cudaFree(h->d_up_planar); cudaFree(h->d_chain); cudaFree(h->d_frame);
  cudaFree(h->d_gmap_st); cudaFree(h->d_gmap_pose); cudaFree(h->d_gmap); cudaFree(h->d_gmap_off); cudaFree(h->d_gmap_reg);
  cudaFree(h->d_gmap_fin);
  cudaFree(h->d_gmi_st); cudaFree(h->d_gmi_map); cudaFree(h->d_gmi_in); cudaFree(h->d_gmi_scratch); cudaFree(h->d_packed);
  for (auto& pr : h->gmap_probes) { if (pr.ev) cudaEventDestroy(pr.ev); if (pr.h_count) cudaFreeHost(pr.h_count); }
  cudaFree(h->d_loop_db); cudaFree(h->d_loop_dirs); cudaFree(h->d_loop_in); cudaFree(h->d_loop_best);
  if (h->h_loop_best) cudaFreeHost(h->h_loop_best);
  if (h->ev_loop) cudaEventDestroy(h->ev_loop);
  cudaFree(h->d_lv_st); cudaFree(h->d_lv_pose); cudaFree(h->d_lv_pts); cudaFree(h->d_lv_off); cudaFree(h->d_lv_reg);
  cudaFree(h->d_lv_fin); cudaFree(h->d_lv_state); cudaFree(h->d_lv_scratch); cudaFree(h->d_lvs_scratch);
  for (auto& pr : h->lv_probes) { if (pr.ev) cudaEventDestroy(pr.ev); if (pr.h_count) cudaFreeHost(pr.h_count); }
  cudaFree(h->d_pg_O); cudaFree(h->d_pg_scratch); cudaFree(h->d_pg_state);
  cudaFree(h->d_gmc_O); cudaFree(h->d_gmc_P); cudaFree(h->d_gmc_scratch);
  cudaFree(h->d_gmd_through); cudaFree(h->d_gmd_hits); cudaFree(h->d_gmd_image); cudaFree(h->d_gmd_window);
  cudaFree(h->d_gmd_bounds); cudaFree(h->d_gmd_scratch);
  cudaFree(h->d_occ_scans); cudaFree(h->d_occ_poses); cudaFree(h->d_occ_dirs); cudaFree(h->d_occ_grid); cudaFree(h->d_occ_small);
  cudaFree(h->d_dist); cudaFree(h->d_dist_bands); cudaFree(h->d_dist_table); cudaFree(h->d_dist_small); cudaFree(h->d_dist_q);
  cudaFree(h->d_plan); cudaFree(h->d_plan_tiles); cudaFree(h->d_plan_state); cudaFree(h->d_plan_q); cudaFree(h->d_plan_cells);
  cudaFree(h->d_fr_labels); cudaFree(h->d_fr_tiles); cudaFree(h->d_fr_small); cudaFree(h->d_fr_sort);
  cudaFree(h->d_ter); cudaFree(h->d_ter_cloud); cudaFree(h->d_ter_state);
  cudaFree(h->d_gmm_scratch); cudaFree(h->d_gmm_out);
  cudaFree(h->d_loc_map); cudaFree(h->d_loc_scratch); cudaFree(h->d_loc_qst); cudaFree(h->d_loc_reg); cudaFree(h->d_loc_fin);
  cudaFree(h->d_loc_q); cudaFree(h->d_loc_in); cudaFree(h->d_loc_run);
  cudaFree(h->d_rl_dirs); cudaFree(h->d_rl_places); cudaFree(h->d_rl_small); cudaFree(h->d_rl_q); cudaFree(h->d_rl_run);
  cudaFree(h->d_mu_tables); cudaFree(h->d_mu_image); cudaFree(h->d_mu_window); cudaFree(h->d_mu_prior); cudaFree(h->d_mu_add);
  cudaFree(h->d_mu_small); cudaFree(h->d_mu_q); cudaFree(h->d_mu_build); cudaFree(h->d_mu_out);
  cudaFree(h->d_gr_side[0]); cudaFree(h->d_gr_side[1]); cudaFree(h->d_gr_scratch); cudaFree(h->d_gr_small);
  cudaFree(h->d_gr_reg); cudaFree(h->d_gr_fin); cudaFree(h->d_gr_q); cudaFree(h->d_gr_in); cudaFree(h->d_gr_run);
  for (void* p : h->mu_retired) cudaFree(p);
  for (int i = 0; i < 2; ++i) if (h->ev_stage_free[i]) cudaEventDestroy(h->ev_stage_free[i]);
  for (int i = 0; i < 2; ++i) if (h->ev_fit[i]) cudaEventDestroy(h->ev_fit[i]);
  for (int i = 0; i < 2; ++i) if (h->ev_res[i]) cudaEventDestroy(h->ev_res[i]);
  if (h->copy_stream) { cudaStreamSynchronize(h->copy_stream); cudaStreamDestroy(h->copy_stream); }
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  delete h;
  return TLOAM_B200_OK;
}

// fills the configuration part of the device context
static void fill_ctx_config(tloam_b200_handle* h) {
  DeviceCtx& c = h->ctx;
  const tloam_tls_config& f = h->cfg;
  for (int k = 0; k < 4; ++k) { const double r = radius_of(f, k); c.r2[k] = r * r; }
  c.maxnum[0] = f.edge_maxnum; c.maxnum[1] = f.sphere_maxnum; c.maxnum[2] = f.planar_maxnum; c.maxnum[3] = f.ground_maxnum;
  c.factor_num = f.factor_num; c.max_iterations = f.max_iterations; c.ceres_max_it = f.ceres_max_num_iterations;
  c.edge_dir_thres = f.edge_dir_thres; c.cost_threshold = f.cost_threshold; c.gnc_factor = f.gnc_factor;
  c.noise_bound = f.noise_bound; c.fitness_thres = f.fitness_thres;
  for (int k = 0; k < 3; ++k) c.reinit_dir[k] = f.reinit_dir[k];
  c.initial_radius = f.initial_trust_region_radius;
  c.st = h->d_state; c.stats = h->d_stats; c.counter = h->d_counter;
}

// fill (optional): the library writes the source itself -- the clouds are enqueued on the handle's stream straight into the
// staging buffer (argument: cloud k starts at point n[0] + ... + n[k-1]), xyz is not read (tloam_b200_process_cloud)
static int set_source_impl(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4], bool on_device,
                           const std::function<int(double*)>* fill = nullptr) {
  if (!h || (!xyz && !fill) || !n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  size_t total = 0, pad = 0;
  int blocks = 0;
  for (int c = 0; c < 4; ++c) {
    if (n[c] > 0 && !fill && !xyz[c]) return TLOAM_B200_ERR_INVALID_ARG;
    if (n[c] > (size_t)1 << 30) return TLOAM_B200_ERR_INVALID_ARG;
    total += n[c];
    pad += round_up(n[c], kBlk);
  }
  if (pad == 0) pad = kBlk;
  blocks = (int)(pad / kBlk);
  // host input is staged; device input is read in place -- unless the device-side submap is in use, whose update
  // appends the staged edge / ground features after the frame (tloam_b200_submap_update)
  const bool stage = !on_device || h->submap_ready || fill;
  // (re)allocations: a pointer is nulled and its capacity zeroed right after the free, and the new capacity is only
  // committed once the allocation succeeded, so a failed cudaMalloc leaves the handle consistent
  h->have_src = false; h->src_staged = false;
  static const bool no_prefetch = getenv("TLOAM_B200_NO_PREFETCH") != nullptr;   // A/B knob
  const bool prefetch = stage && !on_device && h->async_inputs && !no_prefetch;   // upload beside the frame that is still running
  if (prefetch) h->stage_cur ^= 1;
  const int sb = h->stage_cur;
  if (stage && total > h->cap_stage_buf[sb]) {
    cudaFree(h->d_stage_buf[sb]); h->d_stage_buf[sb] = nullptr; h->cap_stage_buf[sb] = 0;   // (cudaFree waits for its readers)
    h->d_stage_src = nullptr; h->cap_stage_src = 0;
    const size_t ncap = total + total / 4 + 1024;
    CU_TRY(cudaMalloc(&h->d_stage_buf[sb], ncap * 3 * sizeof(double)));
    h->cap_stage_buf[sb] = ncap;
  }
  h->d_stage_src = h->d_stage_buf[sb]; h->cap_stage_src = h->cap_stage_buf[sb];
  cudaStream_t up = prefetch ? h->src_stream : h->stream;
  if (prefetch && h->stage_free_valid[sb]) CU_TRY(cudaStreamWaitEvent(up, h->ev_stage_free[sb], 0));
  if (pad > h->cap_pad) {
    cudaFree(h->d_feat); cudaFree(h->d_flags); h->d_feat = nullptr; h->d_flags = nullptr; h->cap_pad = 0;
    const size_t ncap = round_up(pad + pad / 4, kBlk);
    CU_TRY(cudaMalloc(&h->d_feat, ncap * 11 * sizeof(double)));
    CU_TRY(cudaMalloc(&h->d_flags, ncap * 2));
    h->cap_pad = ncap;
  }
  if ((size_t)blocks > h->cap_blocks) {
    cudaFree(h->d_blk_count); cudaFree(h->d_partial); cudaFree(h->d_fit);
    h->d_blk_count = nullptr; h->d_partial = nullptr; h->d_fit = nullptr; h->cap_blocks = 0; h->cap_fit = 0;
    const size_t ncap = h->cap_pad / kBlk + 8;
    CU_TRY(cudaMalloc(&h->d_blk_count, 2 * ncap * sizeof(int)));
    CU_TRY(cudaMemsetAsync(h->d_blk_count, 0, 2 * ncap * sizeof(int), h->stream));
    CU_TRY(cudaMalloc(&h->d_partial, ncap * kNRed * sizeof(double)));
    CU_TRY(cudaMalloc(&h->d_fit, (ncap * 2 + 2) * sizeof(double)));   // + {fitness, rmse} of the side-stream reduction
    h->cap_blocks = ncap; h->cap_fit = ncap;
  }
  DeviceCtx& c = h->ctx;
  fill_ctx_config(h);
  size_t off = 0, poff = 0;
  const double* src[4];
  c.blk_off[0] = 0;
  for (int k = 0; k < 4; ++k) {
    src[k] = stage ? h->d_stage_src + 3 * off : xyz[k];
    h->src_ptr[k] = src[k];
    if (n[k] > 0 && stage && !fill)
    {
      static const bool stage_pageable = getenv("TLOAM_B200_NO_HOST_STAGE") == nullptr;
      if (!on_device && stage_pageable && n[k] * 24 >= (128u << 10) && HostStage::pageable(xyz[k])) {
        CU_TRY(h->hstage.upload(h->d_stage_src + 3 * off, xyz[k], n[k] * 3 * sizeof(double), up));
      } else {
        CU_TRY(cudaMemcpyAsync(h->d_stage_src + 3 * off, xyz[k], n[k] * 3 * sizeof(double),
                               on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, up));
      }
    }
    c.n[k] = (int)n[k];
    c.pad_off[k] = (int)poff;
    off += n[k];
    poff += round_up(n[k], kBlk);
    c.blk_off[k + 1] = (int)(poff / kBlk);
    h->n_src[k] = n[k];
  }
  double* f = h->d_feat;
  const size_t cp = h->cap_pad;
  c.px = f; c.py = f + cp; c.pz = f + 2 * cp; c.w = f + 3 * cp; c.slot = f + 4 * cp;
  for (int j = 0; j < 6; ++j) c.prim[j] = f + (5 + j) * cp;
  c.flags = h->d_flags; c.active = h->d_flags + cp;
  c.blk_count = h->d_blk_count; c.blk_cap = (int)h->cap_blocks; c.partial = h->d_partial;
  h->total_blocks = c.blk_off[4];
  if (fill) {
    const int rc = (*fill)(h->d_stage_src);
    if (rc != TLOAM_B200_OK) return rc;
  }
  if (!on_device) CU_TRY(cudaEventRecord(h->ev_src, up));             // the uploads are in; the caller's buffers are free
  if (prefetch) CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_src, 0));
  if (h->total_blocks > 0) {
    TL_LAUNCH(TLOAM_B200_K_STAGE_SOURCE, (k_stage_source<<<h->total_blocks, kBlk, 0, h->stream>>>(src[0], src[1], src[2], src[3], c, f, f + cp, f + 2 * cp)));
    CU_TRY(cudaGetLastError());
  }
  if (stage) { CU_TRY(cudaEventRecord(h->ev_stage_free[sb], h->stream)); h->stage_free_valid[sb] = true; }
  h->have_src = true;
  h->src_staged = stage;
  if (!on_device && !h->async_inputs) CU_TRY(cudaEventSynchronize(h->ev_src));    // caller buffers may be freed on return
  return TLOAM_B200_OK;
}

int tloam_b200_set_source(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4]) {
  return set_source_impl(h, xyz, n, false);
}
int tloam_b200_set_source_device(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4]) {
  return set_source_impl(h, xyz, n, true);
}

static unsigned next_pow2(size_t v) { unsigned p = 256; while ((size_t)p < v) p <<= 1; return p; }

// the blob layout is a pure function of the configuration and the four point counts (so every rank of a shared-map
// broadcast can lay the incoming blob out without reading its header back)
static size_t layout_header(const tloam_tls_config& cfg, const size_t n[4], MapHeader& hd) {
  memset(&hd, 0, sizeof(hd));
  hd.magic = kMapMagic;
  size_t off = sizeof(MapHeader);
  for (int c = 0; c < 4; ++c) {
    hd.n[c] = (unsigned)n[c];
    hd.tsize[c] = next_pow2(n[c] + 1);      // >= bricks + 1 even if every point sits in its own brick
    hd.cell[c] = radius_of(cfg, c);
    hd.pts_off[c] = off; off += round_up(n[c] * sizeof(float4), 256);
  }
  // second-level tables: at most n / kFineMin dense cells per cloud (written by the build, never zeroed)
  for (int c = 0; c < 4; ++c) { hd.fine_off[c] = off; off += round_up((n[c] / kFineMin + 1) * (size_t)kFineEntryBytes, 256); }
  for (int c = 0; c < 4; ++c) { hd.table_off[c] = off; off += (size_t)hd.tsize[c] * kBrickBytes; }
  for (int d = 0; d < 3; ++d) { hd.bbox_enc[d] = ~0ull; hd.bbox_enc[3 + d] = 0ull; }
  return off;
}

static int layout_map(tloam_b200_handle* h, const size_t n[4]) {
  const size_t off = layout_header(h->cfg, n, h->hdr);
  h->blob_bytes = off;
  if (off > h->cap_blob) {
    cudaFree(h->d_blob); h->d_blob = nullptr; h->cap_blob = 0;
    CU_TRY(cudaMalloc(&h->d_blob, off + off / 4));
    h->cap_blob = off + off / 4;
  }
  return TLOAM_B200_OK;
}

static void bind_map(tloam_b200_handle* h) {
  DeviceCtx& c = h->ctx;
  for (int k = 0; k < 4; ++k) {
    c.grid[k].pts = reinterpret_cast<const float4*>(h->d_blob + h->hdr.pts_off[k]);
    c.grid[k].table = reinterpret_cast<const uint4*>(h->d_blob + h->hdr.table_off[k]);
    c.grid[k].mask = h->hdr.tsize[k] - 1u;
    c.grid[k].n = h->hdr.n[k];
    c.grid[k].cell = h->hdr.cell[k];
    c.grid[k].inv_cell = 1.0 / h->hdr.cell[k];
    c.grid[k].fine = reinterpret_cast<const unsigned short*>(h->d_blob + h->hdr.fine_off[k]);
  }
  c.origin = reinterpret_cast<const double*>(h->d_blob + offsetof(MapHeader, origin));
  c.map_flags = reinterpret_cast<const unsigned long long*>(h->d_blob + offsetof(MapHeader, build_flags));
  c.map_bricks = reinterpret_cast<const unsigned*>(h->d_blob + offsetof(MapHeader, nbricks));
}

// the origin lives in the device header; fetch it once per map (tiny D2H) so that it can be passed by value
// (and the build flags with it: a map whose cell counters overflowed must not be searched)
static int fetch_origin(tloam_b200_handle* h) {
  if (!h->origin_known) {
    CU_TRY(cudaMemcpyAsync(h->h_result + 24, h->d_blob + offsetof(MapHeader, origin), 3 * sizeof(double),
                           cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaMemcpyAsync(h->h_result + 27, h->d_blob + offsetof(MapHeader, build_flags), sizeof(unsigned long long),
                           cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    for (int d = 0; d < 3; ++d) h->hdr.origin[d] = h->h_result[24 + d];
    memcpy(&h->hdr.build_flags, h->h_result + 27, sizeof(unsigned long long));
    h->origin_known = true;
  }
  return (h->hdr.build_flags & 1ull) ? TLOAM_B200_ERR_MAP_DENSITY : TLOAM_B200_OK;
}

static void harvest_map_stats(tloam_b200_handle* h, bool wait);

// Which clouds of the map about to be built get the second level (map_grid.cuh: kFineMin, fine_search.cuh).  The
// build kernel itself finds the dense cells; this only decides whether it is launched at all, so that sparse maps
// (BASELINE config 2: 8-25 points per occupied brick) do not pay for an empty launch.  Either choice leaves every
// search path exact.
constexpr double kFinePointsPerBrick = 256.0;    // config 2 maps: 8-25; config 3: ~1700
constexpr size_t kFineFirstMapPoints = 65536;     // no statistics yet (first map of a handle): big clouds only
static int fine_build_mask(tloam_b200_handle* h, const size_t n[4]) {
  if (h->fine_mode == 0) return 0;
  harvest_map_stats(h, false);
  int mask = 0;
  for (int c = 0; c < 4; ++c) {
    if (n[c] < kFineMin) continue;
    bool on = h->fine_mode == 1;
    if (!on) {
      if (h->stats_known) on = h->nbricks[c] > 0 && (double)h->n_tgt[c] / (double)h->nbricks[c] >= kFinePointsPerBrick;   // previous map
      else on = n[c] >= kFineFirstMapPoints;
    }
    if (on) mask |= 1 << c;
  }
  return mask;
}

static int set_target_impl(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4], bool on_device,
                           const unsigned* const* n_dev = nullptr) {
  if (!h || !xyz || !n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  size_t total = 0;
  for (int c = 0; c < 4; ++c) {
    if (n[c] > 0 && !xyz[c]) return TLOAM_B200_ERR_INVALID_ARG;
    if (n[c] > (size_t)1 << 30) return TLOAM_B200_ERR_INVALID_ARG;
    total += n[c];
  }
  h->have_tgt = false;
  bool all_staged = !on_device;                    // every host cloud went through the pageable staging ring
  if (total > h->cap_scratch) {
    cudaFree(h->d_scratch); h->d_scratch = nullptr; h->cap_scratch = 0;
    const size_t ncap = total + total / 4 + 1024;
    CU_TRY(cudaMalloc(&h->d_scratch, ncap * 2 * sizeof(unsigned)));
    h->cap_scratch = ncap;
  }
  if (!on_device && total > h->cap_stage_tgt) {
    cudaFree(h->d_stage_tgt); h->d_stage_tgt = nullptr; h->cap_stage_tgt = 0;
    const size_t ncap = total + total / 4 + 1024;
    CU_TRY(cudaMalloc(&h->d_stage_tgt, ncap * 3 * sizeof(double)));
    h->cap_stage_tgt = ncap;
  }
  const int fine_mask = fine_build_mask(h, n);
  if (fine_mask && total > h->cap_fine_tmp) {
    cudaFree(h->d_fine_tmp); h->d_fine_tmp = nullptr; h->cap_fine_tmp = 0;
    const size_t ncap = total + total / 4 + 1024;
    CU_TRY(cudaMalloc(&h->d_fine_tmp, ncap * sizeof(float4)));
    h->cap_fine_tmp = ncap;
  }
  int rc = layout_map(h, n);
  if (rc != TLOAM_B200_OK) return rc;
  h->hdr.fine_build = (unsigned)fine_mask;
  MapBuildArgs a;
  a.fine_mask = fine_mask; a.fine_tmp = h->d_fine_tmp;
  a.blob = h->d_blob; a.slot_of = h->d_scratch; a.rank_of = h->d_scratch + h->cap_scratch;
  a.only_cloud = -1;
  for (int c = 0; c < 4; ++c) a.n_dev[c] = n_dev ? n_dev[c] : nullptr;
  for (int c = 0; c < 4; ++c) h->ctx.tgt_cnt[c] = a.n_dev[c];
  size_t off = 0;
  int first = -1;                                  // first non-empty cloud: its bounding box defines the origin
  for (int c = 0; c < 4; ++c) {
    a.stage_off[c] = (unsigned)off;
    // host input is staged; device input is read in place by the build kernels (stream-ordered, no extra copy)
    a.src[c] = on_device ? xyz[c] : h->d_stage_tgt + 3 * off;
    if (first < 0 && n[c] > 0) first = c;
    off += n[c];
    h->n_tgt[c] = n[c];
  }
  a.stage_off[4] = (unsigned)off;
  // header + zeroed tables (key 0 == empty)
  CU_TRY(cudaMemcpyAsync(h->d_blob, &h->hdr, sizeof(MapHeader), cudaMemcpyHostToDevice, h->stream));
  const size_t tables_bytes = h->blob_bytes - h->hdr.table_off[0];
  CU_TRY(cudaMemsetAsync(h->d_blob + h->hdr.table_off[0], 0, tables_bytes, h->stream));
  const unsigned tb = 256;
  auto blocks_for = [&](size_t cnt) { return (unsigned)((cnt + tb - 1) / tb); };
  if (total == 0) {
    TL_LAUNCH(TLOAM_B200_K_MAP_ORIGIN, (k_map_origin<<<1, 32, 0, h->stream>>>(a)));
  } else if (on_device) {
    // inputs already in HBM: one pass over all clouds per kernel
    MapBuildArgs ab = a;
    ab.i_beg = a.stage_off[first]; ab.i_end = a.stage_off[first + 1];
    const unsigned gbb = blocks_for(n[first]);
    TL_LAUNCH(TLOAM_B200_K_MAP_BBOX, (k_map_bbox<<<(gbb < 592u ? gbb : 592u), tb, 0, h->stream>>>(ab)));   // + origin
    a.i_beg = 0; a.i_end = (unsigned)total;
    const unsigned gb = blocks_for(total);
    unsigned tslots = 0;
    for (int c = 0; c < 4; ++c) tslots += h->hdr.tsize[c];
    TL_LAUNCH(TLOAM_B200_K_MAP_INSERT, (k_map_insert<<<gb, tb, 0, h->stream>>>(a)));
    TL_LAUNCH(TLOAM_B200_K_MAP_OFFSETS, (k_map_offsets<<<(tslots + tb - 1) / tb, tb, 0, h->stream>>>(a)));
    TL_LAUNCH(TLOAM_B200_K_MAP_SCATTER, (k_map_scatter<<<gb, tb, 0, h->stream>>>(a)));
    if (fine_mask) TL_LAUNCH(TLOAM_B200_K_MAP_FINE, (k_map_fine<<<4 * h->num_sms, 128, 0, h->stream>>>(a)));
    CU_TRY(cudaGetLastError());
  } else {
    // host inputs: the clouds cross PCIe one after the other on a copy stream; cloud c is inserted, offset and
    // scattered on the compute stream while cloud c+1 is still in flight.  The origin cloud goes first, then the
    // others by descending size, so that the build left exposed after the last copy is the smallest one.
    int order[4], m = 0;
    order[m++] = first;
    for (int c = 0; c < 4; ++c) if (c != first && n[c] > 0) order[m++] = c;
    for (int i = 2; i < m; ++i)
      for (int j = i; j > 1 && n[order[j]] > n[order[j - 1]]; --j) { const int t = order[j]; order[j] = order[j - 1]; order[j - 1] = t; }
    CU_TRY(cudaEventRecord(h->ev_copy[0], h->stream));                  // the staging buffer is free once earlier work is done
    CU_TRY(cudaStreamWaitEvent(h->copy_stream, h->ev_copy[0], 0));
    static const bool stage_pageable = getenv("TLOAM_B200_NO_HOST_STAGE") == nullptr;   // A/B knob
    for (int k = 0; k < m; ++k) {
      const int c = order[k];
      if (stage_pageable && HostStage::pageable(xyz[c])) {
        CU_TRY(h->hstage.upload(h->d_stage_tgt + 3 * (size_t)a.stage_off[c], xyz[c], n[c] * 3 * sizeof(double), h->copy_stream));
      } else {
        CU_TRY(cudaMemcpyAsync(h->d_stage_tgt + 3 * (size_t)a.stage_off[c], xyz[c], n[c] * 3 * sizeof(double), cudaMemcpyHostToDevice, h->copy_stream));
        all_staged = false;
      }
      CU_TRY(cudaEventRecord(h->ev_copy[1 + c], h->copy_stream));
      h->last_uploaded = c;
    }
    for (int k = 0; k < m; ++k) {
      const int c = order[k];
      CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_copy[1 + c], 0));
      MapBuildArgs ac = a;
      ac.i_beg = a.stage_off[c]; ac.i_end = a.stage_off[c + 1]; ac.only_cloud = c;
      const unsigned gb = blocks_for(n[c]);
      if (k == 0) TL_LAUNCH(TLOAM_B200_K_MAP_BBOX, (k_map_bbox<<<(gb < 592u ? gb : 592u), tb, 0, h->stream>>>(ac)));   // + origin
      TL_LAUNCH(TLOAM_B200_K_MAP_INSERT, (k_map_insert<<<gb, tb, 0, h->stream>>>(ac)));
      TL_LAUNCH(TLOAM_B200_K_MAP_OFFSETS, (k_map_offsets<<<(h->hdr.tsize[c] + tb - 1) / tb, tb, 0, h->stream>>>(ac)));
      TL_LAUNCH(TLOAM_B200_K_MAP_SCATTER, (k_map_scatter<<<gb, tb, 0, h->stream>>>(ac)));
      if ((fine_mask >> c) & 1) {
        ac.fine_mask = 1 << c;
        TL_LAUNCH(TLOAM_B200_K_MAP_FINE, (k_map_fine<<<4 * h->num_sms, 128, 0, h->stream>>>(ac)));
      }
    }
    CU_TRY(cudaGetLastError());
  }
  bind_map(h);
  h->map_fine_mask = fine_mask;
  h->origin_known = false;
  h->have_tgt = true;
  // occupied bricks per cloud pick the search path (points per brick).  They come home with every frame's result
  // (FrameState::map_bricks); only the FIRST map of a handle is read back on its own, so that the very first frame can
  // already be routed -- both paths return the same exact neighbours, so the choice never changes a pose
  if (!h->stats_known) {
    CU_TRY(cudaMemcpyAsync(h->h_mapstats, h->d_blob + offsetof(MapHeader, nbricks), 4 * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaEventRecord(h->ev_stats, h->stream));
    h->stats_pending = true;
  }
  // host path: the caller's buffers are free once the LAST upload has landed; the build of the last cloud may
  // still be running on the compute stream (everything that follows is ordered behind it on that stream)
  // (staged pageable inputs have been read completely already: nothing to wait for)
  if (!on_device && total > 0 && !all_staged) CU_TRY(cudaEventSynchronize(h->ev_copy[1 + h->last_uploaded]));
  return TLOAM_B200_OK;
}

int tloam_b200_set_target(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4]) {
  return set_target_impl(h, xyz, n, false);
}
int tloam_b200_set_target_device(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4]) {
  return set_target_impl(h, xyz, n, true);
}

int tloam_b200_get_map_origin(tloam_b200_handle* h, double origin[3]) {
  if (!h || !origin) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  int rc = fetch_origin(h);
  if (rc != TLOAM_B200_OK) return rc;
  for (int d = 0; d < 3; ++d) origin[d] = h->hdr.origin[d];
  return TLOAM_B200_OK;
}

int tloam_b200_map_blob_size(tloam_b200_handle* h, size_t* bytes) {
  if (!h || !bytes) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  *bytes = h->blob_bytes;
  return TLOAM_B200_OK;
}

int tloam_b200_map_export(tloam_b200_handle* h, void* d_dst, size_t bytes) {
  if (!h || !d_dst) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  if (bytes < h->blob_bytes) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(d_dst, h->d_blob, h->blob_bytes, cudaMemcpyDeviceToDevice, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_map_import(tloam_b200_handle* h, const void* d_src, size_t bytes) {
  if (!h || !d_src || bytes < sizeof(MapHeader)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  MapHeader hd;
  CU_TRY(cudaMemcpy(&hd, d_src, sizeof(hd), cudaMemcpyDeviceToHost));
  if (hd.magic != kMapMagic) return TLOAM_B200_ERR_INVALID_ARG;
  size_t need = hd.table_off[3] + (size_t)hd.tsize[3] * kBrickBytes;
  if (bytes < need) return TLOAM_B200_ERR_INVALID_ARG;
  for (int c = 0; c < 4; ++c)
    if (hd.cell[c] != radius_of(h->cfg, c)) return TLOAM_B200_ERR_INVALID_ARG;   // grid cell must equal this handle's radius
  if (need > h->cap_blob) {
    cudaFree(h->d_blob);
    h->cap_blob = need + need / 4;
    CU_TRY(cudaMalloc(&h->d_blob, h->cap_blob));
  }
  CU_TRY(cudaMemcpyAsync(h->d_blob, d_src, need, cudaMemcpyDeviceToDevice, h->stream));
  h->hdr = hd;
  h->blob_bytes = need;
  for (int c = 0; c < 4; ++c) h->n_tgt[c] = hd.n[c];
  fill_ctx_config(h);
  bind_map(h);
  h->origin_known = true;
  h->have_tgt = true;
  for (int c = 0; c < 4; ++c) h->nbricks[c] = hd.nbricks[c];
  h->map_fine_mask = (int)hd.fine_build;
  h->stats_known = true; h->stats_pending = false;
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}


// ---- zero-copy shared-map transport (config 4): ONE collective, no size handshake, no host synchronisation ----
// sender: the built blob itself (no export copy).  The consumer stream must be ordered behind the build:
// tloam_b200_signal_stream(h, consumer_stream).
int tloam_b200_map_send_buffer(tloam_b200_handle* h, void** d_ptr, size_t* bytes) {
  if (!h || !d_ptr || !bytes) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  *d_ptr = h->d_blob; *bytes = h->blob_bytes;
  return TLOAM_B200_OK;
}

int tloam_b200_map_layout_bytes(tloam_b200_handle* h, const size_t n[4], size_t* bytes) {
  if (!h || !n || !bytes) return TLOAM_B200_ERR_INVALID_ARG;
  MapHeader hd;
  *bytes = layout_header(h->cfg, n, hd);
  return TLOAM_B200_OK;
}

// receiver: where the broadcast of a map with these point counts must land -- a SECOND blob of the handle, so frames
// keep registering against the active map while the next one is in flight.
int tloam_b200_map_recv_buffer(tloam_b200_handle* h, const size_t n[4], void** d_ptr, size_t* bytes) {
  if (!h || !n || !d_ptr || !bytes) return TLOAM_B200_ERR_INVALID_ARG;
  for (int c = 0; c < 4; ++c) if (n[c] > (size_t)1 << 30) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  const size_t need = layout_header(h->cfg, n, h->hdr_in);
  if (need > h->cap_blob_in) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_blob_in); h->d_blob_in = nullptr; h->cap_blob_in = 0;
    CU_TRY(cudaMalloc(&h->d_blob_in, need + need / 4));
    h->cap_blob_in = need + need / 4;
  }
  h->blob_in_bytes = need; h->blob_in_ready = true;
  *d_ptr = h->d_blob_in; *bytes = need;
  return TLOAM_B200_OK;
}

// receiver: the collective that fills the receive buffer has been ENQUEUED on producer_stream.  Orders the handle's
// stream behind it (device-side wait) and makes the received blob the active map: no copy, no host synchronisation.
int tloam_b200_map_adopt(tloam_b200_handle* h, void* producer_stream) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->blob_in_ready) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  if ((cudaStream_t)producer_stream != h->stream) {
    CU_TRY(cudaEventRecord(h->ev_copy[0], (cudaStream_t)producer_stream));
    CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_copy[0], 0));
  }
  std::swap(h->d_blob, h->d_blob_in);
  std::swap(h->cap_blob, h->cap_blob_in);
  h->blob_bytes = h->blob_in_bytes;
  h->hdr = h->hdr_in;
  h->blob_in_ready = false;
  for (int c = 0; c < 4; ++c) { h->n_tgt[c] = h->hdr.n[c]; h->ctx.tgt_cnt[c] = nullptr; }
  fill_ctx_config(h);
  bind_map(h);
  h->map_fine_mask = 0xF;                  // unknown without reading the header: bricks without a second level say so themselves
  h->origin_known = false;                 // lives in the received header on the device; fetched lazily if ever asked for
  h->stats_pending = false;                // occupied-brick statistics stay those of the previous map
  h->have_tgt = true;
  return TLOAM_B200_OK;
}

// orders `consumer_stream` behind everything enqueued so far on the handle's stream (device-side wait)
int tloam_b200_signal_stream(tloam_b200_handle* h, void* consumer_stream) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if ((cudaStream_t)consumer_stream == h->stream) return TLOAM_B200_OK;
  CU_TRY(cudaEventRecord(h->ev_copy[1], h->stream));
  CU_TRY(cudaStreamWaitEvent((cudaStream_t)consumer_stream, h->ev_copy[1], 0));
  return TLOAM_B200_OK;
}

static int check_ready(tloam_b200_handle* h) {
  if (!h->have_src || !h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  for (int c = 0; c < 4; ++c)
    if (h->n_src[c] < 10 || h->n_tgt[c] < 10) return TLOAM_B200_ERR_TOO_FEW_POINTS;   // ref: :928-929
  return TLOAM_B200_OK;
}


// ---- dense-map path: decision + scratch ----
static void harvest_map_stats(tloam_b200_handle* h, bool wait) {
  if (!h->stats_pending) return;
  if (wait) cudaEventSynchronize(h->ev_stats);
  else if (cudaEventQuery(h->ev_stats) != cudaSuccess) { cudaGetLastError(); return; }
  for (int c = 0; c < 4; ++c) h->nbricks[c] = h->h_mapstats[c];
  h->stats_pending = false; h->stats_known = true;
}

// exact accumulator counts (device) -> tighter host bounds, whenever an asynchronous read-back has landed
static void harvest_counts(tloam_b200_handle* h) {
  for (int i = 0; i < 4; ++i) {
    tloam_b200_handle::CntProbe& pr = h->probes[i];
    if (!pr.pending) continue;
    if (cudaEventQuery(pr.ev) != cudaSuccess) { cudaGetLastError(); continue; }
    pr.pending = false;
    for (int k = 0; k < 2; ++k)
      if (pr.cum[k] >= h->known_cum[k]) { h->known_cum[k] = pr.cum[k]; h->known_cnt[k] = pr.h_vals[k]; }
  }
  for (int k = 0; k < 2; ++k) {
    const size_t bound = h->known_cnt[k] + (size_t)(h->cum_add[k] - h->known_cum[k]);
    if (bound < h->n_acc[k]) h->n_acc[k] = bound;
  }
}

constexpr double kDensePointsPerBrick = 256.0;   // config 2 maps: 8-25; config 3: ~1700
constexpr size_t kDenseMinQueries = 2048;

// clouds served by the two-level search (k_correspond_fine): built with the second level and dense (or not yet known)
static int fine_mask_of(tloam_b200_handle* h) {
  if (h->fine_mode == 0 || h->map_fine_mask == 0) return 0;
  harvest_map_stats(h, false);
  int mask = 0;
  for (int c = 0; c < 4; ++c) {
    const bool enabled = (c == kPlanar || c == kGround) ? true : (c == kEdge ? h->cfg.factor_num >= 3 : h->cfg.factor_num == 4);
    if (!enabled || h->n_src[c] == 0 || h->n_tgt[c] == 0 || !((h->map_fine_mask >> c) & 1)) continue;
    const bool dense = !h->stats_known || (h->nbricks[c] > 0 && (double)h->n_tgt[c] / (double)h->nbricks[c] >= kFinePointsPerBrick);
    if (h->fine_mode == 1 || dense) mask |= 1 << c;
  }
  return mask;
}

static int dense_mask_of(tloam_b200_handle* h) {
  h->dense_kernel = 0;
  if (h->dense_mode == 0) {
    const int fm = fine_mask_of(h);
    if (fm) h->dense_kernel = 2;
    return fm;
  }
  h->dense_kernel = 1;
  harvest_map_stats(h, !h->stats_known);         // the very first map of a handle: wait once for its statistics
  int mask = 0;
  for (int c = 0; c < 4; ++c) {
    if (c == kSphere) continue;                   // K = 1 search: lane-pair path only
    const bool enabled = (c == kPlanar || c == kGround) ? true : h->cfg.factor_num >= 3;
    if (!enabled || h->n_src[c] == 0 || h->n_tgt[c] == 0) continue;
    const bool dense = h->nbricks[c] > 0 && (double)h->n_tgt[c] / (double)h->nbricks[c] >= kDensePointsPerBrick &&
                       h->n_src[c] >= kDenseMinQueries;
    if (h->dense_mode == 1 || dense) mask |= 1 << c;
  }
  return mask;
}

static int prepare_dense(tloam_b200_handle* h, int mask) {
  DenseArgs a;
  memset(&a, 0, sizeof(a));
  a.mask = mask;
  size_t off = 256;                              // ctl words first
  size_t total_q = 0;
  unsigned toff = 0;
  size_t o_keys[4] = {0, 0, 0, 0}, o_cnt[4] = {0, 0, 0, 0};
  unsigned ts[4] = {0, 0, 0, 0};
  for (int c = 0; c < 4; ++c) {
    if (!((mask >> c) & 1)) continue;
    ts[c] = next_pow2(2 * h->n_src[c] + 1);
    o_keys[c] = off; off += (size_t)ts[c] * 8;
    o_cnt[c] = off; off += (size_t)ts[c] * 4;
    total_q += h->n_src[c];
  }
  const size_t zero_bytes = off;
  size_t o_base[4], o_slot[4], o_rank[4], o_order[4];
  for (int c = 0; c < 4; ++c) {
    if (!((mask >> c) & 1)) continue;
    o_base[c] = off; off += (size_t)ts[c] * 4;
    o_slot[c] = off; off += round_up(h->n_src[c] * 4, 256);
    o_rank[c] = off; off += round_up(h->n_src[c] * 4, 256);
    o_order[c] = off; off += round_up(h->n_src[c] * 4, 256);
  }
  const size_t o_work = off; off += total_q * sizeof(DenseWork);
  if (off > h->cap_dense) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_dense); h->d_dense = nullptr; h->cap_dense = 0;
    CU_TRY(cudaMalloc(&h->d_dense, off + off / 4));
    h->cap_dense = off + off / 4;
  }
  unsigned char* b = h->d_dense;
  for (int c = 0; c < 4; ++c) {
    if (!((mask >> c) & 1)) continue;
    DenseCloud& q = a.cl[c];
    q.keys = (unsigned long long*)(b + o_keys[c]); q.cnt = (unsigned*)(b + o_cnt[c]); q.base = (unsigned*)(b + o_base[c]);
    q.q_slot = (unsigned*)(b + o_slot[c]); q.q_rank = (unsigned*)(b + o_rank[c]); q.q_order = (unsigned*)(b + o_order[c]);
    q.tmask = ts[c] - 1u; q.toff = toff; toff += ts[c];
  }
  a.work = (DenseWork*)(b + o_work);
  a.ctl = (unsigned*)b;
  a.tslots = toff;
  a.dbg = h->dense_check ? h->d_cnt + 16 : nullptr;          // d_cnt[16..23]: self-check counters
  h->dargs = a;
  h->dense_zero_bytes = zero_bytes;
  if (!h->dense_attr_set) {
    CU_TRY(cudaFuncSetAttribute(k_correspond_dense, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDenseSmemBytes));
    h->dense_attr_set = true;
  }
  return TLOAM_B200_OK;
}

// true when no `*_maxnum` cap can bind for any enabled cloud: the fused first evaluation (k_first) applies
static bool caps_cannot_bind(const tloam_b200_handle* h) {
  const DeviceCtx& c = h->ctx;
  for (int k = 0; k < 4; ++k) {
    const bool enabled = (k == kPlanar || k == kGround) ? true : (k == kEdge ? c.factor_num >= 3 : c.factor_num == 4);
    if (enabled && c.maxnum[k] < c.n[k]) return false;
  }
  return true;
}

static constexpr size_t kFrameResultBytes = 16 * sizeof(double) + 2 * sizeof(int) + 2 * sizeof(double) + 4 * sizeof(unsigned);
static BatchTab no_batch() { BatchTab t; memset(&t, 0, sizeof(t)); t.S = 1; return t; }

// correspondence search + fit of one outer iteration as kernels of their own (un-fused sequence, build_factors)
static int enqueue_correspond(tloam_b200_handle* h, const DeviceCtx& c) {
  const int nb = h->total_blocks;
  if (c.dense_mask && h->dense_kernel == 2) {
    // dense map clouds: two-level grid, one thread per feature (fine_search.cuh)
    TL_LAUNCH(TLOAM_B200_K_FINE, (k_correspond_fine<false><<<nb, kBlk, kFineSmemBytes, h->stream>>>(c, no_batch(), h->dense_check ? h->d_cnt + 16 : nullptr)));
  } else if (c.dense_mask) {
    // dense map clouds: bin the queries by map cell, then the TMA-staged block-per-cell search (dense_search.cuh)
    const DenseArgs& da = h->dargs;
    CU_TRY(cudaMemsetAsync(h->d_dense, 0, h->dense_zero_bytes, h->stream));
    TL_LAUNCH(TLOAM_B200_K_DENSE_BIN, (k_qbin_count<<<nb, kBlk, 0, h->stream>>>(c, da)));
    TL_LAUNCH(TLOAM_B200_K_DENSE_BIN, (k_qbin_offsets<<<(da.tslots + 255) / 256, 256, 0, h->stream>>>(c, da)));
    TL_LAUNCH(TLOAM_B200_K_DENSE_BIN, (k_qbin_scatter<<<nb, kBlk, 0, h->stream>>>(c, da)));
    TL_LAUNCH(TLOAM_B200_K_DENSE, (k_correspond_dense<<<h->num_sms, kDenseThreads, kDenseSmemBytes, h->stream>>>(c, da)));
  }
  TL_LAUNCH(TLOAM_B200_K_CORRESPOND, (k_correspond<false><<<nb * 2, kBlk, 0, h->stream>>>(c, no_batch())));
  return TLOAM_B200_OK;
}

// enqueues the frame's fixed launch sequence on h->stream (also used under stream capture)
static int enqueue_frame(tloam_b200_handle* h, const DeviceCtx& c, bool fused) {
  const int nb = h->total_blocks;
  const int ne = eval_grid_of(nb), nf = first_grid_of(nb);
  const BatchTab nt = no_batch();
  // per-frame health metric (ref: registration.cpp:257-296): the reference queries the UNTRANSFORMED scan, so the two
  // kernels depend on the staged scan and the map only -- they run on a side stream beside the registration (a fork /
  // join inside the captured graph; the frame leaves 85 % of the SMs idle) and join before the result is copied.
  // With profiling on (events around every launch on h->stream) they stay in line.
  const bool fit = h->frame_fitness && nb > 0;
  static const bool fit_inline = getenv("TLOAM_B200_FIT_INLINE") != nullptr;      // A/B knob
  cudaStream_t fs = (h->profiling || fit_inline) ? h->stream : h->fit_stream;
  if (fit) {
    if (fs != h->stream) {
      CU_TRY(cudaEventRecord(h->ev_fit[0], h->stream));
      CU_TRY(cudaStreamWaitEvent(fs, h->ev_fit[0], 0));
    }
    TL_LAUNCH(TLOAM_B200_K_FITNESS, (k_fitness<<<nb, kBlk, 0, fs>>>(c, h->cfg.fitness_thres * h->cfg.fitness_thres, h->d_fit)));
    TL_LAUNCH(TLOAM_B200_K_FITNESS, (k_fitness_reduce<<<1, 128, 0, fs>>>(c, h->d_fit, h->d_fit + 2 * h->cap_fit)));
    if (fs != h->stream) CU_TRY(cudaEventRecord(h->ev_fit[1], fs));
  }
  CU_TRY(cudaMemcpyAsync(h->d_predict, h->h_predict, sizeof(Predict), cudaMemcpyHostToDevice, h->stream));
  TL_LAUNCH(TLOAM_B200_K_BEGIN_FRAME, (k_begin_frame<false><<<1, 256, 0, h->stream>>>(c, nt, h->d_predict)));
  for (int outer = 0; outer < h->cfg.max_iterations; ++outer) {
    if (fused) {
      TL_LAUNCH(TLOAM_B200_K_FIRST, (k_first<false><<<nf, kBlk, 0, h->stream>>>(c, nt)));
    } else {
      const int crc = enqueue_correspond(h, c);
      if (crc != TLOAM_B200_OK) return crc;
      TL_LAUNCH(TLOAM_B200_K_EVAL_FIRST, (k_eval<true, false><<<ne, kBlk, 0, h->stream>>>(c, nt)));
    }
    for (int it = 0; it < h->cfg.ceres_max_num_iterations; ++it)
      TL_LAUNCH(TLOAM_B200_K_EVAL, (k_eval<false, false><<<ne, kBlk, 0, h->stream>>>(c, nt)));
  }
  if (fit) {
    if (fs != h->stream) CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_fit[1], 0));        // join
    // into the frame state only now: the solver blocks write the whole state back while the frame runs
    CU_TRY(cudaMemcpyAsync((char*)h->d_state + offsetof(FrameState, fitness), h->d_fit + 2 * h->cap_fit, 2 * sizeof(double),
                           cudaMemcpyDeviceToDevice, h->stream));
  }
  // result[16] + {frame_done, status} + {fitness, rmse}: contiguous in FrameState.  Pipelined handles copy it after the
  // graph launch into alternating slots instead (scan_match_enqueue)
  if (!h->async_inputs)
    CU_TRY(cudaMemcpyAsync(h->h_result, (const char*)h->d_state + offsetof(FrameState, result), kFrameResultBytes,
                           cudaMemcpyDeviceToHost, h->stream));
  return TLOAM_B200_OK;
}

static int scan_match_enqueue(tloam_b200_handle* h, const double* predict);

int tloam_b200_scan_match_async(tloam_b200_handle* h, const double predict[16]) {
  if (!h || !predict) return TLOAM_B200_ERR_INVALID_ARG;
  return scan_match_enqueue(h, predict);
}

// (f)-3: the frame is predicted on the device from the two last results (no host input at all)
int tloam_b200_scan_match_predicted_async(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  return scan_match_enqueue(h, nullptr);
}

int tloam_b200_scan_match_predicted(tloam_b200_handle* h, double result[16], tloam_b200_stats* stats) {
  const int rc = tloam_b200_scan_match_predicted_async(h);
  if (rc != TLOAM_B200_OK) return rc;
  return tloam_b200_get_result(h, result, stats);
}

int tloam_b200_set_pose_history(tloam_b200_handle* h, const double last_pose[16], const double curr_pose[16]) {
  if (!h || !last_pose || !curr_pose) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  CU_TRY(cudaMemcpy((char*)h->d_state + offsetof(FrameState, last_pose), last_pose, 16 * sizeof(double), cudaMemcpyHostToDevice));
  CU_TRY(cudaMemcpy((char*)h->d_state + offsetof(FrameState, curr_pose), curr_pose, 16 * sizeof(double), cudaMemcpyHostToDevice));
  return TLOAM_B200_OK;
}

static int scan_match_enqueue(tloam_b200_handle* h, const double* predict) {
  const int rc = check_ready(h);
  if (rc != TLOAM_B200_OK) return rc;
  if (h->async_inputs && h->frames_enqueued - h->frames_fetched >= 2) return TLOAM_B200_ERR_NOT_READY;   // fetch a result first
  if (h->frame_fitness) {
    if (h->cfg.fitness_thres <= 0.0) return TLOAM_B200_ERR_INVALID_ARG;
    for (int c = 0; c < 4; ++c) if (h->cfg.fitness_thres > radius_of(h->cfg, c)) return TLOAM_B200_ERR_INVALID_ARG;
  }
  CU_TRY(cudaSetDevice(h->device));
  if (predict) { memcpy(h->h_predict->m, predict, 16 * sizeof(double)); h->h_predict->from_state = 0.0; }
  else h->h_predict->from_state = 1.0;
  DeviceCtx c = h->ctx;
  if (!h->trace) c.stats = nullptr;             // skip the per-iteration trace (fewer instructions in the serial solver)
  c.dense_mask = dense_mask_of(h);
  if (c.dense_mask && h->dense_kernel == 1) { const int drc = prepare_dense(h, c.dense_mask); if (drc != TLOAM_B200_OK) return drc; }
  const bool fused = h->use_fused && caps_cannot_bind(h) && c.dense_mask == 0;
  const int per_frame = 1 + h->cfg.max_iterations * ((fused ? 1 : 2) + (c.dense_mask ? (h->dense_kernel == 1 ? 4 : 1) : 0) + h->cfg.ceres_max_num_iterations) +
                        (h->frame_fitness ? 2 : 0);
  CU_TRY(cudaEventRecord(h->ev0, h->stream));
  if (h->use_graph && !h->profiling) {
    // one graph launch per frame; the graph is re-captured only when the device context changed
    if (!h->gvalid || h->gfused != fused || h->gfitness != h->frame_fitness || memcmp(&h->gctx, &c, sizeof(DeviceCtx)) != 0 ||
        h->gdense_kernel != h->dense_kernel ||
        (c.dense_mask && h->dense_kernel == 1 && memcmp(&h->gdargs, &h->dargs, sizeof(DenseArgs)) != 0)) {
      h->gvalid = false;
      cudaGraph_t graph = nullptr;
      CU_TRY(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
      const long long l0 = h->launches;
      const int erc = enqueue_frame(h, c, fused);
      h->launches = l0;                           // capture does not execute anything
      cudaError_t ce = cudaStreamEndCapture(h->stream, &graph);
      if (erc != TLOAM_B200_OK || ce != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        snprintf(h->last_error, sizeof(h->last_error), "graph capture failed: %s", cudaGetErrorString(ce));
        return TLOAM_B200_ERR_CUDA;
      }
      // same topology, new kernel parameters / grid sizes (cloud sizes change from frame to frame in a real
      // stream): update the instantiated graph in place, which is much cheaper than instantiating a new one
      bool updated = false;
      if (h->gexec && h->gfused == fused && h->gfitness == h->frame_fitness && h->gctx.dense_mask == c.dense_mask &&
          h->gdense_kernel == h->dense_kernel) {
        cudaGraphExecUpdateResultInfo info;
        updated = cudaGraphExecUpdate(h->gexec, graph, &info) == cudaSuccess;
        if (!updated) { cudaGetLastError(); cudaGraphExecDestroy(h->gexec); h->gexec = nullptr; }
      }
      if (!updated) ce = cudaGraphInstantiate(&h->gexec, graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) { snprintf(h->last_error, sizeof(h->last_error), "graph instantiate: %s", cudaGetErrorString(ce)); return TLOAM_B200_ERR_CUDA; }
      h->gctx = c;
      h->gdargs = h->dargs;
      h->gdense_kernel = h->dense_kernel;
      h->gfused = fused;
      h->gfitness = h->frame_fitness;
      h->gvalid = true;
    }
    CU_TRY(cudaGraphLaunch(h->gexec, h->stream));
    h->launches += per_frame;
  } else {
    const int erc = enqueue_frame(h, c, fused);
    if (erc != TLOAM_B200_OK) return erc;
    CU_TRY(cudaGetLastError());
  }
  CU_TRY(cudaEventRecord(h->ev1, h->stream));
  if (h->async_inputs) {                         // pipelined: result -> slot (frame & 1), one event per slot
    const int p = (int)(h->frames_enqueued & 1);
    CU_TRY(cudaMemcpyAsync(h->h_result + 32 * p, (const char*)h->d_state + offsetof(FrameState, result), kFrameResultBytes,
                           cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaEventRecord(h->ev_res[p], h->stream));
  }
  h->frames_enqueued++;
  h->launches_frame = per_frame;
  h->traced_last = h->trace;
  h->frame_pending = true;
  return TLOAM_B200_OK;
}

int tloam_b200_get_result(tloam_b200_handle* h, double result[16], tloam_b200_stats* stats) {
  if (!h || !result) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->frame_pending) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  if (stats && !h->traced_last) memset(h->h_stats, 0, sizeof(tloam_b200_stats));
  const double* slot = h->h_result;
  if (h->async_inputs) {
    // pipelined: the OLDEST un-fetched frame; waits for that frame only (the host may already have enqueued the next)
    if (h->frames_fetched >= h->frames_enqueued) return TLOAM_B200_ERR_NOT_READY;
    const int p = (int)(h->frames_fetched & 1);
    CU_TRY(cudaEventSynchronize(h->ev_res[p]));
    slot = h->h_result + 32 * p;
    h->frames_fetched++;
    h->frame_pending = h->frames_fetched < h->frames_enqueued;
    if (stats) memset(h->h_stats, 0, sizeof(tloam_b200_stats));      // no per-iteration trace in pipelined mode
  } else {
    if (stats && h->traced_last) CU_TRY(cudaMemcpyAsync(h->h_stats, h->d_stats, sizeof(tloam_b200_stats), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    h->frame_pending = false;
    h->frames_fetched = h->frames_enqueued;
  }
  harvest_counts(h);
  memcpy(result, slot, 16 * sizeof(double));
  int flags[2];
  memcpy(flags, slot + 16, sizeof(flags));   // frame_done, status
  h->last_fitness = slot[17]; h->last_rmse = slot[18];
  memcpy(h->nbricks, slot + 19, 4 * sizeof(unsigned));   // statistics of the map this frame used: route the next frames
  h->stats_known = true; h->stats_pending = false;
  if (stats) {
    *stats = *h->h_stats;
    stats->gpu_launches = h->launches_frame;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, h->ev0, h->ev1) == cudaSuccess) stats->gpu_ms = ms;
  }
  if (flags[1] != TLOAM_B200_OK) return flags[1];
  if (!flags[0]) { snprintf(h->last_error, sizeof(h->last_error), "frame did not complete"); return TLOAM_B200_ERR_CUDA; }
  return TLOAM_B200_OK;
}

int tloam_b200_scan_match(tloam_b200_handle* h, const double predict[16], double result[16], tloam_b200_stats* stats) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  const bool saved = h->trace;
  if (stats) h->trace = true;                   // the blocking form knows whether the caller wants the trace
  int rc = tloam_b200_scan_match_async(h, predict);
  h->trace = saved;
  if (rc != TLOAM_B200_OK) return rc;
  return tloam_b200_get_result(h, result, stats);
}

int tloam_b200_set_trace(tloam_b200_handle* h, int on) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  h->trace = on != 0;
  return TLOAM_B200_OK;
}

// Orders the handle's stream behind everything enqueued so far on `producer_stream` (a cudaStream_t; NULL = the legacy
// default stream): device inputs (set_*_device) are read IN PLACE by kernels on the handle's stream, so whoever
// produced them on another stream must be waited for -- on the device, the host does not block.
int tloam_b200_wait_stream(tloam_b200_handle* h, void* producer_stream) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if ((cudaStream_t)producer_stream == h->stream) return TLOAM_B200_OK;
  CU_TRY(cudaEventRecord(h->ev_src, (cudaStream_t)producer_stream));
  CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_src, 0));
  return TLOAM_B200_OK;
}

// self-check counters of the dense correspondence path (TLOAM_B200_DENSE_CHECK=1), accumulated since creation:
// [0] queries searched, [1] kNN lists that differ from the plain search, [2] work items, [3] staging passes
int tloam_b200_dense_check_counters(tloam_b200_handle* h, unsigned out[16]) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  CU_TRY(cudaMemcpy(out, h->d_cnt + 16, 16 * sizeof(unsigned), cudaMemcpyDeviceToHost));
  return TLOAM_B200_OK;
}

int tloam_b200_synchronize(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

long long tloam_b200_launch_count(tloam_b200_handle* h) { return h ? h->launches : 0; }

static int read_state_pose(tloam_b200_handle* h, size_t offset, double out[16]) {
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(h->h_result, (const char*)h->d_state + offset, 16 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  memcpy(out, h->h_result, 16 * sizeof(double));
  return TLOAM_B200_OK;
}

int tloam_b200_get_transform(tloam_b200_handle* h, double pose[16]) {   // ref: registration.cpp:370-372
  if (!h || !pose) return TLOAM_B200_ERR_INVALID_ARG;
  return read_state_pose(h, offsetof(FrameState, curr_pose), pose);
}

int tloam_b200_get_pose_increment(tloam_b200_handle* h, double pose[16]) {   // ref: registration.cpp:374-376
  if (!h || !pose) return TLOAM_B200_ERR_INVALID_ARG;
  double L[16], C[16];
  int rc = read_state_pose(h, offsetof(FrameState, last_pose), L);
  if (rc != TLOAM_B200_OK) return rc;
  rc = read_state_pose(h, offsetof(FrameState, curr_pose), C);
  if (rc != TLOAM_B200_OK) return rc;
  double Li[16];
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) Li[c * 4 + r] = L[r * 4 + c];
  for (int r = 0; r < 3; ++r) Li[12 + r] = -(Li[0 * 4 + r] * L[12] + Li[1 * 4 + r] * L[13] + Li[2 * 4 + r] * L[14]);
  Li[3] = Li[7] = Li[11] = 0.0; Li[15] = 1.0;
  for (int c = 0; c < 4; ++c) for (int r = 0; r < 4; ++r) {
    double s = 0.0;
    for (int k = 0; k < 4; ++k) s += Li[k * 4 + r] * C[c * 4 + k];
    pose[c * 4 + r] = s;
  }
  return TLOAM_B200_OK;
}


// ---------------------------------------------------------------------------------------------
// Batched registration: S independent sequences stepped together, ONE launch sequence per batch frame.
// A single 40k-feature frame is 8.5 warps per SM and every evaluation ends in a ~9 us serial tail on one SM
// (DESIGN.md section 4); batching fills the machine with the sequences' parallel phases and runs their tails
// concurrently.  Each sequence keeps its own handle (map, scan, pose history, submap); only the frame kernels
// are shared.  Poses are bit-identical to registering each sequence alone (same per-sequence reduction tree).
// ---------------------------------------------------------------------------------------------
struct tloam_b200_batch {
  int S = 0, device = 0;
  std::vector<tloam_b200_handle*> hs;
  cudaStream_t stream = nullptr;
  FrameState* d_states = nullptr;
  DeviceCtx* d_ctxs = nullptr;
  std::vector<DeviceCtx> ctx_sent;   bool ctx_valid = false;
  Predict* h_pred = nullptr; Predict* d_pred = nullptr;
  unsigned char* h_results = nullptr;          // pinned [S][kResultBytes]
  cudaEvent_t ev_done = nullptr, ev0 = nullptr, ev1 = nullptr;
  std::vector<cudaEvent_t> ev_ready;
  cudaGraphExec_t gexec = nullptr;
  BatchTab g_first, g_corr, g_eval, g_fine; bool gfused = false, gvalid = false;
  bool any_fine = false, gany_fine = false;          // some sequence has clouds served by the two-level search
  bool use_graph = true, use_fused = false, pending = false;
  long long launches = 0; int launches_frame = 0;
  char last_error[512] = {0};
  // optional per-kernel-class timing (CUDA events around every launch of the batch frame; no graph in this mode)
  bool profiling = false;
  std::vector<cudaEvent_t> ev_pool; size_t ev_next = 0;
  struct Span { int cls; cudaEvent_t a, b; };
  std::vector<Span> spans;
  tloam_b200_profile prof;
};
struct BatchLaunchScope {
  tloam_b200_batch* b; int cls; cudaEvent_t a = nullptr, e = nullptr;
  BatchLaunchScope(tloam_b200_batch* bb, int c) : b(bb), cls(c) {
    if (b->profiling) {
      while (b->ev_pool.size() < b->ev_next + 2) { cudaEvent_t ev; if (cudaEventCreate(&ev) != cudaSuccess) { b->profiling = false; return; } b->ev_pool.push_back(ev); }
      a = b->ev_pool[b->ev_next++]; e = b->ev_pool[b->ev_next++];
      cudaEventRecord(a, b->stream);
    }
  }
  ~BatchLaunchScope() { if (a && e) { cudaEventRecord(e, b->stream); b->spans.push_back({cls, a, e}); } }
};
#define TLB_LAUNCH(cls, ...) do { BatchLaunchScope ls__(b, cls); __VA_ARGS__; } while (0)
static constexpr size_t kResultBytes = 16 * sizeof(double) + 2 * sizeof(int);   // result + {frame_done, status}

#define CUB_TRY(expr)                                                                                  \
  do {                                                                                                 \
    cudaError_t e__ = (expr);                                                                          \
    if (e__ != cudaSuccess) {                                                                          \
      snprintf(b->last_error, sizeof(b->last_error), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), \
               __FILE__, __LINE__);                                                                    \
      return TLOAM_B200_ERR_CUDA;                                                                      \
    }                                                                                                  \
  } while (0)

int tloam_b200_batch_destroy(tloam_b200_batch* b) {
  if (!b) return TLOAM_B200_OK;
  cudaSetDevice(b->device);
  if (b->stream) cudaStreamSynchronize(b->stream);
  for (tloam_b200_handle* h : b->hs) tloam_b200_destroy(h);
  if (b->gexec) cudaGraphExecDestroy(b->gexec);
  cudaFree(b->d_states); cudaFree(b->d_ctxs); cudaFree(b->d_pred);
  if (b->h_pred) cudaFreeHost(b->h_pred);
  if (b->h_results) cudaFreeHost(b->h_results);
  for (cudaEvent_t e : b->ev_ready) cudaEventDestroy(e);
  for (cudaEvent_t e : b->ev_pool) cudaEventDestroy(e);
  if (b->ev_done) cudaEventDestroy(b->ev_done);
  if (b->ev0) cudaEventDestroy(b->ev0);
  if (b->ev1) cudaEventDestroy(b->ev1);
  if (b->stream) cudaStreamDestroy(b->stream);
  delete b;
  return TLOAM_B200_OK;
}

int tloam_b200_batch_create(const tloam_tls_config* cfg, int device, int S, tloam_b200_batch** out) {
  if (!cfg || !out || S < 1 || S > kMaxBatch) return TLOAM_B200_ERR_INVALID_ARG;
  *out = nullptr;
  tloam_b200_batch* b = new (std::nothrow) tloam_b200_batch();
  if (!b) return TLOAM_B200_ERR_INVALID_ARG;
  b->S = S; b->device = device;
  auto fail = [&](int code) { tloam_b200_batch_destroy(b); return code; };
  for (int s = 0; s < S; ++s) {
    tloam_b200_handle* h = nullptr;
    const int rc = tloam_b200_create(cfg, device, nullptr, &h);     // own non-blocking stream: map builds of the sequences overlap
    if (rc != TLOAM_B200_OK) return fail(rc);
    b->hs.push_back(h);
  }
  if (cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
  if (cudaMalloc(&b->d_states, S * sizeof(FrameState)) != cudaSuccess || cudaMalloc(&b->d_ctxs, S * sizeof(DeviceCtx)) != cudaSuccess ||
      cudaMalloc(&b->d_pred, S * sizeof(Predict)) != cudaSuccess || cudaMallocHost(&b->h_pred, S * sizeof(Predict)) != cudaSuccess ||
      cudaMallocHost(&b->h_results, S * kResultBytes) != cudaSuccess)
    return fail(TLOAM_B200_ERR_CUDA);
  if (cudaEventCreateWithFlags(&b->ev_done, cudaEventDisableTiming) != cudaSuccess || cudaEventCreate(&b->ev0) != cudaSuccess ||
      cudaEventCreate(&b->ev1) != cudaSuccess)
    return fail(TLOAM_B200_ERR_CUDA);
  for (int s = 0; s < S; ++s) {
    cudaEvent_t e;
    if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
    b->ev_ready.push_back(e);
    // the sequences' frame states live in ONE array (one strided D2H copy fetches every result)
    tloam_b200_handle* h = b->hs[s];
    if (cudaMemcpy(b->d_states + s, h->d_state, sizeof(FrameState), cudaMemcpyDeviceToDevice) != cudaSuccess) return fail(TLOAM_B200_ERR_CUDA);
    cudaFree(h->d_state);
    h->d_state = b->d_states + s; h->own_state = false;
  }
  { const char* e = getenv("TLOAM_B200_NO_GRAPH"); b->use_graph = !(e && e[0] == '1'); }
  { const char* e = getenv("TLOAM_B200_FUSE"); b->use_fused = (e && e[0] == '1'); }
  { const char* e = getenv("TLOAM_B200_NO_FUSE"); if (e && e[0] == '1') b->use_fused = false; }
  *out = b;
  return TLOAM_B200_OK;
}

int tloam_b200_batch_size(tloam_b200_batch* b) { return b ? b->S : 0; }
tloam_b200_handle* tloam_b200_batch_handle(tloam_b200_batch* b, int i) { return (b && i >= 0 && i < b->S) ? b->hs[i] : nullptr; }
const char* tloam_b200_batch_last_error(tloam_b200_batch* b) { return b ? b->last_error : ""; }
long long tloam_b200_batch_launch_count(tloam_b200_batch* b) {
  if (!b) return 0;
  long long n = b->launches;
  for (tloam_b200_handle* h : b->hs) n += h->launches;
  return n;
}

static int batch_set(tloam_b200_batch* b, const double* const* xyz, const size_t* n, bool target, bool on_device) {
  if (!b || !xyz || !n) return TLOAM_B200_ERR_INVALID_ARG;
  for (int s = 0; s < b->S; ++s) {
    const int rc = target ? set_target_impl(b->hs[s], xyz + 4 * s, n + 4 * s, on_device) : set_source_impl(b->hs[s], xyz + 4 * s, n + 4 * s, on_device);
    if (rc != TLOAM_B200_OK) {
      snprintf(b->last_error, sizeof(b->last_error), "sequence %d: %.400s", s, b->hs[s]->last_error);
      return rc;
    }
  }
  return TLOAM_B200_OK;
}
int tloam_b200_batch_set_target(tloam_b200_batch* b, const double* const* xyz, const size_t* n) { return batch_set(b, xyz, n, true, false); }
int tloam_b200_batch_set_source(tloam_b200_batch* b, const double* const* xyz, const size_t* n) { return batch_set(b, xyz, n, false, false); }
int tloam_b200_batch_set_target_device(tloam_b200_batch* b, const double* const* xyz, const size_t* n) { return batch_set(b, xyz, n, true, true); }
int tloam_b200_batch_set_source_device(tloam_b200_batch* b, const double* const* xyz, const size_t* n) { return batch_set(b, xyz, n, false, true); }

static int batch_enqueue_frame(tloam_b200_batch* b, bool fused, const tloam_tls_config& cfg) {
  static const DeviceCtx zero_ctx = {};
  const int S = b->S;
  CUB_TRY(cudaMemcpyAsync(b->d_pred, b->h_pred, S * sizeof(Predict), cudaMemcpyHostToDevice, b->stream));
  TLB_LAUNCH(TLOAM_B200_K_BEGIN_FRAME, (k_begin_frame<true><<<S, 256, 0, b->stream>>>(zero_ctx, b->g_eval, b->d_pred)));
  for (int outer = 0; outer < cfg.max_iterations; ++outer) {
    if (fused) {
      TLB_LAUNCH(TLOAM_B200_K_FIRST, (k_first<true><<<b->g_first.off[S], kBlk, 0, b->stream>>>(zero_ctx, b->g_first)));
    } else {
      if (b->any_fine) TLB_LAUNCH(TLOAM_B200_K_FINE, (k_correspond_fine<true><<<b->g_fine.off[S], kBlk, kFineSmemBytes, b->stream>>>(zero_ctx, b->g_fine, nullptr)));
      TLB_LAUNCH(TLOAM_B200_K_CORRESPOND, (k_correspond<true><<<b->g_corr.off[S], kBlk, 0, b->stream>>>(zero_ctx, b->g_corr)));
      TLB_LAUNCH(TLOAM_B200_K_EVAL_FIRST, (k_eval<true, true><<<b->g_eval.off[S], kBlk, 0, b->stream>>>(zero_ctx, b->g_eval)));
    }
    for (int it = 0; it < cfg.ceres_max_num_iterations; ++it)
      TLB_LAUNCH(TLOAM_B200_K_EVAL, (k_eval<false, true><<<b->g_eval.off[S], kBlk, 0, b->stream>>>(zero_ctx, b->g_eval)));
  }
  CUB_TRY(cudaGetLastError());
  // every sequence's result[16] + {frame_done, status} with ONE strided copy
  CUB_TRY(cudaMemcpy2DAsync(b->h_results, kResultBytes, (const char*)b->d_states + offsetof(FrameState, result), sizeof(FrameState),
                            kResultBytes, S, cudaMemcpyDeviceToHost, b->stream));
  return TLOAM_B200_OK;
}

// predicts: S x 16 doubles (4x4 column-major each), or NULL = device-side constant-velocity prediction per sequence
int tloam_b200_batch_scan_match_async(tloam_b200_batch* b, const double* predicts) {
  if (!b) return TLOAM_B200_ERR_INVALID_ARG;
  const int S = b->S;
  for (int s = 0; s < S; ++s) {
    const int rc = check_ready(b->hs[s]);
    if (rc != TLOAM_B200_OK) { snprintf(b->last_error, sizeof(b->last_error), "sequence %d is not ready", s); return rc; }
  }
  CUB_TRY(cudaSetDevice(b->device));
  const tloam_tls_config& cfg = b->hs[0]->cfg;
  // the frame kernels run behind everything the sequences have enqueued on their own streams (map build, staging)
  std::vector<DeviceCtx> ctxs(S);
  BatchTab tf, tc, te, tq;
  memset(&tf, 0, sizeof(tf)); memset(&tc, 0, sizeof(tc)); memset(&te, 0, sizeof(te)); memset(&tq, 0, sizeof(tq));
  tf.S = tc.S = te.S = tq.S = S; tf.ctxs = tc.ctxs = te.ctxs = tq.ctxs = b->d_ctxs;
  bool fused = b->use_fused;
  bool any_fine = false;
  for (int s = 0; s < S; ++s) {
    tloam_b200_handle* h = b->hs[s];
    CUB_TRY(cudaEventRecord(b->ev_ready[s], h->stream));
    CUB_TRY(cudaStreamWaitEvent(b->stream, b->ev_ready[s], 0));
    ctxs[s] = h->ctx;
    ctxs[s].stats = nullptr; ctxs[s].dbg = nullptr;
    ctxs[s].dense_mask = fine_mask_of(h);            // dense map clouds: two-level search (the TMA-staged path is single-sequence only)
    any_fine = any_fine || ctxs[s].dense_mask != 0;
    fused = fused && caps_cannot_bind(h);
    const int nb = h->total_blocks;
    tq.off[s + 1] = tq.off[s] + nb;
    tf.off[s + 1] = tf.off[s] + first_grid_of(nb);
    tc.off[s + 1] = tc.off[s] + 2 * nb;
    te.off[s + 1] = te.off[s] + eval_grid_of(nb);
    if (predicts) { memcpy(b->h_pred[s].m, predicts + 16 * s, 16 * sizeof(double)); b->h_pred[s].from_state = 0.0; }
    else b->h_pred[s].from_state = 1.0;
  }
  if (!b->ctx_valid || memcmp(b->ctx_sent.data(), ctxs.data(), S * sizeof(DeviceCtx)) != 0) {
    CUB_TRY(cudaMemcpyAsync(b->d_ctxs, ctxs.data(), S * sizeof(DeviceCtx), cudaMemcpyHostToDevice, b->stream));   // pageable source: staged before return
    b->ctx_sent = ctxs; b->ctx_valid = true;
  }
  if (any_fine) fused = false;
  b->any_fine = any_fine;
  const int per_frame = 1 + cfg.max_iterations * ((fused ? 1 : 2) + (any_fine ? 1 : 0) + cfg.ceres_max_num_iterations);
  CUB_TRY(cudaEventRecord(b->ev0, b->stream));
  if (b->use_graph && !b->profiling) {
    const bool same = b->gvalid && b->gfused == fused && b->gany_fine == any_fine && memcmp(&b->g_first, &tf, sizeof(tf)) == 0 &&
                      memcmp(&b->g_corr, &tc, sizeof(tc)) == 0 && memcmp(&b->g_eval, &te, sizeof(te)) == 0;
    if (!same) {
      b->gvalid = false;
      b->g_first = tf; b->g_corr = tc; b->g_eval = te; b->g_fine = tq;
      cudaGraph_t graph = nullptr;
      CUB_TRY(cudaStreamBeginCapture(b->stream, cudaStreamCaptureModeThreadLocal));
      const int erc = batch_enqueue_frame(b, fused, cfg);
      cudaError_t ce = cudaStreamEndCapture(b->stream, &graph);
      if (erc != TLOAM_B200_OK || ce != cudaSuccess || !graph) {
        if (graph) cudaGraphDestroy(graph);
        cudaGetLastError();
        if (erc == TLOAM_B200_OK) snprintf(b->last_error, sizeof(b->last_error), "graph capture failed: %s", cudaGetErrorString(ce));
        return TLOAM_B200_ERR_CUDA;
      }
      bool updated = false;
      if (b->gexec && b->gfused == fused && b->gany_fine == any_fine) {
        cudaGraphExecUpdateResultInfo info;
        updated = cudaGraphExecUpdate(b->gexec, graph, &info) == cudaSuccess;
        if (!updated) { cudaGetLastError(); cudaGraphExecDestroy(b->gexec); b->gexec = nullptr; }
      } else if (b->gexec) { cudaGraphExecDestroy(b->gexec); b->gexec = nullptr; }
      if (!updated) ce = cudaGraphInstantiate(&b->gexec, graph, 0);
      cudaGraphDestroy(graph);
      if (ce != cudaSuccess) { snprintf(b->last_error, sizeof(b->last_error), "graph instantiate: %s", cudaGetErrorString(ce)); return TLOAM_B200_ERR_CUDA; }
      b->gfused = fused; b->gany_fine = any_fine; b->gvalid = true;
    }
    CUB_TRY(cudaGraphLaunch(b->gexec, b->stream));
  } else {
    b->g_first = tf; b->g_corr = tc; b->g_eval = te; b->g_fine = tq;
    const int erc = batch_enqueue_frame(b, fused, cfg);
    if (erc != TLOAM_B200_OK) return erc;
  }
  CUB_TRY(cudaEventRecord(b->ev1, b->stream));
  // whatever the sequences enqueue next on their own streams (the next map build overwrites the map in use) waits
  CUB_TRY(cudaEventRecord(b->ev_done, b->stream));
  for (int s = 0; s < S; ++s) CUB_TRY(cudaStreamWaitEvent(b->hs[s]->stream, b->ev_done, 0));
  b->launches += per_frame; b->launches_frame = per_frame;
  b->pending = true;
  return TLOAM_B200_OK;
}

// results: S x 16 doubles; statuses: S ints (tloam_b200_status per sequence).  Returns OK when every sequence is OK,
// else the first non-OK status.
int tloam_b200_batch_get_results(tloam_b200_batch* b, double* results, int* statuses, float* gpu_ms) {
  if (!b || !results) return TLOAM_B200_ERR_INVALID_ARG;
  if (!b->pending) return TLOAM_B200_ERR_NOT_READY;
  CUB_TRY(cudaSetDevice(b->device));
  CUB_TRY(cudaStreamSynchronize(b->stream));
  b->pending = false;
  int worst = TLOAM_B200_OK;
  for (int s = 0; s < b->S; ++s) {
    const unsigned char* r = b->h_results + s * kResultBytes;
    memcpy(results + 16 * s, r, 16 * sizeof(double));
    int flags[2];
    memcpy(flags, r + 16 * sizeof(double), sizeof(flags));
    int st = flags[1];
    if (st == TLOAM_B200_OK && !flags[0]) st = TLOAM_B200_ERR_CUDA;      // the frame did not complete
    if (statuses) statuses[s] = st;
    if (worst == TLOAM_B200_OK && st != TLOAM_B200_OK) worst = st;
  }
  if (gpu_ms) { float ms = 0.f; if (cudaEventElapsedTime(&ms, b->ev0, b->ev1) == cudaSuccess) *gpu_ms = ms; }
  return worst;
}

int tloam_b200_batch_set_profiling(tloam_b200_batch* b, int on) {
  if (!b) return TLOAM_B200_ERR_INVALID_ARG;
  CUB_TRY(cudaSetDevice(b->device));
  CUB_TRY(cudaStreamSynchronize(b->stream));
  b->profiling = on != 0;
  b->spans.clear(); b->ev_next = 0;
  memset(&b->prof, 0, sizeof(b->prof));
  return TLOAM_B200_OK;
}

int tloam_b200_batch_get_profile(tloam_b200_batch* b, tloam_b200_profile* out) {
  if (!b || !out) return TLOAM_B200_ERR_INVALID_ARG;
  CUB_TRY(cudaSetDevice(b->device));
  CUB_TRY(cudaStreamSynchronize(b->stream));
  for (const auto& sp : b->spans) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, sp.a, sp.b) == cudaSuccess && sp.cls >= 0 && sp.cls < TLOAM_B200_K_COUNT) {
      b->prof.launches[sp.cls] += 1;
      b->prof.total_ms[sp.cls] += ms;
    }
  }
  b->spans.clear(); b->ev_next = 0;
  *out = b->prof;
  return TLOAM_B200_OK;
}

int tloam_b200_batch_scan_match(tloam_b200_batch* b, const double* predicts, double* results, int* statuses) {
  const int rc = tloam_b200_batch_scan_match_async(b, predicts);
  if (rc != TLOAM_B200_OK) return rc;
  return tloam_b200_batch_get_results(b, results, statuses, nullptr);
}

int tloam_b200_fitness(tloam_b200_handle* h, double* fitness, double* rmse) {
  if (!h || !fitness || !rmse) return TLOAM_B200_ERR_INVALID_ARG;
  *fitness = 0.0; *rmse = 0.0;
  if (!h->have_src || !h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  if (h->cfg.fitness_thres <= 0.0) return TLOAM_B200_OK;                 // ref: :258-261
  for (int c = 0; c < 4; ++c) if (h->cfg.fitness_thres > radius_of(h->cfg, c)) return TLOAM_B200_ERR_INVALID_ARG;
  const int nb = h->total_blocks;
  if (nb == 0) return TLOAM_B200_OK;                                     // every source cloud is empty: nothing matches
  CU_TRY(cudaSetDevice(h->device));
  // block partials live in a buffer sized with the source (no allocation on this per-frame health metric); the
  // per-cloud sums are formed on the device in block order and land in the frame state
  TL_LAUNCH(TLOAM_B200_K_FITNESS, (k_fitness<<<nb, kBlk, 0, h->stream>>>(h->ctx, h->cfg.fitness_thres * h->cfg.fitness_thres, h->d_fit)));
  TL_LAUNCH(TLOAM_B200_K_FITNESS, (k_fitness_reduce<<<1, 128, 0, h->stream>>>(h->ctx, h->d_fit, reinterpret_cast<double*>(reinterpret_cast<char*>(h->d_state) + offsetof(FrameState, fitness)))));
  CU_TRY(cudaGetLastError());
  CU_TRY(cudaMemcpyAsync(h->h_result + 20, (const char*)h->d_state + offsetof(FrameState, fitness), 2 * sizeof(double),
                         cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  *fitness = h->h_result[20]; *rmse = h->h_result[21];
  return TLOAM_B200_OK;
}

// per-frame health metric in the asynchronous flow: every scan_match also evaluates getFitnessScore of its scan
// (two more kernels in the frame graph, no allocation); the pair comes back with the frame's result
int tloam_b200_set_frame_fitness(tloam_b200_handle* h, int on) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  h->frame_fitness = on != 0;
  return TLOAM_B200_OK;
}
int tloam_b200_get_frame_fitness(tloam_b200_handle* h, double* fitness, double* rmse) {   // of the last fetched result
  if (!h || !fitness || !rmse) return TLOAM_B200_ERR_INVALID_ARG;
  *fitness = h->last_fitness; *rmse = h->last_rmse;
  return TLOAM_B200_OK;
}
// Pipelined use: set_source / submap_update return without waiting for their uploads (the host buffers must then stay
// valid until the frame's result has been fetched) and get_result waits for the OLDEST un-fetched frame only, so the
// host can enqueue frame k+1 while the GPU still runs frame k (at most 2 frames in flight).
int tloam_b200_set_async_inputs(tloam_b200_handle* h, int on) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->async_inputs = on != 0;
  h->frames_fetched = h->frames_enqueued; h->frame_pending = false;
  h->gvalid = false;                             // the frame graph holds (or not) the result copy
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// piecewise entry points (tests)
// ---------------------------------------------------------------------------------------------
int tloam_b200_knn(tloam_b200_handle* h, int cloud, const double* queries, size_t nq, double radius, int k, int* idx,
                   double* d2, int* count) {
  if (!h || cloud < 0 || cloud > 3 || !queries || !idx || !d2 || !count) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  if (!(radius > 0.0) || radius > h->hdr.cell[cloud] || (k != 1 && k != 3 && k != 5)) return TLOAM_B200_ERR_INVALID_ARG;
  if (nq == 0) return TLOAM_B200_OK;
  CU_TRY(cudaSetDevice(h->device));
  { const int rc = fetch_origin(h); if (rc != TLOAM_B200_OK) return rc; }
  double *dq = nullptr, *dd = nullptr; int *di = nullptr, *dc = nullptr;
  cudaError_t e = cudaMalloc(&dq, nq * 3 * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&dd, nq * k * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&di, nq * k * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&dc, nq * sizeof(int));
  if (e == cudaSuccess) e = cudaMemcpyAsync(dq, queries, nq * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) {
    const unsigned tb = 128, gb = (unsigned)((nq + tb - 1) / tb);
    const GridDesc g = h->ctx.grid[cloud];
    const double* o = h->ctx.origin;
    if (k == 1) k_knn<1><<<gb, tb, 0, h->stream>>>(g, o, dq, (unsigned)nq, radius * radius, di, dd, dc);
    else if (k == 3) k_knn<3><<<gb, tb, 0, h->stream>>>(g, o, dq, (unsigned)nq, radius * radius, di, dd, dc);
    else k_knn<5><<<gb, tb, 0, h->stream>>>(g, o, dq, (unsigned)nq, radius * radius, di, dd, dc);
    h->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(idx, di, nq * k * sizeof(int), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d2, dd, nq * k * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(count, dc, nq * sizeof(int), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(dq); cudaFree(dd); cudaFree(di); cudaFree(dc);
  if (e != cudaSuccess) { snprintf(h->last_error, sizeof(h->last_error), "knn: %s", cudaGetErrorString(e)); return TLOAM_B200_ERR_CUDA; }
  return TLOAM_B200_OK;
}

int tloam_b200_build_factors(tloam_b200_handle* h, int cloud, const double x[6], int* valid, double* prim, size_t n) {
  if (!h || cloud < 0 || cloud > 3 || !x || !valid || !prim) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_src || !h->have_tgt) return TLOAM_B200_ERR_NOT_READY;
  if (n != h->n_src[cloud]) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  { const int rc = fetch_origin(h); if (rc != TLOAM_B200_OK) return rc; }
  Predict pr;
  memset(&pr, 0, sizeof(pr));
  memcpy(pr.m, x, 6 * sizeof(double));
  DeviceCtx c = h->ctx;
  c.factor_num = 4;   // build every cloud regardless of the configured subset
  c.dense_mask = dense_mask_of(h);
  if (c.dense_mask && h->dense_kernel == 1) { const int drc = prepare_dense(h, c.dense_mask); if (drc != TLOAM_B200_OK) return drc; }
  k_set_pose<<<1, 256, 0, h->stream>>>(c, pr);
  { const int crc = enqueue_correspond(h, c); if (crc != TLOAM_B200_OK) return crc; }
  k_caps<<<h->total_blocks, kBlk, 0, h->stream>>>(c);
  h->launches += 2;
  CU_TRY(cudaGetLastError());
  std::vector<unsigned char> act(n);
  std::vector<double> col(n);
  const size_t off = (size_t)h->ctx.pad_off[cloud];
  CU_TRY(cudaMemcpyAsync(act.data(), h->ctx.active + off, n, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (size_t i = 0; i < n; ++i) valid[i] = act[i];
  for (int j = 0; j < 6; ++j) {
    CU_TRY(cudaMemcpyAsync(col.data(), h->ctx.prim[j] + off, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    for (size_t i = 0; i < n; ++i) prim[6 * i + j] = act[i] ? col[i] : 0.0;
  }
  // leave the handle idle
  int one = 1;
  CU_TRY(cudaMemcpyAsync((char*)h->d_state + offsetof(FrameState, frame_done), &one, sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

static int run_functor(tloam_b200_handle* h, int type, const double x[6], size_t m, const double* p, const double* a,
                       const double* b, size_t b_stride, const double* w, double* r, size_t r_stride, double* J,
                       size_t j_stride, double* cost) {
  if (!h || !x || !p || !a || !b || !w || !r || !J || !cost) return TLOAM_B200_ERR_INVALID_ARG;
  if (m == 0) return TLOAM_B200_OK;
  CU_TRY(cudaSetDevice(h->device));
  Predict pr;
  memset(&pr, 0, sizeof(pr));
  memcpy(pr.m, x, 6 * sizeof(double));
  const size_t in_doubles = m * (3 + 3 + b_stride + 1), out_doubles = m * (r_stride + j_stride + 1);
  double* d = nullptr;
  cudaError_t e = cudaMalloc(&d, (in_doubles + out_doubles) * sizeof(double));
  if (e != cudaSuccess) { snprintf(h->last_error, sizeof(h->last_error), "functor: %s", cudaGetErrorString(e)); return TLOAM_B200_ERR_CUDA; }
  double *dp = d, *da = dp + 3 * m, *db = da + 3 * m, *dw = db + b_stride * m, *dr = dw + m, *dJ = dr + r_stride * m, *dc = dJ + j_stride * m;
  e = cudaMemcpyAsync(dp, p, 3 * m * sizeof(double), cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(da, a, 3 * m * sizeof(double), cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(db, b, b_stride * m * sizeof(double), cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(dw, w, m * sizeof(double), cudaMemcpyHostToDevice, h->stream);
  if (e == cudaSuccess) {
    k_functor<<<(unsigned)((m + 127) / 128), 128, 0, h->stream>>>(type, pr, (unsigned)m, dp, da, db, dw, dr, dJ, dc);
    h->launches++;
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(r, dr, r_stride * m * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(J, dJ, j_stride * m * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(cost, dc, m * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(d);
  if (e != cudaSuccess) { snprintf(h->last_error, sizeof(h->last_error), "functor: %s", cudaGetErrorString(e)); return TLOAM_B200_ERR_CUDA; }
  return TLOAM_B200_OK;
}

int tloam_b200_eval_point_to_point(tloam_b200_handle* h, const double x[6], size_t m, const double* p, const double* q,
                                   const double* w, double* r, double* J, double* cost) {
  return run_functor(h, 0, x, m, p, q, q, 3, w, r, 3, J, 18, cost);
}
int tloam_b200_eval_point_to_line(tloam_b200_handle* h, const double x[6], size_t m, const double* p, const double* a,
                                  const double* b, const double* w, double* r, double* J, double* cost) {
  return run_functor(h, 1, x, m, p, a, b, 3, w, r, 3, J, 18, cost);
}
int tloam_b200_eval_point_to_plane(tloam_b200_handle* h, const double x[6], size_t m, const double* p, const double* n,
                                   const double* d, const double* w, double* r, double* J, double* cost) {
  return run_functor(h, 2, x, m, p, n, d, 1, w, r, 1, J, 6, cost);
}

static int run_se3(tloam_b200_handle* h, int op, const double* in, int nin, double* out, int nout, double* extra) {
  if (!h || !in || !out) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  Predict pr;
  memset(&pr, 0, sizeof(pr));
  memcpy(pr.m, in, nin * sizeof(double));
  double* d = nullptr;
  CU_TRY(cudaMalloc(&d, 32 * sizeof(double)));
  k_se3<<<1, 32, 0, h->stream>>>(op, pr, d);
  h->launches++;
  double tmp[32];
  cudaError_t e = cudaMemcpyAsync(tmp, d, 32 * sizeof(double), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  cudaFree(d);
  if (e != cudaSuccess) { snprintf(h->last_error, sizeof(h->last_error), "se3: %s", cudaGetErrorString(e)); return TLOAM_B200_ERR_CUDA; }
  memcpy(out, tmp, nout * sizeof(double));
  if (extra) *extra = tmp[6];
  return TLOAM_B200_OK;
}

int tloam_b200_se3_exp(tloam_b200_handle* h, const double a[6], double T[16]) { return run_se3(h, 0, a, 6, T, 16, nullptr); }
int tloam_b200_se3_log(tloam_b200_handle* h, const double T[16], double a[6]) {
  double ok = 1.0;
  int rc = run_se3(h, 1, T, 16, a, 6, &ok);
  if (rc != TLOAM_B200_OK) return rc;
  return ok != 0.0 ? TLOAM_B200_OK : TLOAM_B200_ERR_BAD_POSE;
}
int tloam_b200_se3_plus(tloam_b200_handle* h, const double x[6], const double delta[6], double out[6]) {
  double in[12];
  memcpy(in, x, 48); memcpy(in + 6, delta, 48);
  return run_se3(h, 2, in, 12, out, 6, nullptr);
}

int tloam_b200_min_on_boundary_2d(tloam_b200_handle* h, const double B[4], const double g[2], double radius, double y[2]) {
  if (!B || !g || !y) return TLOAM_B200_ERR_INVALID_ARG;
  double in[7] = {B[0], B[1], B[2], B[3], g[0], g[1], radius};
  return run_se3(h, 3, in, 7, y, 2, nullptr);
}

// ---------------------------------------------------------------------------------------------
// (f)-1 device-side submap maintenance
// ---------------------------------------------------------------------------------------------
void tloam_b200_submap_default_config(tloam_submap_config* c) {   // ref: config/mapping/lidar_odometry.yaml:6-17
  c->ground_down_sample = 0.3; c->ground_down_sample_submap = 0.45; c->edge_down_sample_submap = 0.3;
  c->planar_frame_size = 3; c->sphere_frame_size = 3;
  c->edge_crop_box_length = 100.0; c->ground_crop_box_length = 100.0;
}

static int ensure_dev(tloam_b200_handle* h, double** p, size_t* cap, size_t need_points, bool keep) {
  if (need_points <= *cap) return TLOAM_B200_OK;
  const size_t ncap = need_points + need_points / 2 + 1024;
  double* q = nullptr;
  CU_TRY(cudaMalloc(&q, ncap * 3 * sizeof(double)));
  if (keep && *p && *cap) CU_TRY(cudaMemcpyAsync(q, *p, *cap * 3 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  if (*p) { CU_TRY(cudaStreamSynchronize(h->stream)); cudaFree(*p); }
  *p = q; *cap = ncap;
  return TLOAM_B200_OK;
}

// ---- limits of the voxel kernels, checked on the host for clouds that come from the host (nothing is launched when a
//      cloud fails them: the caller returns VOXEL_RANGE) ----
//   key range: k_vox_accum packs each axis's index into kGMapKeyBits bits (cell_key), so an index of 2^21 or more would
//     land in the voxel of index mod 2^21 and vox_average would write its mean there.  k_gmap_guard's expression on the
//     finite rows' bounds gives the largest index exactly: floor((p - min_bound) / voxel) is monotone in p.
//   headroom: each row adds llrint(offset * 2^40) to a signed 64-bit sum, with offset = p - (voxel's base) at most the
//     voxel plus rounding: below 2^-52 (3 |p| + 4 voxel) for a keyable index, padded here to 2^-49 (|p| + voxel), plus the
//     half unit of llrint.  n rows times that stays below 2^63 / 2^40 = 2^23 m whatever voxel they share.
static void vox_extent_add(VoxExtent& e, double x, double y, double z) {
  if (!std::isfinite(x) || !std::isfinite(y) || !std::isfinite(z)) return;
  const double p[3] = {x, y, z};
  for (int d = 0; d < 3; ++d) {
    e.lo[d] = e.n ? std::fmin(e.lo[d], p[d]) : p[d];
    e.hi[d] = e.n ? std::fmax(e.hi[d], p[d]) : p[d];
  }
  ++e.n;
}
static VoxExtent vox_extent(const double* p, size_t n) {
  VoxExtent e;
  for (size_t i = 0; i < n; ++i) vox_extent_add(e, p[3 * i], p[3 * i + 1], p[3 * i + 2]);
  return e;
}
static VoxExtent vox_extent_packed(const tloam_packed_scan* s) {   // the FLOAT32 fields, as unpack_packed widens them
  VoxExtent e;
  const unsigned char* r = static_cast<const unsigned char*>(s->data);
  for (size_t i = 0; i < s->n; ++i, r += s->point_step) {
    float f[3];
    memcpy(&f[0], r + s->x_offset, 4); memcpy(&f[1], r + s->y_offset, 4); memcpy(&f[2], r + s->z_offset, 4);
    vox_extent_add(e, f[0], f[1], f[2]);
  }
  return e;
}
static bool vox_fits(const VoxExtent& e, double voxel) {
  if (!e.known || e.n == 0) return true;
  double big = 0.0;
  for (int d = 0; d < 3; ++d) {
    const double mb = e.lo[d] - voxel * 0.5;
    const double ref = (e.hi[d] - mb) / voxel;
    if (!(ref < (double)(1u << kGMapKeyBits))) return false;
    big = std::fmax(big, std::fmax(std::fabs(e.lo[d]), std::fabs(e.hi[d])));
  }
  return (double)e.n * (voxel + 0x1p-49 * (big + voxel) + 0x1p-40) < 0x1p23;
}

// crop + VoxelDownSample of d_in into d_out, enqueued without any host round trip: the voxel count lands in
// *out_count (device).  The input holds n_bound points at most; its exact count is n_bound itself (n_dev == nullptr)
// or *n_dev + n_add.  The crop box is lo/hi (host values; nullptr = none) or pose.t +- box_len with the pose in
// device memory.
// sorted (optional): the voxels are put in ascending key order instead of being emitted (the scan features of
// tloam_b200_process_cloud, see submap.cuh); voxel_emit_sorted writes them once the count is known.
struct VoxSorted { VoxArgs a; unsigned* slots = nullptr; const unsigned long long* keys = nullptr; /* ~key, descending */ };
static int voxel_pipeline(tloam_b200_handle* h, const double* d_in, size_t n_bound, const unsigned* n_dev, unsigned n_add,
                          const double* lo, const double* hi, const double* box_pose, double box_len, double voxel,
                          double* d_out, unsigned* out_count, cudaStream_t stream = nullptr, int scratch = 0,
                          VoxSorted* sorted = nullptr) {
  if (!stream) stream = h->stream;
  if (sorted) sorted->slots = nullptr;
  if (n_bound == 0) { CU_TRY(cudaMemsetAsync(out_count, 0, sizeof(unsigned), stream)); return TLOAM_B200_OK; }
  if (!(voxel > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  const unsigned tsize = next_pow2(2 * n_bound + 1);
  size_t npad = 1;                                     // the bitonic network pads the list to a power of two
  while (npad < n_bound) npad <<= 1;
  const size_t o_sort = 256 + (size_t)tsize * (8 + 24 + 4);
  const size_t bytes = o_sort + (sorted ? npad * (8 + 8 + 4 + 4 + 4) : 0);
  unsigned char*& d_vox = scratch ? h->d_vox1 : h->d_vox;
  size_t& cap_vox = scratch ? h->cap_vox1 : h->cap_vox;
  if (bytes > cap_vox) {
    CU_TRY(cudaStreamSynchronize(stream));
    cudaFree(d_vox); d_vox = nullptr; cap_vox = 0;
    CU_TRY(cudaMalloc(&d_vox, bytes + bytes / 2));
    cap_vox = bytes + bytes / 2;
  }
  VoxArgs a;
  a.in = d_in; a.n = (unsigned)n_bound; a.voxel = voxel;
  a.n_dev = n_dev; a.n_add = n_add; a.box_pose = box_pose; a.box_len = box_len;
  for (int d = 0; d < 3; ++d) { a.lo[d] = lo ? lo[d] : -DBL_MAX; a.hi[d] = hi ? hi[d] : DBL_MAX; }
  a.minenc = reinterpret_cast<unsigned long long*>(d_vox);            // [0..2] min bound
  a.out_count = out_count;
  a.keys = reinterpret_cast<unsigned long long*>(d_vox + 256);
  a.sums = reinterpret_cast<long long*>(d_vox + 256 + (size_t)tsize * 8);
  a.cnt = reinterpret_cast<unsigned*>(d_vox + 256 + (size_t)tsize * 32);
  a.mask = tsize - 1u;
  a.out = d_out;
  CU_TRY(cudaMemsetAsync(d_vox, 0, 256 + (size_t)tsize * 36, stream));   // ONE memset: min bound (complemented), keys, sums, counts
  const unsigned tb = 256, gb = (unsigned)((n_bound + tb - 1) / tb);
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_vox_min<<<(gb < 592u ? gb : 592u), tb, 0, stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_vox_accum<<<gb, tb, 0, stream>>>(a)));
  if (!sorted) {
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_vox_emit<<<(tsize + tb - 1) / tb, tb, 0, stream>>>(a)));
    CU_TRY(cudaGetLastError());
    return TLOAM_B200_OK;
  }
  // ordered: (~key, slot) pairs sorted by the PCA selection's rank sort / bitonic network, one list (grid y = 1, one block)
  unsigned long long* key_raw = reinterpret_cast<unsigned long long*>(d_vox + o_sort);
  unsigned long long* key_sorted = key_raw + npad;
  unsigned* slot_raw = reinterpret_cast<unsigned*>(key_sorted + npad);
  unsigned* slot_sorted = slot_raw + npad;
  unsigned* rank = slot_sorted + npad;
  CU_TRY(cudaMemsetAsync(rank, 0, npad * sizeof(unsigned), stream));
  if (!h->fe_sort_attr_set) {
    CU_TRY(cudaFuncSetAttribute(k_fe_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFeSortSmemBytes));
    h->fe_sort_attr_set = true;
  }
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_vox_keys<<<(tsize + tb - 1) / tb, tb, 0, stream>>>(a, key_raw, slot_raw)));
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_fe_rank<<<dim3(gb, 1, kFeRankSplit), 256, 0, stream>>>(key_raw, slot_raw, key_raw, slot_raw, rank, rank,
                                                                                           out_count)));
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_fe_rank_scatter<<<dim3(gb, 1), 256, 0, stream>>>(key_raw, slot_raw, key_raw, slot_raw, rank, rank, key_sorted,
                                                                                   slot_sorted, key_sorted, slot_sorted, out_count)));
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_fe_sort<<<1, 1024, kFeSortSmemBytes, stream>>>(key_sorted, slot_sorted, key_sorted, slot_sorted, out_count)));
  CU_TRY(cudaGetLastError());
  sorted->a = a;
  sorted->slots = slot_sorted;
  sorted->keys = key_sorted;
  return TLOAM_B200_OK;
}

// the n voxels sorted by voxel_pipeline into out (n: the count it left in out_count, read back by the caller)
static int voxel_emit_sorted(tloam_b200_handle* h, const VoxSorted& s, size_t n, double* out) {
  if (n == 0) return TLOAM_B200_OK;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_vox_emit_sorted<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(s.a, s.slots, out)));
  CU_TRY(cudaGetLastError());
  return TLOAM_B200_OK;
}

static int upload_points(tloam_b200_handle* h, const double* host, size_t n) {
  int rc = ensure_dev(h, &h->d_up, &h->cap_up, n, false);
  if (rc != TLOAM_B200_OK) return rc;
  if (n) CU_TRY(cudaMemcpyAsync(h->d_up, host, n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  return TLOAM_B200_OK;
}

static unsigned* acc_count(tloam_b200_handle* h, int k) { return h->d_cnt + 4 + 2 * k + h->acc_cur[k]; }

static int submap_set_target(tloam_b200_handle* h) {
  // order at the ABI: edge, sphere, planar, ground.  After the first update the sphere map IS the planar window
  // (ref: front_end.cpp:220-230 iterates submap_planar_buffer).  Edge / ground: the host knows an upper bound, the
  // exact counts are read on the device.
  const double* xyz[4] = {h->d_acc[0], h->sphere_is_init ? h->d_sphere0 : h->d_cat, h->d_cat, h->d_acc[1]};
  const size_t n[4] = {h->n_acc[0], h->sphere_is_init ? h->n_sphere0 : h->n_cat, h->n_cat, h->n_acc[1]};
  const unsigned* nd[4] = {acc_count(h, 0), nullptr, nullptr, acc_count(h, 1)};
  return set_target_impl(h, xyz, n, true, nd);
}

// ---------------------------------------------------------------------------------------------
// "next" row (f)-2: PCA feature extraction (feature_extract.cuh)
// ---------------------------------------------------------------------------------------------
void tloam_b200_feature_default_config(tloam_feature_config* c) {   // ref: config/mapping/feature.yaml
  c->radius = 0.2; c->K = 20; c->min_neigh = 10; c->planar_num = 500; c->sphere_num = 300;
  c->cvr_scan = 0.25; c->cvr_submap = 0.15; c->planar_scan_thres = 0.75; c->planar_submap_thres = 0.65;
  c->planar_vertic_thres = 0.25;
}

namespace {
struct FeArena {
  const double* stage; unsigned* scratch; unsigned char* blob; MapHeader hdr;
  FeOut out;
  unsigned long long *key_p_sorted, *key_s_sorted;
  unsigned *val_p_sorted, *val_s_sorted, *counts;
  unsigned *host_val_p = nullptr, *host_val_s = nullptr;   // optional: the sorted index lists land here (one sync)
};
}  // namespace

// carves the arena for n points and enqueues grid build + k_fe_pca (+ classification and sorts when `select`).
// on_device: xyz is a device cloud, read in place on the handle's stream (no upload)
static int fe_run(tloam_b200_handle* h, const tloam_feature_config* cfg, const double* xyz, size_t n, bool select, FeArena& A,
                  bool on_device = false) {
  if (n == 0 || n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!(cfg->radius > 0.0) || cfg->K < 3 || cfg->K > kFeK) return TLOAM_B200_ERR_INVALID_ARG;   // :56 asserts K >= 3
  CU_TRY(cudaSetDevice(h->device));
  MapHeader& hd = A.hdr;
  memset(&hd, 0, sizeof(hd));
  hd.magic = kMapMagic;
  size_t boff = sizeof(MapHeader);
  for (int c = 0; c < 4; ++c) {
    hd.n[c] = c == 0 ? (unsigned)n : 0u;
    hd.tsize[c] = next_pow2((c == 0 ? n : 0) + 1);
    hd.cell[c] = cfg->radius;                       // cell edge == search radius: the 27-cell search is exact
    hd.pts_off[c] = boff; boff += round_up(hd.n[c] * sizeof(FePoint), 256);
  }
  for (int c = 0; c < 4; ++c) { hd.table_off[c] = boff; boff += (size_t)hd.tsize[c] * kBrickBytes; }
  for (int d = 0; d < 3; ++d) { hd.bbox_enc[d] = ~0ull; hd.bbox_enc[3 + d] = 0ull; }
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += round_up(bytes, 256); return o; };
  const size_t o_stage = on_device ? 0 : take(n * 3 * sizeof(double)), o_scr = take(n * 2 * sizeof(unsigned)), o_blob = take(boff);
  const size_t o_cvr = take(n * 8), o_flat = take(n * 8), o_sph = take(n * 8), o_nrm = take(n * 24), o_num = take(n * 4),
               o_nei = take(n * kFeK * 4);
  size_t npad = 1;                                     // the bitonic network pads each candidate list to a power of two
  while (npad < n) npad <<= 1;
  const size_t o_kps = take(npad * 8), o_kss = take(npad * 8), o_vps = take(npad * 4), o_vss = take(npad * 4), o_cnt = take(256);
  const size_t o_kpr = take(npad * 8), o_ksr = take(npad * 8), o_vpr = take(npad * 4), o_vsr = take(npad * 4);   // compacted, unsorted
  const size_t o_rk = take(npad * 8);                  // ranks of the two lists
  if (off > h->cap_fe) {
    cudaFree(h->d_fe);
    h->cap_fe = off + off / 4;
    CU_TRY(cudaMalloc(&h->d_fe, h->cap_fe));
  }
  unsigned char* b = h->d_fe;
  A.stage = on_device ? xyz : (const double*)(b + o_stage); A.scratch = (unsigned*)(b + o_scr); A.blob = b + o_blob;
  A.out.cvr = (double*)(b + o_cvr); A.out.flatness = (double*)(b + o_flat); A.out.sphericity = (double*)(b + o_sph);
  A.out.normal = (double*)(b + o_nrm); A.out.num_sum = (int*)(b + o_num); A.out.neigh = (int*)(b + o_nei);
  A.key_p_sorted = (unsigned long long*)(b + o_kps); A.key_s_sorted = (unsigned long long*)(b + o_kss);
  A.val_p_sorted = (unsigned*)(b + o_vps); A.val_s_sorted = (unsigned*)(b + o_vss);
  A.counts = (unsigned*)(b + o_cnt);
  unsigned long long* key_p_raw = (unsigned long long*)(b + o_kpr); unsigned long long* key_s_raw = (unsigned long long*)(b + o_ksr);
  unsigned* val_p_raw = (unsigned*)(b + o_vpr); unsigned* val_s_raw = (unsigned*)(b + o_vsr);
  unsigned* rank_p = (unsigned*)(b + o_rk); unsigned* rank_s = rank_p + npad;

  if (!on_device) CU_TRY(cudaMemcpyAsync(b + o_stage, xyz, n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CU_TRY(cudaMemcpyAsync(A.blob, &hd, sizeof(MapHeader), cudaMemcpyHostToDevice, h->stream));
  CU_TRY(cudaMemsetAsync(A.blob + hd.table_off[0], 0, boff - hd.table_off[0], h->stream));
  CU_TRY(cudaMemsetAsync(A.counts, 0, 256, h->stream));
  MapBuildArgs ma;
  ma.blob = A.blob; ma.slot_of = A.scratch; ma.rank_of = A.scratch + n;
  ma.i_beg = 0; ma.i_end = (unsigned)n; ma.only_cloud = -1;
  ma.fine_mask = 0; ma.fine_tmp = nullptr;
  for (int c = 0; c < 4; ++c) ma.n_dev[c] = nullptr;
  for (int c = 0; c < 4; ++c) ma.src[c] = A.stage;
  ma.stage_off[0] = 0;
  for (int c = 1; c <= 4; ++c) ma.stage_off[c] = (unsigned)n;
  FeBuildArgs fa;
  fa.stage = A.stage; fa.n = (unsigned)n; fa.blob = A.blob; fa.slot_of = A.scratch; fa.rank_of = A.scratch + n;
  const unsigned tb = 256, gb = (unsigned)((n + tb - 1) / tb);
  unsigned tslots = 0;
  for (int c = 0; c < 4; ++c) tslots += hd.tsize[c];
  TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_map_bbox<<<(gb < 592u ? gb : 592u), tb, 0, h->stream>>>(ma)));   // + origin
  TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_insert<<<gb, tb, 0, h->stream>>>(fa)));
  TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_map_offsets<<<(tslots + tb - 1) / tb, tb, 0, h->stream>>>(ma)));
  TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_scatter<<<gb, tb, 0, h->stream>>>(fa)));
  FeGrid g;
  g.pts = reinterpret_cast<const FePoint*>(A.blob + hd.pts_off[0]);
  g.table = reinterpret_cast<const uint4*>(A.blob + hd.table_off[0]);
  g.mask = hd.tsize[0] - 1u; g.n = (unsigned)n; g.cell = cfg->radius; g.inv_cell = 1.0 / cfg->radius;
  g.origin = reinterpret_cast<const double*>(A.blob + offsetof(MapHeader, origin));
  FeParams prm;
  prm.dbg = h->profiling ? h->d_dbg + 8 : nullptr;     // slots 8..11 (k_correspond uses them in frame profiling)
  prm.r2 = cfg->radius * cfg->radius; prm.K = cfg->K; prm.min_neigh = cfg->min_neigh;
  prm.cvr_submap = cfg->cvr_submap; prm.planar_submap_thres = cfg->planar_submap_thres;
  prm.planar_vertic_thres = cfg->planar_vertic_thres;
  if (!h->fe_attr_set) {
    CU_TRY(cudaFuncSetAttribute(k_fe_pca, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFeSmemBytes));
    h->fe_attr_set = true;
  }
  TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_pca<<<(unsigned)((n + kFeBlk - 1) / kFeBlk), kFeBlk, kFeSmemBytes, h->stream>>>(g, prm, A.out)));
  if (select) {
    TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_classify<<<gb, tb, 0, h->stream>>>((unsigned)n, prm, A.out, key_p_raw, key_s_raw, val_p_raw, val_s_raw,
                                                                              A.counts)));
    // candidates first compacted, then ordered by (flatness descending, point index ascending): rank sort over the whole
    // GPU for lists up to 32 768 candidates, the shared-memory bitonic network for longer ones (each is a no-op otherwise)
    CU_TRY(cudaMemsetAsync(rank_p, 0, npad * 8, h->stream));
    TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_rank<<<dim3(gb, 2, kFeRankSplit), 256, 0, h->stream>>>(key_p_raw, val_p_raw, key_s_raw, val_s_raw, rank_p,
                                                                                                  rank_s, A.counts)));
    TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_rank_scatter<<<dim3(gb, 2), 256, 0, h->stream>>>(key_p_raw, val_p_raw, key_s_raw, val_s_raw, rank_p, rank_s,
                                                                                            A.key_p_sorted, A.val_p_sorted, A.key_s_sorted,
                                                                                            A.val_s_sorted, A.counts)));
    if (!h->fe_sort_attr_set) {
      CU_TRY(cudaFuncSetAttribute(k_fe_sort, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFeSortSmemBytes));
      h->fe_sort_attr_set = true;
    }
    TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_sort<<<2, 1024, kFeSortSmemBytes, h->stream>>>(A.key_p_sorted, A.val_p_sorted, A.key_s_sorted, A.val_s_sorted, A.counts)));
    TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_fe_counts<<<1, 32, 0, h->stream>>>(A.key_p_sorted, A.key_s_sorted, A.counts, cfg->planar_num,
                                                                           cfg->sphere_num, cfg->planar_scan_thres, cfg->cvr_scan)));
  }
  CU_TRY(cudaGetLastError());
  // counts + build flags -> pinned scratch (h_result[28..31])
  CU_TRY(cudaMemcpyAsync(h->h_result + 28, A.counts, 4 * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaMemcpyAsync(h->h_result + 30, A.blob + offsetof(MapHeader, build_flags), sizeof(unsigned long long),
                         cudaMemcpyDeviceToHost, h->stream));
  if (select && A.host_val_p) CU_TRY(cudaMemcpyAsync(A.host_val_p, A.val_p_sorted, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  if (select && A.host_val_s) CU_TRY(cudaMemcpyAsync(A.host_val_s, A.val_s_sorted, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  unsigned long long flags;
  memcpy(&flags, h->h_result + 30, sizeof(flags));
  return (flags & 1ull) ? TLOAM_B200_ERR_MAP_DENSITY : TLOAM_B200_OK;
}

int tloam_b200_extract_planar_sphere(tloam_b200_handle* h, const tloam_feature_config* cfg, const double* xyz, size_t n,
                                     size_t* planar_scan_index, size_t* n_planar_scan, size_t* planar_submap_index,
                                     size_t* n_planar_submap, size_t* sphere_scan_index, size_t* n_sphere_scan,
                                     size_t* sphere_submap_index, size_t* n_sphere_submap, size_t* sphere_candidates) {
  if (!h || !cfg || !planar_scan_index || !n_planar_scan || !planar_submap_index || !n_planar_submap || !sphere_scan_index ||
      !n_sphere_scan || !sphere_submap_index || !n_sphere_submap)
    return TLOAM_B200_ERR_INVALID_ARG;
  *n_planar_scan = *n_planar_submap = *n_sphere_scan = *n_sphere_submap = 0;
  if (n == 0) return TLOAM_B200_OK;              // calculatePCAInfo fails on an empty cloud: nothing is selected (:49-54, :141)
  if (!xyz) return TLOAM_B200_ERR_INVALID_ARG;
  FeArena A;
  std::vector<unsigned> vp(n), vs(n);            // sorted point indices (candidates first), fetched with the counts
  A.host_val_p = vp.data(); A.host_val_s = vs.data();
  const int rc = fe_run(h, cfg, xyz, n, true, A);
  if (rc != TLOAM_B200_OK) return rc;
  unsigned counts[4];
  memcpy(counts, h->h_result + 28, sizeof(counts));
  const unsigned np = counts[0], ns = counts[1], nps = counts[2], nss = counts[3];
  for (unsigned i = 0; i < np; ++i) planar_submap_index[i] = vp[i];                    // :180
  for (unsigned i = 0; i < nps; ++i) planar_scan_index[i] = vp[i];                     // :177-178
  *n_planar_submap = np; *n_planar_scan = nps;
  for (unsigned i = 0; i < ns; ++i) sphere_submap_index[i] = i;                          // :187 (rank, not index)
  for (unsigned i = 0; i < nss; ++i) sphere_scan_index[i] = i;                           // :184-185
  *n_sphere_submap = ns; *n_sphere_scan = nss;
  if (sphere_candidates) for (unsigned i = 0; i < ns; ++i) sphere_candidates[i] = vs[i];
  return TLOAM_B200_OK;
}

int tloam_b200_pca_info(tloam_b200_handle* h, const tloam_feature_config* cfg, const double* xyz, size_t n, double* cvr,
                        double* flatness, double* sphericity, double* normal, int* num_sum, int* neigh) {
  if (!h || !cfg || !xyz || n == 0) return TLOAM_B200_ERR_INVALID_ARG;
  FeArena A;
  const int rc = fe_run(h, cfg, xyz, n, false, A);
  if (rc != TLOAM_B200_OK) return rc;
  if (cvr) CU_TRY(cudaMemcpyAsync(cvr, A.out.cvr, n * 8, cudaMemcpyDeviceToHost, h->stream));
  if (flatness) CU_TRY(cudaMemcpyAsync(flatness, A.out.flatness, n * 8, cudaMemcpyDeviceToHost, h->stream));
  if (sphericity) CU_TRY(cudaMemcpyAsync(sphericity, A.out.sphericity, n * 8, cudaMemcpyDeviceToHost, h->stream));
  if (normal) CU_TRY(cudaMemcpyAsync(normal, A.out.normal, n * 24, cudaMemcpyDeviceToHost, h->stream));
  if (num_sum) CU_TRY(cudaMemcpyAsync(num_sum, A.out.num_sum, n * 4, cudaMemcpyDeviceToHost, h->stream));
  std::vector<int> nb;
  if (neigh) {
    nb.resize(n * kFeK);
    CU_TRY(cudaMemcpyAsync(nb.data(), A.out.neigh, n * kFeK * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (neigh)
    for (size_t i = 0; i < n; ++i)
      for (int j = 0; j < cfg->K; ++j) neigh[i * cfg->K + j] = nb[i * kFeK + j];
  return TLOAM_B200_OK;
}

int tloam_b200_voxel_down_sample(tloam_b200_handle* h, const double* pts, size_t n, double voxel, double* out, size_t* n_out) {
  if (!h || (!pts && n) || !out || !n_out) return TLOAM_B200_ERR_INVALID_ARG;
  *n_out = 0;
  if (n && !(voxel > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!vox_fits(vox_extent(pts, n), voxel)) return TLOAM_B200_ERR_VOXEL_RANGE;
  CU_TRY(cudaSetDevice(h->device));
  int rc = upload_points(h, pts, n);
  if (rc != TLOAM_B200_OK) return rc;
  rc = ensure_dev(h, &h->d_acc_tmp, &h->cap_acc_tmp, n, false);
  if (rc != TLOAM_B200_OK) return rc;
  rc = voxel_pipeline(h, h->d_up, n, nullptr, 0u, nullptr, nullptr, nullptr, 0.0, voxel, h->d_acc_tmp, h->d_cnt + 8);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(h->h_result + 28, h->d_cnt + 8, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  unsigned cnt;
  memcpy(&cnt, h->h_result + 28, sizeof(cnt));
  *n_out = cnt;
  if (cnt) CU_TRY(cudaMemcpyAsync(out, h->d_acc_tmp, (size_t)cnt * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// on_device: the four clouds are device buffers (tloam_b200_submap_init_frame: the last processed frame), copied D2D
static int submap_init_impl(tloam_b200_handle* h, const tloam_submap_config* cfg, const double* edge, size_t ne,
                            const double* ground_raw, size_t ng, const double* planar_sub, size_t np,
                            const double* sphere_sub, size_t ns, bool on_device) {
  if (!h || !cfg || (!edge && ne) || (!ground_raw && ng) || (!planar_sub && np) || (!sphere_sub && ns)) return TLOAM_B200_ERR_INVALID_ARG;
  if (cfg->planar_frame_size < 1 || cfg->planar_frame_size > 64) return TLOAM_B200_ERR_INVALID_ARG;
  // every submap_update crops to pose.t +- L before its voxel pass, so 2 L / voxel + 1 < 2^21 keeps each cropped cloud's
  // indices keyable (the extra voxel covers the min bound's half-voxel margin and the rounding of the box)
  const double crop_len[2] = {cfg->edge_crop_box_length, cfg->ground_crop_box_length};
  const double crop_vox[2] = {cfg->edge_down_sample_submap, cfg->ground_down_sample_submap};
  for (int k = 0; k < 2; ++k)
    if (!(crop_vox[k] > 0.0) || !(2.0 * crop_len[k] / crop_vox[k] + 1.0 < (double)(1u << kGMapKeyBits))) return TLOAM_B200_ERR_INVALID_ARG;
  if (ng && !(cfg->ground_down_sample > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!vox_fits(on_device ? h->fr_ground_ext : vox_extent(ground_raw, ng), cfg->ground_down_sample)) return TLOAM_B200_ERR_VOXEL_RANGE;
  CU_TRY(cudaSetDevice(h->device));
  h->scfg = *cfg;
  if (!h->d_pose) CU_TRY(cudaMalloc(&h->d_pose, 16 * sizeof(double)));
  int rc;
  const cudaMemcpyKind kind = on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  h->acc_cur[0] = h->acc_cur[1] = 0;
  // edge: raw copy (front_end.cpp:286)
  if ((rc = ensure_dev(h, &h->d_acc[0], &h->cap_acc[0], ne, false)) != TLOAM_B200_OK) return rc;
  if (ne) CU_TRY(cudaMemcpyAsync(h->d_acc[0], edge, ne * 3 * sizeof(double), kind, h->stream));
  h->n_acc[0] = ne;
  k_set_counts<<<1, 32, 0, h->stream>>>(h->d_cnt + 4, 0, (unsigned)ne, -1, 0u);
  // ground: VoxelDownSample(ground_down_sample) (:287)
  if (!on_device && (rc = upload_points(h, ground_raw, ng)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, &h->d_acc[1], &h->cap_acc[1], ng, false)) != TLOAM_B200_OK) return rc;
  if ((rc = voxel_pipeline(h, on_device ? ground_raw : h->d_up, ng, nullptr, 0u, nullptr, nullptr, nullptr, 0.0, cfg->ground_down_sample,
                           h->d_acc[1], acc_count(h, 1))) != TLOAM_B200_OK) return rc;
  // planar / sphere: the submap-index selections (:291-292); the sliding-window buffers stay empty (:285-305)
  if ((rc = ensure_dev(h, &h->d_cat, &h->cap_cat, np, false)) != TLOAM_B200_OK) return rc;
  if (np) CU_TRY(cudaMemcpyAsync(h->d_cat, planar_sub, np * 3 * sizeof(double), kind, h->stream));
  h->n_cat = np;
  cudaFree(h->d_sphere0); h->d_sphere0 = nullptr;
  if (ns) {
    CU_TRY(cudaMalloc(&h->d_sphere0, ns * 3 * sizeof(double)));
    CU_TRY(cudaMemcpyAsync(h->d_sphere0, sphere_sub, ns * 3 * sizeof(double), kind, h->stream));
  }
  h->n_sphere0 = ns; h->sphere_is_init = true;
  for (double* p : h->ring) cudaFree(p);
  h->ring.clear(); h->ring_n.clear(); h->ring_cap.clear();
  // once per sequence: wait for the uploads and read the exact ground count
  CU_TRY(cudaMemcpyAsync(h->h_result + 28, acc_count(h, 1), sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  unsigned gcnt;
  memcpy(&gcnt, h->h_result + 28, sizeof(gcnt));
  h->n_acc[1] = gcnt;
  for (int k = 0; k < 2; ++k) { h->cum_add[k] = h->known_cum[k] = 0; h->known_cnt[k] = h->n_acc[k]; }
  for (auto& pr : h->probes) pr.pending = false;
  h->submap_ready = true;
  return submap_set_target(h);
}

int tloam_b200_submap_init(tloam_b200_handle* h, const tloam_submap_config* cfg, const double* edge, size_t ne,
                           const double* ground_raw, size_t ng, const double* planar_sub, size_t np,
                           const double* sphere_sub, size_t ns) {
  return submap_init_impl(h, cfg, edge, ne, ground_raw, ng, planar_sub, np, sphere_sub, ns, false);
}

// FrontEnd::updateSubmap (ref: front_end.cpp:201-267) enqueued WITHOUT a host round trip: the voxel counts that size the
// next map stay on the device (the host only tracks upper bounds, tightened by asynchronous read-backs), and in the
// chained form the pose is the device-resident result of the frame that was just enqueued.
// planar_on_device: planar_sub is a device buffer written on the handle's stream (the last processed frame's selection), read in place
static int submap_update_impl(tloam_b200_handle* h, const double* pose_host, const double* planar_sub, size_t np,
                              bool planar_on_device = false) {
  if (!h || (!planar_sub && np)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->submap_ready || !h->have_src) return TLOAM_B200_ERR_NOT_READY;
  if (!h->src_staged) return TLOAM_B200_ERR_NOT_READY;           // the staged source is what gets appended
  CU_TRY(cudaSetDevice(h->device));
  harvest_counts(h);
  const tloam_submap_config& cf = h->scfg;
  int rc;
  const double* d_pose = h->d_pose;
  if (pose_host) {
    double tmp[16];
    memcpy(tmp, pose_host, sizeof(tmp));
    CU_TRY(cudaMemcpyAsync(h->d_pose, tmp, sizeof(tmp), cudaMemcpyHostToDevice, h->stream));   // pageable source: staged before return
  } else {
    d_pose = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, result));
  }
  const unsigned tb = 256;
  // ---- planar sliding window (:207-217, 232-242): newest frame transformed by its pose ----
  // pipelined handles: the upload runs on src_stream (it does not depend on the frame that is still being registered);
  // its buffer is free again once the transform below has read it
  static const bool no_prefetch = getenv("TLOAM_B200_NO_PREFETCH") != nullptr;
  const bool side = h->async_inputs && !h->profiling && !no_prefetch;
  const double* d_planar_in = nullptr;
  if (planar_on_device) {
    d_planar_in = planar_sub;                                     // ordered by the fork below (ps waits for the handle's stream)
  } else if (side) {
    if (np > h->cap_up_planar) {
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_up_planar); h->d_up_planar = nullptr; h->cap_up_planar = 0;
      CU_TRY(cudaMalloc(&h->d_up_planar, (np + np / 2 + 1024) * 3 * sizeof(double)));
      h->cap_up_planar = np + np / 2 + 1024;
      h->planar_free_valid = false;
    }
    if (h->planar_free_valid) CU_TRY(cudaStreamWaitEvent(h->src_stream, h->ev_planar_free, 0));
    if (np) CU_TRY(cudaMemcpyAsync(h->d_up_planar, planar_sub, np * 3 * sizeof(double), cudaMemcpyHostToDevice, h->src_stream));
    CU_TRY(cudaEventRecord(h->ev_planar_in, h->src_stream));
    d_planar_in = h->d_up_planar;
  } else {
    if ((rc = upload_points(h, planar_sub, np)) != TLOAM_B200_OK) return rc;
    d_planar_in = h->d_up;
  }
  // ---- fork: the ground accumulator (k = 1 below) is appended, cropped and down-sampled on sub_stream, the planar
  //      window is assembled on fit_stream (idle between frames), the edge accumulator stays on the handle's stream ----
  cudaStream_t gs = side ? h->sub_stream : h->stream;
  cudaStream_t ps = side ? h->fit_stream : h->stream;
  if (side) {
    CU_TRY(cudaEventRecord(h->ev_sub[0], h->stream));
    CU_TRY(cudaStreamWaitEvent(gs, h->ev_sub[0], 0));
    CU_TRY(cudaStreamWaitEvent(ps, h->ev_sub[0], 0));
    if (!planar_on_device) CU_TRY(cudaStreamWaitEvent(ps, h->ev_planar_in, 0));
  }
  double* slot = nullptr; size_t slot_cap = 0;
  if ((int)h->ring.size() >= cf.planar_frame_size) {            // recycle the oldest buffer
    slot = h->ring.front(); slot_cap = h->ring_cap.front();
    h->ring.erase(h->ring.begin()); h->ring_n.erase(h->ring_n.begin()); h->ring_cap.erase(h->ring_cap.begin());
  }
  if ((rc = ensure_dev(h, &slot, &slot_cap, np, false)) != TLOAM_B200_OK) return rc;
  if (np) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_transform_append<<<(unsigned)((np + tb - 1) / tb), tb, 0, ps>>>(d_planar_in, (unsigned)np, slot, d_pose, nullptr)));
  if (side) { CU_TRY(cudaEventRecord(h->ev_planar_free, ps)); h->planar_free_valid = true; }
  h->ring.push_back(slot); h->ring_n.push_back(np); h->ring_cap.push_back(slot_cap);
  size_t tot = 0;
  for (size_t k : h->ring_n) tot += k;
  if ((rc = ensure_dev(h, &h->d_cat, &h->cap_cat, tot, false)) != TLOAM_B200_OK) return rc;
  size_t off = 0;
  for (size_t f = 0; f < h->ring.size(); ++f) {
    if (h->ring_n[f]) CU_TRY(cudaMemcpyAsync(h->d_cat + 3 * off, h->ring[f], h->ring_n[f] * 3 * sizeof(double), cudaMemcpyDeviceToDevice, ps));
    off += h->ring_n[f];
  }
  if (side) CU_TRY(cudaEventRecord(h->ev_planar_done, ps));     // the planar window is assembled
  h->n_cat = tot;
  h->sphere_is_init = false;
  // ---- edge / ground: append the current source features in the world frame (:245-246), crop (:248-264),
  //      VoxelDownSample ----
  const int src_cloud[2] = {0, 3};
  const double vox[2] = {cf.edge_down_sample_submap, cf.ground_down_sample_submap};
  const double len[2] = {cf.edge_crop_box_length, cf.ground_crop_box_length};
  size_t soff[4], o = 0;
  for (int c = 0; c < 4; ++c) { soff[c] = o; o += h->n_src[c]; }
  for (int k = 0; k < 2; ++k) {
    const size_t nadd = h->n_src[src_cloud[k]];
    const size_t nall = h->n_acc[k] + nadd;                       // bound
    cudaStream_t ks = k == 1 ? gs : h->stream;                    // ground on the side stream, own scratch + output buffer
    double*& tmp = (k == 1 && side) ? h->d_acc_tmp1 : h->d_acc_tmp;
    size_t& tmp_cap = (k == 1 && side) ? h->cap_acc_tmp1 : h->cap_acc_tmp;
    if ((rc = ensure_dev(h, &h->d_acc[k], &h->cap_acc[k], nall, true)) != TLOAM_B200_OK) return rc;
    if ((rc = ensure_dev(h, &tmp, &tmp_cap, nall, false)) != TLOAM_B200_OK) return rc;
    unsigned* cur = acc_count(h, k);
    if (nadd) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_transform_append<<<(unsigned)((nadd + tb - 1) / tb), tb, 0, ks>>>(
        h->d_stage_src + 3 * soff[src_cloud[k]], (unsigned)nadd, h->d_acc[k], d_pose, cur)));
    h->acc_cur[k] ^= 1;
    if ((rc = voxel_pipeline(h, h->d_acc[k], nall, cur, (unsigned)nadd, nullptr, nullptr, d_pose, len[k], vox[k], tmp,
                             acc_count(h, k), ks, (k == 1 && side) ? 1 : 0)) != TLOAM_B200_OK) return rc;
    // the down-sampled cloud becomes the accumulator (swap buffers)
    double* t = h->d_acc[k]; h->d_acc[k] = tmp; tmp = t;
    size_t tc = h->cap_acc[k]; h->cap_acc[k] = tmp_cap; tmp_cap = tc;
    h->n_acc[k] = nall;
    h->cum_add[k] += nadd;
  }
  if (side) {                                                     // join
    CU_TRY(cudaEventRecord(h->ev_sub[1], gs));
    CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_sub[1], 0));
    CU_TRY(cudaStreamWaitEvent(h->stream, h->ev_planar_done, 0));
  }
  CU_TRY(cudaEventRecord(h->ev_stage_free[h->stage_cur], h->stream));   // the staged source has been appended: its buffer is free
  // asynchronous read-back of the two exact counts (tightens the bounds of later frames)
  {
    tloam_b200_handle::CntProbe& pr = h->probes[h->probe_next];
    if (!pr.pending || cudaEventQuery(pr.ev) == cudaSuccess) {
      if (pr.pending) { pr.pending = false; for (int k = 0; k < 2; ++k) if (pr.cum[k] >= h->known_cum[k]) { h->known_cum[k] = pr.cum[k]; h->known_cnt[k] = pr.h_vals[k]; } }
      for (int k = 0; k < 2; ++k) {
        CU_TRY(cudaMemcpyAsync(pr.h_vals + k, acc_count(h, k), sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
        pr.cum[k] = h->cum_add[k];
      }
      CU_TRY(cudaEventRecord(pr.ev, h->stream));
      pr.pending = true;
      h->probe_next = (h->probe_next + 1) & 3;
    } else {
      cudaGetLastError();
    }
  }
  return submap_set_target(h);                                   // :267
}

int tloam_b200_submap_update(tloam_b200_handle* h, const double pose[16], const double* planar_sub, size_t np,
                             const double* sphere_sub, size_t ns) {
  (void)sphere_sub; (void)ns;   // stored but never used by the reference (front_end.cpp:202-205, 220-230)
  if (!pose) return TLOAM_B200_ERR_INVALID_ARG;
  return submap_update_impl(h, pose, planar_sub, np);
}

// pose = the result of the frame that was just enqueued on this handle, read on the device: frames chain with no host
// round trip (set_source -> scan_match_predicted_async -> submap_update_chained -> next frame)
int tloam_b200_submap_update_chained(tloam_b200_handle* h, const double* planar_sub, size_t np) {
  return submap_update_impl(h, nullptr, planar_sub, np);
}

// exact sizes (synchronises: inspection / tests)
int tloam_b200_submap_sizes(tloam_b200_handle* h, size_t n[4]) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->submap_ready) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  unsigned cnt[2];
  for (int k = 0; k < 2; ++k) CU_TRY(cudaMemcpyAsync(h->h_result + 28 + k, acc_count(h, k), sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (int k = 0; k < 2; ++k) memcpy(&cnt[k], h->h_result + 28 + k, sizeof(unsigned));
  n[0] = cnt[0]; n[1] = h->sphere_is_init ? h->n_sphere0 : h->n_cat; n[2] = h->n_cat; n[3] = cnt[1];
  return TLOAM_B200_OK;
}

int tloam_b200_submap_download(tloam_b200_handle* h, int cloud, double* out, size_t capacity_points) {
  if (!h || !out || cloud < 0 || cloud > 3) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->submap_ready) return TLOAM_B200_ERR_NOT_READY;
  size_t n[4];
  const int rc = tloam_b200_submap_sizes(h, n);
  if (rc != TLOAM_B200_OK) return rc;
  if (capacity_points < n[cloud]) return TLOAM_B200_ERR_INVALID_ARG;
  const double* src = cloud == 0 ? h->d_acc[0] : cloud == 3 ? h->d_acc[1] : (cloud == 1 && h->sphere_is_init) ? h->d_sphere0 : h->d_cat;
  CU_TRY(cudaSetDevice(h->device));
  if (n[cloud]) CU_TRY(cudaMemcpyAsync(out, src, n[cloud] * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}


// ---------------------------------------------------------------------------------------------
// "next" row (f)-4, first part: multi-region ground extraction (ground_extract.cuh)
// ---------------------------------------------------------------------------------------------
void tloam_b200_ground_default_config(tloam_ground_config* c) {   // ref: config/mapping/segmentation.yaml
  c->sensor_model = 64; c->sensor_height = 1.73; c->vertical_res = 0.4; c->init_angle = -24.9;
  c->sensor_min_range = 1.0; c->sensor_max_range = 120.0;
  c->quadrant = 4; c->num_sec = 3; c->plane_dis = 0.3; c->max_iter = 3; c->ground_seed_num = 20;
}

// Segmentation::initSections, ref: segmentation.cpp:174-221 (host side: 64 iterations of scalar arithmetic).  Restated
// literally: the `continue` at :203-206 also skips the angle increment, so the table stalls at the first >= 5 m jump and
// only two section bounds are produced with the shipped configuration.
static int ground_section_bounds(const tloam_ground_config& c, float out[4]) {
  int nb = 0;
  int boundary[4] = {0, 0, 0, 0};
  const int section_width = static_cast<int>(std::ceil(1.0 * c.sensor_model) / c.num_sec);
  for (int i = 0; i < c.num_sec; ++i) boundary[i] = section_width * (i + 1) - 1;
  double prev_radius = 0.0, angle = c.init_angle;
  int sec = 0;
  for (int i = 0; i < c.sensor_model; ++i) {
    if (c.sensor_model == 64 && i == 31) angle += 1.7;
    double cur = c.sensor_height / std::tan(std::fabs(angle) / 180.0 * M_PI);
    cur = cur < c.sensor_max_range ? cur : c.sensor_max_range;
    if (i >= 1) {
      const double dis = std::fabs(cur - prev_radius);
      if (dis >= 5.0 || dis <= 0.0) continue;
    }
    if (sec < c.num_sec && i == boundary[sec] && sec <= 3) {
      const double theta = std::fabs(angle / 180 * M_PI);
      out[nb++] = (theta != 0 && i < c.sensor_model) ? static_cast<float>(c.sensor_height / std::tan(theta))
                                                      : static_cast<float>(c.sensor_max_range);
      ++sec;
    }
    prev_radius = cur;
    angle += c.vertical_res;
  }
  return nb;
}

// groundRemove with both forms of the per-point channel: beam = (int)intensity, intensity = the reference's FP64 value
static int ground_run(tloam_b200_handle* h, const tloam_ground_config* cfg, const double* xyz, size_t n, size_t* ground_index,
                      size_t* n_ground, size_t* object_index, size_t* n_object, int* beam, double* intensity, int* region,
                      double* height_threshold, double* planes) {
  if (!h || !cfg || !ground_index || !n_ground || !object_index || !n_object) return TLOAM_B200_ERR_INVALID_ARG;
  h->seg_gen++;                                                            // the last raw scan may no longer be in place
  *n_ground = *n_object = 0;
  if ((cfg->sensor_model != 64 && cfg->sensor_model != 16) || cfg->quadrant != 4 || cfg->num_sec < 1 || cfg->num_sec > 3 ||
      cfg->max_iter < 1 || cfg->max_iter > kGeMaxIter || cfg->ground_seed_num < 1)
    return TLOAM_B200_ERR_INVALID_ARG;                            // the HDL-64E and VLP-16 branches (:433-442); others: `default:`
  if (planes) for (int i = 0; i < 12 * kGeMaxIter * 4; ++i) planes[i] = std::nan("");
  if (n == 0) { if (height_threshold) *height_threshold = 1.0; return TLOAM_B200_OK; }   // :335-338
  if (!xyz || n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  GeArgs a;
  memset(&a, 0, sizeof(a));
  a.n = (unsigned)n; a.nchunk = (unsigned)((n + kGeChunk - 1) / kGeChunk);
  a.sensor_model = cfg->sensor_model; a.num_sec = cfg->num_sec; a.max_iter = cfg->max_iter; a.seed_num = cfg->ground_seed_num;
  a.sensor_height = cfg->sensor_height; a.min_range = cfg->sensor_min_range; a.max_range = cfg->sensor_max_range;
  a.plane_dis = cfg->plane_dis;
  a.ang_bot = std::fabs(cfg->init_angle) + 0.1; a.vertical_res = cfg->vertical_res;
  a.nbounds = ground_section_bounds(*cfg, a.bounds);              // VLP-16 with the shipped values: ONE bound (see DESIGN.md §4d)
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += round_up(bytes, 256); return o; };
  const size_t o_pts = take(n * 24), o_ct = take(a.nchunk * 4), o_cs = take(a.nchunk * 8), o_sc = take(64), o_beam = take(n * 4),
               o_key = take(n), o_cc = take((size_t)a.nchunk * kGeKeys * 4), o_kb = take((kGeKeys + 1) * 4), o_ord = take(n * 4),
               o_flag = take(n), o_lists = take(2 * n * 4), o_rc = take(12 * 2 * 4), o_pl = take(12 * kGeMaxIter * 4 * 8),
               o_og = take(n * 4), o_oo = take(n * 4), o_oc = take(64), o_int = take(n * 8);
  if (off > h->cap_ge) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ge); h->d_ge = nullptr; h->cap_ge = 0;
    CU_TRY(cudaMalloc(&h->d_ge, off + off / 4));
    h->cap_ge = off + off / 4;
  }
  unsigned char* b = h->d_ge;
  a.pts = (const double*)(b + o_pts); a.chunk_trans = (unsigned*)(b + o_ct); a.chunk_sum = (double*)(b + o_cs);
  a.scal = (double*)(b + o_sc); a.beam = (int*)(b + o_beam); a.key = b + o_key; a.chunk_cnt = (unsigned*)(b + o_cc);
  a.key_base = (unsigned*)(b + o_kb); a.order = (unsigned*)(b + o_ord); a.flag = b + o_flag; a.lists = (unsigned*)(b + o_lists);
  a.reg_cnt = (unsigned*)(b + o_rc); a.planes = (double*)(b + o_pl); a.out_ground = (unsigned*)(b + o_og);
  a.out_object = (unsigned*)(b + o_oo); a.out_counts = (unsigned*)(b + o_oc);
  a.intensity = (double*)(b + o_int); a.first_trans = (unsigned*)(a.scal + 4);
  if (h->seg.active) a.pts = h->seg.dev_xyz;
  else CU_TRY(cudaMemcpyAsync(b + o_pts, xyz, n * 24, cudaMemcpyHostToDevice, h->stream));
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_pre<<<a.nchunk, kGeChunk, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_scan1<<<1, 1024, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_region<<<a.nchunk, kGeChunk, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_scan2<<<1, 1024, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_scatter<<<a.nchunk, kGeChunk, 0, h->stream>>>(a)));
  constexpr size_t kGeFitSmem = (6 * kGeTile + kGeSeedCache) * sizeof(double);
  if (!h->ge_attr_set) {
    CU_TRY(cudaFuncSetAttribute(k_ge_fit, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGeFitSmem));
    h->ge_attr_set = true;
  }
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_fit<<<4 * cfg->num_sec, kGeFitThreads, kGeFitSmem, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_GROUND, (k_ge_emit<<<dim3(32, 25), 256, 0, h->stream>>>(a)));
  CU_TRY(cudaGetLastError());
  // counts + threshold first (one small copy each, one synchronisation), then exactly the list prefixes
  CU_TRY(cudaMemcpyAsync(h->h_result + 28, a.out_counts, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaMemcpyAsync(h->h_result + 29, a.scal, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  unsigned counts[2];
  memcpy(counts, h->h_result + 28, sizeof(counts));
  if (height_threshold) *height_threshold = h->h_result[29];
  if (h->seg.active) {                                                     // chained: the lists stay on the device
    h->seg.ground = a.out_ground; h->seg.object = a.out_object; h->seg.beam = a.beam; h->seg.intensity = a.intensity;
    h->seg.n_ground = counts[0]; h->seg.n_object = counts[1];
    *n_ground = counts[0]; *n_object = counts[1];
    return TLOAM_B200_OK;
  }
  std::vector<unsigned> gi(counts[0]), oi(counts[1]);
  if (counts[0]) CU_TRY(cudaMemcpyAsync(gi.data(), a.out_ground, counts[0] * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  if (counts[1]) CU_TRY(cudaMemcpyAsync(oi.data(), a.out_object, counts[1] * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  if (beam) CU_TRY(cudaMemcpyAsync(beam, a.beam, n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (intensity) CU_TRY(cudaMemcpyAsync(intensity, a.intensity, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  std::vector<unsigned char> keys;
  if (region) { keys.resize(n); CU_TRY(cudaMemcpyAsync(keys.data(), a.key, n, cudaMemcpyDeviceToHost, h->stream)); }
  if (planes) CU_TRY(cudaMemcpyAsync(planes, a.planes, 12 * kGeMaxIter * 4 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (unsigned i = 0; i < counts[0]; ++i) ground_index[i] = gi[i];
  for (unsigned i = 0; i < counts[1]; ++i) object_index[i] = oi[i];
  if (region) for (size_t i = 0; i < n; ++i) region[i] = keys[i];
  *n_ground = counts[0]; *n_object = counts[1];
  return TLOAM_B200_OK;
}

int tloam_b200_ground_remove(tloam_b200_handle* h, const tloam_ground_config* cfg, const double* xyz, size_t n, size_t* ground_index,
                             size_t* n_ground, size_t* object_index, size_t* n_object, double* intensity, int* region,
                             double* height_threshold, double* planes) {
  return ground_run(h, cfg, xyz, n, ground_index, n_ground, object_index, n_object, nullptr, intensity, region, height_threshold, planes);
}

int tloam_b200_ground_extract(tloam_b200_handle* h, const tloam_ground_config* cfg, const double* xyz, size_t n,
                              size_t* ground_index, size_t* n_ground, size_t* object_index, size_t* n_object, int* beam,
                              int* region, double* height_threshold, double* planes) {
  return ground_run(h, cfg, xyz, n, ground_index, n_ground, object_index, n_object, beam, nullptr, region, height_threshold, planes);
}

// ---------------------------------------------------------------------------------------------
// "next" row (f)-4, second part: LOAM-style edge extraction (edge_extract.cuh)
// ---------------------------------------------------------------------------------------------
int tloam_b200_extract_edge(tloam_b200_handle* h, int sensor_model, int ring_min_num, const double* xyz, const double* intensity,
                            size_t n, size_t* edge_index, size_t* n_edge, size_t* non_edge_index, size_t* n_non_edge) {
  if (!h || !edge_index || !n_edge || !non_edge_index || !n_non_edge) return TLOAM_B200_ERR_INVALID_ARG;
  h->seg_gen++;
  *n_edge = *n_non_edge = 0;
  if (sensor_model < 1 || sensor_model > kEeKeys || ring_min_num < 0) return TLOAM_B200_ERR_INVALID_ARG;
  if (n == 0) return TLOAM_B200_OK;                                        // ref: :1222-1225 (empty input: nothing extracted)
  if (!xyz || !intensity || n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  EeArgs a;
  memset(&a, 0, sizeof(a));
  a.n = (unsigned)n; a.nchunk = (unsigned)((n + kEeChunk - 1) / kEeChunk);
  a.sensor_model = sensor_model; a.ring_min = ring_min_num;
  const int nsec = kEeKeys * kEeSectors;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += round_up(bytes, 256); return o; };
  const size_t o_pts = take(n * 24), o_int = take(n * 8), o_key = take(n), o_cc = take((size_t)a.nchunk * kEeKeys * 4),
               o_rb = take((kEeKeys + 1) * 4), o_ord = take(n * 4), o_se = take(n * 4), o_sn = take(n * 4), o_sc = take(nsec * 2 * 4),
               o_so = take((nsec + 1) * 2 * 4), o_oe = take(n * 8), o_on = take(n * 8), o_st = take(64);
  if (off > h->cap_ge) {                                                   // shares the segmentation arena
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ge); h->d_ge = nullptr; h->cap_ge = 0;
    CU_TRY(cudaMalloc(&h->d_ge, off + off / 4));
    h->cap_ge = off + off / 4;
  }
  unsigned char* b = h->d_ge;
  a.pts = (const double*)(b + o_pts); a.intensity = (const double*)(b + o_int); a.key = b + o_key;
  a.chunk_cnt = (unsigned*)(b + o_cc); a.ring_base = (unsigned*)(b + o_rb); a.order = (unsigned*)(b + o_ord);
  a.sec_edge = (unsigned*)(b + o_se); a.sec_non = (unsigned*)(b + o_sn); a.sec_cnt = (unsigned*)(b + o_sc);
  a.sec_off = (unsigned*)(b + o_so); a.out_edge = (unsigned long long*)(b + o_oe); a.out_non = (unsigned long long*)(b + o_on);
  a.status = (int*)(b + o_st);
  if (!h->ee_attr_set) {
    CU_TRY(cudaFuncSetAttribute(k_ee_section, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kEeSmemBytes));
    h->ee_attr_set = true;
  }
  if (h->seg.active) { a.pts = h->seg.dev_xyz; a.intensity = h->seg.dev_intensity; }
  else {
    CU_TRY(cudaMemcpyAsync(b + o_pts, xyz, n * 24, cudaMemcpyHostToDevice, h->stream));
    CU_TRY(cudaMemcpyAsync(b + o_int, intensity, n * 8, cudaMemcpyHostToDevice, h->stream));
  }
  CU_TRY(cudaMemsetAsync(b + o_sc, 0, nsec * 2 * 4, h->stream));         // beams >= sensor_model have no sections
  TL_LAUNCH(TLOAM_B200_K_EDGE, (k_ee_key<<<a.nchunk, kEeChunk, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_EDGE, (k_ee_scan<<<1, kEeKeys, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_EDGE, (k_ee_scatter<<<a.nchunk, kEeChunk, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_EDGE, (k_ee_section<<<dim3(kEeSectors, sensor_model), kEeThreads, kEeSmemBytes, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_EDGE, (k_ee_offsets<<<1, 32, 0, h->stream>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_EDGE, (k_ee_copy<<<dim3(kEeSectors, sensor_model), kEeThreads, 0, h->stream>>>(a)));
  CU_TRY(cudaGetLastError());
  unsigned tot[2];
  int st = 0;
  CU_TRY(cudaMemcpyAsync(tot, a.sec_off + 2 * (sensor_model * kEeSectors), sizeof(tot), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaMemcpyAsync(&st, a.status, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (st != 0) {
    snprintf(h->last_error, sizeof(h->last_error), "extract_edge: a beam sector holds more than %d curvature values", kEeMaxSection);
    return TLOAM_B200_ERR_INVALID_ARG;
  }
  static_assert(sizeof(size_t) == sizeof(unsigned long long), "index lists are copied straight into size_t arrays");
  if (h->seg.active) {                                                     // chained: the lists stay on the device
    h->seg.edge = a.out_edge; h->seg.non_edge = a.out_non; h->seg.n_edge = tot[0]; h->seg.n_non = tot[1];
    *n_edge = tot[0]; *n_non_edge = tot[1];
    return TLOAM_B200_OK;
  }
  if (tot[0]) CU_TRY(cudaMemcpyAsync(edge_index, a.out_edge, tot[0] * sizeof(size_t), cudaMemcpyDeviceToHost, h->stream));
  if (tot[1]) CU_TRY(cudaMemcpyAsync(non_edge_index, a.out_non, tot[1] * sizeof(size_t), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  *n_edge = tot[0]; *n_non_edge = tot[1];
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// "next" row (f)-4, third part: object segmentation = DCVC (object_segment.cuh)
// ---------------------------------------------------------------------------------------------
void tloam_b200_dcvc_default_config(tloam_dcvc_config* c) {                  // ref: config/mapping/segmentation.yaml
  if (!c) return;
  c->start_r = 0.35; c->delta_r = 0.0004; c->delta_p = 1.2; c->delta_a = 1.2; c->min_seg = 80;
  c->sensor_min_range = 1.0; c->sensor_max_range = 120.0;
  c->min_pitch_init = 0.0; c->max_pitch_init = 0.0; c->min_polar_init = 0.0; c->max_polar_init = 0.0;
}

int tloam_b200_object_segmentation(tloam_b200_handle* h, const tloam_dcvc_config* cfg, const double* xyz, size_t n,
                                   size_t* seg_index, size_t* n_seg, int* n_clusters, int* sizes, double* boxes, int* root,
                                   int* cluster, int* voxel, double* polar) {
  if (!h || !cfg || !seg_index || !n_seg || !n_clusters) return TLOAM_B200_ERR_INVALID_ARG;
  h->seg_gen++;
  *n_seg = 0; *n_clusters = 0;
  if (!(cfg->delta_p > 0.0) || !(cfg->delta_a > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (n == 0) return TLOAM_B200_OK;                                         // ref: :1088-1093 (nothing to convert)
  if (!xyz || n > ((size_t)1 << 26)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  OsArgs a;
  memset(&a, 0, sizeof(a));
  a.n = (unsigned)n; a.nchunk = (unsigned)((n + kOsChunk - 1) / kOsChunk);
  a.start_r = cfg->start_r; a.delta_r = cfg->delta_r; a.delta_p = cfg->delta_p; a.delta_a = cfg->delta_a;
  a.min_range = cfg->sensor_min_range; a.max_range = cfg->sensor_max_range; a.min_seg = cfg->min_seg;
  a.init[0] = cfg->min_pitch_init; a.init[1] = cfg->max_pitch_init; a.init[2] = cfg->min_polar_init; a.init[3] = cfg->max_polar_init;
  size_t cap = 1024;
  while (cap < 2 * n) cap <<= 1;
  a.cap_mask = (unsigned)(cap - 1);
  const size_t n32 = round_up(n, 32);
  const size_t state_words = (n + 15) / 16 + 1;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += round_up(bytes, 256); return o; };
  const size_t o_pts = take(n * 24), o_pol = take(n * 24), o_enc = take(64), o_ext = take(64), o_par = take(64),
               o_bnd = take(kOsMaxBounds * 8), o_key = take(n * 4), o_crd = take(n * 12), o_tab = take(cap * 8), o_sv = take(cap * 4),
               o_ps = take(n * 4), o_vid = take(n * 4), o_f1 = take(n * 4), o_f2 = take(n * 4),
               o_ek = take(n * 4), o_ept = take(n * 4), o_ei = take(n32 * 4), o_rows = take((n32 + 32 * kOsSeqStages) * kOsRowStride * 4), o_ep = take(n32),
               o_stg = take(state_words * 4), o_par2 = take(n * 4), o_root = take(n * 4), o_cnt = take(n * 4), o_clr = take(n * 4),
               o_crr = take(n * 4), o_cl = take(n * 4), o_sz = take(n * 4), o_pk = take(n * 4), o_box = take(n * 48), o_benc = take(n * 48),
               o_cc = take((size_t)a.nchunk * kOsKeys * 4), o_kb = take((kOsKeys + 1) * 4), o_pa = take(n * 4), o_pb = take(n * 4),
               o_seg = take(n * 8);
  if (off > h->cap_ge) {                                                   // shares the segmentation arena
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ge); h->d_ge = nullptr; h->cap_ge = 0;
    CU_TRY(cudaMalloc(&h->d_ge, off + off / 4));
    h->cap_ge = off + off / 4;
  }
  unsigned char* b = h->d_ge;
  a.pts = (const double*)(b + o_pts); a.polar = (double*)(b + o_pol); a.ext_enc = (unsigned long long*)(b + o_enc);
  a.ext = (double*)(b + o_ext); a.params = (int*)(b + o_par); a.bounds = (double*)(b + o_bnd); a.key = (int*)(b + o_key);
  a.coord = (int*)(b + o_crd); a.table = (unsigned long long*)(b + o_tab); a.slot_vid = (int*)(b + o_sv); a.pslot = (int*)(b + o_ps);
  a.vid = (int*)(b + o_vid); a.f1 = (int*)(b + o_f1); a.f2 = (int*)(b + o_f2); a.evkey = (int*)(b + o_ek);
  a.ev_pt = (int*)(b + o_ept); a.ev_info = (int*)(b + o_ei); a.rows = (int*)(b + o_rows); a.ev_p = (signed char*)(b + o_ep);
  a.state_g = (unsigned*)(b + o_stg); a.parent = (int*)(b + o_par2); a.root = (int*)(b + o_root); a.cnt = (int*)(b + o_cnt);
  a.cl_root = (int*)(b + o_clr); a.cl_rank_of_root = (int*)(b + o_crr); a.cluster = (int*)(b + o_cl); a.sizes = (int*)(b + o_sz);
  a.pkey = (int*)(b + o_pk); a.boxes = (double*)(b + o_box); a.box_enc = (unsigned long long*)(b + o_benc); a.chunk_cnt = (unsigned*)(b + o_cc); a.key_base = (unsigned*)(b + o_kb);
  a.perm_a = (int*)(b + o_pa); a.perm_b = (int*)(b + o_pb); a.out_seg = (unsigned long long*)(b + o_seg);
  const size_t seq_fixed = (size_t)kOsSeqStages * 32 * kOsRowStride * sizeof(int);
  const size_t state_bytes = round_up(n, 4) + 8;                           // one byte per voxel (at most n voxels)
  const bool seq_bytes = seq_fixed + state_bytes <= (size_t)kOsSeqSmemBytes && !getenv("TLOAM_B200_DCVC_PACKED");
  const int use_smem = seq_fixed + state_words * 4 <= (size_t)kOsSeqSmemBytes && !getenv("TLOAM_B200_DCVC_GLOBAL") ? 1 : 0;
  const size_t seq_smem = seq_fixed + (seq_bytes ? state_bytes : (use_smem ? state_words * 4 : 0));
  if (!h->os_attr_set) {
    CU_TRY(cudaFuncSetAttribute(k_os_seq<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kOsSeqSmemBytes));
    CU_TRY(cudaFuncSetAttribute(k_os_seq<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kOsSeqSmemBytes));
    h->os_attr_set = true;
  }
  cudaStream_t st = h->stream;
  if (h->seg.active) a.pts = h->seg.dev_xyz;
  else CU_TRY(cudaMemcpyAsync(b + o_pts, xyz, n * 24, cudaMemcpyHostToDevice, st));
  CU_TRY(cudaMemsetAsync(b + o_tab, 0, cap * 8, st));
  if (!seq_bytes && !use_smem) CU_TRY(cudaMemsetAsync(b + o_stg, 0, state_words * 4, st));
  const unsigned ev_blocks = (unsigned)((n32 * 32 + 255) / 256);
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_init<<<1, 32, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_polar<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_bounds<<<1, 32, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_key<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_vid<<<(unsigned)(cap / 256), 256, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_first<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_second<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_evkey<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  auto partition = [&](const int* keys, const int* perm_in, int* perm_out, const int* n_items, int shift, int* total_out) {
    OsPart p;
    p.keys = keys; p.perm_in = perm_in; p.perm_out = perm_out; p.n_items = n_items; p.n_fixed = a.n; p.shift = shift;
    p.chunk_cnt = a.chunk_cnt; p.key_base = a.key_base; p.nchunk = a.nchunk; p.total_out = total_out;
    TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_part_hist<<<a.nchunk, kOsChunk, 0, st>>>(p)));
    TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_part_scan<<<1, kOsKeys, 0, st>>>(p)));
    TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_part_scatter<<<a.nchunk, kOsChunk, 0, st>>>(p)));
    return 0;
  };
  partition(a.evkey, nullptr, a.ev_pt, nullptr, 0, a.params + 5);          // events in point order
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_rows<<<ev_blocks, 256, 0, st>>>(a)));
  if (seq_bytes) TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_seq<true><<<1, 32, seq_smem, st>>>(a, 1)));
  else TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_seq<false><<<1, 32, seq_smem, st>>>(a, use_smem)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_union<<<ev_blocks, 256, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_label<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_clusters<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  const size_t cl_bound = cfg->min_seg >= 0 ? n / ((size_t)cfg->min_seg + 1) + 1 : n;   // classes with > min_seg points
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_rank<<<(unsigned)((cl_bound + 255) / 256), 256, 0, st>>>(a)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_pkey<<<a.nchunk, kOsChunk, 0, st>>>(a)));
  partition(a.pkey, nullptr, a.perm_a, nullptr, 0, a.params + 7);           // stable LSD partition by cluster rank
  const int* seg = a.perm_a;
  if (cl_bound > 256) { partition(a.pkey, a.perm_a, a.perm_b, a.params + 7, 8, nullptr); seg = a.perm_b; }
  if (cl_bound > 65536) { partition(a.pkey, a.perm_b, a.perm_a, a.params + 7, 16, nullptr); seg = a.perm_a; }
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_boxes_acc<<<a.nchunk, 256, 0, st>>>(a, seg)));
  TL_LAUNCH(TLOAM_B200_K_OBJECT, (k_os_boxes_fin<<<(unsigned)((cl_bound + 255) / 256), 256, 0, st>>>(a)));
  CU_TRY(cudaGetLastError());
  int par[8];
  CU_TRY(cudaMemcpyAsync(par, a.params, sizeof(par), cudaMemcpyDeviceToHost, st));
  CU_TRY(cudaStreamSynchronize(st));
  if (par[3] != 0) {
    snprintf(h->last_error, sizeof(h->last_error), "object_segmentation: more than %d polar rings", kOsMaxBounds);
    return TLOAM_B200_ERR_INVALID_ARG;
  }
  static_assert(sizeof(size_t) == sizeof(unsigned long long), "index lists are copied straight into size_t arrays");
  const size_t nc = (size_t)par[6], ns = (size_t)par[7];
  if (h->seg.active) { h->seg.seg = a.out_seg; h->seg.n_seg = (unsigned)ns; }   // chained: the scan stays on the device
  else if (ns) CU_TRY(cudaMemcpyAsync(seg_index, a.out_seg, ns * sizeof(size_t), cudaMemcpyDeviceToHost, st));
  if (sizes && nc) CU_TRY(cudaMemcpyAsync(sizes, a.sizes, nc * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (boxes && nc) CU_TRY(cudaMemcpyAsync(boxes, a.boxes, nc * 6 * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (root) CU_TRY(cudaMemcpyAsync(root, a.root, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (cluster) CU_TRY(cudaMemcpyAsync(cluster, a.cluster, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (voxel) CU_TRY(cudaMemcpyAsync(voxel, a.key, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (polar) {
    CU_TRY(cudaMemcpyAsync(polar, a.polar, n * 24, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaMemcpyAsync(polar + 3 * n, a.ext, 4 * sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  CU_TRY(cudaStreamSynchronize(st));
  *n_seg = ns; *n_clusters = (int)nc;
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// "next" row (f)-4: the three steps of Segmentation::spinOnce (ref: segmentation.cpp:47-66) as ONE call: the scan is
// uploaded once, every stage is fed by a gather kernel from the previous stage's device-side index list, and only the
// final lists come home -- as indices into the ORIGINAL scan.
// ---------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(256) k_chain_gather_object(const double* pts, const double* intensity, const unsigned* idx, unsigned n,
                                                             double* out_pts, double* out_beam) {
  const unsigned j = blockIdx.x * 256 + threadIdx.x;
  if (j >= n) return;
  const unsigned i = idx[j];
  out_pts[3ull * j] = pts[3ull * i]; out_pts[3ull * j + 1] = pts[3ull * i + 1]; out_pts[3ull * j + 2] = pts[3ull * i + 2];
  out_beam[j] = intensity[i];                                              // the object points carry the channel (:707-709)
}
__global__ void __launch_bounds__(256) k_chain_gather_segmented(const double* obj_pts, const double* obj_beam, const unsigned* obj_idx,
                                                                const unsigned long long* seg, unsigned n, double* out_pts, double* out_beam,
                                                                unsigned* out_orig) {
  const unsigned j = blockIdx.x * 256 + threadIdx.x;
  if (j >= n) return;
  const unsigned i = (unsigned)seg[j];
  out_pts[3ull * j] = obj_pts[3ull * i]; out_pts[3ull * j + 1] = obj_pts[3ull * i + 1]; out_pts[3ull * j + 2] = obj_pts[3ull * i + 2];
  out_beam[j] = obj_beam[i];
  out_orig[j] = obj_idx[i];
}
// blockIdx.y: 0 ground, 1 edge, 2 general -- index lists into the original scan, as 64-bit values (raw_of: kept -> raw
// index after the removal step, null = no removal step); 3: the channel of kept point j into slot raw_of[j] of out_intensity
__global__ void __launch_bounds__(256) k_chain_final(const unsigned* ground, unsigned n_ground, const unsigned long long* edge, unsigned n_edge,
                                                     const unsigned long long* non_edge, unsigned n_non, const unsigned* seg_orig,
                                                     const unsigned* raw_of, const double* intensity, unsigned n_kept,
                                                     unsigned long long* out_ground, unsigned long long* out_edge, unsigned long long* out_general,
                                                     double* out_intensity) {
  const unsigned j = blockIdx.x * 256 + threadIdx.x;
  auto raw = [&](unsigned k) { return raw_of ? raw_of[k] : k; };
  if (blockIdx.y == 0) { if (j < n_ground) out_ground[j] = raw(ground[j]); }
  else if (blockIdx.y == 1) { if (j < n_edge) out_edge[j] = raw(seg_orig[(unsigned)edge[j]]); }
  else if (blockIdx.y == 2) { if (j < n_non) out_general[j] = raw(seg_orig[(unsigned)non_edge[j]]); }
  else { if (j < n_kept) out_intensity[raw(j)] = intensity[j]; }
}
}  // namespace

// a library that ships next to this one (libtloam_b200_gmi.so, libtloam_b200_unpack.so): its path in this library's directory
static std::string sibling_path(const char* file) {
  Dl_info info;
  std::string path = file;
  if (dladdr(reinterpret_cast<void*>(&tloam_b200_last_error), &info) && info.dli_fname) {
    const std::string self = info.dli_fname;
    const size_t slash = self.rfind('/');
    if (slash != std::string::npos) path = self.substr(0, slash + 1) + path;
  }
  return path;
}

// host staging of a copy to the device: pageable memory through HostStage, pinned / registered memory by DMA
static int upload_host(tloam_b200_handle* h, void* dst, const void* src, size_t bytes) {
  if (HostStage::pageable(src) && getenv("TLOAM_B200_NO_HOST_STAGE") == nullptr) CU_TRY(h->hstage.upload(dst, src, bytes, h->stream));
  else CU_TRY(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
  return TLOAM_B200_OK;
}

// ---- packed raw scans (tloam_packed_scan): k_unpack_scan lives in libtloam_b200_unpack.so (unpack_scan.cu), loaded on the
//      first packed call so that the kernels of this library keep their SASS ----
static std::mutex g_unpack_mu;
static tloam_unpack_scan_fn g_unpack = nullptr;

static int unpack_load(tloam_b200_handle* h, tloam_unpack_scan_fn* out) {
  std::lock_guard<std::mutex> lk(g_unpack_mu);
  if (!g_unpack) {
    const std::string path = sibling_path("libtloam_b200_unpack.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    tloam_unpack_scan_fn fn = so ? reinterpret_cast<tloam_unpack_scan_fn>(dlsym(so, "tloam_unpack_scan")) : nullptr;
    if (!fn) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "packed scan: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_unpack = fn;
  }
  *out = g_unpack;
  return TLOAM_B200_OK;
}

static bool packed_valid(const tloam_packed_scan* s) {
  if (!s || (!s->data && s->n) || s->point_step < 12 || s->n > ((size_t)1 << 26)) return false;
  if (s->n && s->point_step > SIZE_MAX / s->n) return false;                 // no such host buffer
  const int off[4] = {s->x_offset, s->y_offset, s->z_offset, s->intensity_offset};
  for (int k = 0; k < 4; ++k) {
    if (k == 3 && off[k] == -1) continue;
    if (off[k] < 0 || (size_t)off[k] + 4 > s->point_step) return false;
  }
  return true;
}

// one upload of the packed records, then (double)float of every field on the device: xyz (n x 3) and, when `intensity` is
// not null and the layout has the field, the intensity (n).  The layout has been validated.
static int unpack_packed(tloam_b200_handle* h, const tloam_packed_scan* s, double* xyz, double* intensity) {
  if (!s->n) return TLOAM_B200_OK;
  tloam_unpack_scan_fn unpack;
  int rc = unpack_load(h, &unpack);
  if (rc != TLOAM_B200_OK) return rc;
  const size_t bytes = s->n * s->point_step, padded = round_up(bytes, 16);   // the kernel loads whole 16-byte chunks
  if (padded > h->cap_packed) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_packed); h->d_packed = nullptr; h->cap_packed = 0;
    CU_TRY(cudaMalloc(&h->d_packed, padded + padded / 4));
    h->cap_packed = padded + padded / 4;
  }
  if ((rc = upload_host(h, h->d_packed, s->data, bytes)) != TLOAM_B200_OK) return rc;
  const int off[4] = {s->x_offset, s->y_offset, s->z_offset, s->intensity_offset};
  int e = 0;
  TL_LAUNCH(TLOAM_B200_K_GROUND, (e = unpack(h->d_packed, s->n, s->point_step, off, xyz, intensity, h->device, h->stream)));
  if (e != cudaSuccess) {
    snprintf(h->last_error, sizeof(h->last_error), "packed scan: k_unpack_scan: %s", cudaGetErrorString((cudaError_t)e));
    return TLOAM_B200_ERR_CUDA;
  }
  return TLOAM_B200_OK;
}

// ---- deskewing (the *_timed calls): the kernels live in libtloam_b200_deskew.so (deskew.cu), loaded on the first timed call
//      so that the kernels of this library keep their SASS ----
static std::mutex g_deskew_mu;
struct DeskewLib { tloam_deskew_fn motion = nullptr, tend = nullptr, apply = nullptr; };
static DeskewLib g_deskew;

static int deskew_load(tloam_b200_handle* h, DeskewLib* out) {
  std::lock_guard<std::mutex> lk(g_deskew_mu);
  if (!g_deskew.apply) {
    const std::string path = sibling_path("libtloam_b200_deskew.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    DeskewLib l;
    if (so) {
      l.motion = reinterpret_cast<tloam_deskew_fn>(dlsym(so, "tloam_deskew_motion"));
      l.tend = reinterpret_cast<tloam_deskew_fn>(dlsym(so, "tloam_deskew_tend"));
      l.apply = reinterpret_cast<tloam_deskew_fn>(dlsym(so, "tloam_deskew_apply"));
    }
    if (!l.motion || !l.tend || !l.apply) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "deskew: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_deskew = l;
  }
  *out = g_deskew;
  return TLOAM_B200_OK;
}

static bool packed_time_valid(const tloam_packed_time* t, size_t point_step) {
  const int bytes = t->datatype == 8 ? 8 : (t->datatype == 6 || t->datatype == 7) ? 4 : 0;
  return bytes && t->offset >= 0 && (size_t)t->offset + bytes <= point_step && std::isfinite(t->unit) && t->unit > 0.0;
}

// the raw scan a chain call starts from: FP64 AoS rows (xyz), or a packed scan unpacked on the device.  timed: deskew it
// (process_raw only) with the FP64 times `time` or, for a packed scan, its field `ptime`, over the frame period `period`.
struct RawScanIn {
  const double* xyz = nullptr; const tloam_packed_scan* packed = nullptr; size_t n = 0;
  bool timed = false; const double* time = nullptr; const tloam_packed_time* ptime = nullptr; double period = 0.0;
};

// k_deskew_motion -> k_deskew_tend -> k_deskew on the handle's stream: scan (n x 3, on the device) corrected into out.  The
// times are d_time (uploaded) or the packed records where unpack_packed uploaded them.  scratch: TLOAM_DESKEW_SCRATCH_DOUBLES.
static int deskew_scan(tloam_b200_handle* h, const RawScanIn& in, const double* scan, const double* d_time, double* scratch,
                       double* out) {
  DeskewLib lib;
  int rc = deskew_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  tloam_deskew_args a;
  a.last_pose = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, last_pose));
  a.curr_pose = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, curr_pose));
  a.time = d_time; a.records = nullptr; a.point_step = 0; a.offset = 0; a.datatype = 0; a.unit = 1.0;
  if (!d_time) {
    a.records = h->d_packed; a.point_step = in.packed->point_step;
    a.offset = in.ptime->offset; a.datatype = in.ptime->datatype; a.unit = in.ptime->unit;
  }
  a.n = in.n; a.period = in.period; a.xyz = scan; a.out = out; a.scratch = scratch; a.device = h->device; a.stream = h->stream;
  const tloam_deskew_fn step[3] = {lib.motion, lib.tend, lib.apply};
  static const char* const names[3] = {"k_deskew_motion", "k_deskew_tend", "k_deskew"};
  for (int k = 0; k < 3; ++k) {
    int e = 0;
    TL_LAUNCH(TLOAM_B200_K_FEATURE, (e = step[k](&a)));
    if (e != cudaSuccess) {
      snprintf(h->last_error, sizeof(h->last_error), "deskew: %s: %s", names[k], cudaGetErrorString((cudaError_t)e));
      return TLOAM_B200_ERR_CUDA;
    }
  }
  return TLOAM_B200_OK;
}

// The one implementation of the chained segmentation; only the way the scan reaches the device depends on its form (in).
// remove: run RemoveClosedNonFinitePoints(near_dis) on the device first (tloam_b200_segment_raw_scan); tloam_b200_segment_scan
// runs without that step.  beam / intensity (optional, n values): the channel of every point of the scan as int / FP64 (NaN
// for removed points).  keep (optional): the three final lists stay on the device (tloam_b200_process_raw_scan) -- the index
// arrays are not written, *keep receives the uploaded scan, the intensity of a packed scan with that field (else null), the
// deskewed scan of a timed call (else null) and the lists (valid until the handle's next segmentation call); the counts
// still land in *n_ground / *n_edge / *n_general.  The segmentation itself always reads the uploaded (raw) scan.
struct ChainKeep {
  const double* scan = nullptr; const double* intensity = nullptr; const double* deskewed = nullptr;
  const unsigned long long *ground = nullptr, *edge = nullptr, *general = nullptr;
};
static int segment_chain(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num, bool remove,
                         double near_dis, const RawScanIn& in, size_t* ground_index, size_t* n_ground, size_t* edge_index,
                         size_t* n_edge, size_t* general_index, size_t* n_general, int* n_clusters, int* sizes, double* boxes, int* beam,
                         double* intensity, ChainKeep* keep = nullptr) {
  if (!h || !gcfg || !dcfg || !ground_index || !n_ground || !edge_index || !n_edge || !general_index || !n_general || !n_clusters)
    return TLOAM_B200_ERR_INVALID_ARG;
  h->seg_gen++;                                           // d_chain (the raw scan of the last process_raw_scan) is rewritten
  *n_ground = *n_edge = *n_general = 0; *n_clusters = 0;
  if (remove && gcfg->sensor_model != 64 && gcfg->sensor_model != 16) return TLOAM_B200_ERR_INVALID_ARG;
  if (in.packed && !packed_valid(in.packed)) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t n = in.n;
  if (n == 0) return TLOAM_B200_OK;
  if ((!in.packed && !in.xyz) || n > ((size_t)1 << 26)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  // chain buffer: what must outlive a stage's arena
  const unsigned nchunk = (unsigned)((n + kGeChunk - 1) / kGeChunk);
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += round_up(bytes, 256); return o; };
  const size_t o_scan = take(n * 24), o_gnd = take(n * 4), o_oidx = take(n * 4), o_opts = take(n * 24), o_obeam = take(n * 8),
               o_spts = take(n * 24), o_sbeam = take(n * 8), o_sorig = take(n * 4), o_fg = take(n * 8), o_fe = take(n * 8), o_fn = take(n * 8),
               o_beam = take(n * 4), o_kept = remove ? take(n * 24) : 0, o_map = remove ? take(n * 4) : 0,
               o_rmc = remove ? take(nchunk * 4 + 64) : 0, o_int = intensity ? take(n * 8) : 0, o_fi = intensity ? take(n * 8) : 0;
  const bool keep_int = keep && in.packed && in.packed->intensity_offset >= 0;
  const size_t o_pint = keep_int ? take(n * 8) : 0;
  const bool timed = keep && in.timed;
  const size_t o_dsk = timed ? take(n * 24) : 0, o_time = timed && !in.packed ? take(n * 8) : 0,
               o_dscr = timed ? take(TLOAM_DESKEW_SCRATCH_DOUBLES * 8) : 0;
  if (off > h->cap_chain) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_chain); h->d_chain = nullptr; h->cap_chain = 0;
    CU_TRY(cudaMalloc(&h->d_chain, off + off / 4));
    h->cap_chain = off + off / 4;
  }
  unsigned char* c = h->d_chain;
  double* d_scan = (double*)(c + o_scan);
  unsigned* d_gnd = (unsigned*)(c + o_gnd); unsigned* d_oidx = (unsigned*)(c + o_oidx);
  double* d_opts = (double*)(c + o_opts); double* d_obeam = (double*)(c + o_obeam);
  double* d_spts = (double*)(c + o_spts); double* d_sbeam = (double*)(c + o_sbeam); unsigned* d_sorig = (unsigned*)(c + o_sorig);
  unsigned long long* d_fg = (unsigned long long*)(c + o_fg); unsigned long long* d_fe = (unsigned long long*)(c + o_fe);
  unsigned long long* d_fn = (unsigned long long*)(c + o_fn);
  double* d_pint = keep_int ? (double*)(c + o_pint) : nullptr;
  int rc = in.packed ? unpack_packed(h, in.packed, d_scan, d_pint) : upload_host(h, d_scan, in.xyz, n * 24);
  if (rc != TLOAM_B200_OK) return rc;
  double* d_dsk = timed ? (double*)(c + o_dsk) : nullptr;
  if (timed) {
    double* d_time = in.packed ? nullptr : (double*)(c + o_time);
    if (d_time && (rc = upload_host(h, d_time, in.time, n * 8)) != TLOAM_B200_OK) return rc;
    if ((rc = deskew_scan(h, in, d_scan, d_time, (double*)(c + o_dscr), d_dsk)) != TLOAM_B200_OK) return rc;
  }
  struct Reset { tloam_b200_handle* h; ~Reset() { h->seg = tloam_b200_handle::SegChain(); } } reset{h};
  // ---- 0. RemoveClosedNonFinitePoints (:48, :472-499): kept points + kept -> raw map ----
  const double* pts = d_scan;
  const unsigned* raw_of = nullptr;
  size_t nk = n;
  if (remove) {
    RmArgs r;
    r.raw = d_scan; r.n = (unsigned)n; r.nchunk = nchunk; r.norm_min = near_dis * near_dis;
    r.chunk_cnt = (unsigned*)(c + o_rmc); r.total = r.chunk_cnt + round_up(nchunk, 16);
    r.kept = (double*)(c + o_kept); r.map = (unsigned*)(c + o_map);
    TL_LAUNCH(TLOAM_B200_K_GROUND, (k_rm_count<<<nchunk, kGeChunk, 0, h->stream>>>(r)));
    TL_LAUNCH(TLOAM_B200_K_GROUND, (k_rm_scan<<<1, 1024, 0, h->stream>>>(r)));
    TL_LAUNCH(TLOAM_B200_K_GROUND, (k_rm_scatter<<<nchunk, kGeChunk, 0, h->stream>>>(r)));
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpyAsync(h->h_result + 28, r.total, sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    unsigned kept;
    memcpy(&kept, h->h_result + 28, sizeof(kept));
    pts = r.kept; raw_of = r.map; nk = kept;
  }
  if (intensity) CU_TRY(cudaMemsetAsync(c + o_fi, 0xFF, n * 8, h->stream));   // all-ones: NaN for the removed points
  size_t ng = 0, no = 0, ne = 0, nn = 0;
  if (nk) {
    h->seg.active = true;
    // ---- 1. groundRemove ----
    h->seg.dev_xyz = pts;
    rc = ground_run(h, gcfg, pts /*placeholder: read on the device*/, nk, ground_index, &ng, general_index /*scratch: not written when
                    chained*/, &no, nullptr, nullptr, nullptr, nullptr, nullptr);
    if (rc != TLOAM_B200_OK) return rc;
    if (ng) CU_TRY(cudaMemcpyAsync(d_gnd, h->seg.ground, ng * 4, cudaMemcpyDeviceToDevice, h->stream));
    if (beam) CU_TRY(cudaMemcpyAsync(c + o_beam, h->seg.beam, nk * 4, cudaMemcpyDeviceToDevice, h->stream));
    if (intensity) CU_TRY(cudaMemcpyAsync(c + o_int, h->seg.intensity, nk * 8, cudaMemcpyDeviceToDevice, h->stream));
    if (no) {
      CU_TRY(cudaMemcpyAsync(d_oidx, h->seg.object, no * 4, cudaMemcpyDeviceToDevice, h->stream));
      k_chain_gather_object<<<(unsigned)((no + 255) / 256), 256, 0, h->stream>>>(pts, h->seg.intensity, h->seg.object, (unsigned)no, d_opts, d_obeam);
      CU_TRY(cudaGetLastError());
      // ---- 2. objectSegmentation ----
      h->seg.dev_xyz = d_opts;
      size_t ns = 0;
      rc = tloam_b200_object_segmentation(h, dcfg, d_opts /*placeholder: read on the device*/, no, general_index, &ns, n_clusters, sizes, boxes,
                                          nullptr, nullptr, nullptr, nullptr);
      if (rc != TLOAM_B200_OK) return rc;
      if (ns) {
        k_chain_gather_segmented<<<(unsigned)((ns + 255) / 256), 256, 0, h->stream>>>(d_opts, d_obeam, d_oidx, h->seg.seg, (unsigned)ns, d_spts,
                                                                                       d_sbeam, d_sorig);
        CU_TRY(cudaGetLastError());
        // ---- 3. extractEdgePoint ----
        h->seg.dev_xyz = d_spts; h->seg.dev_intensity = d_sbeam;
        rc = tloam_b200_extract_edge(h, gcfg->sensor_model, ring_min_num, d_spts, d_sbeam, ns, edge_index, &ne, general_index, &nn);
        if (rc != TLOAM_B200_OK) return rc;
      }
    }
  }
  const size_t nki = intensity ? nk : 0;
  size_t most = ng > ne ? (ng > nn ? ng : nn) : (ne > nn ? ne : nn);
  most = most > nki ? most : nki;
  if (most) {
    k_chain_final<<<dim3((unsigned)((most + 255) / 256), intensity ? 4 : 3), 256, 0, h->stream>>>(
        d_gnd, (unsigned)ng, h->seg.edge, (unsigned)ne, h->seg.non_edge, (unsigned)nn, d_sorig, raw_of, (const double*)(c + o_int), (unsigned)nki,
        d_fg, d_fe, d_fn, (double*)(c + o_fi));
    CU_TRY(cudaGetLastError());
    static_assert(sizeof(size_t) == sizeof(unsigned long long), "index lists are copied straight into size_t arrays");
    if (ng && !keep) CU_TRY(cudaMemcpyAsync(ground_index, d_fg, ng * 8, cudaMemcpyDeviceToHost, h->stream));
    if (ne && !keep) CU_TRY(cudaMemcpyAsync(edge_index, d_fe, ne * 8, cudaMemcpyDeviceToHost, h->stream));
    if (nn && !keep) CU_TRY(cudaMemcpyAsync(general_index, d_fn, nn * 8, cudaMemcpyDeviceToHost, h->stream));
  }
  if (keep) {
    keep->scan = d_scan; keep->intensity = d_pint; keep->deskewed = d_dsk;
    keep->ground = d_fg; keep->edge = d_fe; keep->general = d_fn;
  }
  if (beam) CU_TRY(cudaMemcpyAsync(beam, c + o_beam, n * 4, cudaMemcpyDeviceToHost, h->stream));
  if (intensity) CU_TRY(cudaMemcpyAsync(intensity, c + o_fi, n * 8, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  *n_ground = ng; *n_edge = ne; *n_general = nn;
  return TLOAM_B200_OK;
}

int tloam_b200_segment_scan(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                            const double* xyz, size_t n, size_t* ground_index, size_t* n_ground, size_t* edge_index, size_t* n_edge,
                            size_t* general_index, size_t* n_general, int* n_clusters, int* sizes, double* boxes, int* beam) {
  RawScanIn in;
  in.xyz = xyz; in.n = n;
  return segment_chain(h, gcfg, dcfg, ring_min_num, false, 0.0, in, ground_index, n_ground, edge_index, n_edge, general_index, n_general,
                       n_clusters, sizes, boxes, beam, nullptr);
}

int tloam_b200_segment_raw_scan(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                                double near_dis, const double* xyz, size_t n, size_t* ground_index, size_t* n_ground, size_t* edge_index,
                                size_t* n_edge, size_t* general_index, size_t* n_general, int* n_clusters, int* sizes, double* boxes,
                                double* intensity) {
  RawScanIn in;
  in.xyz = xyz; in.n = n;
  return segment_chain(h, gcfg, dcfg, ring_min_num, true, near_dis, in, ground_index, n_ground, edge_index, n_edge, general_index, n_general,
                       n_clusters, sizes, boxes, nullptr, intensity);
}

int tloam_b200_segment_raw_scan_packed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                       int ring_min_num, double near_dis, const tloam_packed_scan* scan, size_t* ground_index,
                                       size_t* n_ground, size_t* edge_index, size_t* n_edge, size_t* general_index, size_t* n_general,
                                       int* n_clusters, int* sizes, double* boxes, double* intensity) {
  if (!scan) return TLOAM_B200_ERR_INVALID_ARG;
  RawScanIn in;
  in.packed = scan; in.n = scan->n;
  return segment_chain(h, gcfg, dcfg, ring_min_num, true, near_dis, in, ground_index, n_ground, edge_index, n_edge, general_index, n_general,
                       n_clusters, sizes, boxes, nullptr, intensity);
}

// ---------------------------------------------------------------------------------------------
// FrontEnd::processCloud (ref: src/front_end/front_end.cpp:181-199) + setInputSource on the device: the frame's ground /
// edge / general clouds sit in h->d_frame, and the four features are written straight into the registration's staging
// buffer.  Every launch and copy goes on the handle's stream.  That stream order is what lets process_* of frame k+1
// overwrite d_frame (the planar-submap selection of frame k) and the staging buffer: the submap update of frame k reads
// them on side streams that it joins back into the handle's stream before it returns.
// ---------------------------------------------------------------------------------------------
static int reserve_frame(tloam_b200_handle* h, size_t ng, size_t ne, size_t nn) {
  const size_t need = ng + ne + 2 * nn;                   // raw ground | raw edge | general | planar-submap selection (<= nn)
  if (need <= h->cap_frame) return TLOAM_B200_OK;
  CU_TRY(cudaStreamSynchronize(h->stream));
  cudaFree(h->d_frame); h->d_frame = nullptr; h->cap_frame = 0;
  const size_t ncap = need + need / 4 + 1024;
  CU_TRY(cudaMalloc(&h->d_frame, ncap * 3 * sizeof(double)));
  h->cap_frame = ncap;
  return TLOAM_B200_OK;
}

static int process_frame(tloam_b200_handle* h, const tloam_feature_config* fcfg, double ground_down_sample, double edge_down_sample,
                         size_t ng, size_t ne, size_t nn, size_t n_source[4]) {
  const double* d_ground = h->d_frame;
  const double* d_edge = d_ground + 3 * ng;
  const double* d_general = d_edge + 3 * ne;
  double* d_planar_sub = h->d_frame + 3 * (ng + ne + nn);
  int rc;
  // VoxelDownSample of the ground (:183) and edge (:186) clouds, sorted by voxel key (the caps take features in index
  // order); each keeps its own voxel scratch until the emission below
  VoxSorted vg, ve;
  if ((rc = voxel_pipeline(h, d_ground, ng, nullptr, 0u, nullptr, nullptr, nullptr, 0.0, ground_down_sample, nullptr, h->d_cnt + 12,
                           h->stream, 0, &vg)) != TLOAM_B200_OK) return rc;
  if ((rc = voxel_pipeline(h, d_edge, ne, nullptr, 0u, nullptr, nullptr, nullptr, 0.0, edge_down_sample, nullptr, h->d_cnt + 13,
                           h->stream, 1, &ve)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(h->h_result + 22, h->d_cnt + 12, 2 * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  // extractPlanarSphere (:194); an empty general cloud selects nothing (feature_extract.cpp:49-54, 140).  fe_run ends with
  // the one synchronisation of the call.
  FeArena A;
  unsigned fc[4] = {0u, 0u, 0u, 0u};                     // planar_submap, sphere_submap, planar_scan, sphere_scan counts
  if (nn) {
    if ((rc = fe_run(h, fcfg, d_general, nn, true, A, true)) != TLOAM_B200_OK) return rc;
    memcpy(fc, h->h_result + 28, sizeof(fc));
  } else {
    CU_TRY(cudaStreamSynchronize(h->stream));
  }
  unsigned vc[2];
  memcpy(vc, h->h_result + 22, sizeof(vc));
  const size_t n[4] = {vc[1], fc[3], fc[2], vc[0]};     // edge, sphere, planar, ground
  const unsigned tb = 256;
  // SelectByIndex (:197-198): planar = general[planar_scan_index]; sphere = general[sphere_scan_index] where the reference's
  // sphere list holds RANKS 0..n-1 (feature_extract.cpp:183-188, SURVEY Q12), so the sphere feature is the general cloud's
  // first n points -- restated literally, like tloam_b200_extract_planar_sphere's lists
  const std::function<int(double*)> fill = [&](double* stage) -> int {
    int r;
    if ((r = voxel_emit_sorted(h, ve, n[0], stage)) != TLOAM_B200_OK) return r;
    if (n[1]) TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_select_by_index<unsigned><<<(unsigned)((n[1] + tb - 1) / tb), tb, 0, h->stream>>>(
                                                   d_general, nullptr, (unsigned)n[1], stage + 3 * n[0])));
    if (n[2]) TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_select_by_index<unsigned><<<(unsigned)((n[2] + tb - 1) / tb), tb, 0, h->stream>>>(
                                                   d_general, A.val_p_sorted, (unsigned)n[2], stage + 3 * (n[0] + n[1]))));
    if ((r = voxel_emit_sorted(h, vg, n[3], stage + 3 * (n[0] + n[1] + n[2]))) != TLOAM_B200_OK) return r;
    // the frame's planar-submap selection general[planar_submap_index] (:291, :207), kept for submap_init_frame / _update_frame
    if (fc[0]) TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_select_by_index<unsigned><<<(fc[0] + tb - 1) / tb, tb, 0, h->stream>>>(
                                                    d_general, A.val_p_sorted, fc[0], d_planar_sub)));
    CU_TRY(cudaGetLastError());
    return TLOAM_B200_OK;
  };
  if ((rc = set_source_impl(h, nullptr, n, true, &fill)) != TLOAM_B200_OK) return rc;
  h->fr_ng = ng; h->fr_ne = ne; h->fr_nn = nn; h->fr_np_sub = fc[0]; h->fr_ns_sub = fc[1];
  h->have_frame = true;
  for (int k = 0; k < 4; ++k) n_source[k] = n[k];
  return TLOAM_B200_OK;
}

int tloam_b200_process_cloud(tloam_b200_handle* h, const tloam_feature_config* fcfg, double ground_down_sample, double edge_down_sample,
                             const double* ground, size_t ng, const double* edge, size_t ne, const double* general, size_t nn,
                             size_t n_source[4]) {
  if (!h || !fcfg || !n_source || (!ground && ng) || (!edge && ne) || (!general && nn)) return TLOAM_B200_ERR_INVALID_ARG;
  h->seg_gen++;                                           // the last raw scan no longer belongs to the processed frame
  for (int k = 0; k < 4; ++k) n_source[k] = 0;
  if (!(ground_down_sample > 0.0) || !(edge_down_sample > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (ng > ((size_t)1 << 30) || ne > ((size_t)1 << 30) || nn > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  const VoxExtent ground_ext = vox_extent(ground, ng);
  if (!vox_fits(ground_ext, ground_down_sample) || !vox_fits(vox_extent(edge, ne), edge_down_sample)) return TLOAM_B200_ERR_VOXEL_RANGE;
  CU_TRY(cudaSetDevice(h->device));
  h->have_frame = false;
  h->fr_ground_ext = ground_ext;
  int rc = reserve_frame(h, ng, ne, nn);
  if (rc != TLOAM_B200_OK) return rc;
  const double* src[3] = {ground, edge, general};
  const size_t cnt[3] = {ng, ne, nn};
  size_t off = 0;
  for (int c = 0; c < 3; ++c) {                           // the only point data that crosses PCIe
    if (cnt[c]) {
      if (HostStage::pageable(src[c]) && getenv("TLOAM_B200_NO_HOST_STAGE") == nullptr)
        CU_TRY(h->hstage.upload(h->d_frame + 3 * off, src[c], cnt[c] * 24, h->stream));
      else
        CU_TRY(cudaMemcpyAsync(h->d_frame + 3 * off, src[c], cnt[c] * 24, cudaMemcpyHostToDevice, h->stream));
    }
    off += cnt[c];
  }
  return process_frame(h, fcfg, ground_down_sample, edge_down_sample, ng, ne, nn, n_source);
}

static int process_raw(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                       double near_dis, const tloam_feature_config* fcfg, double ground_down_sample, double edge_down_sample,
                       const RawScanIn& in, size_t n_source[4]) {
  if (!h || !gcfg || !dcfg || !fcfg || !n_source || (!in.packed && !in.xyz && in.n)) return TLOAM_B200_ERR_INVALID_ARG;
  for (int k = 0; k < 4; ++k) n_source[k] = 0;
  if (!(ground_down_sample > 0.0) || !(edge_down_sample > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (in.timed) {
    if (!std::isfinite(in.period) || !(in.period > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
    if (in.packed ? (in.ptime ? !packed_time_valid(in.ptime, in.packed->point_step) : in.n > 0) : (!in.time && in.n))
      return TLOAM_B200_ERR_INVALID_ARG;
  }
  // the ground and edge clouds are subsets of the scan's finite rows, so the scan's extent bounds theirs; a timed call
  // moves rows on the device after this check (not covered: see Deskewing in the header)
  if (in.packed && !packed_valid(in.packed)) return TLOAM_B200_ERR_INVALID_ARG;
  VoxExtent scan_ext = in.packed ? vox_extent_packed(in.packed) : vox_extent(in.xyz, in.n);
  if (!vox_fits(scan_ext, ground_down_sample) || !vox_fits(scan_ext, edge_down_sample)) return TLOAM_B200_ERR_VOXEL_RANGE;
  scan_ext.known = !in.timed;
  CU_TRY(cudaSetDevice(h->device));
  h->have_frame = false;
  h->fr_ground_ext = scan_ext;
  size_t unused[1];                                       // the index lists stay on the device (ChainKeep)
  size_t ng = 0, ne = 0, nn = 0;
  int n_clusters = 0;
  ChainKeep keep;
  int rc = segment_chain(h, gcfg, dcfg, ring_min_num, true, near_dis, in, unused, &ng, unused, &ne, unused, &nn, &n_clusters, nullptr,
                         nullptr, nullptr, nullptr, &keep);
  if (rc != TLOAM_B200_OK) return rc;
  if ((rc = reserve_frame(h, ng, ne, nn)) != TLOAM_B200_OK) return rc;
  const unsigned long long* lists[3] = {keep.ground, keep.edge, keep.general};
  const size_t cnt[3] = {ng, ne, nn};
  size_t off = 0;
  const double* rows = keep.deskewed ? keep.deskewed : keep.scan;   // the corrected scan of a timed call
  for (int c = 0; c < 3; ++c) {                           // ground / edge / general clouds gathered from the uploaded raw scan
    if (cnt[c]) TL_LAUNCH(TLOAM_B200_K_FEATURE, (k_select_by_index<unsigned long long><<<(unsigned)((cnt[c] + 255) / 256), 256, 0, h->stream>>>(
                                                    rows, lists[c], (unsigned)cnt[c], h->d_frame + 3 * off)));
    off += cnt[c];
  }
  CU_TRY(cudaGetLastError());
  if ((rc = process_frame(h, fcfg, ground_down_sample, edge_down_sample, ng, ne, nn, n_source)) != TLOAM_B200_OK) return rc;
  h->raw_scan = rows; h->raw_int = keep.intensity; h->raw_n = in.n; h->raw_gen = h->seg_gen;   // for global_map_append_frame*
  return TLOAM_B200_OK;
}

int tloam_b200_process_raw_scan(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                                double near_dis, const tloam_feature_config* fcfg, double ground_down_sample, double edge_down_sample,
                                const double* xyz, size_t n, size_t n_source[4]) {
  RawScanIn in;
  in.xyz = xyz; in.n = n;
  return process_raw(h, gcfg, dcfg, ring_min_num, near_dis, fcfg, ground_down_sample, edge_down_sample, in, n_source);
}

int tloam_b200_process_raw_scan_packed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                       int ring_min_num, double near_dis, const tloam_feature_config* fcfg, double ground_down_sample,
                                       double edge_down_sample, const tloam_packed_scan* scan, size_t n_source[4]) {
  if (!scan) return TLOAM_B200_ERR_INVALID_ARG;
  RawScanIn in;
  in.packed = scan; in.n = scan->n;
  return process_raw(h, gcfg, dcfg, ring_min_num, near_dis, fcfg, ground_down_sample, edge_down_sample, in, n_source);
}

int tloam_b200_process_raw_scan_timed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                      int ring_min_num, double near_dis, const tloam_feature_config* fcfg, double ground_down_sample,
                                      double edge_down_sample, const double* xyz, const double* time, size_t n, double frame_period,
                                      size_t n_source[4]) {
  RawScanIn in;
  in.xyz = xyz; in.n = n; in.timed = true; in.time = time; in.period = frame_period;
  return process_raw(h, gcfg, dcfg, ring_min_num, near_dis, fcfg, ground_down_sample, edge_down_sample, in, n_source);
}

int tloam_b200_process_raw_scan_packed_timed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                             int ring_min_num, double near_dis, const tloam_feature_config* fcfg,
                                             double ground_down_sample, double edge_down_sample, const tloam_packed_scan* scan,
                                             const tloam_packed_time* time, double frame_period, size_t n_source[4]) {
  if (!scan) return TLOAM_B200_ERR_INVALID_ARG;
  RawScanIn in;
  in.packed = scan; in.n = scan->n; in.timed = true; in.ptime = time; in.period = frame_period;
  return process_raw(h, gcfg, dcfg, ring_min_num, near_dis, fcfg, ground_down_sample, edge_down_sample, in, n_source);
}

int tloam_b200_source_download(tloam_b200_handle* h, int cloud, double* out, size_t capacity_points) {
  if (!h || !out || cloud < 0 || cloud > 3) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_src) return TLOAM_B200_ERR_NOT_READY;
  if (capacity_points < h->n_src[cloud]) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (h->n_src[cloud]) CU_TRY(cudaMemcpyAsync(out, h->src_ptr[cloud], h->n_src[cloud] * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// first-frame seeding (ref: front_end.cpp:285-305) from the last processed frame, through submap_init's body
int tloam_b200_submap_init_frame(tloam_b200_handle* h, const tloam_submap_config* scfg) {
  if (!h || !scfg) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_frame) return TLOAM_B200_ERR_NOT_READY;
  const double* ground = h->d_frame;
  const double* edge = ground + 3 * h->fr_ng;
  const double* general = edge + 3 * h->fr_ne;
  const double* planar_sub = general + 3 * h->fr_nn;
  return submap_init_impl(h, scfg, edge, h->fr_ne, ground, h->fr_ng, planar_sub, h->fr_np_sub, general, h->fr_ns_sub, true);
}

int tloam_b200_submap_update_frame(tloam_b200_handle* h, const double pose[16]) {
  if (!h || !pose) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_frame) return TLOAM_B200_ERR_NOT_READY;
  return submap_update_impl(h, pose, h->d_frame + 3 * (h->fr_ng + h->fr_ne + h->fr_nn), h->fr_np_sub, true);
}

int tloam_b200_submap_update_frame_chained(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->have_frame) return TLOAM_B200_ERR_NOT_READY;
  return submap_update_impl(h, nullptr, h->d_frame + 3 * (h->fr_ng + h->fr_ne + h->fr_nn), h->fr_np_sub, true);
}

// ---------------------------------------------------------------------------------------------
// Global map (FrontEnd::updateSubmap with mapping_flag, ref: front_end.cpp:269-274; kernels in submap.cuh).  Every append
// is enqueued on the handle's stream.  The map's size stays on the device; the host keeps an upper bound (an exact count
// read back asynchronously, plus the rows appended since) and synchronises only to grow the buffer.
// ---------------------------------------------------------------------------------------------
void tloam_b200_global_map_default_config(tloam_global_map_config* c) {
  c->voxel = 1.0;                          // front_end.cpp:273: VoxelDownSample(1.0)
  c->initial_capacity_points = (size_t)1 << 20;
}

static void gmap_harvest(tloam_b200_handle* h) {
  for (auto& pr : h->gmap_probes) {
    if (!pr.pending) continue;
    if (cudaEventQuery(pr.ev) != cudaSuccess) { cudaGetLastError(); continue; }
    pr.pending = false;
    if (pr.cum >= h->gmap_known_cum) { h->gmap_known_cum = pr.cum; h->gmap_known = *pr.h_count; }
  }
}

static int gmap_clear(tloam_b200_handle* h) {
  CU_TRY(cudaMemsetAsync(h->d_gmap_st, 0, sizeof(GMapState), h->stream));
  CU_TRY(cudaMemsetAsync(h->d_gmap_off, 0, sizeof(unsigned long long), h->stream));
  h->gmap_cum = h->gmap_known_cum = h->gmap_known = h->gmap_calls = 0;
  for (auto& pr : h->gmap_probes) pr.pending = false;
  h->gmap_reg_valid = false; h->gmap_reg_n = 0;
  h->gmi_used = false;                     // re-arms the intensity channel (the next intensity frame starts it afresh)
  for (int k = 0; k < 16; ++k) h->gmc_M[k] = k % 5 == 0 ? 1.0 : 0.0;
  h->gmc_M_identity = true;                // the pose tables are empty with the frame table; tracking stays as it is
  h->gmm_valid = false;                    // the merged snapshot belonged to the map before
  h->occ_built = false;                    // the grid too; the captures are indexed by the frame count, now 0
  if (h->gmd_on) {                         // every row starts at (0, 0); removal stays on
    CU_TRY(cudaMemsetAsync(h->d_gmd_through, 0, h->cap_gmd * sizeof(unsigned), h->stream));
    CU_TRY(cudaMemsetAsync(h->d_gmd_hits, 0, h->cap_gmd * sizeof(unsigned), h->stream));
  }
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_enable(tloam_b200_handle* h, const tloam_global_map_config* cfg) {
  if (!h || !cfg || !(cfg->voxel > 0.0) || !std::isfinite(cfg->voxel)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!h->d_gmap_st) {
    CU_TRY(cudaMalloc(&h->d_gmap_st, sizeof(GMapState)));
    CU_TRY(cudaMalloc(&h->d_gmap_pose, 16 * sizeof(double)));
    for (auto& pr : h->gmap_probes) {
      CU_TRY(cudaEventCreateWithFlags(&pr.ev, cudaEventDisableTiming));
      CU_TRY(cudaMallocHost(&pr.h_count, sizeof(unsigned long long)));
    }
  }
  const size_t cap = cfg->initial_capacity_points ? cfg->initial_capacity_points : 1;
  if (cap != h->cap_gmap) {
    cudaFree(h->d_gmap); h->d_gmap = nullptr; h->cap_gmap = 0;
    cudaFree(h->d_gmi_map); h->d_gmi_map = nullptr;                       // reallocated by the next intensity append
    CU_TRY(cudaMalloc(&h->d_gmap, cap * 3 * sizeof(double)));
    h->cap_gmap = cap;
  }
  if (!h->d_gmap_off) {
    CU_TRY(cudaMalloc(&h->d_gmap_off, 1024 * sizeof(unsigned long long)));
    h->cap_gmap_off = 1024;
  }
  h->gmap_voxel = cfg->voxel;
  h->gmap_growths = 0;
  h->gmap_on = true;
  h->gmc_on = false;
  h->gmd_on = false;
  h->occ_on = false;
  return gmap_clear(h);
}

int tloam_b200_global_map_reset(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  return gmap_clear(h);
}

// the one place an append synchronises: the map (or its frame table) may not hold the next frame.  The exact size is read,
// and the buffer grows to max(1.5 x capacity, exact size + n rows); the frame table likewise.
static int gmap_grow(tloam_b200_handle* h, size_t n) {
  CU_TRY(cudaStreamSynchronize(h->stream));
  GMapState st;
  CU_TRY(cudaMemcpyAsync(&st, h->d_gmap_st, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->gmap_known = st.count; h->gmap_known_cum = h->gmap_cum;
  for (auto& pr : h->gmap_probes) pr.pending = false;
  if (st.count + n > h->cap_gmap) {
    size_t ncap = h->cap_gmap + h->cap_gmap / 2;
    if (ncap < st.count + n) ncap = st.count + n;
    double* q = nullptr;
    CU_TRY(cudaMalloc(&q, ncap * 3 * sizeof(double)));
    if (st.count) CU_TRY(cudaMemcpyAsync(q, h->d_gmap, st.count * 3 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gmap);
    h->d_gmap = q; h->cap_gmap = ncap;
    if (h->d_gmi_map) {                    // the intensity channel grows with the map
      double* qi = nullptr;
      CU_TRY(cudaMalloc(&qi, ncap * sizeof(double)));
      if (st.count) CU_TRY(cudaMemcpyAsync(qi, h->d_gmi_map, st.count * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_gmi_map);
      h->d_gmi_map = qi;
    }
    if (h->gmd_on) {                       // the removal counters grow with the map; rows past the count stay (0, 0)
      for (unsigned** t : {&h->d_gmd_through, &h->d_gmd_hits}) {
        unsigned* qt = nullptr;
        CU_TRY(cudaMalloc(&qt, ncap * sizeof(unsigned)));
        CU_TRY(cudaMemsetAsync(qt, 0, ncap * sizeof(unsigned), h->stream));
        if (st.count) CU_TRY(cudaMemcpyAsync(qt, *t, st.count * sizeof(unsigned), cudaMemcpyDeviceToDevice, h->stream));
        CU_TRY(cudaStreamSynchronize(h->stream));
        cudaFree(*t);
        *t = qt;
      }
      h->cap_gmd = ncap;
    }
  }
  if (h->gmap_calls + 2 > h->cap_gmap_off) {
    size_t ncap = h->cap_gmap_off + h->cap_gmap_off / 2;
    if (ncap < h->gmap_calls + 2) ncap = h->gmap_calls + 2;
    unsigned long long* q = nullptr;
    CU_TRY(cudaMalloc(&q, ncap * sizeof(unsigned long long)));
    CU_TRY(cudaMemcpyAsync(q, h->d_gmap_off, (st.frames + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gmap_off);
    h->d_gmap_off = q; h->cap_gmap_off = ncap;
    if (h->gmc_on) {                       // the pose tables grow with the frame table
      for (double** t : {&h->d_gmc_O, &h->d_gmc_P}) {
        double* qt = nullptr;
        CU_TRY(cudaMalloc(&qt, ncap * 16 * sizeof(double)));
        if (st.frames) CU_TRY(cudaMemcpyAsync(qt, *t, st.frames * 16 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
        CU_TRY(cudaStreamSynchronize(h->stream));
        cudaFree(*t);
        *t = qt;
      }
      h->cap_gmc = ncap;
    }
    if (h->occ_on) {                       // the captures grow with the frame table
      const size_t per[2] = {(size_t)h->occ_cfg.n_cols * TLOAM_OCC_SLOT, 16};
      double** tabs[2] = {&h->d_occ_scans, &h->d_occ_poses};
      for (int k = 0; k < 2; ++k) {
        double* qt = nullptr;
        CU_TRY(cudaMalloc(&qt, ncap * per[k] * sizeof(double)));
        if (st.frames) CU_TRY(cudaMemcpyAsync(qt, *tabs[k], st.frames * per[k] * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
        CU_TRY(cudaStreamSynchronize(h->stream));
        cudaFree(*tabs[k]);
        *tabs[k] = qt;
      }
      h->cap_occ = ncap;
    }
  }
  h->gmap_growths++;
  return TLOAM_B200_OK;
}

// ---- the intensity channel's kernels live in libtloam_b200_gmi.so (gmap_intensity.cu), next to this library: loaded on the
//      first intensity call, so that the kernels of this library keep their SASS and a process that never asks for
//      intensity never loads it ----
struct GmiLib { tloam_gmi_scratch_bytes_fn scratch_bytes = nullptr; tloam_gmi_append_fn append = nullptr; tloam_gmi_plain_fn plain = nullptr; };
static std::mutex g_gmi_mu;
static GmiLib g_gmi;

static int gmi_load(tloam_b200_handle* h, GmiLib* out) {
  std::lock_guard<std::mutex> lk(g_gmi_mu);
  if (!g_gmi.append) {
    const std::string path = sibling_path("libtloam_b200_gmi.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    GmiLib l;
    if (so) {
      l.scratch_bytes = reinterpret_cast<tloam_gmi_scratch_bytes_fn>(dlsym(so, "tloam_gmi_scratch_bytes"));
      l.append = reinterpret_cast<tloam_gmi_append_fn>(dlsym(so, "tloam_gmi_append"));
      l.plain = reinterpret_cast<tloam_gmi_plain_fn>(dlsym(so, "tloam_gmi_plain"));
    }
    if (!so || !l.scratch_bytes || !l.append || !l.plain) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "global map intensity: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_gmi = l;
  }
  *out = g_gmi;
  return TLOAM_B200_OK;
}

static int gmi_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "global map intensity: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

// ---- the pose tables' and the correction's kernels live in libtloam_b200_gmc.so (map_correct.cu), next to this library:
//      loaded by tloam_b200_global_map_correction_enable, so that the kernels of this library keep their SASS and an append
//      with tracking on cannot meet a missing library ----
struct GmcLib { tloam_gmc_pose_fn pose = nullptr; tloam_gmc_correct_fn correct = nullptr; };
static std::mutex g_gmc_mu;
static GmcLib g_gmc;

static int gmc_load(tloam_b200_handle* h, GmcLib* out) {
  std::lock_guard<std::mutex> lk(g_gmc_mu);
  if (!g_gmc.pose) {
    const std::string path = sibling_path("libtloam_b200_gmc.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    GmcLib l;
    if (so) {
      l.pose = reinterpret_cast<tloam_gmc_pose_fn>(dlsym(so, "tloam_gmc_pose"));
      l.correct = reinterpret_cast<tloam_gmc_correct_fn>(dlsym(so, "tloam_gmc_correct"));
    }
    if (!l.pose || !l.correct) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "global map correction: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_gmc = l;
  }
  *out = g_gmc;
  return TLOAM_B200_OK;
}

static int gmc_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "global map correction: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

// ---- the removal's kernels live in libtloam_b200_gmd.so (map_dynamic.cu), next to this library: loaded by
//      tloam_b200_global_map_dynamic_enable, so that the kernels of this library keep their SASS and an append with removal
//      on cannot meet a missing library ----
struct GmdLib { tloam_gmd_vote_fn vote = nullptr; tloam_gmd_static_blocks_fn blocks = nullptr; tloam_gmd_static_fn compact = nullptr; };
static std::mutex g_gmd_mu;
static GmdLib g_gmd;

static int gmd_load(tloam_b200_handle* h, GmdLib* out) {
  std::lock_guard<std::mutex> lk(g_gmd_mu);
  if (!g_gmd.vote) {
    const std::string path = sibling_path("libtloam_b200_gmd.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    GmdLib l;
    if (so) {
      l.vote = reinterpret_cast<tloam_gmd_vote_fn>(dlsym(so, "tloam_gmd_vote"));
      l.blocks = reinterpret_cast<tloam_gmd_static_blocks_fn>(dlsym(so, "tloam_gmd_static_blocks"));
      l.compact = reinterpret_cast<tloam_gmd_static_fn>(dlsym(so, "tloam_gmd_static"));
    }
    if (!l.vote || !l.blocks || !l.compact) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "global map dynamic removal: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_gmd = l;
  }
  *out = g_gmd;
  return TLOAM_B200_OK;
}

static int gmd_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "global map dynamic removal: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

// ---- the occupancy grid's kernels live in libtloam_b200_occ.so (occupancy.cu), next to this library: loaded by
//      tloam_b200_occupancy_enable, so that the kernels of this library keep their SASS and an append with the grid on
//      cannot meet a missing library ----
struct OccLib { tloam_occ_capture_fn capture = nullptr; tloam_occ_build_fn extent = nullptr, rasterise = nullptr; };
static std::mutex g_occ_mu;
static OccLib g_occ;

static int occ_load(tloam_b200_handle* h, OccLib* out) {
  std::lock_guard<std::mutex> lk(g_occ_mu);
  if (!g_occ.capture) {
    const std::string path = sibling_path("libtloam_b200_occ.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    OccLib l;
    if (so) {
      l.capture = reinterpret_cast<tloam_occ_capture_fn>(dlsym(so, "tloam_occ_capture"));
      l.extent = reinterpret_cast<tloam_occ_build_fn>(dlsym(so, "tloam_occ_extent"));
      l.rasterise = reinterpret_cast<tloam_occ_build_fn>(dlsym(so, "tloam_occ_rasterise"));
    }
    if (!l.capture || !l.extent || !l.rasterise) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "occupancy grid: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_occ = l;
  }
  *out = g_occ;
  return TLOAM_B200_OK;
}

static int occ_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "occupancy grid: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

static tloam_occ_params occ_params(const tloam_b200_handle* h) {
  tloam_occ_params p;
  const tloam_occupancy_config& c = h->occ_cfg;
  p.n_cols = c.n_cols; p.z_lo = c.z_lo; p.z_hi = c.z_hi; p.min_range = c.min_range; p.max_range = c.max_range;
  p.dirs = h->d_occ_dirs;
  return p;
}

// device buffers of an intensity frame of n rows (after gmap_grow: d_gmi_map takes the map's current capacity)
static int gmi_prepare(tloam_b200_handle* h, const GmiLib& lib, size_t n) {
  if (!h->d_gmi_st) {
    CU_TRY(cudaMalloc(&h->d_gmi_st, 2 * sizeof(unsigned)));
    CU_TRY(cudaMemsetAsync(h->d_gmi_st, 0, 2 * sizeof(unsigned), h->stream));
  }
  if (!h->d_gmi_map) CU_TRY(cudaMalloc(&h->d_gmi_map, h->cap_gmap * sizeof(double)));
  const size_t bytes = lib.scratch_bytes((unsigned)n);
  if (bytes > h->cap_gmi_scratch) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gmi_scratch); h->d_gmi_scratch = nullptr; h->cap_gmi_scratch = 0;
    CU_TRY(cudaMalloc(&h->d_gmi_scratch, bytes + bytes / 2));
    h->cap_gmi_scratch = bytes + bytes / 2;
  }
  return TLOAM_B200_OK;
}

// d_gmi_in holds the intensity of a host frame of n rows (uploaded or unpacked there)
static int gmi_reserve_in(tloam_b200_handle* h, size_t n) {
  if (n <= h->cap_gmi_in) return TLOAM_B200_OK;
  const size_t ncap = n + n / 2 + 1024;
  CU_TRY(cudaStreamSynchronize(h->stream));
  cudaFree(h->d_gmi_in); h->d_gmi_in = nullptr; h->cap_gmi_in = 0;
  CU_TRY(cudaMalloc(&h->d_gmi_in, ncap * sizeof(double)));
  h->cap_gmi_in = ncap;
  return TLOAM_B200_OK;
}

// global_map += (T . raw).VoxelDownSample(voxel).  d_in: the raw scan on the device -- read in place, or the registered-scan
// buffer the host frame was staged into (transformed there).  pose_host == nullptr: the device-side result of the frame just
// enqueued (as submap_update_impl's chained form).  d_int: the raw scan's intensity on the device (n values), or nullptr: the
// frame has no intensity channel.
static int gmap_append_impl(tloam_b200_handle* h, const double* pose_host, const double* d_in, size_t n, const double* d_int) {
  CU_TRY(cudaSetDevice(h->device));
  int rc;
  GmiLib gmi;
  const bool with_int = d_int && n;        // an empty frame adds nothing: the channel is left as it is
  if ((with_int || h->gmi_used) && (rc = gmi_load(h, &gmi)) != TLOAM_B200_OK) return rc;
  gmap_harvest(h);
  const unsigned long long bound = h->gmap_known + (h->gmap_cum - h->gmap_known_cum) + n;   // voxels <= finite rows <= rows
  if (bound > h->cap_gmap || h->gmap_calls + 2 > h->cap_gmap_off)
    if ((rc = gmap_grow(h, n)) != TLOAM_B200_OK) return rc;
  if (with_int && (rc = gmi_prepare(h, gmi, n)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, &h->d_gmap_reg, &h->cap_gmap_reg, n, false)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, &h->d_gmap_fin, &h->cap_gmap_fin, n, false)) != TLOAM_B200_OK) return rc;
  const double* d_pose = h->d_gmap_pose;
  if (pose_host) {
    double tmp[16];
    memcpy(tmp, pose_host, sizeof(tmp));
    CU_TRY(cudaMemcpyAsync(h->d_gmap_pose, tmp, sizeof(tmp), cudaMemcpyHostToDevice, h->stream));   // pageable source: staged before return
  } else {
    d_pose = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, result));
  }
  GMapState* st = h->d_gmap_st;
  if (h->gmc_on) {                         // O_f, P_f = M O_f recorded at the frame's slot; the transform reads P_f
    GmcLib gmc;
    if ((rc = gmc_load(h, &gmc)) != TLOAM_B200_OK) return rc;
    tloam_gmc_mat M;
    memcpy(M.m, h->gmc_M, sizeof(M.m));
    int e = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = gmc.pose(d_pose, h->d_gmap_pose, h->d_gmc_O, h->d_gmc_P, &st->frames, h->cap_gmc,
                                                 h->gmc_M_identity ? nullptr : &M, h->device, h->stream)));
    if ((rc = gmc_status(h, e, "k_gmc_pose")) != TLOAM_B200_OK) return rc;
    d_pose = h->d_gmap_pose;
  }
  if (h->gmd_on && n) {                    // free-space votes of the sensor-frame rows (before the transform below) at the
    GmdLib gmd;                            // block's pose, on the rows [0, count) present before this append
    if ((rc = gmd_load(h, &gmd)) != TLOAM_B200_OK) return rc;
    const tloam_global_map_dynamic_config& c = h->gmd_cfg;
    tloam_gmd_vote_args a;
    memset(&a, 0, sizeof(a));
    a.p.n_rows = c.n_rows; a.p.n_cols = c.n_cols; a.p.wr = c.window_rows; a.p.wc = c.window_cols;
    a.p.margin_abs = c.margin_abs; a.p.margin_rel = c.margin_rel; a.p.min_range = c.min_range; a.p.max_range = c.max_range;
    a.p.row_bounds = h->d_gmd_bounds; a.p.col_bounds = h->d_gmd_bounds + (c.n_rows + 1);
    a.scan = d_in; a.n = (unsigned)n; a.pose = d_pose; a.map = h->d_gmap; a.count = &st->count;
    a.through = h->d_gmd_through; a.hits = h->d_gmd_hits; a.image = h->d_gmd_image; a.window = h->d_gmd_window;
    a.device = h->device; a.stream = h->stream;
    int launches = 0, e = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = gmd.vote(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = gmd_status(h, e, "k_gmd_vote")) != TLOAM_B200_OK) return rc;
  }
  if (h->occ_on) {                         // the 2D scan of the sensor-frame rows (before the transform below) and the
    OccLib occ;                            // block's pose, into the slot of the device frame count
    if ((rc = occ_load(h, &occ)) != TLOAM_B200_OK) return rc;
    tloam_occ_capture_args a;
    memset(&a, 0, sizeof(a));
    a.p = occ_params(h);
    a.scan = d_in; a.n = (unsigned)n; a.pose = d_pose; a.frames = &st->frames; a.cap = h->cap_occ;
    a.scans = h->d_occ_scans; a.poses = h->d_occ_poses;
    a.device = h->device; a.stream = h->stream;
    int launches = 0, e = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = occ.capture(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = occ_status(h, e, "k_occ_clear / _bin / _pick / _final")) != TLOAM_B200_OK) return rc;
  }
  CU_TRY(cudaMemsetAsync(&st->n_fin, 0, sizeof(GMapState) - offsetof(GMapState, n_fin), h->stream));
  const unsigned tb = 256, gb = (unsigned)((n + tb - 1) / tb);
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_transform<<<gb, tb, 0, h->stream>>>(d_in, (unsigned)n, d_pose, h->d_gmap_reg, h->d_gmap_fin, st)));
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_guard<<<1, 32, 0, h->stream>>>(st, h->gmap_voxel)));
  VoxSorted vs;
  if ((rc = voxel_pipeline(h, h->d_gmap_fin, n, &st->n_fin, 0u, nullptr, nullptr, nullptr, 0.0, h->gmap_voxel, nullptr, &st->n_vox,
                           h->stream, 0, &vs)) != TLOAM_B200_OK) return rc;
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_emit<<<gb, tb, 0, h->stream>>>(vs.a, vs.slots, h->d_gmap, st, h->cap_gmap)));
  // the intensity channel, while st->count is still the frame's base (gmap_intensity.cu)
  if (with_int) {
    tloam_gmi_frame f;
    f.reg = h->d_gmap_reg; f.intensity = d_int; f.n = (unsigned)n;
    f.minenc = vs.a.minenc; f.voxel = h->gmap_voxel; f.keys_sorted = vs.keys; f.n_vox = &st->n_vox; f.refused = &st->refused;
    f.count = &st->count; f.frames = &st->frames; f.cap = h->cap_gmap; f.frame_cap = h->cap_gmap_off;
    f.map_intensity = h->d_gmi_map; f.state = h->d_gmi_st; f.fresh = h->gmi_used ? 0 : 1; f.scratch = h->d_gmi_scratch;
    int launches = 0, e = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = gmi.append(&f, h->device, h->stream, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = gmi_status(h, e, "append")) != TLOAM_B200_OK) return rc;
    h->gmi_used = true;
  } else if (n && h->gmi_used) {
    int e = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = gmi.plain(h->d_gmi_st, &st->n_vox, &st->refused, &st->count, &st->frames, h->cap_gmap,
                                                  h->cap_gmap_off, h->device, h->stream)));
    if ((rc = gmi_status(h, e, "plain")) != TLOAM_B200_OK) return rc;
  }
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_commit<<<1, 32, 0, h->stream>>>(st, h->d_gmap_off, h->cap_gmap, h->cap_gmap_off)));
  CU_TRY(cudaGetLastError());
  h->gmap_cum += n;
  h->gmap_calls++;
  h->gmap_reg_n = n; h->gmap_reg_valid = true;
  // asynchronous read-back of the exact size (tightens the bound of later frames)
  tloam_b200_handle::GMapProbe& pr = h->gmap_probes[h->gmap_probe_next];
  if (!pr.pending) {
    CU_TRY(cudaMemcpyAsync(pr.h_count, &st->count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaEventRecord(pr.ev, h->stream));
    pr.cum = h->gmap_cum; pr.pending = true;
    h->gmap_probe_next = (h->gmap_probe_next + 1) & 3;
  }
  return TLOAM_B200_OK;
}

// a host frame: its rows are staged in the registered-scan buffer (transformed there) and its intensity, if any, in
// d_gmi_in -- uploaded as FP64 (xyz, inten), or uploaded packed and unpacked on the device (packed, n == packed->n).  The
// only point data that crosses PCIe.
static int gmap_append_host(tloam_b200_handle* h, const double* pose_host, const double* xyz, const double* inten,
                            const tloam_packed_scan* packed, size_t n) {
  if (n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  const bool with_int = packed ? packed->intensity_offset >= 0 : inten != nullptr;
  int rc;
  if ((rc = ensure_dev(h, &h->d_gmap_reg, &h->cap_gmap_reg, n, false)) != TLOAM_B200_OK) return rc;
  if (with_int && (rc = gmi_reserve_in(h, n)) != TLOAM_B200_OK) return rc;
  if (packed) {
    if ((rc = unpack_packed(h, packed, h->d_gmap_reg, with_int ? h->d_gmi_in : nullptr)) != TLOAM_B200_OK) return rc;
  } else if (n) {
    if ((rc = upload_host(h, h->d_gmap_reg, xyz, n * 24)) != TLOAM_B200_OK) return rc;
    if (with_int && (rc = upload_host(h, h->d_gmi_in, inten, n * 8)) != TLOAM_B200_OK) return rc;
  }
  return gmap_append_impl(h, pose_host, h->d_gmap_reg, n, with_int ? h->d_gmi_in : nullptr);
}

int tloam_b200_global_map_append(tloam_b200_handle* h, const double pose[16], const double* xyz, size_t n) {
  if (!h || !pose || (!xyz && n)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  return gmap_append_host(h, pose, xyz, nullptr, nullptr, n);
}

int tloam_b200_global_map_append_chained(tloam_b200_handle* h, const double* xyz, size_t n) {
  if (!h || (!xyz && n)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  return gmap_append_host(h, nullptr, xyz, nullptr, nullptr, n);
}

// the raw scan is read where process_raw_scan uploaded it (d_chain); any segmentation / process call since may have
// reused that buffer, so the generation must still match.  inten: an explicit host intensity (n values, uploaded), else the
// intensity a packed process_raw_scan left beside the raw scan (read in place), if any.
static int gmap_append_frame(tloam_b200_handle* h, const double* pose, const double* inten = nullptr) {
  if (!h->gmap_on || h->raw_gen != h->seg_gen) return TLOAM_B200_ERR_NOT_READY;
  const double* d_int = h->raw_int;
  if (inten) {
    CU_TRY(cudaSetDevice(h->device));
    int rc;
    if ((rc = gmi_reserve_in(h, h->raw_n)) != TLOAM_B200_OK) return rc;
    if (h->raw_n && (rc = upload_host(h, h->d_gmi_in, inten, h->raw_n * 8)) != TLOAM_B200_OK) return rc;
    d_int = h->d_gmi_in;
  }
  return gmap_append_impl(h, pose, h->raw_scan, h->raw_n, d_int);
}

int tloam_b200_global_map_append_frame(tloam_b200_handle* h, const double pose[16]) {
  if (!h || !pose) return TLOAM_B200_ERR_INVALID_ARG;
  return gmap_append_frame(h, pose);
}

int tloam_b200_global_map_append_frame_chained(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  return gmap_append_frame(h, nullptr);
}

// synchronises and reads the device-side state; a pending refusal / overflow flag is cleared and returned as a status
static int gmap_read(tloam_b200_handle* h, GMapState* st, int* flag_status) {
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(st, h->d_gmap_st, sizeof(*st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  *flag_status = TLOAM_B200_OK;
  if (st->flags) {
    CU_TRY(cudaMemsetAsync(&h->d_gmap_st->flags, 0, sizeof(unsigned), h->stream));
    if (st->flags & kGMapOverflow) {       // the host sizes the buffer from an upper bound: this is a bug, not an input error
      snprintf(h->last_error, sizeof(h->last_error), "global map: the device-side capacity check refused a frame");
      *flag_status = TLOAM_B200_ERR_CUDA;
    } else {
      *flag_status = TLOAM_B200_ERR_VOXEL_RANGE;
    }
  }
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_size(tloam_b200_handle* h, size_t* n_points, size_t* n_frames) {
  if (!h || !n_points || !n_frames) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int flag = TLOAM_B200_OK;
  const int rc = gmap_read(h, &st, &flag);
  if (rc != TLOAM_B200_OK) return rc;
  *n_points = st.count; *n_frames = st.frames;
  return flag;
}

int tloam_b200_global_map_download(tloam_b200_handle* h, size_t first, size_t count, double* out) {
  if (!h || (!out && count)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int flag = TLOAM_B200_OK;
  const int rc = gmap_read(h, &st, &flag);
  if (rc != TLOAM_B200_OK) return rc;
  if (first > st.count || count > st.count - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (count) CU_TRY(cudaMemcpyAsync(out, h->d_gmap + 3 * first, count * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return flag;
}

int tloam_b200_global_map_frame_offsets(tloam_b200_handle* h, size_t* offsets, size_t capacity) {
  if (!h || !offsets) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int flag = TLOAM_B200_OK;
  const int rc = gmap_read(h, &st, &flag);
  if (rc != TLOAM_B200_OK) return rc;
  if (capacity < st.frames + 1) return TLOAM_B200_ERR_INVALID_ARG;
  static_assert(sizeof(size_t) == sizeof(unsigned long long), "the frame table is copied straight into a size_t array");
  CU_TRY(cudaMemcpyAsync(offsets, h->d_gmap_off, (st.frames + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return flag;
}

int tloam_b200_global_map_capacity(tloam_b200_handle* h, size_t* capacity_points, size_t* growths) {
  if (!h || !capacity_points || !growths) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  *capacity_points = h->cap_gmap; *growths = h->gmap_growths;
  return TLOAM_B200_OK;
}

int tloam_b200_registered_scan_download(tloam_b200_handle* h, double* out, size_t capacity_points, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->gmap_reg_valid) return TLOAM_B200_ERR_NOT_READY;
  *n = h->gmap_reg_n;
  if (capacity_points < h->gmap_reg_n || (!out && h->gmap_reg_n)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (h->gmap_reg_n) CU_TRY(cudaMemcpyAsync(out, h->d_gmap_reg, h->gmap_reg_n * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---- the intensity channel (kernels in gmap_intensity.cu): the same appends with the raw scan's intensity ----
int tloam_b200_global_map_append_intensity(tloam_b200_handle* h, const double pose[16], const double* xyz, const double* intensity,
                                           size_t n) {
  if (!h || !pose || (!xyz && n) || !intensity) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  return gmap_append_host(h, pose, xyz, intensity, nullptr, n);
}

int tloam_b200_global_map_append_intensity_chained(tloam_b200_handle* h, const double* xyz, const double* intensity, size_t n) {
  if (!h || (!xyz && n) || !intensity) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  return gmap_append_host(h, nullptr, xyz, intensity, nullptr, n);
}

int tloam_b200_global_map_append_frame_intensity(tloam_b200_handle* h, const double pose[16], const double* intensity) {
  if (!h || !pose || !intensity) return TLOAM_B200_ERR_INVALID_ARG;
  return gmap_append_frame(h, pose, intensity);
}

int tloam_b200_global_map_append_frame_intensity_chained(tloam_b200_handle* h, const double* intensity) {
  if (!h || !intensity) return TLOAM_B200_ERR_INVALID_ARG;
  return gmap_append_frame(h, nullptr, intensity);
}

int tloam_b200_global_map_append_packed(tloam_b200_handle* h, const double pose[16], const tloam_packed_scan* scan) {
  if (!h || !pose || !packed_valid(scan)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  return gmap_append_host(h, pose, nullptr, nullptr, scan, scan->n);
}

int tloam_b200_global_map_append_packed_chained(tloam_b200_handle* h, const tloam_packed_scan* scan) {
  if (!h || !packed_valid(scan)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  return gmap_append_host(h, nullptr, nullptr, nullptr, scan, scan->n);
}

// synchronises (gmap_read: the sticky flags of the xyz map) and reads whether the map has the channel (PointCloud2::
// HasIntensity: a non-empty map whose every point has an intensity)
static int gmi_read(tloam_b200_handle* h, GMapState* st, int* flag_status, bool* has) {
  int rc = gmap_read(h, st, flag_status);
  if (rc != TLOAM_B200_OK) return rc;
  *has = false;
  if (!h->gmi_used) return TLOAM_B200_OK;
  unsigned s[2];
  CU_TRY(cudaMemcpyAsync(s, h->d_gmi_st, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (s[1]) {                              // a finite row found no voxel of its frame: a bug, not an input error
    CU_TRY(cudaMemsetAsync(h->d_gmi_st + 1, 0, sizeof(unsigned), h->stream));
    snprintf(h->last_error, sizeof(h->last_error), "global map intensity: a finite row found no voxel of its frame");
    *flag_status = TLOAM_B200_ERR_CUDA;
  }
  *has = s[0] != 0u && st->count > 0;
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_has_intensity(tloam_b200_handle* h, int* has) {
  if (!h || !has) return TLOAM_B200_ERR_INVALID_ARG;
  *has = 0;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int flag = TLOAM_B200_OK;
  bool b = false;
  const int rc = gmi_read(h, &st, &flag, &b);
  if (rc != TLOAM_B200_OK) return rc;
  *has = b ? 1 : 0;
  return flag;
}

int tloam_b200_global_map_intensity_download(tloam_b200_handle* h, size_t first, size_t count, double* out) {
  if (!h || (!out && count)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int flag = TLOAM_B200_OK;
  bool has = false;
  const int rc = gmi_read(h, &st, &flag, &has);
  if (rc != TLOAM_B200_OK) return rc;
  if (flag == TLOAM_B200_ERR_CUDA) return flag;
  if (!has) return TLOAM_B200_ERR_NOT_READY;
  if (first > st.count || count > st.count - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (count) CU_TRY(cudaMemcpyAsync(out, h->d_gmi_map + first, count * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return flag;
}

// ---------------------------------------------------------------------------------------------
// Loop closure (Scan Context descriptors and an exact search; kernels in scan_context.cu, loaded from libtloam_b200_loop.so
// on the first loop call so that the kernels of this library keep their SASS).  Every add is enqueued on the handle's
// stream; the host keeps the frame count and synchronises only to grow the database.
// ---------------------------------------------------------------------------------------------
struct LoopLib { tloam_sc_fn bin = nullptr, finish = nullptr, search = nullptr; };
static std::mutex g_loop_mu;
static LoopLib g_loop;

static int loop_load(tloam_b200_handle* h, LoopLib* out) {
  std::lock_guard<std::mutex> lk(g_loop_mu);
  if (!g_loop.search) {
    const std::string path = sibling_path("libtloam_b200_loop.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    LoopLib l;
    if (so) {
      l.bin = reinterpret_cast<tloam_sc_fn>(dlsym(so, "tloam_sc_bin"));
      l.finish = reinterpret_cast<tloam_sc_fn>(dlsym(so, "tloam_sc_finish"));
      l.search = reinterpret_cast<tloam_sc_fn>(dlsym(so, "tloam_sc_search"));
    }
    if (!l.bin || !l.finish || !l.search) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "loop closure: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_loop = l;
  }
  *out = g_loop;
  return TLOAM_B200_OK;
}

void tloam_b200_loop_default_config(tloam_loop_config* c) {   // Scan Context's published parameters
  c->lidar_height = 2.0; c->n_ring = 20; c->n_sector = 60; c->max_radius = 80.0;
  c->exclude_recent = 50; c->dist_threshold = 0.13;
  c->initial_capacity_frames = 1024;
}

int tloam_b200_loop_enable(tloam_b200_handle* h, const tloam_loop_config* cfg) {
  if (!h || !cfg || cfg->n_ring < 1 || cfg->n_sector < 1 || (long long)cfg->n_ring * cfg->n_sector > 4096 ||
      !std::isfinite(cfg->max_radius) || !(cfg->max_radius > 0.0) || cfg->exclude_recent < 0 || !std::isfinite(cfg->lidar_height) ||
      !std::isfinite(cfg->dist_threshold))
    return TLOAM_B200_ERR_INVALID_ARG;
  LoopLib lib;
  int rc = loop_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!h->d_loop_best) {
    CU_TRY(cudaMalloc(&h->d_loop_best, (TLOAM_SC_MAX_BLOCKS + 1) * sizeof(tloam_sc_best)));
    CU_TRY(cudaMallocHost(&h->h_loop_best, sizeof(tloam_sc_best)));
    CU_TRY(cudaEventCreateWithFlags(&h->ev_loop, cudaEventDisableTiming));
  }
  cudaFree(h->d_loop_db); h->d_loop_db = nullptr; h->loop_cap = 0;
  cudaFree(h->d_loop_dirs); h->d_loop_dirs = nullptr;
  const size_t cap = cfg->initial_capacity_frames ? cfg->initial_capacity_frames : 1;
  CU_TRY(cudaMalloc(&h->d_loop_db, cap * TLOAM_SC_SLOT_DOUBLES(cfg->n_ring, cfg->n_sector) * sizeof(double)));
  h->loop_cap = cap;
  // the sector boundaries: (cos, sin) of 2 pi k / n_sector, k = 1 .. n_sector - 1, by the C library (the oracle calls the same)
  std::vector<double> dirs(2 * (size_t)cfg->n_sector);
  for (int k = 1; k < cfg->n_sector; ++k) {
    const double t = 2.0 * M_PI * k / cfg->n_sector;
    dirs[2 * (k - 1)] = std::cos(t);
    dirs[2 * (k - 1) + 1] = std::sin(t);
  }
  CU_TRY(cudaMalloc(&h->d_loop_dirs, dirs.size() * sizeof(double)));
  CU_TRY(cudaMemcpy(h->d_loop_dirs, dirs.data(), dirs.size() * sizeof(double), cudaMemcpyHostToDevice));
  h->loop_cfg = *cfg;
  h->loop_frames = 0; h->loop_growths = 0; h->loop_has_result = false; h->loop_query = -1;
  h->loop_on = true;
  h->lv_on = false;                        // verification is enabled anew on the empty database
  h->lvs_on = false;
  return TLOAM_B200_OK;
}

static int lv_clear(tloam_b200_handle* h);

int tloam_b200_loop_reset(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on) return TLOAM_B200_ERR_NOT_READY;
  h->loop_frames = 0; h->loop_has_result = false; h->loop_query = -1;
  if (h->lv_on) {
    CU_TRY(cudaSetDevice(h->device));
    return lv_clear(h);
  }
  return TLOAM_B200_OK;
}

// the one place an add synchronises: the database is full.  It grows to 1.5 x its capacity; the slots keep their bits.
static int loop_grow(tloam_b200_handle* h) {
  const size_t slot = TLOAM_SC_SLOT_DOUBLES(h->loop_cfg.n_ring, h->loop_cfg.n_sector);
  size_t ncap = h->loop_cap + h->loop_cap / 2;
  if (ncap < h->loop_cap + 1) ncap = h->loop_cap + 1;
  double* q = nullptr;
  CU_TRY(cudaMalloc(&q, ncap * slot * sizeof(double)));
  if (h->loop_frames)
    CU_TRY(cudaMemcpyAsync(q, h->d_loop_db, h->loop_frames * slot * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  cudaFree(h->d_loop_db);
  h->d_loop_db = q; h->loop_cap = ncap;
  h->loop_growths++;
  return TLOAM_B200_OK;
}

static int lv_append(tloam_b200_handle* h, const double* d_in, size_t n);

// the descriptor of the n rows at d_xyz (device) into the next slot, then its query over every slot <= frame - exclude_recent;
// the result lands in the pinned slot, ev_loop marks it
static int loop_add_impl(tloam_b200_handle* h, const double* d_xyz, size_t n) {
  LoopLib lib;
  int rc = loop_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  if (h->loop_frames == h->loop_cap && (rc = loop_grow(h)) != TLOAM_B200_OK) return rc;
  if (h->lv_on && (rc = lv_append(h, d_xyz, n)) != TLOAM_B200_OK) return rc;
  const tloam_loop_config& c = h->loop_cfg;
  tloam_sc_args a;
  a.n_ring = c.n_ring; a.n_sector = c.n_sector; a.lidar_height = c.lidar_height; a.max_radius = c.max_radius;
  a.dirs = h->d_loop_dirs; a.xyz = d_xyz; a.n = n; a.db = h->d_loop_db; a.frame = h->loop_frames;
  const size_t E = (size_t)c.exclude_recent;
  a.n_candidates = h->loop_frames >= E ? h->loop_frames - E + 1 : 0;
  a.partial = h->d_loop_best; a.best = h->d_loop_best + TLOAM_SC_MAX_BLOCKS;
  a.device = h->device; a.stream = h->stream;
  const tloam_sc_fn step[3] = {lib.bin, lib.finish, lib.search};
  static const char* const names[3] = {"k_sc_bin", "k_sc_finish", "k_sc_search"};
  for (int k = 0; k < 3; ++k) {
    int e = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = step[k](&a)));
    if (e != cudaSuccess) {
      snprintf(h->last_error, sizeof(h->last_error), "loop closure: %s: %s", names[k], cudaGetErrorString((cudaError_t)e));
      return TLOAM_B200_ERR_CUDA;
    }
  }
  CU_TRY(cudaMemcpyAsync(h->h_loop_best, a.best, sizeof(tloam_sc_best), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaEventRecord(h->ev_loop, h->stream));
  h->loop_query = (long long)h->loop_frames;
  h->loop_frames++;
  h->loop_has_result = true;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_add_frame(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on || h->raw_gen != h->seg_gen) return TLOAM_B200_ERR_NOT_READY;
  return loop_add_impl(h, h->raw_scan, h->raw_n);
}

int tloam_b200_loop_add(tloam_b200_handle* h, const double* xyz, size_t n) {
  if (!h || (!xyz && n) || n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  int rc;
  if ((rc = ensure_dev(h, &h->d_loop_in, &h->cap_loop_in, n, false)) != TLOAM_B200_OK) return rc;
  if (n && (rc = upload_host(h, h->d_loop_in, xyz, n * 24)) != TLOAM_B200_OK) return rc;
  return loop_add_impl(h, h->d_loop_in, n);
}

int tloam_b200_loop_result(tloam_b200_handle* h, tloam_loop_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on || !h->loop_has_result) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaEventSynchronize(h->ev_loop));
  const tloam_sc_best b = *h->h_loop_best;
  const int S = h->loop_cfg.n_sector;
  out->query = h->loop_query;
  out->candidate = b.candidate;
  out->shift = (int)b.shift;
  const int k = 2 * out->shift >= S ? S - out->shift : -out->shift;      // yaw = -shift sectors, wrapped to (-pi, pi]
  out->yaw = b.candidate >= 0 ? (double)k * (2.0 * M_PI / S) : 0.0;
  out->distance = b.distance;
  out->is_loop = b.candidate >= 0 && b.distance < h->loop_cfg.dist_threshold ? 1 : 0;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_size(tloam_b200_handle* h, size_t* n_frames) {
  if (!h || !n_frames) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on) return TLOAM_B200_ERR_NOT_READY;
  *n_frames = h->loop_frames;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_descriptor_download(tloam_b200_handle* h, size_t frame, double* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on) return TLOAM_B200_ERR_NOT_READY;
  if (frame >= h->loop_frames) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t slot = TLOAM_SC_SLOT_DOUBLES(h->loop_cfg.n_ring, h->loop_cfg.n_sector);
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(out, h->d_loop_db + frame * slot, slot * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_loop_descriptors_download(tloam_b200_handle* h, size_t first, size_t count, double* out) {
  if (!h || (!out && count)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on) return TLOAM_B200_ERR_NOT_READY;
  if (first > h->loop_frames || count > h->loop_frames - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (!count) return TLOAM_B200_OK;
  const size_t slot = TLOAM_SC_SLOT_DOUBLES(h->loop_cfg.n_ring, h->loop_cfg.n_sector);
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(out, h->d_loop_db + first * slot, count * slot * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Loop verification (a keyframe per loop frame, by the global map's ordered path into buffers of its own; the commit and
// the ICP kernels in loop_verify.cu, loaded from libtloam_b200_loopv.so on the first verification call).
// ---------------------------------------------------------------------------------------------
struct LoopvLib { tloam_lv_verify_fn verify = nullptr; tloam_lv_commit_fn commit = nullptr; };
static std::mutex g_loopv_mu;
static LoopvLib g_loopv;

static int loopv_load(tloam_b200_handle* h, LoopvLib* out) {
  std::lock_guard<std::mutex> lk(g_loopv_mu);
  if (!g_loopv.verify) {
    const std::string path = sibling_path("libtloam_b200_loopv.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    LoopvLib l;
    if (so) {
      l.verify = reinterpret_cast<tloam_lv_verify_fn>(dlsym(so, "tloam_lv_verify"));
      l.commit = reinterpret_cast<tloam_lv_commit_fn>(dlsym(so, "tloam_lv_commit"));
    }
    if (!l.verify || !l.commit) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "loop verification: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_loopv = l;
  }
  *out = g_loopv;
  return TLOAM_B200_OK;
}

static int lv_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "loop verification: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

void tloam_b200_loop_verify_default_config(tloam_loop_verify_config* c) {
  c->voxel = 0.5;
  c->corr_dist_coarse = 4.0; c->corr_dist_fine = 1.0;
  c->max_iterations = 40;
  c->eps_translation = 1e-4; c->eps_rotation = 1e-5;
  c->max_fitness = 1.0;
  c->initial_capacity_points = (size_t)1 << 21;
}

// an empty store (keyframe table offsets[0] = 0)
static int lv_clear(tloam_b200_handle* h) {
  CU_TRY(cudaMemsetAsync(h->d_lv_st, 0, sizeof(GMapState), h->stream));
  CU_TRY(cudaMemsetAsync(h->d_lv_off, 0, sizeof(unsigned long long), h->stream));
  h->lv_cum = h->lv_known_cum = h->lv_known = 0;
  for (auto& pr : h->lv_probes) pr.pending = false;
  h->lv_ran = false; h->lv_passes = 0; h->lv_nq = 0;
  h->lvs_ran = false; h->lvs_passes = 0;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_verify_enable(tloam_b200_handle* h, const tloam_loop_verify_config* c) {
  if (!h || !c) return TLOAM_B200_ERR_INVALID_ARG;
  const double v[6] = {c->voxel, c->corr_dist_coarse, c->corr_dist_fine, c->eps_translation, c->eps_rotation, c->max_fitness};
  for (double x : v)
    if (!std::isfinite(x) || !(x > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (c->corr_dist_fine > c->corr_dist_coarse || c->max_iterations < 1 || c->max_iterations > 200) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loop_on || h->loop_frames != 0) return TLOAM_B200_ERR_NOT_READY;
  LoopvLib lib;
  int rc = loopv_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!h->d_lv_st) {
    CU_TRY(cudaMalloc(&h->d_lv_st, sizeof(GMapState)));
    CU_TRY(cudaMalloc(&h->d_lv_pose, 16 * sizeof(double)));
    const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    CU_TRY(cudaMemcpy(h->d_lv_pose, eye, sizeof(eye), cudaMemcpyHostToDevice));
    CU_TRY(cudaMalloc(&h->d_lv_state, sizeof(tloam_lv_state)));
    for (auto& pr : h->lv_probes) {
      CU_TRY(cudaEventCreateWithFlags(&pr.ev, cudaEventDisableTiming));
      CU_TRY(cudaMallocHost(&pr.h_count, sizeof(unsigned long long)));
    }
  }
  const size_t cap = c->initial_capacity_points ? c->initial_capacity_points : 1;
  if (cap != h->cap_lv) {
    cudaFree(h->d_lv_pts); h->d_lv_pts = nullptr; h->cap_lv = 0;
    CU_TRY(cudaMalloc(&h->d_lv_pts, cap * 3 * sizeof(double)));
    h->cap_lv = cap;
  }
  const size_t cap_off = h->loop_cap + 2;    // the descriptor database's capacity, plus the closing entry
  if (cap_off > h->cap_lv_off) {
    cudaFree(h->d_lv_off); h->d_lv_off = nullptr; h->cap_lv_off = 0;
    CU_TRY(cudaMalloc(&h->d_lv_off, cap_off * sizeof(unsigned long long)));
    h->cap_lv_off = cap_off;
  }
  h->lv_cfg = *c;
  h->lv_growths = 0;
  h->lv_on = true;
  return lv_clear(h);
}

static void lv_harvest(tloam_b200_handle* h) {
  for (auto& pr : h->lv_probes) {
    if (!pr.pending) continue;
    if (cudaEventQuery(pr.ev) != cudaSuccess) { cudaGetLastError(); continue; }
    pr.pending = false;
    if (pr.cum >= h->lv_known_cum) { h->lv_known_cum = pr.cum; h->lv_known = *pr.h_count; }
  }
}

// the one place a keyframe add synchronises: the store (or its table) may not hold the next keyframe.  The exact size is
// read, and the store grows to max(1.5 x capacity, exact size + n rows); the table x1.5.
static int lv_grow(tloam_b200_handle* h, size_t n) {
  CU_TRY(cudaStreamSynchronize(h->stream));
  GMapState st;
  CU_TRY(cudaMemcpyAsync(&st, h->d_lv_st, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->lv_known = st.count; h->lv_known_cum = h->lv_cum;
  for (auto& pr : h->lv_probes) pr.pending = false;
  if (st.count + n > h->cap_lv) {
    size_t ncap = h->cap_lv + h->cap_lv / 2;
    if (ncap < st.count + n) ncap = st.count + n;
    double* q = nullptr;
    CU_TRY(cudaMalloc(&q, ncap * 3 * sizeof(double)));
    if (st.count) CU_TRY(cudaMemcpyAsync(q, h->d_lv_pts, st.count * 3 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_lv_pts);
    h->d_lv_pts = q; h->cap_lv = ncap;
  }
  if (h->loop_frames + 2 > h->cap_lv_off) {
    size_t ncap = h->cap_lv_off + h->cap_lv_off / 2;
    if (ncap < h->loop_frames + 2) ncap = h->loop_frames + 2;
    unsigned long long* q = nullptr;
    CU_TRY(cudaMalloc(&q, ncap * sizeof(unsigned long long)));
    CU_TRY(cudaMemcpyAsync(q, h->d_lv_off, (h->loop_frames + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_lv_off);
    h->d_lv_off = q; h->cap_lv_off = ncap;
  }
  h->lv_growths++;
  return TLOAM_B200_OK;
}

// keyframe loop_frames = VoxelDownSample(voxel) of the finite rows of the n rows at d_in: gmap_append_impl's transform ->
// guard -> voxel_pipeline(sorted) -> emit at pose I, then a commit that closes the slot whatever the frame held
static int lv_append(tloam_b200_handle* h, const double* d_in, size_t n) {
  LoopvLib lib;
  int rc = loopv_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  lv_harvest(h);
  const unsigned long long bound = h->lv_known + (h->lv_cum - h->lv_known_cum) + n;   // voxels <= finite rows <= rows
  if (bound > h->cap_lv || h->loop_frames + 2 > h->cap_lv_off)
    if ((rc = lv_grow(h, n)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, &h->d_lv_reg, &h->cap_lv_reg, n, false)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, &h->d_lv_fin, &h->cap_lv_fin, n, false)) != TLOAM_B200_OK) return rc;
  GMapState* st = h->d_lv_st;
  const double voxel = h->lv_cfg.voxel;
  CU_TRY(cudaMemsetAsync(&st->n_fin, 0, sizeof(GMapState) - offsetof(GMapState, n_fin), h->stream));
  const unsigned tb = 256, gb = (unsigned)((n + tb - 1) / tb);
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_transform<<<gb, tb, 0, h->stream>>>(d_in, (unsigned)n, h->d_lv_pose, h->d_lv_reg, h->d_lv_fin, st)));
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_guard<<<1, 32, 0, h->stream>>>(st, voxel)));
  VoxSorted vs;
  if ((rc = voxel_pipeline(h, h->d_lv_fin, n, &st->n_fin, 0u, nullptr, nullptr, nullptr, 0.0, voxel, nullptr, &st->n_vox,
                           h->stream, 0, &vs)) != TLOAM_B200_OK) return rc;
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_emit<<<gb, tb, 0, h->stream>>>(vs.a, vs.slots, h->d_lv_pts, st, h->cap_lv)));
  int e = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.commit(&st->n_vox, &st->refused, &st->count, &st->frames, &st->flags, h->d_lv_off, h->cap_lv,
                                                 h->device, h->stream)));
  if ((rc = lv_status(h, e, "k_lv_commit")) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaGetLastError());
  h->lv_cum += n;
  tloam_b200_handle::GMapProbe& pr = h->lv_probes[h->lv_probe_next];
  if (!pr.pending) {
    CU_TRY(cudaMemcpyAsync(pr.h_count, &st->count, sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaEventRecord(pr.ev, h->stream));
    pr.cum = h->lv_cum; pr.pending = true;
    h->lv_probe_next = (h->lv_probe_next + 1) & 3;
  }
  return TLOAM_B200_OK;
}

// synchronises and reads keyframe f's range; a store that refused a keyframe for want of room is a bug, not an input error
static int lv_range(tloam_b200_handle* h, size_t f, unsigned long long* first, unsigned long long* n) {
  unsigned long long off[2];
  unsigned flags = 0;
  CU_TRY(cudaMemcpyAsync(off, h->d_lv_off + f, sizeof(off), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaMemcpyAsync(&flags, &h->d_lv_st->flags, sizeof(flags), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (flags & kGMapOverflow) {
    snprintf(h->last_error, sizeof(h->last_error), "loop verification: the device-side capacity check refused a keyframe");
    return TLOAM_B200_ERR_CUDA;
  }
  *first = off[0]; *n = off[1] - off[0];
  return TLOAM_B200_OK;
}

int tloam_b200_loop_keyframe_download(tloam_b200_handle* h, size_t frame, double* out, size_t capacity_points, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on) return TLOAM_B200_ERR_NOT_READY;
  if (frame >= h->loop_frames) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  unsigned long long first = 0, cnt = 0;
  int rc = lv_range(h, frame, &first, &cnt);
  if (rc != TLOAM_B200_OK) return rc;
  *n = cnt;
  if (capacity_points < cnt || (!out && cnt)) return TLOAM_B200_ERR_INVALID_ARG;
  if (cnt) CU_TRY(cudaMemcpyAsync(out, h->d_lv_pts + 3 * first, cnt * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_loop_verify(tloam_b200_handle* h, long long query, long long candidate, const double guess[16],
                           tloam_loop_verify_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on) return TLOAM_B200_ERR_NOT_READY;
  if (query < 0 || candidate < 0 || (size_t)query >= h->loop_frames || (size_t)candidate >= h->loop_frames)
    return TLOAM_B200_ERR_INVALID_ARG;
  double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if (guess) memcpy(T, guess, sizeof(T));
  Pose7 p7;
  if (!pose_from_matrix(T, p7) || T[3] != 0.0 || T[7] != 0.0 || T[11] != 0.0 || T[15] != 1.0) return TLOAM_B200_ERR_BAD_POSE;
  LoopvLib lib;
  int rc = loopv_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  unsigned long long q0 = 0, nq = 0, m0 = 0, nm = 0;
  if ((rc = lv_range(h, (size_t)query, &q0, &nq)) != TLOAM_B200_OK) return rc;
  if ((rc = lv_range(h, (size_t)candidate, &m0, &nm)) != TLOAM_B200_OK) return rc;
  const tloam_loop_verify_config& c = h->lv_cfg;
  memset(out, 0, sizeof(*out));
  out->query = query; out->candidate = candidate;
  memcpy(out->T, T, sizeof(T));
  out->n_query_points = (long long)nq; out->n_candidate_points = (long long)nm;
  h->lv_ran = true; h->lv_passes = 0; h->lv_nq = nq;
  if (nq == 0 || nm == 0) {
    out->termination = TLOAM_LOOP_VERIFY_EMPTY;
    out->fitness = INFINITY;
    return TLOAM_B200_OK;
  }
  // M is split over grid y until the search has about four blocks per SM of an H100 SXM (132)
  const unsigned long long qb = (nq + TLOAM_LV_THREADS - 1) / TLOAM_LV_THREADS, tiles = (nm + TLOAM_LV_THREADS - 1) / TLOAM_LV_THREADS;
  unsigned long long splits = (4 * 132 + qb - 1) / qb;
  if (splits > tiles) splits = tiles;
  if (splits < 1) splits = 1;
  const size_t passes = (size_t)c.max_iterations + 1;
  const size_t o_sums = round_up(splits * nq * sizeof(tloam_lv_best), 256);
  const size_t o_idx = o_sums + round_up(qb * TLOAM_LV_SUMS * sizeof(double), 256);
  const size_t o_d2 = o_idx + round_up(passes * nq * sizeof(int), 256);
  const size_t bytes = o_d2 + passes * nq * sizeof(double);
  if (bytes > h->cap_lv_scratch) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_lv_scratch); h->d_lv_scratch = nullptr; h->cap_lv_scratch = 0;
    CU_TRY(cudaMalloc(&h->d_lv_scratch, bytes));
    h->cap_lv_scratch = bytes;
  }
  tloam_lv_state s;
  memset(&s, 0, sizeof(s));
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) s.R[3 * r + k] = T[4 * k + r];
    s.t[r] = T[12 + r];
  }
  s.r = c.corr_dist_coarse;
  s.term = TLOAM_LOOP_VERIFY_ITERATION_LIMIT;
  CU_TRY(cudaMemcpyAsync(h->d_lv_state, &s, sizeof(s), cudaMemcpyHostToDevice, h->stream));   // pageable: staged before return
  tloam_lv_args a;
  a.pts = h->d_lv_pts; a.q0 = q0; a.nq = nq; a.m0 = m0; a.nm = nm;
  a.corr_dist_coarse = c.corr_dist_coarse; a.corr_dist_fine = c.corr_dist_fine;
  a.eps_translation = c.eps_translation; a.eps_rotation = c.eps_rotation; a.max_iterations = c.max_iterations;
  a.splits = (unsigned)splits; a.state = h->d_lv_state;
  a.part = reinterpret_cast<tloam_lv_best*>(h->d_lv_scratch);
  a.sums = reinterpret_cast<double*>(h->d_lv_scratch + o_sums);
  a.match_index = reinterpret_cast<int*>(h->d_lv_scratch + o_idx);
  a.match_d2 = reinterpret_cast<double*>(h->d_lv_scratch + o_d2);
  a.device = h->device; a.stream = h->stream;
  h->lv_match_index = a.match_index; h->lv_match_d2 = a.match_d2;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.verify(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = lv_status(h, e, "k_lv_*")) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(&s, h->d_lv_state, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (int r = 0; r < 3; ++r) {
    for (int k = 0; k < 3; ++k) out->T[4 * k + r] = s.R[3 * r + k];
    out->T[12 + r] = s.t[r];
  }
  out->fitness = s.fitness; out->rmse = s.rmse; out->inliers = (long long)s.inliers;
  out->iterations = s.iter; out->termination = s.term;
  out->accepted = s.term == TLOAM_LOOP_VERIFY_CONVERGED && s.fitness <= c.max_fitness ? 1 : 0;
  h->lv_passes = s.iter + 1;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_verify_matches(tloam_b200_handle* h, int pass, int* index, double* d2, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on || !h->lv_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = h->lv_nq;
  if (pass < 0 || pass >= h->lv_passes || capacity < h->lv_nq) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t nq = h->lv_nq;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (index) CU_TRY(cudaMemcpyAsync(index, h->lv_match_index + (size_t)pass * nq, nq * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (d2) CU_TRY(cudaMemcpyAsync(d2, h->lv_match_d2 + (size_t)pass * nq, nq * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Pose graph (the node store and the loop edges here; the Gauss-Newton kernels in pose_graph.cu, loaded from
// libtloam_b200_pg.so on the first optimisation).
// ---------------------------------------------------------------------------------------------
struct PgLib { tloam_pg_optimize_fn optimize = nullptr; tloam_pg_chol_blocks_fn chol_blocks = nullptr; };
static std::mutex g_pg_mu;
static PgLib g_pg;

static int pg_load(tloam_b200_handle* h, PgLib* out) {
  std::lock_guard<std::mutex> lk(g_pg_mu);
  if (!g_pg.optimize) {
    const std::string path = sibling_path("libtloam_b200_pg.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    PgLib l;
    if (so) {
      l.optimize = reinterpret_cast<tloam_pg_optimize_fn>(dlsym(so, "tloam_pg_optimize"));
      l.chol_blocks = reinterpret_cast<tloam_pg_chol_blocks_fn>(dlsym(so, "tloam_pg_chol_blocks"));
    }
    if (!l.optimize || !l.chol_blocks) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "pose graph: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_pg = l;
  }
  *out = g_pg;
  return TLOAM_B200_OK;
}

static int pg_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "pose graph: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

static bool pg_rigid(const double T[16]) {
  Pose7 p7;
  return pose_from_matrix(T, p7) && T[3] == 0.0 && T[7] == 0.0 && T[11] == 0.0 && T[15] == 1.0;
}

void tloam_b200_pose_graph_default_config(tloam_pose_graph_config* c) {
  c->sigma_odom_translation = 0.02; c->sigma_odom_rotation = 0.001;
  c->sigma_loop_translation = 0.3; c->sigma_loop_rotation = 0.002;
  c->max_iterations = 20;
  c->eps_translation = 1e-4; c->eps_rotation = 1e-6;
  c->max_loop_edges = 1024;
  c->initial_capacity_nodes = 4096;
}

int tloam_b200_pose_graph_enable(tloam_b200_handle* h, const tloam_pose_graph_config* c) {
  if (!h || !c) return TLOAM_B200_ERR_INVALID_ARG;
  const double v[6] = {c->sigma_odom_translation, c->sigma_odom_rotation, c->sigma_loop_translation, c->sigma_loop_rotation,
                       c->eps_translation, c->eps_rotation};
  for (double x : v)
    if (!std::isfinite(x) || !(x > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (c->max_iterations < 1 || c->max_iterations > 100 || c->max_loop_edges == 0) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  const size_t cap = c->initial_capacity_nodes ? c->initial_capacity_nodes : 1;
  if (cap != h->cap_pg) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_pg_O); h->d_pg_O = nullptr; h->cap_pg = 0;
    CU_TRY(cudaMalloc(&h->d_pg_O, cap * 16 * sizeof(double)));
    h->cap_pg = cap;
  }
  if (!h->d_pg_state) CU_TRY(cudaMalloc(&h->d_pg_state, sizeof(tloam_pg_state)));
  h->pg_cfg = *c;
  h->pg_growths = 0;
  h->pg_on = true;
  return tloam_b200_pose_graph_reset(h);
}

int tloam_b200_pose_graph_reset(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  h->pg_nodes = 0;
  h->pg_ij.clear(); h->pg_Z.clear();
  h->d_pg_T = nullptr; h->pg_opt_nodes = 0;
  h->d_pgr_w = nullptr; h->pgr_w_edges = 0;
  return TLOAM_B200_OK;
}

// the one place an add synchronises: the store is full and grows x1.5
static int pg_reserve(tloam_b200_handle* h) {
  if (h->pg_nodes < h->cap_pg) return TLOAM_B200_OK;
  const size_t ncap = h->cap_pg + (h->cap_pg + 1) / 2;
  double* q = nullptr;
  CU_TRY(cudaMalloc(&q, ncap * 16 * sizeof(double)));
  CU_TRY(cudaMemcpyAsync(q, h->d_pg_O, h->pg_nodes * 16 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  cudaFree(h->d_pg_O);
  h->d_pg_O = q; h->cap_pg = ncap;
  h->pg_growths++;
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_add_node(tloam_b200_handle* h, const double pose[16]) {
  if (!h || !pose) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  if (!pg_rigid(pose)) return TLOAM_B200_ERR_BAD_POSE;
  CU_TRY(cudaSetDevice(h->device));
  int rc = pg_reserve(h);
  if (rc != TLOAM_B200_OK) return rc;
  double tmp[16];
  memcpy(tmp, pose, sizeof(tmp));
  CU_TRY(cudaMemcpyAsync(h->d_pg_O + 16 * h->pg_nodes, tmp, sizeof(tmp), cudaMemcpyHostToDevice, h->stream));   // pageable: staged before return
  h->pg_nodes++;
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_add_node_chained(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  int rc = pg_reserve(h);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(h->d_pg_O + 16 * h->pg_nodes, reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, result),
                         16 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  h->pg_nodes++;
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_add_loop(tloam_b200_handle* h, const tloam_loop_verify_result* v) {
  if (!h || !v) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  if (!v->accepted || v->candidate < 0 || v->query < 0 || (size_t)v->candidate >= h->pg_nodes ||
      (size_t)v->query >= h->pg_nodes || v->candidate == v->query || h->pg_ij.size() / 2 >= h->pg_cfg.max_loop_edges)
    return TLOAM_B200_ERR_INVALID_ARG;
  if (!pg_rigid(v->T)) return TLOAM_B200_ERR_BAD_POSE;
  h->pg_ij.push_back(v->candidate); h->pg_ij.push_back(v->query);
  h->pg_Z.insert(h->pg_Z.end(), v->T, v->T + 16);
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_size(tloam_b200_handle* h, size_t* nodes, size_t* loop_edges) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  if (nodes) *nodes = h->pg_nodes;
  if (loop_edges) *loop_edges = h->pg_ij.size() / 2;
  return TLOAM_B200_OK;
}

// the device buffers of one optimisation over the graph as it stands, the loop edges uploaded and T[0] = O; robust: after
// them, the loop edges' weights (set to 1), residuals and the GNC state
struct PgrBufs { double* w = nullptr; double* rho = nullptr; tloam_pgr_state* state = nullptr; };

static int pg_prepare(tloam_b200_handle* h, const PgLib& lib, tloam_pg_args* ap, PgrBufs* robust) {
  const size_t N = h->pg_nodes, L = h->pg_ij.size() / 2;
  CU_TRY(cudaSetDevice(h->device));
  const tloam_pose_graph_config& c = h->pg_cfg;
  const size_t nl = 6 * L, ncol = nl + 1, E = N - 1 + L;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += round_up(bytes, 256); return at; };
  const size_t o_T = take(2 * N * 16 * sizeof(double)), o_ij = take(2 * L * sizeof(long long)), o_Z = take(16 * L * sizeof(double));
  const size_t o_edge = take(E * TLOAM_PG_EDGE * sizeof(double)), o_chain = take(N * TLOAM_PG_CHAIN * sizeof(double));
  const size_t o_b = take(N * 6 * sizeof(double)), o_Y = take(6 * (N - 1) * ncol * sizeof(double));
  const size_t o_S = take(nl * ncol * sizeof(double)), o_z = take(nl * sizeof(double)), o_n = take(N * 2 * sizeof(double));
  size_t o_w = 0, o_rho = 0, o_g = 0;
  if (robust) { o_w = take(L * sizeof(double)); o_rho = take(L * sizeof(double)); o_g = take(sizeof(tloam_pgr_state)); }
  if (o > h->cap_pg_scratch) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_pg_scratch); h->d_pg_scratch = nullptr; h->cap_pg_scratch = 0;
    CU_TRY(cudaMalloc(&h->d_pg_scratch, o));
    h->cap_pg_scratch = o;
  }
  unsigned char* base = h->d_pg_scratch;
  tloam_pg_args& a = *ap;
  memset(&a, 0, sizeof(a));
  a.O = h->d_pg_O;
  a.T = reinterpret_cast<double*>(base + o_T);
  a.loop_ij = reinterpret_cast<const long long*>(base + o_ij);
  a.loop_Z = reinterpret_cast<const double*>(base + o_Z);
  a.N = N; a.L = L;
  for (int k = 0; k < 3; ++k) {
    a.w_odom[k] = 1.0 / (c.sigma_odom_translation * c.sigma_odom_translation);
    a.w_odom[3 + k] = 1.0 / (c.sigma_odom_rotation * c.sigma_odom_rotation);
    a.w_loop[k] = 1.0 / (c.sigma_loop_translation * c.sigma_loop_translation);
    a.w_loop[3 + k] = 1.0 / (c.sigma_loop_rotation * c.sigma_loop_rotation);
  }
  a.eps_translation = c.eps_translation; a.eps_rotation = c.eps_rotation; a.max_iterations = c.max_iterations;
  int rc;
  if ((rc = pg_status(h, lib.chol_blocks(h->device, &a.chol_blocks), "occupancy")) != TLOAM_B200_OK) return rc;
  a.state = h->d_pg_state;
  a.edge = reinterpret_cast<double*>(base + o_edge);
  a.chain = reinterpret_cast<double*>(base + o_chain);
  a.b = reinterpret_cast<double*>(base + o_b);
  a.Y = reinterpret_cast<double*>(base + o_Y);
  a.S = reinterpret_cast<double*>(base + o_S);
  a.z = reinterpret_cast<double*>(base + o_z);
  a.norms = reinterpret_cast<double*>(base + o_n);
  a.device = h->device; a.stream = h->stream;
  // pageable sources: staged before each call returns
  CU_TRY(cudaMemcpyAsync(base + o_ij, h->pg_ij.data(), 2 * L * sizeof(long long), cudaMemcpyHostToDevice, h->stream));
  CU_TRY(cudaMemcpyAsync(base + o_Z, h->pg_Z.data(), 16 * L * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CU_TRY(cudaMemcpyAsync(a.T, h->d_pg_O, N * 16 * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  if (robust) {
    robust->w = reinterpret_cast<double*>(base + o_w);
    robust->rho = reinterpret_cast<double*>(base + o_rho);
    robust->state = reinterpret_cast<tloam_pgr_state*>(base + o_g);
    const std::vector<double> ones(L, 1.0);
    CU_TRY(cudaMemcpyAsync(robust->w, ones.data(), L * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  }
  return TLOAM_B200_OK;
}

// enqueues one Gauss-Newton stage of up to max_iterations steps from T[cur]: the state reset (cost and initial_cost are
// evaluated at T[cur] by the stage), then the launcher
static int pg_stage(tloam_b200_handle* h, const PgLib& lib, tloam_pg_args& a, int cur, int max_iterations) {
  tloam_pg_state s;
  memset(&s, 0, sizeof(s));
  s.cur = cur;
  s.term = TLOAM_POSE_GRAPH_ITERATION_LIMIT;
  CU_TRY(cudaMemcpyAsync(h->d_pg_state, &s, sizeof(s), cudaMemcpyHostToDevice, h->stream));
  a.max_iterations = max_iterations;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.optimize(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  return pg_status(h, e, "k_pg_*");
}

static void pg_forget(tloam_b200_handle* h) {
  h->d_pg_T = nullptr; h->pg_opt_nodes = 0;
  h->d_pgr_w = nullptr; h->pgr_w_edges = 0;
}

int tloam_b200_pose_graph_optimize(tloam_b200_handle* h, tloam_pose_graph_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  const size_t N = h->pg_nodes, L = h->pg_ij.size() / 2;
  memset(out, 0, sizeof(*out));
  out->nodes = (long long)N; out->loop_edges = (long long)L;
  pg_forget(h);
  if (L == 0) {
    out->termination = TLOAM_POSE_GRAPH_NO_LOOPS;
    return TLOAM_B200_OK;
  }
  PgLib lib;
  int rc = pg_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  tloam_pg_args a;
  if ((rc = pg_prepare(h, lib, &a, nullptr)) != TLOAM_B200_OK) return rc;
  if ((rc = pg_stage(h, lib, a, 0, h->pg_cfg.max_iterations)) != TLOAM_B200_OK) return rc;
  tloam_pg_state s;
  CU_TRY(cudaMemcpyAsync(&s, h->d_pg_state, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  out->iterations = s.iter; out->termination = s.term;
  out->initial_cost = s.initial_cost; out->final_cost = s.cost;
  out->step_translation = s.step_t; out->step_rotation = s.step_r;
  h->d_pg_T = a.T + 16 * N * (size_t)s.cur;
  h->pg_opt_nodes = N;
  return TLOAM_B200_OK;
}

// ---- robust pose graph (the outer GNC loop here; the residual and weight kernels in pose_graph_robust.cu, loaded from
//      libtloam_b200_pgr.so on the first robust optimisation) ----
struct PgrLib { tloam_pgr_update_fn update = nullptr; };
static std::mutex g_pgr_mu;
static PgrLib g_pgr;

static int pgr_load(tloam_b200_handle* h, PgrLib* out) {
  std::lock_guard<std::mutex> lk(g_pgr_mu);
  if (!g_pgr.update) {
    const std::string path = sibling_path("libtloam_b200_pgr.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    PgrLib l;
    if (so) l.update = reinterpret_cast<tloam_pgr_update_fn>(dlsym(so, "tloam_pgr_update"));
    if (!l.update) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "robust pose graph: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_pgr = l;
  }
  *out = g_pgr;
  return TLOAM_B200_OK;
}

void tloam_b200_pose_graph_robust_default_config(tloam_pose_graph_robust_config* c) {
  c->chi2_threshold = 16.81;
  c->gnc_factor = 1.4;
  c->inner_iterations = 2;
  c->max_outer_iterations = 100;
}

int tloam_b200_pose_graph_optimize_robust(tloam_b200_handle* h, const tloam_pose_graph_robust_config* cfg,
                                          tloam_pose_graph_robust_result* out) {
  if (!h || !cfg || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  if (!std::isfinite(cfg->chi2_threshold) || !(cfg->chi2_threshold > 0.0) || !std::isfinite(cfg->gnc_factor) ||
      !(cfg->gnc_factor > 1.0) || cfg->inner_iterations < 1 || cfg->inner_iterations > 100 || cfg->max_outer_iterations < 1 ||
      cfg->max_outer_iterations > 1000)
    return TLOAM_B200_ERR_INVALID_ARG;
  const size_t N = h->pg_nodes, L = h->pg_ij.size() / 2;
  memset(out, 0, sizeof(*out));
  out->pg.nodes = (long long)N; out->pg.loop_edges = (long long)L;
  pg_forget(h);
  if (L == 0) {
    out->pg.termination = TLOAM_POSE_GRAPH_NO_LOOPS;
    out->gnc_termination = TLOAM_POSE_GRAPH_GNC_NO_LOOPS;
    return TLOAM_B200_OK;
  }
  PgLib lib;
  PgrLib rlib;
  int rc = pg_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  if ((rc = pgr_load(h, &rlib)) != TLOAM_B200_OK) return rc;
  tloam_pg_args a;
  PgrBufs buf;
  if ((rc = pg_prepare(h, lib, &a, &buf)) != TLOAM_B200_OK) return rc;
  a.loop_w = buf.w;
  tloam_pgr_args r;
  memset(&r, 0, sizeof(r));
  r.T = a.T; r.pg_state = a.state; r.loop_ij = a.loop_ij; r.loop_Z = a.loop_Z; r.N = N; r.L = L;
  memcpy(r.w_loop, a.w_loop, sizeof(r.w_loop));
  r.chi2_threshold = cfg->chi2_threshold; r.gnc_factor = cfg->gnc_factor;
  r.rho = buf.rho; r.w = buf.w; r.state = buf.state;
  r.device = h->device; r.stream = h->stream;
  const int max_iterations = h->pg_cfg.max_iterations;
  tloam_pg_state s;
  tloam_pgr_state g;
  memset(&g, 0, sizeof(g));
  // one stage; update: then the weights at its poses (nothing when the stage was singular); then both states home
  auto stage = [&](int cur, int iterations, int update, int first) -> int {
    int rc2 = pg_stage(h, lib, a, cur, iterations);
    if (rc2 != TLOAM_B200_OK) return rc2;
    if (update) {
      int e = 0, launches = 0;
      TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = rlib.update(&r, first, &launches)));
      h->launches += launches > 0 ? launches - 1 : 0;
      if (e != cudaSuccess) {
        snprintf(h->last_error, sizeof(h->last_error), "robust pose graph: k_pgr_*: %s", cudaGetErrorString((cudaError_t)e));
        return TLOAM_B200_ERR_CUDA;
      }
      CU_TRY(cudaMemcpyAsync(&g, buf.state, sizeof(g), cudaMemcpyDeviceToHost, h->stream));
    }
    CU_TRY(cudaMemcpyAsync(&s, h->d_pg_state, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    out->pg.iterations += s.iter;
    return TLOAM_B200_OK;
  };
  if ((rc = stage(0, max_iterations, 1, 1)) != TLOAM_B200_OK) return rc;
  out->pg.initial_cost = s.initial_cost;
  int gnc = -1;
  if (s.term == TLOAM_POSE_GRAPH_SINGULAR) gnc = TLOAM_POSE_GRAPH_GNC_SINGULAR;
  else if (g.all_inliers) { gnc = TLOAM_POSE_GRAPH_GNC_ALL_INLIERS; out->inliers = (long long)L; }
  while (gnc < 0) {
    // g holds the weights the next stage runs with
    out->outer_iterations++;
    out->mu_final = g.mu; out->inliers = g.inliers; out->rejected = g.rejected;
    if (g.binary) {
      if ((rc = stage(s.cur, max_iterations, 0, 0)) != TLOAM_B200_OK) return rc;
      gnc = s.term == TLOAM_POSE_GRAPH_SINGULAR ? TLOAM_POSE_GRAPH_GNC_SINGULAR : TLOAM_POSE_GRAPH_GNC_CONVERGED;
      break;
    }
    const bool last = out->outer_iterations >= cfg->max_outer_iterations;
    if ((rc = stage(s.cur, cfg->inner_iterations, !last, 0)) != TLOAM_B200_OK) return rc;
    if (s.term == TLOAM_POSE_GRAPH_SINGULAR) gnc = TLOAM_POSE_GRAPH_GNC_SINGULAR;
    else if (last) gnc = TLOAM_POSE_GRAPH_GNC_OUTER_LIMIT;
  }
  out->gnc_termination = gnc;
  out->pg.termination = s.term;
  out->pg.final_cost = s.cost;
  out->pg.step_translation = s.step_t; out->pg.step_rotation = s.step_r;
  h->d_pg_T = a.T + 16 * N * (size_t)s.cur;
  h->pg_opt_nodes = N;
  h->d_pgr_w = buf.w; h->pgr_w_edges = L;
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_loop_weights(tloam_b200_handle* h, size_t first, size_t count, double* w) {
  if (!h || (!w && count)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  const size_t L = h->pg_ij.size() / 2;
  if (first > L || count > L - first) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  const size_t split = first + count < h->pgr_w_edges ? first + count : (first > h->pgr_w_edges ? first : h->pgr_w_edges);
  if (split > first)
    CU_TRY(cudaMemcpyAsync(w, h->d_pgr_w + first, (split - first) * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  for (size_t l = split; l < first + count; ++l) w[l - first] = 1.0;
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_download(tloam_b200_handle* h, size_t first, size_t count, double* out) {
  if (!h || (!out && count)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  if (first > h->pg_nodes || count > h->pg_nodes - first) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  const size_t split = first + count < h->pg_opt_nodes ? first + count : (first > h->pg_opt_nodes ? first : h->pg_opt_nodes);
  if (split > first)
    CU_TRY(cudaMemcpyAsync(out, h->d_pg_T + 16 * first, (split - first) * 16 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (first + count > split)
    CU_TRY(cudaMemcpyAsync(out + 16 * (split - first), h->d_pg_O + 16 * split, (first + count - split) * 16 * sizeof(double),
                           cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_pose_graph_correction(tloam_b200_handle* h, double T[16]) {
  if (!h || !T) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  for (int k = 0; k < 16; ++k) T[k] = k % 5 == 0 ? 1.0 : 0.0;
  if (!h->pg_opt_nodes) return TLOAM_B200_OK;
  const size_t last = h->pg_opt_nodes - 1;
  double A[16], O[16];
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(A, h->d_pg_T + 16 * last, sizeof(A), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaMemcpyAsync(O, h->d_pg_O + 16 * last, sizeof(O), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  // T = A O^-1: R_A R_O^T, t_A - R_A R_O^T t_O (column-major)
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[4 * c + r] = A[r] * O[c] + A[4 + r] * O[4 + c] + A[8 + r] * O[8 + c];
  }
  for (int r = 0; r < 3; ++r) T[12 + r] = A[12 + r] - (T[r] * O[12] + T[4 + r] * O[13] + T[8 + r] * O[14]);
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Loop-corrected global map (the pose tables here and in gmap_append_impl; the kernels in map_correct.cu, loaded from
// libtloam_b200_gmc.so when tracking is enabled).
// ---------------------------------------------------------------------------------------------
int tloam_b200_global_map_correction_enable(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || h->gmap_calls != 0) return TLOAM_B200_ERR_NOT_READY;
  GmcLib lib;
  int rc = gmc_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  if (h->cap_gmc != h->cap_gmap_off) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gmc_O); cudaFree(h->d_gmc_P); h->d_gmc_O = h->d_gmc_P = nullptr; h->cap_gmc = 0;
    CU_TRY(cudaMalloc(&h->d_gmc_O, h->cap_gmap_off * 16 * sizeof(double)));
    CU_TRY(cudaMalloc(&h->d_gmc_P, h->cap_gmap_off * 16 * sizeof(double)));
    h->cap_gmc = h->cap_gmap_off;
  }
  h->gmc_on = true;
  return TLOAM_B200_OK;
}

// the map's exact size, without touching its sticky flags (the next size / download call still reports them)
static int gmc_read(tloam_b200_handle* h, GMapState* st) {
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(st, h->d_gmap_st, sizeof(*st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_correct(tloam_b200_handle* h, const long long* node, size_t n_frames) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->gmc_on || !h->pg_on) return TLOAM_B200_ERR_NOT_READY;
  GmcLib lib;
  int rc = gmc_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  GMapState st;
  if ((rc = gmc_read(h, &st)) != TLOAM_B200_OK) return rc;
  if (n_frames != st.frames || (!node && n_frames)) return TLOAM_B200_ERR_INVALID_ARG;
  for (size_t f = 0; f < n_frames; ++f)
    if (node[f] < -1 || (node[f] >= 0 && (size_t)node[f] >= h->pg_nodes)) return TLOAM_B200_ERR_INVALID_ARG;
  double D[16];
  if ((rc = tloam_b200_pose_graph_correction(h, D)) != TLOAM_B200_OK) return rc;
  bool ident = true;                       // bit for bit: M = I keeps the appends' copy path
  for (int k = 0; k < 16; ++k) {
    const double e = k % 5 == 0 ? 1.0 : 0.0;
    ident &= memcmp(&D[k], &e, sizeof(double)) == 0;
  }
  if (n_frames) {
    size_t o = 0;
    auto take = [&](size_t bytes) { const size_t at = o; o += round_up(bytes, 256); return at; };
    const size_t o_node = take(n_frames * sizeof(long long)), o_M = take(n_frames * 16 * sizeof(double));
    const size_t o_moved = take(n_frames * sizeof(unsigned));
    if (o > h->cap_gmc_scratch) {
      cudaFree(h->d_gmc_scratch); h->d_gmc_scratch = nullptr; h->cap_gmc_scratch = 0;
      CU_TRY(cudaMalloc(&h->d_gmc_scratch, o + o / 2));
      h->cap_gmc_scratch = o + o / 2;
    }
    unsigned char* base = h->d_gmc_scratch;
    tloam_gmc_args a;
    memset(&a, 0, sizeof(a));
    a.node = reinterpret_cast<const long long*>(base + o_node);
    a.node_O = h->d_pg_O; a.node_T = h->d_pg_T; a.n_opt = h->pg_opt_nodes;
    memcpy(a.delta_new.m, D, sizeof(D));
    a.O = h->d_gmc_O; a.P = h->d_gmc_P;
    a.M = reinterpret_cast<double*>(base + o_M);
    a.moved = reinterpret_cast<unsigned*>(base + o_moved);
    a.frames = st.frames; a.points = st.count;
    a.offsets = h->d_gmap_off; a.map = h->d_gmap;
    a.device = h->device; a.stream = h->stream;
    // pageable source: staged before the call returns
    CU_TRY(cudaMemcpyAsync(base + o_node, node, n_frames * sizeof(long long), cudaMemcpyHostToDevice, h->stream));
    int e = 0, launches = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.correct(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = gmc_status(h, e, "k_gmc_*")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaStreamSynchronize(h->stream));
  }
  memcpy(h->gmc_M, D, sizeof(D));
  h->gmc_M_identity = ident;
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_frame_poses(tloam_b200_handle* h, size_t first, size_t count, double* odom, double* current) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->gmc_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int rc = gmc_read(h, &st);
  if (rc != TLOAM_B200_OK) return rc;
  if (first > st.frames || count > st.frames - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (count && odom)
    CU_TRY(cudaMemcpyAsync(odom, h->d_gmc_O + 16 * first, count * 16 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (count && current)
    CU_TRY(cudaMemcpyAsync(current, h->d_gmc_P + 16 * first, count * 16 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Dynamic-point removal (the counters, images and tables here and in gmap_append_impl / gmap_grow / gmap_clear; the kernels
// in map_dynamic.cu, loaded from libtloam_b200_gmd.so when removal is enabled).
// ---------------------------------------------------------------------------------------------
void tloam_b200_global_map_dynamic_default_config(tloam_global_map_dynamic_config* c) {
  c->n_rows = 64; c->fov_up = 2.0; c->fov_down = -24.9; c->n_cols = 1024;   // an HDL-64E at the map's 1 m voxel
  c->window_rows = 1; c->window_cols = 2;
  c->margin_abs = 1.0; c->margin_rel = 0.02;
  c->min_range = 3.0; c->max_range = 60.0;
  c->min_through = 3;
}

static bool gmd_config_valid(const tloam_global_map_dynamic_config* c) {
  const auto fin = [](double v) { return std::isfinite(v); };
  if (c->n_rows < 1 || c->n_rows > 1024 || c->n_cols < 1 || c->n_cols > 16384) return false;
  if (!fin(c->fov_up) || !fin(c->fov_down) || !(c->fov_down < c->fov_up) || c->fov_down < -90.0 || c->fov_up > 90.0) return false;
  if (c->window_rows < 0 || c->window_rows >= c->n_rows || c->window_cols < 0 || 2 * c->window_cols + 1 > c->n_cols) return false;
  if (!fin(c->margin_abs) || !(c->margin_abs >= 0.0) || !fin(c->margin_rel) || !(c->margin_rel >= 0.0)) return false;
  if (!fin(c->min_range) || !fin(c->max_range) || !(c->min_range > 0.0) || !(c->min_range <= c->max_range)) return false;
  return c->min_through >= 1;
}

// the host tables: b_k = sin(lo + k (hi - lo) / n_rows) and Scan Context's sector boundaries (cos, sin of 2 pi k / n_cols);
// false when the row table is not non-decreasing (the row search needs it so)
static bool gmd_tables(const tloam_global_map_dynamic_config* cfg, std::vector<double>* out) {
  std::vector<double>& tab = *out;
  tab.assign((size_t)(cfg->n_rows + 1) + 2 * (size_t)(cfg->n_cols - 1), 0.0);
  const double lo = cfg->fov_down * (M_PI / 180.0), hi = cfg->fov_up * (M_PI / 180.0);
  for (int k = 0; k <= cfg->n_rows; ++k) tab[k] = std::sin(lo + k * (hi - lo) / cfg->n_rows);
  for (int k = 1; k <= cfg->n_rows; ++k)
    if (!(tab[k] >= tab[k - 1])) return false;
  double* dirs = tab.data() + (cfg->n_rows + 1);
  for (int k = 1; k < cfg->n_cols; ++k) {
    const double t = 2.0 * M_PI * k / cfg->n_cols;
    dirs[2 * (k - 1)] = std::cos(t);
    dirs[2 * (k - 1) + 1] = std::sin(t);
  }
  return true;
}

int tloam_b200_global_map_dynamic_enable(tloam_b200_handle* h, const tloam_global_map_dynamic_config* cfg) {
  if (!h || !cfg) return TLOAM_B200_ERR_INVALID_ARG;
  if (!gmd_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || h->gmap_calls != 0) return TLOAM_B200_ERR_NOT_READY;
  GmdLib lib;
  int rc = gmd_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  std::vector<double> tab;
  if (!gmd_tables(cfg, &tab)) return TLOAM_B200_ERR_INVALID_ARG;
  if (tab.size() > h->cap_gmd_bounds) {
    cudaFree(h->d_gmd_bounds); h->d_gmd_bounds = nullptr; h->cap_gmd_bounds = 0;
    CU_TRY(cudaMalloc(&h->d_gmd_bounds, tab.size() * sizeof(double)));
    h->cap_gmd_bounds = tab.size();
  }
  CU_TRY(cudaMemcpy(h->d_gmd_bounds, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice));
  const size_t pix = (size_t)cfg->n_rows * cfg->n_cols;
  if (pix > h->cap_gmd_image) {
    cudaFree(h->d_gmd_image); cudaFree(h->d_gmd_window); h->d_gmd_image = nullptr; h->d_gmd_window = nullptr;
    h->cap_gmd_image = 0;
    CU_TRY(cudaMalloc(&h->d_gmd_image, pix * sizeof(unsigned long long)));
    CU_TRY(cudaMalloc(&h->d_gmd_window, pix * sizeof(double)));
    h->cap_gmd_image = pix;
  }
  if (h->cap_gmd != h->cap_gmap) {
    cudaFree(h->d_gmd_through); cudaFree(h->d_gmd_hits); h->d_gmd_through = h->d_gmd_hits = nullptr; h->cap_gmd = 0;
    CU_TRY(cudaMalloc(&h->d_gmd_through, h->cap_gmap * sizeof(unsigned)));
    CU_TRY(cudaMalloc(&h->d_gmd_hits, h->cap_gmap * sizeof(unsigned)));
    h->cap_gmd = h->cap_gmap;
  }
  CU_TRY(cudaMemsetAsync(h->d_gmd_through, 0, h->cap_gmd * sizeof(unsigned), h->stream));
  CU_TRY(cudaMemsetAsync(h->d_gmd_hits, 0, h->cap_gmd * sizeof(unsigned), h->stream));
  h->gmd_cfg = *cfg;
  h->gmd_on = true;
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_votes_download(tloam_b200_handle* h, size_t first, size_t count, unsigned* through, unsigned* hits) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->gmd_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int rc = gmc_read(h, &st);
  if (rc != TLOAM_B200_OK) return rc;
  if (first > st.count || count > st.count - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (count && through)
    CU_TRY(cudaMemcpyAsync(through, h->d_gmd_through + first, count * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  if (count && hits)
    CU_TRY(cudaMemcpyAsync(hits, h->d_gmd_hits + first, count * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_static_download(tloam_b200_handle* h, double* xyz, double* intensity, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  *n = 0;
  if (!h->gmap_on || !h->gmd_on) return TLOAM_B200_ERR_NOT_READY;
  GmdLib lib;
  int rc = gmd_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  GMapState st;
  if ((rc = gmc_read(h, &st)) != TLOAM_B200_OK) return rc;   // the sticky flags stay for the next size / download call
  bool has = false;                                           // the map has the intensity channel (gmi_read's rule)
  if (h->gmi_used && st.count) {
    unsigned s0 = 0;
    CU_TRY(cudaMemcpyAsync(&s0, h->d_gmi_st, sizeof(s0), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    has = s0 != 0u;
  }
  const size_t count = st.count;
  const unsigned blocks = lib.blocks(count);
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t at = o; o += round_up(bytes, 256); return at; };
  const size_t o_blocks = take((size_t)blocks * sizeof(unsigned)), o_total = take(sizeof(unsigned long long));
  const size_t o_xyz = take(count * 3 * sizeof(double)), o_int = take(has ? count * sizeof(double) : 0);
  if (o > h->cap_gmd_scratch) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gmd_scratch); h->d_gmd_scratch = nullptr; h->cap_gmd_scratch = 0;
    CU_TRY(cudaMalloc(&h->d_gmd_scratch, o + o / 2));
    h->cap_gmd_scratch = o + o / 2;
  }
  unsigned char* base = h->d_gmd_scratch;
  tloam_gmd_static_args a;
  memset(&a, 0, sizeof(a));
  a.map = h->d_gmap; a.intensity = has ? h->d_gmi_map : nullptr;
  a.through = h->d_gmd_through; a.hits = h->d_gmd_hits;
  a.count = count; a.min_through = (unsigned)h->gmd_cfg.min_through;
  a.block_counts = reinterpret_cast<unsigned*>(base + o_blocks);
  a.total = reinterpret_cast<unsigned long long*>(base + o_total);
  a.out_xyz = reinterpret_cast<double*>(base + o_xyz);
  a.out_intensity = has ? reinterpret_cast<double*>(base + o_int) : nullptr;
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.compact(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = gmd_status(h, e, "k_gmd_count / k_gmd_scatter")) != TLOAM_B200_OK) return rc;
  unsigned long long total = 0;
  CU_TRY(cudaMemcpyAsync(&total, a.total, sizeof(total), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  *n = (size_t)total;
  if (capacity < *n || (!xyz && *n)) return TLOAM_B200_ERR_INVALID_ARG;
  if (*n) CU_TRY(cudaMemcpyAsync(xyz, a.out_xyz, *n * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (*n && intensity && has)
    CU_TRY(cudaMemcpyAsync(intensity, a.out_intensity, *n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Occupancy grid (the captures, the build's extent and the grid here and in gmap_append_impl / gmap_grow / gmap_clear; the
// kernels in occupancy.cu, loaded from libtloam_b200_occ.so when the grid is enabled).
// ---------------------------------------------------------------------------------------------
void tloam_b200_occupancy_default_config(tloam_occupancy_config* c) {
  c->resolution = 0.1; c->n_cols = 1024;   // an HDL-64E at 1.73 m
  c->z_lo = -1.2; c->z_hi = 0.5;
  c->min_range = 3.0; c->max_range = 30.0;
  c->free_margin = 0.1;
}

static bool occ_config_valid(const tloam_occupancy_config* c) {
  const auto fin = [](double v) { return std::isfinite(v); };
  if (!fin(c->resolution) || !(c->resolution > 0.0) || c->n_cols < 1 || c->n_cols > 4096) return false;
  if (!fin(c->z_lo) || !fin(c->z_hi) || !(c->z_lo < c->z_hi)) return false;
  if (!fin(c->min_range) || !fin(c->max_range) || !(c->min_range > 0.0) || !(c->min_range <= c->max_range)) return false;
  return fin(c->free_margin) && c->free_margin >= 0.0;
}

int tloam_b200_occupancy_enable(tloam_b200_handle* h, const tloam_occupancy_config* cfg) {
  if (!h || !cfg || !occ_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || h->gmap_calls != 0) return TLOAM_B200_ERR_NOT_READY;
  OccLib lib;
  int rc = occ_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  std::vector<double> dirs(2 * (size_t)(cfg->n_cols - 1) + 1, 0.0);   // Scan Context's boundaries, as gmd_tables
  for (int k = 1; k < cfg->n_cols; ++k) {
    const double t = 2.0 * M_PI * k / cfg->n_cols;
    dirs[2 * (k - 1)] = std::cos(t);
    dirs[2 * (k - 1) + 1] = std::sin(t);
  }
  if (dirs.size() > h->cap_occ_dirs) {
    cudaFree(h->d_occ_dirs); h->d_occ_dirs = nullptr; h->cap_occ_dirs = 0;
    CU_TRY(cudaMalloc(&h->d_occ_dirs, dirs.size() * sizeof(double)));
    h->cap_occ_dirs = dirs.size();
  }
  CU_TRY(cudaMemcpy(h->d_occ_dirs, dirs.data(), dirs.size() * sizeof(double), cudaMemcpyHostToDevice));
  cudaFree(h->d_occ_scans); cudaFree(h->d_occ_poses); h->d_occ_scans = h->d_occ_poses = nullptr; h->cap_occ = 0;
  CU_TRY(cudaMalloc(&h->d_occ_scans, h->cap_gmap_off * (size_t)cfg->n_cols * TLOAM_OCC_SLOT * sizeof(double)));
  CU_TRY(cudaMalloc(&h->d_occ_poses, h->cap_gmap_off * 16 * sizeof(double)));
  h->cap_occ = h->cap_gmap_off;
  if (!h->d_occ_small) CU_TRY(cudaMalloc(&h->d_occ_small, 128));
  h->occ_cfg = *cfg;
  h->occ_on = true;
  h->occ_built = false;
  return TLOAM_B200_OK;
}

int tloam_b200_occupancy_build(tloam_b200_handle* h, tloam_occupancy_info* info) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->occ_on) return TLOAM_B200_ERR_NOT_READY;
  OccLib lib;
  int rc = occ_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  GMapState st;
  if ((rc = gmc_read(h, &st)) != TLOAM_B200_OK) return rc;   // the sticky flags stay for the next size / download call
  h->occ_built = false;
  const tloam_occupancy_config& c = h->occ_cfg;
  tloam_occupancy_info out;
  memset(&out, 0, sizeof(out));
  out.resolution = c.resolution;
  out.frames = st.frames;
  if (st.frames) {
    tloam_occ_build_args a;
    memset(&a, 0, sizeof(a));
    a.p = occ_params(h);
    a.free_margin = c.free_margin; a.resolution = c.resolution;
    const double za = std::fabs(c.z_lo) > std::fabs(c.z_hi) ? std::fabs(c.z_lo) : std::fabs(c.z_hi);
    a.W = (c.max_range + za) + c.resolution;
    a.scans = h->d_occ_scans;
    a.poses = h->gmc_on ? h->d_gmc_P : h->d_occ_poses;
    a.n_frames = st.frames;
    a.extent = reinterpret_cast<double*>(h->d_occ_small);
    a.dropped = reinterpret_cast<unsigned long long*>(h->d_occ_small + 64);
    a.device = h->device; a.stream = h->stream;
    int e = 0, launches = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.extent(&a, &launches)));
    if ((rc = occ_status(h, e, "k_occ_extent")) != TLOAM_B200_OK) return rc;
    double ext[4];
    CU_TRY(cudaMemcpyAsync(ext, a.extent, sizeof(ext), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    const double r = c.resolution;
    const double ox = r * std::floor((ext[0] - a.W) / r), oy = r * std::floor((ext[1] - a.W) / r);
    const double fw = std::floor(((ext[2] + a.W) - ox) / r) + 1.0, fh = std::floor(((ext[3] + a.W) - oy) / r) + 1.0;
    if (!std::isfinite(ox) || !std::isfinite(oy) || !std::isfinite(fw) || !std::isfinite(fh) || !(fw >= 1.0) || !(fh >= 1.0) ||
        fw > (double)(1u << 28) || fh > (double)(1u << 28) || fw * fh > (double)(1u << 28))
      return TLOAM_B200_ERR_VOXEL_RANGE;
    a.origin_x = ox; a.origin_y = oy;
    a.width = (unsigned)fw; a.height = (unsigned)fh;
    a.nwin = (int)std::ceil(2.0 * a.W / r) + 3;          // any cell with |c - t| <= W lies in these candidates
    const size_t cells = (size_t)a.width * a.height;
    if (cells > h->cap_occ_grid) {
      cudaFree(h->d_occ_grid); h->d_occ_grid = nullptr; h->cap_occ_grid = 0;
      const size_t cap = cells + cells / 2;
      CU_TRY(cudaMalloc(&h->d_occ_grid, cap * (2 * sizeof(unsigned) + 1)));
      h->cap_occ_grid = cap;
    }
    a.occupied = reinterpret_cast<unsigned*>(h->d_occ_grid);
    a.free_count = a.occupied + h->cap_occ_grid;
    a.cells = reinterpret_cast<signed char*>(a.free_count + h->cap_occ_grid);
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.rasterise(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = occ_status(h, e, "k_occ_free / _hits / _value")) != TLOAM_B200_OK) return rc;
    unsigned long long dropped = 0;
    CU_TRY(cudaMemcpyAsync(&dropped, a.dropped, sizeof(dropped), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    out.origin_x = ox; out.origin_y = oy; out.width = a.width; out.height = a.height;
    out.dropped = dropped;
    out.cell_tests = (unsigned long long)st.frames * (unsigned long long)a.nwin * (unsigned long long)a.nwin;
  }
  h->occ_info = out;
  h->occ_built = true;
  if (info) *info = out;
  return TLOAM_B200_OK;
}

int tloam_b200_occupancy_download(tloam_b200_handle* h, signed char* cells, unsigned* occupied, unsigned* free_count,
                                  size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->occ_on || !h->occ_built) return TLOAM_B200_ERR_NOT_READY;
  const size_t n = h->occ_info.width * h->occ_info.height;
  if (capacity < n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (n) {
    const unsigned* occ = reinterpret_cast<const unsigned*>(h->d_occ_grid);
    const unsigned* fr = occ + h->cap_occ_grid;
    const signed char* v = reinterpret_cast<const signed char*>(fr + h->cap_occ_grid);
    if (cells) CU_TRY(cudaMemcpyAsync(cells, v, n, cudaMemcpyDeviceToHost, h->stream));
    if (occupied) CU_TRY(cudaMemcpyAsync(occupied, occ, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    if (free_count) CU_TRY(cudaMemcpyAsync(free_count, fr, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  }
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_occupancy_scans_download(tloam_b200_handle* h, size_t first, size_t count, double* scans, double* poses) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->occ_on) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int rc = gmc_read(h, &st);
  if (rc != TLOAM_B200_OK) return rc;
  if (first > st.frames || count > st.frames - first) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t per = (size_t)h->occ_cfg.n_cols * TLOAM_OCC_SLOT;
  if (count && scans)
    CU_TRY(cudaMemcpyAsync(scans, h->d_occ_scans + per * first, count * per * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (count && poses)
    CU_TRY(cudaMemcpyAsync(poses, h->d_occ_poses + 16 * first, count * 16 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Distance field and costmap (the checks, the cost table and the buffers here; the kernels in distance.cu, loaded from
// libtloam_b200_dist.so by the first distance call, so that the kernels of this library keep their SASS).
// ---------------------------------------------------------------------------------------------
struct DistLib { tloam_dist_build_fn build = nullptr; tloam_dist_query_fn query = nullptr; };
static std::mutex g_dist_mu;
static DistLib g_dist;

static int dist_load(tloam_b200_handle* h, DistLib* out) {
  std::lock_guard<std::mutex> lk(g_dist_mu);
  if (!g_dist.build) {
    const std::string path = sibling_path("libtloam_b200_dist.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    DistLib l;
    if (so) {
      l.build = reinterpret_cast<tloam_dist_build_fn>(dlsym(so, "tloam_dist_build"));
      l.query = reinterpret_cast<tloam_dist_query_fn>(dlsym(so, "tloam_dist_query"));
    }
    if (!l.build || !l.query) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "distance field: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_dist = l;
  }
  *out = g_dist;
  return TLOAM_B200_OK;
}

static int dist_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "distance field: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

void tloam_b200_distance_default_config(tloam_distance_config* c) {
  c->inscribed_radius = 0.9;               // half of a 1.8 m-wide car; robot parameters, not calibrated
  c->inflation_radius = 3.0;
  c->cost_scaling_factor = 3.0;            // nav2's inflation-layer default
}

static bool dist_config_valid(const tloam_distance_config* c) {
  const auto fin = [](double v) { return std::isfinite(v); };
  if (!fin(c->inscribed_radius) || !fin(c->inflation_radius) || !fin(c->cost_scaling_factor)) return false;
  return c->inscribed_radius >= 0.0 && c->inscribed_radius <= c->inflation_radius && c->cost_scaling_factor >= 0.0;
}

// R_c^2 of cfg at this resolution; false when R_c > 4096
static bool dist_r2(const tloam_distance_config* c, double resolution, unsigned* r2) {
  const double rc = std::ceil(c->inflation_radius / resolution);
  if (!(rc <= 4096.0)) return false;
  *r2 = (unsigned)rc * (unsigned)rc;
  return true;
}

// the build of a grid whose cells are on the device at `cells` (width x height, checked); info may be null
static int dist_run(tloam_b200_handle* h, const DistLib& lib, const tloam_distance_config* cfg, const signed char* cells,
                    bool upload_from_host, size_t width, size_t height, double ox, double oy, double res, unsigned r2,
                    tloam_distance_info* info) {
  h->dist_built = false;
  const size_t n = width * height;
  tloam_distance_info out;
  memset(&out, 0, sizeof(out));
  out.origin_x = ox; out.origin_y = oy; out.resolution = res; out.width = width; out.height = height;
  CU_TRY(cudaSetDevice(h->device));
  if (n) {
    if (n > h->cap_dist) {
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_dist); h->d_dist = nullptr; h->cap_dist = 0;
      CU_TRY(cudaMalloc(&h->d_dist, n * 19));
      h->cap_dist = n;
    }
    const size_t nb = width * ((height + TLOAM_DIST_BAND - 1) / TLOAM_DIST_BAND);
    if (nb > h->cap_dist_bands) {
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_dist_bands); h->d_dist_bands = nullptr; h->cap_dist_bands = 0;
      CU_TRY(cudaMalloc(&h->d_dist_bands, nb * 4 * sizeof(unsigned)));
      h->cap_dist_bands = nb;
    }
    if ((size_t)r2 + 1 > h->cap_dist_table) {
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_dist_table); h->d_dist_table = nullptr; h->cap_dist_table = 0;
      CU_TRY(cudaMalloc(&h->d_dist_table, (size_t)r2 + 1));
      h->cap_dist_table = (size_t)r2 + 1;
    }
    if (!h->d_dist_small) CU_TRY(cudaMalloc(&h->d_dist_small, 64));
    // c by sq: InflationLayer::computeCost of the distance sqrt(sq) in cells
    std::vector<unsigned char> table((size_t)r2 + 1);
    table[0] = 254;
    for (unsigned s = 1; s <= r2; ++s) {
      const double dist = std::sqrt((double)s);
      table[s] = dist * res <= cfg->inscribed_radius ? (unsigned char)253
               : (unsigned char)(252.0 * std::exp(-cfg->cost_scaling_factor * (dist * res - cfg->inscribed_radius)));
    }
    CU_TRY(cudaMemcpyAsync(h->d_dist_table, table.data(), table.size(), cudaMemcpyHostToDevice, h->stream));
    const size_t cap = h->cap_dist;
    tloam_dist_build_args a;
    memset(&a, 0, sizeof(a));
    a.sq = reinterpret_cast<unsigned*>(h->d_dist);
    a.sd = reinterpret_cast<float*>(h->d_dist + 4 * cap);
    a.g = reinterpret_cast<unsigned*>(h->d_dist + 8 * cap);
    a.stack = reinterpret_cast<unsigned short*>(h->d_dist + 12 * cap);
    signed char* grid = reinterpret_cast<signed char*>(h->d_dist + 16 * cap);
    a.costs = h->d_dist + 17 * cap;
    a.values = reinterpret_cast<signed char*>(h->d_dist + 18 * cap);
    if (upload_from_host) CU_TRY(cudaMemcpyAsync(grid, cells, n, cudaMemcpyHostToDevice, h->stream));
    a.cells = upload_from_host ? grid : cells;   // the kernels read the source only during the build
    a.width = (unsigned)width; a.height = (unsigned)height; a.resolution = res;
    a.bands = h->d_dist_bands;
    a.table = h->d_dist_table; a.r2 = r2;
    a.obstacles = h->d_dist_small;
    a.device = h->device; a.stream = h->stream;
    int e = 0, launches = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.build(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    int rc = dist_status(h, e, "k_dist_bands / _cols / _rows / _cost");
    if (rc != TLOAM_B200_OK) return rc;
    unsigned long long obstacles = 0;
    CU_TRY(cudaMemcpyAsync(&obstacles, h->d_dist_small, sizeof(obstacles), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    out.obstacles = (size_t)obstacles;
  }
  h->dist_info = out;
  h->dist_built = true;
  ++h->dist_serial;
  if (info) *info = out;
  return TLOAM_B200_OK;
}

static bool dist_shape_ok(size_t width, size_t height) {   // (width - 1)^2 + (height - 1)^2 < 2^32 - 1
  if (width == 0 || height == 0) return true;
  if (width > 65537 || height > 65537) return false;
  const unsigned long long a = width - 1, b = height - 1;
  return a * a + b * b < 0xFFFFFFFFull;
}

int tloam_b200_distance_build(tloam_b200_handle* h, const tloam_distance_config* cfg, tloam_distance_info* info) {
  if (!h || !cfg || !dist_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || !h->occ_on || !h->occ_built) return TLOAM_B200_ERR_NOT_READY;
  const tloam_occupancy_info& g = h->occ_info;
  unsigned r2 = 0;
  if (!dist_r2(cfg, g.resolution, &r2)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!dist_shape_ok(g.width, g.height)) return TLOAM_B200_ERR_VOXEL_RANGE;
  DistLib lib;
  int rc = dist_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  const unsigned* occ = reinterpret_cast<const unsigned*>(h->d_occ_grid);
  const signed char* values = reinterpret_cast<const signed char*>(occ + 2 * h->cap_occ_grid);
  return dist_run(h, lib, cfg, values, false, g.width, g.height, g.origin_x, g.origin_y, g.resolution, r2, info);
}

int tloam_b200_distance_build_grid(tloam_b200_handle* h, const tloam_distance_config* cfg, const signed char* cells,
                                   size_t width, size_t height, double origin_x, double origin_y, double resolution,
                                   tloam_distance_info* info) {
  if (!h || !cfg || !dist_config_valid(cfg) || !cells || width == 0 || height == 0 || width > (1u << 28) ||
      height > (1u << 28) || width * height > (1u << 28) || !std::isfinite(origin_x) || !std::isfinite(origin_y) ||
      !std::isfinite(resolution) || !(resolution > 0.0))
    return TLOAM_B200_ERR_INVALID_ARG;
  unsigned r2 = 0;
  if (!dist_r2(cfg, resolution, &r2)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!dist_shape_ok(width, height)) return TLOAM_B200_ERR_VOXEL_RANGE;
  DistLib lib;
  int rc = dist_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  return dist_run(h, lib, cfg, cells, true, width, height, origin_x, origin_y, resolution, r2, info);
}

int tloam_b200_distance_download(tloam_b200_handle* h, float* sd, unsigned* sq, unsigned char* costs, signed char* values,
                                 size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->dist_built) return TLOAM_B200_ERR_NOT_READY;
  const size_t n = h->dist_info.width * h->dist_info.height;
  if (capacity < n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (n) {
    const size_t cap = h->cap_dist;
    if (sq) CU_TRY(cudaMemcpyAsync(sq, h->d_dist, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    if (sd) CU_TRY(cudaMemcpyAsync(sd, h->d_dist + 4 * cap, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    if (costs) CU_TRY(cudaMemcpyAsync(costs, h->d_dist + 17 * cap, n, cudaMemcpyDeviceToHost, h->stream));
    if (values) CU_TRY(cudaMemcpyAsync(values, h->d_dist + 18 * cap, n, cudaMemcpyDeviceToHost, h->stream));
  }
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_distance_query(tloam_b200_handle* h, const double* xy, size_t n, double* distance, double* gradient) {
  if (!h || (n && !xy)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->dist_built) return TLOAM_B200_ERR_NOT_READY;
  DistLib lib;
  int rc = dist_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  if (n) {
    if (n > h->cap_dist_q) {
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_dist_q); h->d_dist_q = nullptr; h->cap_dist_q = 0;
      CU_TRY(cudaMalloc(&h->d_dist_q, n * 5 * sizeof(double)));
      h->cap_dist_q = n;
    }
    const tloam_distance_info& f = h->dist_info;
    const size_t cells = f.width * f.height;
    tloam_dist_query_args a;
    memset(&a, 0, sizeof(a));
    a.sd = reinterpret_cast<const float*>(h->d_dist + 4 * h->cap_dist);
    a.width = (unsigned)f.width; a.height = (unsigned)f.height;
    a.origin_x = f.origin_x; a.origin_y = f.origin_y; a.resolution = f.resolution;
    a.finite = f.obstacles > 0 && f.obstacles < cells;          // else every sd is +inf or -inf
    a.xy = h->d_dist_q; a.n = n;
    a.distance = h->d_dist_q + 2 * n; a.gradient = h->d_dist_q + 3 * n;
    a.device = h->device; a.stream = h->stream;
    CU_TRY(cudaMemcpyAsync(h->d_dist_q, xy, n * 2 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
    int e = 0, launches = 0;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.query(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = dist_status(h, e, "k_dist_query")) != TLOAM_B200_OK) return rc;
    if (distance) CU_TRY(cudaMemcpyAsync(distance, a.distance, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (gradient) CU_TRY(cudaMemcpyAsync(gradient, a.gradient, n * 2 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  }
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Path planning (the checks, the host loop over rounds and the buffers here; the kernels in plan.cu, loaded from
// libtloam_b200_plan.so by the first plan call, so that the kernels of this library keep their SASS).
// ---------------------------------------------------------------------------------------------
struct PlanLib {
  tloam_plan_init_fn init = nullptr; tloam_plan_rounds_fn rounds = nullptr; tloam_plan_count_fn count = nullptr;
  tloam_plan_path_fn length = nullptr; tloam_plan_path_fn walk = nullptr;
};
static std::mutex g_plan_mu;
static PlanLib g_plan;

static int plan_load(tloam_b200_handle* h, PlanLib* out) {
  std::lock_guard<std::mutex> lk(g_plan_mu);
  if (!g_plan.init) {
    const std::string path = sibling_path("libtloam_b200_plan.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    PlanLib l;
    if (so) {
      l.init = reinterpret_cast<tloam_plan_init_fn>(dlsym(so, "tloam_plan_init"));
      l.rounds = reinterpret_cast<tloam_plan_rounds_fn>(dlsym(so, "tloam_plan_rounds"));
      l.count = reinterpret_cast<tloam_plan_count_fn>(dlsym(so, "tloam_plan_count"));
      l.length = reinterpret_cast<tloam_plan_path_fn>(dlsym(so, "tloam_plan_length"));
      l.walk = reinterpret_cast<tloam_plan_path_fn>(dlsym(so, "tloam_plan_walk"));
    }
    if (!l.init || !l.rounds || !l.count || !l.length || !l.walk) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "path planning: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_plan = l;
  }
  *out = g_plan;
  return TLOAM_B200_OK;
}

static int plan_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "path planning: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

void tloam_b200_plan_default_config(tloam_plan_config* c) {
  c->neutral_cost = 50;                    // global_planner's defaults
  c->cost_factor = 3;
  c->allow_unknown = 1;
}

static bool plan_config_valid(const tloam_plan_config* c) {
  return c->neutral_cost >= 1 && (unsigned long long)c->neutral_cost + 252ull * c->cost_factor <= 65535ull &&
         (c->allow_unknown == 0 || c->allow_unknown == 1);
}

// the cell of (x, y) in the last distance field: (floor((x - origin_x) / resolution), likewise for y); false when x or y
// is not finite or the cell lies outside the grid
static bool plan_cell(const tloam_distance_info& f, double x, double y, long long* i, long long* j) {
  if (!std::isfinite(x) || !std::isfinite(y)) return false;
  const double u = std::floor((x - f.origin_x) / f.resolution), v = std::floor((y - f.origin_y) / f.resolution);
  if (!(u >= 0.0 && u < (double)f.width && v >= 0.0 && v < (double)f.height)) return false;
  *i = (long long)u; *j = (long long)v;
  return true;
}

int tloam_b200_plan_build(tloam_b200_handle* h, const tloam_plan_config* cfg, double goal_x, double goal_y,
                          tloam_plan_info* info) {
  if (!h || !cfg || !plan_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->dist_built) return TLOAM_B200_ERR_NOT_READY;
  const tloam_distance_info f = h->dist_info;
  long long gi = 0, gj = 0;
  if (!plan_cell(f, goal_x, goal_y, &gi, &gj)) return TLOAM_B200_ERR_INVALID_ARG;
  PlanLib lib;
  int rc = plan_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  const unsigned char* costs = h->d_dist + 17 * h->cap_dist;
  const size_t n = f.width * f.height;
  unsigned char code = 0;
  CU_TRY(cudaMemcpyAsync(&code, costs + (size_t)gj * f.width + (size_t)gi, 1, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!(code <= 252 || (code == 255 && cfg->allow_unknown))) return TLOAM_B200_ERR_INVALID_ARG;   // the goal is impassable
  h->plan_built = false;
  h->plan_paths_kept = false;
  if (n > h->cap_plan) {
    cudaFree(h->d_plan); h->d_plan = nullptr; h->cap_plan = 0;
    CU_TRY(cudaMalloc(&h->d_plan, n * 10));
    h->cap_plan = n;
  }
  const size_t ntiles = ((f.width + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE) * ((f.height + TLOAM_PLAN_TILE - 1) / TLOAM_PLAN_TILE);
  if (ntiles > h->cap_plan_tiles) {
    cudaFree(h->d_plan_tiles); h->d_plan_tiles = nullptr; h->cap_plan_tiles = 0;
    CU_TRY(cudaMalloc(&h->d_plan_tiles, ntiles * 3 * sizeof(unsigned)));
    h->cap_plan_tiles = ntiles;
  }
  if (!h->d_plan_state) CU_TRY(cudaMalloc(&h->d_plan_state, sizeof(tloam_plan_state)));
  tloam_plan_args a;
  memset(&a, 0, sizeof(a));
  a.costs = costs;
  a.width = (unsigned)f.width; a.height = (unsigned)f.height;
  a.neutral_cost = cfg->neutral_cost; a.cost_factor = cfg->cost_factor; a.allow_unknown = cfg->allow_unknown;
  a.goal_i = (unsigned)gi; a.goal_j = (unsigned)gj;
  a.P = reinterpret_cast<unsigned long long*>(h->d_plan);
  a.t = reinterpret_cast<unsigned short*>(h->d_plan + 8 * h->cap_plan);
  a.stamp = h->d_plan_tiles;
  a.list = h->d_plan_tiles + ntiles;
  a.state = h->d_plan_state;
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.init(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = plan_status(h, e, "k_plan_init")) != TLOAM_B200_OK) return rc;
  // rounds in batches; after each, the next round's work count decides whether to go on (an empty round exits at once)
  const unsigned kBatch = 32;
  tloam_plan_state st;
  for (unsigned first = 1;; first += kBatch) {
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.rounds(&a, first, kBatch, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = plan_status(h, e, "k_plan_round")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaMemcpyAsync(&st, h->d_plan_state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    if (st.count[(first + kBatch) % 3] == 0) break;
  }
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.count(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = plan_status(h, e, "k_plan_count")) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(&st, h->d_plan_state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  tloam_plan_info out;
  memset(&out, 0, sizeof(out));
  out.origin_x = f.origin_x; out.origin_y = f.origin_y; out.resolution = f.resolution;
  out.width = f.width; out.height = f.height;
  out.goal_i = (size_t)gi; out.goal_j = (size_t)gj;
  out.reachable = (size_t)st.reachable;
  out.rounds = st.rounds; out.tiles = st.tiles;
  h->plan_info = out;
  h->plan_built = true;
  h->plan_serial = h->dist_serial;
  h->plan_cfg = *cfg;
  if (info) *info = out;
  return TLOAM_B200_OK;
}

int tloam_b200_plan_download(tloam_b200_handle* h, unsigned long long* potential, size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->plan_built) return TLOAM_B200_ERR_NOT_READY;
  const size_t n = h->plan_info.width * h->plan_info.height;
  if (capacity < n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (potential) CU_TRY(cudaMemcpyAsync(potential, h->d_plan, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_plan_paths(tloam_b200_handle* h, const double* starts_xy, size_t n, size_t* offsets, int* statuses,
                          unsigned long long* costs) {
  if (!h || (n && !starts_xy) || n > (size_t(1) << 24)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->plan_built) return TLOAM_B200_ERR_NOT_READY;
  PlanLib lib;
  int rc = plan_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  h->plan_paths_kept = false;
  const tloam_plan_info& f = h->plan_info;
  tloam_distance_info g;
  memset(&g, 0, sizeof(g));
  g.origin_x = f.origin_x; g.origin_y = f.origin_y; g.resolution = f.resolution; g.width = f.width; g.height = f.height;
  // per start: the cell (2 int), the status (int), the length (unsigned), the cost and the offset (8 B each)
  if (n > h->cap_plan_q) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_plan_q); h->d_plan_q = nullptr; h->cap_plan_q = 0;
    CU_TRY(cudaMalloc(&h->d_plan_q, n * 32));
    h->cap_plan_q = n;
  }
  std::vector<int> start(2 * n);
  for (size_t s = 0; s < n; ++s) {
    long long i = -1, j = -1;
    if (!plan_cell(g, starts_xy[2 * s], starts_xy[2 * s + 1], &i, &j)) i = j = -1;
    start[2 * s] = (int)i; start[2 * s + 1] = (int)j;
  }
  const size_t cap = h->cap_plan_q;
  tloam_plan_path_args a;
  memset(&a, 0, sizeof(a));
  a.P = reinterpret_cast<const unsigned long long*>(h->d_plan);
  a.t = reinterpret_cast<const unsigned short*>(h->d_plan + 8 * h->cap_plan);
  a.width = (unsigned)f.width; a.height = (unsigned)f.height;
  a.n = (unsigned)n;
  unsigned long long* cost = reinterpret_cast<unsigned long long*>(h->d_plan_q);
  unsigned long long* offset = cost + cap;
  int* cell = reinterpret_cast<int*>(offset + cap);
  a.cost = cost; a.offset = offset; a.start = cell;
  a.status = cell + 2 * cap;
  a.length = reinterpret_cast<unsigned*>(cell + 3 * cap);
  a.device = h->device; a.stream = h->stream;
  std::vector<int> status(n);
  std::vector<unsigned long long> cost_h(n);
  std::vector<unsigned> length(n);
  std::vector<unsigned long long> offset_h(n + 1, 0);
  int e = 0, launches = 0;
  if (n) {
    CU_TRY(cudaMemcpyAsync(cell, start.data(), 2 * n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.length(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = plan_status(h, e, "k_plan_length")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaMemcpyAsync(status.data(), a.status, n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaMemcpyAsync(cost_h.data(), cost, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaMemcpyAsync(length.data(), a.length, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    for (size_t s = 0; s < n; ++s) offset_h[s + 1] = offset_h[s] + length[s];
    const size_t total = (size_t)offset_h[n];
    if (total > h->cap_plan_cells) {
      cudaFree(h->d_plan_cells); h->d_plan_cells = nullptr; h->cap_plan_cells = 0;
      CU_TRY(cudaMalloc(&h->d_plan_cells, total * 2 * sizeof(int)));
      h->cap_plan_cells = total;
    }
    a.cells = h->d_plan_cells;
    CU_TRY(cudaMemcpyAsync(offset, offset_h.data(), n * sizeof(unsigned long long), cudaMemcpyHostToDevice, h->stream));
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.walk(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = plan_status(h, e, "k_plan_walk")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaStreamSynchronize(h->stream));
  }
  for (size_t s = 0; s <= n; ++s)
    if (offsets) offsets[s] = (size_t)offset_h[s];
  if (statuses) std::copy(status.begin(), status.end(), statuses);
  if (costs) std::copy(cost_h.begin(), cost_h.end(), costs);
  h->plan_path_total = (size_t)offset_h[n];
  h->plan_paths_kept = true;
  return TLOAM_B200_OK;
}

int tloam_b200_plan_path_cells(tloam_b200_handle* h, int* ij, double* xy, size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->plan_paths_kept) return TLOAM_B200_ERR_NOT_READY;
  const size_t m = h->plan_path_total;
  if (capacity < m) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  std::vector<int> cells(xy ? 2 * m : 0);
  int* dst = ij ? ij : cells.data();
  if (m && (ij || xy)) CU_TRY(cudaMemcpyAsync(dst, h->d_plan_cells, m * 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (xy) {
    const tloam_plan_info& f = h->plan_info;
    for (size_t k = 0; k < 2 * m; ++k)        // the centre, each operation rounded on its own
      xy[k] = (k % 2 ? f.origin_y : f.origin_x) + ((double)dst[k] + 0.5) * f.resolution;
  }
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Frontiers (the checks, the buffers, the cost, the filter and the order here; the kernels in frontier.cu, loaded from
// libtloam_b200_frontier.so by the first frontier call, so that the kernels of this library keep their SASS).
// ---------------------------------------------------------------------------------------------
struct FrontierLib {
  tloam_fr_fn label = nullptr; tloam_fr_fn group = nullptr;
  tloam_fr_sort_bytes_fn sort_bytes = nullptr; tloam_fr_sort_layout_fn sort_layout = nullptr;
};
static std::mutex g_fr_mu;
static FrontierLib g_fr;

static int fr_load(tloam_b200_handle* h, FrontierLib* out) {
  std::lock_guard<std::mutex> lk(g_fr_mu);
  if (!g_fr.label) {
    const std::string path = sibling_path("libtloam_b200_frontier.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    FrontierLib l;
    if (so) {
      l.label = reinterpret_cast<tloam_fr_fn>(dlsym(so, "tloam_fr_label"));
      l.group = reinterpret_cast<tloam_fr_fn>(dlsym(so, "tloam_fr_group"));
      l.sort_bytes = reinterpret_cast<tloam_fr_sort_bytes_fn>(dlsym(so, "tloam_fr_sort_bytes"));
      l.sort_layout = reinterpret_cast<tloam_fr_sort_layout_fn>(dlsym(so, "tloam_fr_sort_layout"));
    }
    if (!l.label || !l.group || !l.sort_bytes || !l.sort_layout) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "frontiers: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_fr = l;
  }
  *out = g_fr;
  return TLOAM_B200_OK;
}

static int fr_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "frontiers: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

void tloam_b200_frontier_default_config(tloam_frontier_config* c) {
  c->free_max = 252;                       // every cell a plan can enter
  c->min_frontier_size = 0.5;              // explore_lite's defaults; robot parameters, not calibrated
  c->potential_scale = 3.0;
  c->gain_scale = 1.0;
}

static bool fr_config_valid(const tloam_frontier_config* c) {
  const auto ok = [](double v) { return std::isfinite(v) && v >= 0.0; };
  return c->free_max <= 252 && ok(c->min_frontier_size) && ok(c->potential_scale) && ok(c->gain_scale);
}

int tloam_b200_frontier_search(tloam_b200_handle* h, const tloam_frontier_config* cfg, tloam_frontier_info* info) {
  if (!h || !cfg || !fr_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->dist_built || !h->plan_built || h->plan_serial != h->dist_serial) return TLOAM_B200_ERR_NOT_READY;
  FrontierLib lib;
  int rc = fr_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  h->fr_kept = false;
  const tloam_plan_info& f = h->plan_info;
  const size_t n = f.width * f.height;     // >= 1: a plan has a goal cell
  const size_t ntiles = ((f.width + TLOAM_FR_TILE - 1) / TLOAM_FR_TILE) * ((f.height + TLOAM_FR_TILE - 1) / TLOAM_FR_TILE);
  if (n > h->cap_fr_labels) {
    cudaFree(h->d_fr_labels); h->d_fr_labels = nullptr; h->cap_fr_labels = 0;
    CU_TRY(cudaMalloc(&h->d_fr_labels, n * sizeof(unsigned)));
    h->cap_fr_labels = n;
  }
  if (ntiles > h->cap_fr_tiles) {
    cudaFree(h->d_fr_tiles); h->d_fr_tiles = nullptr; h->cap_fr_tiles = 0;
    CU_TRY(cudaMalloc(&h->d_fr_tiles, ntiles));
    h->cap_fr_tiles = ntiles;
  }
  const size_t small_state = TLOAM_FR_BLOCKS * sizeof(unsigned);
  if (!h->d_fr_small) CU_TRY(cudaMalloc(&h->d_fr_small, small_state + sizeof(tloam_fr_state)));
  tloam_fr_args a;
  memset(&a, 0, sizeof(a));
  a.costs = h->d_dist + 17 * h->cap_dist;
  a.P = reinterpret_cast<const unsigned long long*>(h->d_plan);
  a.width = (unsigned)f.width; a.height = (unsigned)f.height;
  a.free_max = cfg->free_max;
  a.labels = h->d_fr_labels;
  a.tile_any = h->d_fr_tiles;
  a.block_counts = reinterpret_cast<unsigned*>(h->d_fr_small);
  a.state = reinterpret_cast<tloam_fr_state*>(h->d_fr_small + small_state);
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.label(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = fr_status(h, e, "k_fr_tile / _border / _flatten")) != TLOAM_B200_OK) return rc;
  tloam_fr_state st;
  CU_TRY(cudaMemcpyAsync(&st, a.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  const size_t m = (size_t)st.cells;
  size_t components = 0;
  std::vector<tloam_fr_stat> stats;
  if (m) {
    if (m > h->cap_fr_sort) {
      cudaFree(h->d_fr_sort); h->d_fr_sort = nullptr; h->cap_fr_sort = 0;
      CU_TRY(cudaMalloc(&h->d_fr_sort, lib.sort_bytes(m)));
      h->cap_fr_sort = m;
    }
    lib.sort_layout(h->d_fr_sort, h->cap_fr_sort, &a);
    a.cells = m;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.group(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = fr_status(h, e, "k_fr_compact / radix sort / heads / k_fr_stats")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaMemcpyAsync(&st, a.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    components = (size_t)st.gmm.n_vox;
    stats.resize(components);
    CU_TRY(cudaMemcpyAsync(stats.data(), a.stats, components * sizeof(tloam_fr_stat), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
  }
  // the cost of each kept frontier in FP64, each operation rounded on its own; then the order
  const double res = f.resolution;
  const double per_m = 70.0 * (double)h->plan_cfg.neutral_cost;
  std::vector<tloam_frontier> kept;
  for (size_t j = 0; j < components; ++j) {
    const tloam_fr_stat& s = stats[j];
    const double size_m = (double)s.n * res;
    if (!(size_m >= cfg->min_frontier_size)) continue;
    tloam_frontier o;
    memset(&o, 0, sizeof(o));
    o.id = (unsigned)j;
    o.size = s.n;
    o.sum_i = s.sum_i; o.sum_j = s.sum_j;
    o.min_i = s.min_i; o.min_j = s.min_j; o.max_i = s.max_i; o.max_j = s.max_j;
    o.centroid_x = f.origin_x + ((double)s.sum_i / (double)s.n + 0.5) * res;
    o.centroid_y = f.origin_y + ((double)s.sum_j / (double)s.n + 0.5) * res;
    o.approach_i = s.approach % f.width; o.approach_j = s.approach / f.width;
    o.approach_x = f.origin_x + ((double)o.approach_i + 0.5) * res;
    o.approach_y = f.origin_y + ((double)o.approach_j + 0.5) * res;
    o.approach_potential = s.approach_p;
    o.status = s.approach_p == TLOAM_PLAN_INF ? 1 : 0;
    if (o.status == 0) {
      o.distance = ((double)s.approach_p / per_m) * res;
      const double pot = cfg->potential_scale * o.distance;
      const double gain = cfg->gain_scale * size_m;
      o.cost = pot - gain;
    } else {
      o.distance = o.cost = HUGE_VAL;
    }
    kept.push_back(o);
  }
  // reachable by (cost, id), a NaN cost after every number; then unreachable by id
  std::stable_sort(kept.begin(), kept.end(), [](const tloam_frontier& x, const tloam_frontier& y) {
    if (x.status != y.status) return x.status < y.status;
    if (x.status == 1) return false;
    const bool xn = std::isnan(x.cost), yn = std::isnan(y.cost);
    if (xn != yn) return yn;
    return !xn && x.cost < y.cost;
  });
  tloam_frontier_info out;
  memset(&out, 0, sizeof(out));
  out.origin_x = f.origin_x; out.origin_y = f.origin_y; out.resolution = res;
  out.width = f.width; out.height = f.height;
  out.goal_i = f.goal_i; out.goal_j = f.goal_j;
  out.cells = m; out.components = components; out.kept = kept.size();
  for (const tloam_frontier& o : kept) out.reachable += o.status == 0 ? 1 : 0;
  h->fr_ranked.swap(kept);
  h->fr_info = out;
  h->fr_sorted = (unsigned)(tloam_fr_passes(n) & 1);
  h->fr_kept = true;
  if (info) *info = out;
  return TLOAM_B200_OK;
}

int tloam_b200_frontier_download(tloam_b200_handle* h, tloam_frontier* out, size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->fr_kept) return TLOAM_B200_ERR_NOT_READY;
  if (capacity < h->fr_ranked.size()) return TLOAM_B200_ERR_INVALID_ARG;
  if (out) std::copy(h->fr_ranked.begin(), h->fr_ranked.end(), out);
  return TLOAM_B200_OK;
}

int tloam_b200_frontier_cells(tloam_b200_handle* h, size_t* offsets, int* ij, double* xy, size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->fr_kept) return TLOAM_B200_ERR_NOT_READY;
  const std::vector<tloam_frontier>& R = h->fr_ranked;
  std::vector<size_t> off(R.size() + 1, 0);
  for (size_t k = 0; k < R.size(); ++k) off[k + 1] = off[k] + R[k].size;
  if (capacity < off.back()) return TLOAM_B200_ERR_INVALID_ARG;
  if (offsets) std::copy(off.begin(), off.end(), offsets);
  if (off.back() && (ij || xy)) {
    // the sorted cells and the heads of the last search, each kept frontier's run copied in rank order
    const tloam_frontier_info& f = h->fr_info;
    tloam_fr_args a;
    memset(&a, 0, sizeof(a));
    FrontierLib lib;
    int rc = fr_load(h, &lib);
    if (rc != TLOAM_B200_OK) return rc;
    lib.sort_layout(h->d_fr_sort, h->cap_fr_sort, &a);
    CU_TRY(cudaSetDevice(h->device));
    std::vector<unsigned> start(f.components + 1), rows(f.cells);
    CU_TRY(cudaMemcpyAsync(start.data(), a.start, start.size() * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaMemcpyAsync(rows.data(), a.row[h->fr_sorted], rows.size() * sizeof(unsigned), cudaMemcpyDeviceToHost,
                           h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    for (size_t k = 0; k < R.size(); ++k) {
      const unsigned lo = start[R[k].id];
      for (size_t q = 0; q < R[k].size; ++q) {
        const unsigned c = rows[lo + q];
        const size_t i = c % f.width, j = c / f.width, o = 2 * (off[k] + q);
        if (ij) { ij[o] = (int)i; ij[o + 1] = (int)j; }
        if (xy) {                        // the centre, each operation rounded on its own
          xy[o] = f.origin_x + ((double)i + 0.5) * f.resolution;
          xy[o + 1] = f.origin_y + ((double)j + 0.5) * f.resolution;
        }
      }
    }
  }
  return TLOAM_B200_OK;
}

int tloam_b200_frontier_labels(tloam_b200_handle* h, unsigned* labels, size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->fr_kept) return TLOAM_B200_ERR_NOT_READY;
  const size_t n = h->fr_info.width * h->fr_info.height;
  if (capacity < n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (labels) CU_TRY(cudaMemcpyAsync(labels, h->d_fr_labels, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Terrain (the checks, the grid's geometry and the buffers here; the kernels in terrain.cu, loaded from
// libtloam_b200_terrain.so by the first terrain call, so that the kernels of this library keep their SASS).
// ---------------------------------------------------------------------------------------------
struct TerrainLib { tloam_ter_fn bounds = nullptr; tloam_ter_fn build = nullptr; };
static std::mutex g_ter_mu;
static TerrainLib g_ter;

static int ter_load(tloam_b200_handle* h, TerrainLib* out) {
  std::lock_guard<std::mutex> lk(g_ter_mu);
  if (!g_ter.bounds) {
    const std::string path = sibling_path("libtloam_b200_terrain.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    TerrainLib l;
    if (so) {
      l.bounds = reinterpret_cast<tloam_ter_fn>(dlsym(so, "tloam_ter_bounds"));
      l.build = reinterpret_cast<tloam_ter_fn>(dlsym(so, "tloam_ter_build"));
    }
    if (!l.bounds || !l.build) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "terrain: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_ter = l;
  }
  *out = g_ter;
  return TLOAM_B200_OK;
}

static int ter_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "terrain: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

void tloam_b200_terrain_default_config(tloam_terrain_config* c) {
  c->resolution = 0.2;                     // a car with an HDL-64E; robot parameters, not calibrated
  c->clearance = 2.0;
  c->ground_radius = 1.6; c->step_radius = 0.3; c->slope_radius = 0.4;
  c->max_step = 0.10; c->max_slope = 15.0 * M_PI / 180.0; c->max_roughness = 0.10;
  c->min_points = 1; c->min_fit = 6;
  c->static_only = 0; c->combine_occupancy = 0;
}

static bool ter_config_valid(const tloam_terrain_config* c) {
  const auto ok = [](double v) { return std::isfinite(v) && v >= 0.0; };
  return std::isfinite(c->resolution) && c->resolution > 0.0 && ok(c->clearance) && ok(c->ground_radius) &&
         ok(c->step_radius) && ok(c->slope_radius) && ok(c->max_step) && ok(c->max_slope) && c->max_slope < M_PI / 2 &&
         ok(c->max_roughness) && c->min_points >= 1 && c->min_fit >= 1;
}

// the radius in cells, false past `limit`
static bool ter_cells(double radius, double resolution, unsigned limit, unsigned* r) {
  const double v = std::ceil(radius / resolution);
  if (!(v <= (double)limit)) return false;
  *r = (unsigned)v;
  return true;
}

// the build over `count` rows at `rows` (device), the selection's counters or null; cfg checked
static int ter_run(tloam_b200_handle* h, const tloam_terrain_config* cfg, const double* rows, size_t count,
                   const unsigned* through, const unsigned* hits, tloam_terrain_info* info) {
  const bool combine = cfg->combine_occupancy != 0;
  const double res = combine ? h->occ_info.resolution : cfg->resolution;
  tloam_ter_args a;
  memset(&a, 0, sizeof(a));
  if (!ter_cells(cfg->ground_radius, res, 1024, &a.rg) || !ter_cells(cfg->step_radius, res, TLOAM_TER_HALO_MAX, &a.rs) ||
      !ter_cells(cfg->slope_radius, res, TLOAM_TER_HALO_MAX, &a.rp))
    return TLOAM_B200_ERR_INVALID_ARG;
  TerrainLib lib;
  int rc = ter_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  if (!h->d_ter_state) CU_TRY(cudaMalloc(&h->d_ter_state, sizeof(tloam_ter_state)));
  a.rows = rows; a.count = count;
  if (through) { a.through = through; a.hits = hits; a.min_through = (unsigned)h->gmd_cfg.min_through; }
  a.resolution = res;
  a.state = h->d_ter_state;
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  tloam_ter_state st;
  if (combine) {
    a.origin_x = h->occ_info.origin_x; a.origin_y = h->occ_info.origin_y;
    a.width = (unsigned)h->occ_info.width; a.height = (unsigned)h->occ_info.height;
    a.occupancy = reinterpret_cast<const signed char*>(reinterpret_cast<const unsigned*>(h->d_occ_grid) + 2 * h->cap_occ_grid);
  } else {
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.bounds(&a, &launches)));
    if ((rc = ter_status(h, e, "k_ter_bounds")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaMemcpyAsync(&st, a.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    if (st.hi[0]) {                        // origin = res floor(min / res), width = floor((max - origin) / res) + 1
      const double ox = res * std::floor(dec_ordered(~st.lo[0]) / res), oy = res * std::floor(dec_ordered(~st.lo[1]) / res);
      const double fw = std::floor((dec_ordered(st.hi[0]) - ox) / res) + 1.0;
      const double fh = std::floor((dec_ordered(st.hi[1]) - oy) / res) + 1.0;
      if (!(fw <= (double)(1u << 28)) || !(fh <= (double)(1u << 28)) || !(fw * fh <= (double)(1u << 28)))
        return TLOAM_B200_ERR_VOXEL_RANGE;
      a.origin_x = ox; a.origin_y = oy;
      a.width = (unsigned)fw; a.height = (unsigned)fh;
    }
  }
  // from here on the last build is replaced
  h->ter_built = false;
  const size_t n = (size_t)a.width * a.height;
  if (n > h->cap_ter) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ter); h->d_ter = nullptr; h->cap_ter = 0;
    CU_TRY(cudaMalloc(&h->d_ter, n * 65));
    h->cap_ter = n;
  }
  const size_t cap = h->cap_ter;
  unsigned char* b = h->d_ter;
  a.lo = reinterpret_cast<unsigned long long*>(b);
  a.gx = a.lo + cap; a.g = a.gx + cap; a.e = a.g + cap;
  a.step = reinterpret_cast<double*>(a.e + cap); a.slope = a.step + cap; a.roughness = a.slope + cap;
  a.n = reinterpret_cast<unsigned*>(a.roughness + cap); a.m = a.n + cap;
  a.values = reinterpret_cast<signed char*>(a.m + cap);
  a.clearance = cfg->clearance; a.max_step = cfg->max_step; a.max_roughness = cfg->max_roughness;
  a.tan_max_slope = std::tan(cfg->max_slope);
  a.min_points = cfg->min_points; a.min_fit = cfg->min_fit;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.build(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = ter_status(h, e, "k_ter_low / _ground / _high / _layers")) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(&st, a.state, sizeof(st), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  tloam_terrain_info out;
  memset(&out, 0, sizeof(out));
  out.origin_x = a.origin_x; out.origin_y = a.origin_y; out.resolution = res;
  out.width = a.width; out.height = a.height;
  out.ground_cells = a.rg; out.step_cells = a.rs; out.slope_cells = a.rp;
  out.used = st.used; out.skipped = st.skipped; out.overhang = st.overhang;
  out.dropped = st.dropped;
  out.known = st.known; out.lethal = st.lethal;
  out.combined = combine ? 1 : 0;
  out.rows = out.used + out.skipped + out.dropped;
  h->ter_info = out;
  h->ter_built = true;
  if (info) *info = out;
  return TLOAM_B200_OK;
}

int tloam_b200_terrain_build(tloam_b200_handle* h, const tloam_terrain_config* cfg, tloam_terrain_info* info) {
  if (!h || !cfg || !ter_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || (cfg->static_only && !h->gmd_on)) return TLOAM_B200_ERR_NOT_READY;
  if (cfg->combine_occupancy && (!h->occ_on || !h->occ_built)) return TLOAM_B200_ERR_NOT_READY;
  GMapState st;
  int rc = gmc_read(h, &st);               // the sticky flags stay for the next size / download call
  if (rc != TLOAM_B200_OK) return rc;
  return ter_run(h, cfg, h->d_gmap, st.count, cfg->static_only ? h->d_gmd_through : nullptr,
                 cfg->static_only ? h->d_gmd_hits : nullptr, info);
}

int tloam_b200_terrain_build_cloud(tloam_b200_handle* h, const tloam_terrain_config* cfg, const double* xyz, size_t n,
                                   tloam_terrain_info* info) {
  if (!h || !cfg || !ter_config_valid(cfg) || cfg->static_only || (n && !xyz)) return TLOAM_B200_ERR_INVALID_ARG;
  if (cfg->combine_occupancy && (!h->gmap_on || !h->occ_on || !h->occ_built)) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  if (n > h->cap_ter_cloud) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_ter_cloud); h->d_ter_cloud = nullptr; h->cap_ter_cloud = 0;
    CU_TRY(cudaMalloc(&h->d_ter_cloud, n * 3 * sizeof(double)));
    h->cap_ter_cloud = n;
  }
  if (n) CU_TRY(cudaMemcpyAsync(h->d_ter_cloud, xyz, n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  return ter_run(h, cfg, h->d_ter_cloud, n, nullptr, nullptr, info);
}

int tloam_b200_terrain_download(tloam_b200_handle* h, signed char* values, double* ground, double* elevation, double* step,
                                double* slope, double* roughness, unsigned* points, size_t capacity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->ter_built) return TLOAM_B200_ERR_NOT_READY;
  const size_t n = h->ter_info.width * h->ter_info.height;
  if (capacity < n) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (n) {
    const size_t cap = h->cap_ter;
    const unsigned long long* g = reinterpret_cast<const unsigned long long*>(h->d_ter) + 2 * cap;
    const unsigned long long* e = g + cap;
    const double* st = reinterpret_cast<const double*>(e + cap);
    const unsigned* m = reinterpret_cast<const unsigned*>(st + 3 * cap) + cap;
    const signed char* v = reinterpret_cast<const signed char*>(m + cap);
    if (values) CU_TRY(cudaMemcpyAsync(values, v, n, cudaMemcpyDeviceToHost, h->stream));
    if (step) CU_TRY(cudaMemcpyAsync(step, st, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (slope) CU_TRY(cudaMemcpyAsync(slope, st + cap, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    if (roughness) CU_TRY(cudaMemcpyAsync(roughness, st + 2 * cap, n * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
    std::vector<unsigned> mm(n);
    std::vector<unsigned long long> gk(ground ? n : 0), ek(elevation ? n : 0);
    CU_TRY(cudaMemcpyAsync(mm.data(), m, n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
    if (ground) CU_TRY(cudaMemcpyAsync(gk.data(), g, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    if (elevation) CU_TRY(cudaMemcpyAsync(ek.data(), e, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    for (size_t c = 0; c < n; ++c) {      // the encodings decoded: G +inf without a row, e NaN without a ground-side row
      if (ground) ground[c] = gk[c] ? dec_ordered(~gk[c]) : HUGE_VAL;
      if (elevation) elevation[c] = mm[c] ? dec_ordered(ek[c]) : std::nan("");
    }
    if (points) std::copy(mm.begin(), mm.end(), points);
  }
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_distance_build_terrain(tloam_b200_handle* h, const tloam_distance_config* cfg, tloam_distance_info* info) {
  if (!h || !cfg || !dist_config_valid(cfg)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->ter_built) return TLOAM_B200_ERR_NOT_READY;
  const tloam_terrain_info& g = h->ter_info;
  unsigned r2 = 0;
  if (!dist_r2(cfg, g.resolution, &r2)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!dist_shape_ok(g.width, g.height)) return TLOAM_B200_ERR_VOXEL_RANGE;
  DistLib lib;
  int rc = dist_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  const signed char* values = reinterpret_cast<const signed char*>(h->d_ter + 64 * h->cap_ter);
  return dist_run(h, lib, cfg, values, false, g.width, g.height, g.origin_x, g.origin_y, g.resolution, r2, info);
}

// ---------------------------------------------------------------------------------------------
// Merged global map (the checks, the key range and the buffers here; the kernels in map_merge.cu, loaded from
// libtloam_b200_gmm.so by the first merge, so that the kernels of this library keep their SASS).
// ---------------------------------------------------------------------------------------------
struct GmmLib {
  tloam_gmm_scratch_bytes_fn scratch_bytes = nullptr; tloam_gmm_state_of_fn state_of = nullptr;
  tloam_gmm_launch_fn bounds = nullptr, sort = nullptr, average = nullptr;
};
static std::mutex g_gmm_mu;
static GmmLib g_gmm;

static int gmm_load(tloam_b200_handle* h, GmmLib* out) {
  std::lock_guard<std::mutex> lk(g_gmm_mu);
  if (!g_gmm.bounds) {
    const std::string path = sibling_path("libtloam_b200_gmm.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    GmmLib l;
    if (so) {
      l.scratch_bytes = reinterpret_cast<tloam_gmm_scratch_bytes_fn>(dlsym(so, "tloam_gmm_scratch_bytes"));
      l.state_of = reinterpret_cast<tloam_gmm_state_of_fn>(dlsym(so, "tloam_gmm_state_of"));
      l.bounds = reinterpret_cast<tloam_gmm_launch_fn>(dlsym(so, "tloam_gmm_bounds"));
      l.sort = reinterpret_cast<tloam_gmm_launch_fn>(dlsym(so, "tloam_gmm_sort"));
      l.average = reinterpret_cast<tloam_gmm_launch_fn>(dlsym(so, "tloam_gmm_average"));
    }
    if (!l.scratch_bytes || !l.state_of || !l.bounds || !l.sort || !l.average) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "global map merge: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_gmm = l;
  }
  *out = g_gmm;
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_merge(tloam_b200_handle* h, double voxel, int static_only, size_t* n_voxels) {
  if (!h || !n_voxels) return TLOAM_B200_ERR_INVALID_ARG;
  *n_voxels = 0;
  if (!(voxel > 0.0) || !std::isfinite(voxel)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmap_on || (static_only && !h->gmd_on)) return TLOAM_B200_ERR_NOT_READY;
  GmmLib lib;
  int rc = gmm_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  h->gmm_valid = false;                                       // a refused merge leaves no snapshot
  GMapState st;
  if ((rc = gmc_read(h, &st)) != TLOAM_B200_OK) return rc;   // the sticky flags stay for the next size / download call
  const size_t count = st.count;
  if (count >> 32) {                                          // the sort's row payload is a u32 (2^32 rows: 103 GB of xyz)
    snprintf(h->last_error, sizeof(h->last_error), "global map merge: %zu rows do not fit a 32-bit row index", count);
    return TLOAM_B200_ERR_CUDA;
  }
  bool has = false;                                           // the map has the intensity channel (gmi_read's rule)
  if (h->gmi_used && count) {
    unsigned s0 = 0;
    CU_TRY(cudaMemcpyAsync(&s0, h->d_gmi_st, sizeof(s0), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    has = s0 != 0u;
  }
  size_t n_vox = 0;
  if (count) {
    const size_t bytes = lib.scratch_bytes(count);
    if (bytes > h->cap_gmm_scratch) {
      CU_TRY(cudaStreamSynchronize(h->stream));
      cudaFree(h->d_gmm_scratch); h->d_gmm_scratch = nullptr; h->cap_gmm_scratch = 0;
      CU_TRY(cudaMalloc(&h->d_gmm_scratch, bytes + bytes / 2));
      h->cap_gmm_scratch = bytes + bytes / 2;
    }
    tloam_gmm_args a;
    memset(&a, 0, sizeof(a));
    a.map = h->d_gmap; a.intensity = has ? h->d_gmi_map : nullptr;
    if (static_only) { a.through = h->d_gmd_through; a.hits = h->d_gmd_hits; a.min_through = (unsigned)h->gmd_cfg.min_through; }
    a.count = count; a.voxel = voxel;
    a.scratch = h->d_gmm_scratch; a.state = lib.state_of(h->d_gmm_scratch, count);
    a.device = h->device; a.stream = h->stream;
    auto run = [&](tloam_gmm_launch_fn f, const char* where) -> int {
      int e = 0, launches = 0;
      TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = f(&a, &launches)));
      h->launches += launches > 0 ? launches - 1 : 0;
      if (e == cudaSuccess) return TLOAM_B200_OK;
      snprintf(h->last_error, sizeof(h->last_error), "global map merge: %s: %s", where, cudaGetErrorString((cudaError_t)e));
      return TLOAM_B200_ERR_CUDA;
    };
    if ((rc = run(lib.bounds, "k_gmm_bounds")) != TLOAM_B200_OK) return rc;
    tloam_gmm_state gs;
    CU_TRY(cudaMemcpyAsync(&gs, a.state, sizeof(gs), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    if (gs.nonfinite) return TLOAM_B200_ERR_VOXEL_RANGE;        // an infinite extent (no append produces such a row)
    if (gs.n_sel) {
      // voxel_min_bound = min - voxel * 0.5 (ref: PointCloud2.cpp:367); the max row has the largest index per axis, as in
      // k_gmap_guard, and fixes the bits of that axis in the key
      for (int d = 0; d < 3; ++d) {
        const double half = voxel * 0.5;
        a.mb[d] = dec_ordered(~gs.lo[d]) - half;
        const double ref = (dec_ordered(gs.hi[d]) - a.mb[d]) / voxel;
        if (!(ref < (double)(1u << kGMapKeyBits))) return TLOAM_B200_ERR_VOXEL_RANGE;
        const unsigned long long top = (unsigned long long)std::floor(ref);
        int bits = 0;
        while (bits < 64 && (top >> bits)) ++bits;
        a.bits[d] = bits;
      }
      a.n_sel = gs.n_sel;
      if ((rc = run(lib.sort, "k_gmm_keys / k_gmm_hist / k_gmm_offsets / k_gmm_scatter / k_gmm_head_*")) != TLOAM_B200_OK) return rc;
      unsigned long long nv = 0;
      CU_TRY(cudaMemcpyAsync(&nv, &a.state->n_vox, sizeof(nv), cudaMemcpyDeviceToHost, h->stream));
      CU_TRY(cudaStreamSynchronize(h->stream));
      n_vox = (size_t)nv;
      if (4 * n_vox > h->cap_gmm_out) {
        cudaFree(h->d_gmm_out); h->d_gmm_out = nullptr; h->cap_gmm_out = 0;
        CU_TRY(cudaMalloc(&h->d_gmm_out, (4 * n_vox + 2 * n_vox) * sizeof(double)));
        h->cap_gmm_out = 4 * n_vox + 2 * n_vox;
      }
      a.n_vox = nv; a.out_xyz = h->d_gmm_out; a.out_intensity = has ? h->d_gmm_out + 3 * n_vox : nullptr;
      if ((rc = run(lib.average, "k_gmm_average")) != TLOAM_B200_OK) return rc;
      CU_TRY(cudaStreamSynchronize(h->stream));
    }
  }
  h->gmm_n = n_vox; h->gmm_has = has; h->gmm_valid = true;
  *n_voxels = n_vox;
  return TLOAM_B200_OK;
}

int tloam_b200_global_map_merged_download(tloam_b200_handle* h, size_t first, size_t count, double* xyz, double* intensity) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gmm_valid) return TLOAM_B200_ERR_NOT_READY;
  if (first > h->gmm_n || count > h->gmm_n - first || (count && !xyz)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  const size_t n = h->gmm_n;
  if (count) CU_TRY(cudaMemcpyAsync(xyz, h->d_gmm_out + 3 * first, count * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (count && intensity && h->gmm_has)
    CU_TRY(cudaMemcpyAsync(intensity, h->d_gmm_out + 3 * n + first, count * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Loop verification against a submap (the window, the checks and the scratch here; the kernels in loop_verify_submap.cu,
// loaded from libtloam_b200_loopvs.so on the first call).
// ---------------------------------------------------------------------------------------------
static std::mutex g_loopvs_mu;
static tloam_lvs_verify_fn g_loopvs = nullptr;

static int loopvs_load(tloam_b200_handle* h, tloam_lvs_verify_fn* out) {
  std::lock_guard<std::mutex> lk(g_loopvs_mu);
  if (!g_loopvs) {
    const std::string path = sibling_path("libtloam_b200_loopvs.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    tloam_lvs_verify_fn f = so ? reinterpret_cast<tloam_lvs_verify_fn>(dlsym(so, "tloam_lvs_verify")) : nullptr;
    if (!f) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "loop verification against a submap: cannot load %s: %s", path.c_str(),
               why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_loopvs = f;
  }
  *out = g_loopvs;
  return TLOAM_B200_OK;
}

void tloam_b200_loop_verify_submap_default_config(tloam_loop_verify_submap_config* c) {
  c->half_window = 5;
  c->normal_radius = 1.0; c->min_normal_neighbours = 5; c->max_planarity = 0.1;
  c->corr_dist_coarse = 4.0; c->corr_dist_fine = 1.0;
  c->max_iterations = 40;
  c->eps_translation = 1e-4; c->eps_rotation = 1e-5;
  c->max_fitness = 0.5;
}

int tloam_b200_loop_verify_submap_enable(tloam_b200_handle* h, const tloam_loop_verify_submap_config* c) {
  if (!h || !c) return TLOAM_B200_ERR_INVALID_ARG;
  const double v[7] = {c->normal_radius, c->max_planarity, c->corr_dist_coarse, c->corr_dist_fine, c->eps_translation,
                       c->eps_rotation, c->max_fitness};
  for (double x : v)
    if (!std::isfinite(x) || !(x > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (c->half_window < 0 || c->half_window > TLOAM_LVS_MAX_HALF_WINDOW || c->min_normal_neighbours < 3 ||
      c->corr_dist_fine > c->corr_dist_coarse || c->max_iterations < 1 || c->max_iterations > 200)
    return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on) return TLOAM_B200_ERR_NOT_READY;
  tloam_lvs_verify_fn fn;
  int rc = loopvs_load(h, &fn);
  if (rc != TLOAM_B200_OK) return rc;
  h->lvs_cfg = *c;
  h->lvs_on = true;
  h->lvs_ran = false; h->lvs_passes = 0;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_verify_submap(tloam_b200_handle* h, long long query, long long candidate, const double guess[16],
                                  const double* poses, tloam_loop_verify_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on || !h->lvs_on) return TLOAM_B200_ERR_NOT_READY;
  if (query < 0 || candidate < 0 || (size_t)query >= h->loop_frames || (size_t)candidate >= h->loop_frames)
    return TLOAM_B200_ERR_INVALID_ARG;
  double T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if (guess) memcpy(T, guess, sizeof(T));
  if (!pg_rigid(T)) return TLOAM_B200_ERR_BAD_POSE;
  const tloam_loop_verify_submap_config& c = h->lvs_cfg;
  const size_t k = (size_t)c.half_window, cand = (size_t)candidate;
  const size_t lo = cand > k ? cand - k : 0, hi = cand + k < h->loop_frames - 1 ? cand + k : h->loop_frames - 1;
  const size_t n_win = hi - lo + 1;
  if (poses) {
    for (size_t w = 0; w < n_win; ++w)
      if (!pg_rigid(poses + 16 * w)) return TLOAM_B200_ERR_BAD_POSE;
  } else if (!h->pg_on || h->pg_nodes < hi + 1) {
    return TLOAM_B200_ERR_NOT_READY;
  }
  tloam_lvs_verify_fn fn;
  int rc = loopvs_load(h, &fn);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  // the window's slice of the keyframe table and the query's range (synchronises, as tloam_b200_loop_verify does)
  unsigned long long off[2 * TLOAM_LVS_MAX_HALF_WINDOW + 2], q0 = 0, nq = 0;
  if ((rc = lv_range(h, (size_t)query, &q0, &nq)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(off, h->d_lv_off + lo, (n_win + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  const bool inside = (size_t)query >= lo && (size_t)query <= hi;
  const unsigned long long nm = off[n_win] - off[0] - (inside ? nq : 0);
  memset(out, 0, sizeof(*out));
  out->query = query; out->candidate = candidate;
  memcpy(out->T, T, sizeof(T));
  out->n_query_points = (long long)nq; out->n_candidate_points = (long long)nm;
  h->lvs_ran = true; h->lvs_passes = 0; h->lvs_nq = nq; h->lvs_nm = 0;
  if (nq == 0 || nm == 0) {
    out->termination = TLOAM_LOOP_VERIFY_EMPTY;
    out->fitness = INFINITY;
    return TLOAM_B200_OK;
  }
  // the target is split over grid y until the search has about four blocks per SM of an H100 SXM (132)
  const unsigned long long qb = (nq + TLOAM_LVS_THREADS - 1) / TLOAM_LVS_THREADS, tiles = (nm + TLOAM_LVS_THREADS - 1) / TLOAM_LVS_THREADS;
  unsigned long long splits = (4 * 132 + qb - 1) / qb;
  if (splits > tiles) splits = tiles;
  if (splits < 1) splits = 1;
  const size_t passes = (size_t)c.max_iterations + 1;
  size_t o = round_up(sizeof(tloam_lv_state), 256);
  const size_t o_poses = o;   o += round_up(n_win * 16 * sizeof(double), 256);
  const size_t o_A = o;       o += round_up(n_win * 16 * sizeof(double), 256);
  const size_t o_target = o;  o += round_up(nm * 3 * sizeof(double), 256);
  const size_t o_normal = o;  o += round_up(nm * 3 * sizeof(double), 256);
  const size_t o_neigh = o;   o += round_up(nm * sizeof(int), 256);
  const size_t o_valid = o;   o += round_up(nm, 256);
  const size_t o_part = o;    o += round_up(splits * nq * sizeof(tloam_lv_best), 256);
  const size_t o_sums = o;    o += round_up(qb * TLOAM_LVS_SUMS * sizeof(double), 256);
  const size_t o_idx = o;     o += round_up(passes * nq * sizeof(int), 256);
  const size_t o_d2 = o;      o += passes * nq * sizeof(double);
  if (o > h->cap_lvs_scratch) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_lvs_scratch); h->d_lvs_scratch = nullptr; h->cap_lvs_scratch = 0;
    const size_t bytes = o + o / 2;
    CU_TRY(cudaMalloc(&h->d_lvs_scratch, bytes));
    h->cap_lvs_scratch = bytes;
  }
  unsigned char* base = h->d_lvs_scratch;
  tloam_lv_state s;
  memset(&s, 0, sizeof(s));
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) s.R[3 * r + j] = T[4 * j + r];
    s.t[r] = T[12 + r];
  }
  s.r = c.corr_dist_coarse;
  s.term = TLOAM_LOOP_VERIFY_ITERATION_LIMIT;
  CU_TRY(cudaMemcpyAsync(base, &s, sizeof(s), cudaMemcpyHostToDevice, h->stream));   // pageable: staged before return
  if (poses) CU_TRY(cudaMemcpyAsync(base + o_poses, poses, n_win * 16 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  tloam_lvs_args a;
  memset(&a, 0, sizeof(a));
  a.pts = h->d_lv_pts; a.offsets = h->d_lv_off;
  a.lo = lo; a.hi = hi; a.candidate = cand;
  a.q0 = q0; a.nq = nq; a.query_in_window = inside ? 1 : 0; a.base = off[0]; a.nm = nm;
  a.poses = poses ? reinterpret_cast<const double*>(base + o_poses) : h->d_pg_O + 16 * lo;
  a.A = reinterpret_cast<double*>(base + o_A);
  a.target = reinterpret_cast<double*>(base + o_target);
  a.normal = reinterpret_cast<double*>(base + o_normal);
  a.neighbours = reinterpret_cast<int*>(base + o_neigh);
  a.valid = base + o_valid;
  a.normal_radius = c.normal_radius; a.max_planarity = c.max_planarity; a.min_normal_neighbours = c.min_normal_neighbours;
  a.corr_dist_coarse = c.corr_dist_coarse; a.corr_dist_fine = c.corr_dist_fine;
  a.eps_translation = c.eps_translation; a.eps_rotation = c.eps_rotation; a.max_iterations = c.max_iterations;
  a.splits = (unsigned)splits;
  a.state = reinterpret_cast<tloam_lv_state*>(base);
  a.part = reinterpret_cast<tloam_lv_best*>(base + o_part);
  a.sums = reinterpret_cast<double*>(base + o_sums);
  a.match_index = reinterpret_cast<int*>(base + o_idx);
  a.match_d2 = reinterpret_cast<double*>(base + o_d2);
  a.device = h->device; a.stream = h->stream;
  h->lvs_last = a; h->lvs_nm = nm;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = fn(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = lv_status(h, e, "k_lvs_*")) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(&s, a.state, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) out->T[4 * j + r] = s.R[3 * r + j];
    out->T[12 + r] = s.t[r];
  }
  out->fitness = s.fitness; out->rmse = s.rmse; out->inliers = (long long)s.inliers;
  out->iterations = s.iter; out->termination = s.term;
  out->accepted = s.term == TLOAM_LOOP_VERIFY_CONVERGED && s.fitness <= c.max_fitness ? 1 : 0;
  h->lvs_passes = s.iter + 1;
  return TLOAM_B200_OK;
}

int tloam_b200_loop_verify_submap_target(tloam_b200_handle* h, double* xyz, double* normal, unsigned char* valid, int* neighbours,
                                         size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on || !h->lvs_on || !h->lvs_ran) return TLOAM_B200_ERR_NOT_READY;
  const size_t nm = h->lvs_nm;
  *n = nm;
  if (capacity < nm) return TLOAM_B200_ERR_INVALID_ARG;
  if (!nm) return TLOAM_B200_OK;
  const tloam_lvs_args& a = h->lvs_last;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (xyz) CU_TRY(cudaMemcpyAsync(xyz, a.target, nm * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (normal) CU_TRY(cudaMemcpyAsync(normal, a.normal, nm * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (valid) CU_TRY(cudaMemcpyAsync(valid, a.valid, nm, cudaMemcpyDeviceToHost, h->stream));
  if (neighbours) CU_TRY(cudaMemcpyAsync(neighbours, a.neighbours, nm * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_loop_verify_submap_matches(tloam_b200_handle* h, int pass, int* index, double* d2, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->lv_on || !h->lvs_on || !h->lvs_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = h->lvs_nq;
  if (pass < 0 || pass >= h->lvs_passes || capacity < h->lvs_nq) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t nq = h->lvs_nq;
  const tloam_lvs_args& a = h->lvs_last;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (index) CU_TRY(cudaMemcpyAsync(index, a.match_index + (size_t)pass * nq, nq * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (d2) CU_TRY(cudaMemcpyAsync(d2, a.match_d2 + (size_t)pass * nq, nq * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Localization in a prior map (the checks, the query's down-sample and the buffers here; the kernels in localize.cu,
// loaded from libtloam_b200_loc.so by the enable call).
// ---------------------------------------------------------------------------------------------
struct LocLib {
  tloam_loc_scratch_bytes_fn scratch_bytes = nullptr;
  tloam_loc_index_fn bounds = nullptr, index = nullptr;
  tloam_loc_run_fn run = nullptr;
};
static std::mutex g_loc_mu;
static LocLib g_loc;

static int loc_load(tloam_b200_handle* h, LocLib* out) {
  std::lock_guard<std::mutex> lk(g_loc_mu);
  if (!g_loc.run) {
    const std::string path = sibling_path("libtloam_b200_loc.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    LocLib l;
    if (so) {
      l.scratch_bytes = reinterpret_cast<tloam_loc_scratch_bytes_fn>(dlsym(so, "tloam_loc_scratch_bytes"));
      l.bounds = reinterpret_cast<tloam_loc_index_fn>(dlsym(so, "tloam_loc_bounds"));
      l.index = reinterpret_cast<tloam_loc_index_fn>(dlsym(so, "tloam_loc_index"));
      l.run = reinterpret_cast<tloam_loc_run_fn>(dlsym(so, "tloam_loc_run"));
    }
    if (!l.scratch_bytes || !l.bounds || !l.index || !l.run) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "localization: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_loc = l;
  }
  *out = g_loc;
  return TLOAM_B200_OK;
}

static int loc_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "localization: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

// the small block: the query's GMapState at 0, the identity pose at 256, the prediction's memory at 512
static GMapState* loc_qst(tloam_b200_handle* h) { return h->d_loc_qst; }
static double* loc_eye(tloam_b200_handle* h) { return reinterpret_cast<double*>(reinterpret_cast<char*>(h->d_loc_qst) + 256); }
static tloam_loc_memory* loc_memory(tloam_b200_handle* h) {
  return reinterpret_cast<tloam_loc_memory*>(reinterpret_cast<char*>(h->d_loc_qst) + 512);
}

void tloam_b200_localize_default_config(tloam_localize_config* c) {
  c->voxel = 0.5; c->cell = 1.0;
  c->normal_radius = 1.0; c->min_normal_neighbours = 5; c->max_planarity = 0.1;
  c->corr_dist_coarse = 2.0; c->corr_dist_fine = 0.5;
  c->max_iterations = 30;
  c->eps_translation = 1e-4; c->eps_rotation = 1e-5;
  c->max_fitness = 0.5;
}

int tloam_b200_localize_enable(tloam_b200_handle* h, const tloam_localize_config* c) {
  if (!h || !c) return TLOAM_B200_ERR_INVALID_ARG;
  const double v[9] = {c->voxel, c->cell, c->normal_radius, c->max_planarity, c->corr_dist_coarse, c->corr_dist_fine,
                       c->eps_translation, c->eps_rotation, c->max_fitness};
  for (double x : v)
    if (!std::isfinite(x) || !(x > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (c->min_normal_neighbours < 3 || c->corr_dist_fine > c->corr_dist_coarse || c->max_iterations < 1 || c->max_iterations > 200 ||
      c->corr_dist_coarse > 3.0 * c->cell || c->normal_radius > 3.0 * c->cell)
    return TLOAM_B200_ERR_INVALID_ARG;
  LocLib lib;
  int rc = loc_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!h->d_loc_qst) {
    CU_TRY(cudaMalloc(&h->d_loc_qst, 512 + sizeof(tloam_loc_memory)));
    const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    CU_TRY(cudaMemcpy(loc_eye(h), eye, sizeof(eye), cudaMemcpyHostToDevice));
  }
  h->loc_cfg = *c;
  h->loc_on = true;
  h->mu_on = false;                                             // updating a prior map is off until enabled again
  h->loc_loaded = false; h->loc_n = 0; h->loc_have_prev = false;
  h->loc_ran = false; h->loc_passes = 0; h->loc_nq = 0;
  return TLOAM_B200_OK;
}

// an n-row index laid out from b: the map, the sorted map, normals, cell keys, sorted rows, cell starts, neighbour counts,
// validity and the state; the pointers into a (a->map is the first n x 3 FP64 block).  Returns the bytes it spans.
static size_t loc_carve_index(unsigned char* b, size_t n, tloam_loc_index_args* a) {
  size_t o = 0;
  if (a) a->map = reinterpret_cast<const double*>(b + o);          o += round_up(n * 24, 256);
  if (a) a->sxyz = reinterpret_cast<double*>(b + o);               o += round_up(n * 24, 256);
  if (a) a->normal = reinterpret_cast<double*>(b + o);             o += round_up(n * 24, 256);
  if (a) a->ckey = reinterpret_cast<unsigned long long*>(b + o);   o += round_up(n * 8, 256);
  if (a) a->srow = reinterpret_cast<unsigned*>(b + o);             o += round_up(n * 4, 256);
  if (a) a->cstart = reinterpret_cast<unsigned*>(b + o);           o += round_up((n + 1) * 4, 256);
  if (a) a->neighbours = reinterpret_cast<int*>(b + o);            o += round_up(n * 4, 256);
  if (a) a->valid = b + o;                                          o += round_up(n, 256);
  if (a) a->st = reinterpret_cast<tloam_gmm_state*>(b + o);        o += round_up(sizeof(tloam_gmm_state), 256);
  return o;
}

// the index of the n rows at a->map (carved by loc_carve_index) with the given cell and normal rule: bounds (synchronises),
// the key range and rounding checks, then keys, sort, cells and normals, enqueued; the radix sort's scratch grown in
// *scratch.  INVALID_ARG for a non-finite row, VOXEL_RANGE for an extent or coordinates the grid cannot hold.
static int loc_index_build(tloam_b200_handle* h, const LocLib& lib, tloam_loc_index_args& a, size_t n, double cell,
                           double normal_radius, double max_planarity, int min_normal_neighbours, unsigned char** scratch,
                           size_t* cap_scratch) {
  a.n = n;
  a.normal_radius = normal_radius; a.max_planarity = max_planarity;
  a.min_normal_neighbours = min_normal_neighbours;
  a.grid.sxyz = a.sxyz; a.grid.srow = a.srow; a.grid.ckey = a.ckey; a.grid.cstart = a.cstart; a.grid.st = a.st;
  a.grid.cell = cell;
  a.device = h->device; a.stream = h->stream;
  const size_t bytes = lib.scratch_bytes(n ? n : 1);
  if (bytes > *cap_scratch) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(*scratch); *scratch = nullptr; *cap_scratch = 0;
    CU_TRY(cudaMalloc(scratch, bytes));
    *cap_scratch = bytes;
  }
  a.scratch = *scratch;
  int e = 0, launches = 0, rc;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.bounds(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = loc_status(h, e, "k_loc_bounds")) != TLOAM_B200_OK) return rc;
  tloam_gmm_state gs;
  CU_TRY(cudaMemcpyAsync(&gs, a.st, sizeof(gs), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (gs.nonfinite) return TLOAM_B200_ERR_INVALID_ARG;
  if (n) {
    for (int d = 0; d < 3; ++d) {                // cell index floor((x - min) / cell), monotone in x: the max row has the top
      a.grid.mb[d] = dec_ordered(~gs.lo[d]);
      const double ref = std::floor((dec_ordered(gs.hi[d]) - a.grid.mb[d]) / a.grid.cell);
      if (!(ref < (double)(1u << kGMapKeyBits))) return TLOAM_B200_ERR_VOXEL_RANGE;
      // the search's cell ranges (k_loc_normals keeps at most TLOAM_LOC_MAX_SPAN per axis) assume that a coordinate's
      // rounding is far below a cell: radius <= 3 cells spans at most 6 (1 + 1e-7) cells plus that rounding
      const double big = std::fmax(std::fabs(dec_ordered(~gs.lo[d])), std::fabs(dec_ordered(gs.hi[d])));
      if (!(big * 0x1p-52 < 1e-6 * a.grid.cell)) return TLOAM_B200_ERR_VOXEL_RANGE;
      a.grid.top[d] = (long long)ref;
      int bits = 0;
      while (bits < 64 && ((unsigned long long)a.grid.top[d] >> bits)) ++bits;
      a.grid.bits[d] = bits;
    }
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.index(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = loc_status(h, e, "k_loc_keys / k_gmm_* / k_loc_cells / k_loc_normals")) != TLOAM_B200_OK) return rc;
  }
  return TLOAM_B200_OK;
}

// the map (already at the start of d_loc_map) indexed: bounds, key range, sort, cells, normals; synchronises
static int loc_build(tloam_b200_handle* h, size_t n) {
  LocLib lib;
  int rc = loc_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  tloam_loc_index_args a;
  memset(&a, 0, sizeof(a));
  loc_carve_index(h->d_loc_map, n, &a);
  if ((rc = loc_index_build(h, lib, a, n, h->loc_cfg.cell, h->loc_cfg.normal_radius, h->loc_cfg.max_planarity,
                            h->loc_cfg.min_normal_neighbours, &h->d_loc_scratch, &h->cap_loc_scratch)) != TLOAM_B200_OK)
    return rc;
  if (n) CU_TRY(cudaStreamSynchronize(h->stream));
  h->loc_index = a;
  h->loc_n = n; h->loc_loaded = true;
  return TLOAM_B200_OK;
}

// room for an n-row map and its index at the start of d_loc_map (the old map is dropped)
static int loc_reserve_map(tloam_b200_handle* h, size_t n) {
  const size_t need = loc_carve_index(nullptr, n, nullptr);
  if (need > h->cap_loc_map) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_loc_map); h->d_loc_map = nullptr; h->cap_loc_map = 0;
    CU_TRY(cudaMalloc(&h->d_loc_map, need));
    h->cap_loc_map = need;
  }
  return TLOAM_B200_OK;
}

static int mu_after_load(tloam_b200_handle* h, int rc);   // updating a prior map: its counters sized to the new map

int tloam_b200_localize_set_map(tloam_b200_handle* h, const double* xyz, size_t n) {
  if (!h || (!xyz && n)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on) return TLOAM_B200_ERR_NOT_READY;
  if (n >> 32) return TLOAM_B200_ERR_INVALID_ARG;             // the sort's row payload is a u32
  CU_TRY(cudaSetDevice(h->device));
  h->loc_loaded = false; h->loc_have_prev = false; h->loc_ran = false; h->loc_passes = 0;
  h->mu_fresh = true; h->mu_frames = 0;                         // an update belongs to the map it was made on
  int rc;
  if ((rc = loc_reserve_map(h, n)) != TLOAM_B200_OK) return rc;
  if (n && (rc = upload_host(h, h->d_loc_map, xyz, n * 24)) != TLOAM_B200_OK) return rc;
  return mu_after_load(h, loc_build(h, n));
}

int tloam_b200_localize_set_map_merged(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || !h->gmm_valid) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  const size_t n = h->gmm_n;
  h->loc_loaded = false; h->loc_have_prev = false; h->loc_ran = false; h->loc_passes = 0;
  h->mu_fresh = true; h->mu_frames = 0;                         // an update belongs to the map it was made on
  int rc;
  if ((rc = loc_reserve_map(h, n)) != TLOAM_B200_OK) return rc;
  if (n) CU_TRY(cudaMemcpyAsync(h->d_loc_map, h->d_gmm_out, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  return mu_after_load(h, loc_build(h, n));
}

// the query: VoxelDownSample(voxel) of the finite rows of the n rows at d_in by the global map's ordered path at pose I
// (the keyframe path of loop verification, in buffers of its own) into *q with its state at st (the localization's, or
// relocalization's own); synchronises and returns its row count
// the same down-sample at `voxel` into the given buffers (reg, fin: the transform's scratch; eye: the identity on the device)
static int ordered_query(tloam_b200_handle* h, const double* d_in, size_t n, double voxel, const double* eye, double** reg,
                         size_t* cap_reg, double** fin, size_t* cap_fin, GMapState* st, double** q, size_t* cap_q, size_t* nq) {
  int rc;
  if ((rc = ensure_dev(h, reg, cap_reg, n, false)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, fin, cap_fin, n, false)) != TLOAM_B200_OK) return rc;
  if ((rc = ensure_dev(h, q, cap_q, n, false)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemsetAsync(st, 0, sizeof(GMapState), h->stream));
  const unsigned tb = 256, gb = (unsigned)((n + tb - 1) / tb);
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_transform<<<gb, tb, 0, h->stream>>>(d_in, (unsigned)n, eye, *reg, *fin, st)));
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_guard<<<1, 32, 0, h->stream>>>(st, voxel)));
  VoxSorted vs;
  if ((rc = voxel_pipeline(h, *fin, n, &st->n_fin, 0u, nullptr, nullptr, nullptr, 0.0, voxel, nullptr, &st->n_vox,
                           h->stream, 0, &vs)) != TLOAM_B200_OK) return rc;
  if (n) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (k_gmap_emit<<<gb, tb, 0, h->stream>>>(vs.a, vs.slots, *q, st, *cap_q)));
  CU_TRY(cudaGetLastError());
  GMapState s;
  CU_TRY(cudaMemcpyAsync(&s, st, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (s.refused) return TLOAM_B200_ERR_VOXEL_RANGE;
  *nq = s.refused ? 0 : s.n_vox;
  return TLOAM_B200_OK;
}

static int loc_query(tloam_b200_handle* h, const double* d_in, size_t n, size_t* nq, GMapState* st, double** q, size_t* cap_q) {
  return ordered_query(h, d_in, n, h->loc_cfg.voxel, loc_eye(h), &h->d_loc_reg, &h->cap_loc_reg, &h->d_loc_fin, &h->cap_loc_fin,
                       st, q, cap_q, nq);
}

static int loc_run(tloam_b200_handle* h, const double* d_in, size_t n, const double* guess, tloam_localize_result* out) {
  if (!h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  if (!guess && !h->loc_have_prev) return TLOAM_B200_ERR_NOT_READY;
  if (guess && !pg_rigid(guess)) return TLOAM_B200_ERR_BAD_POSE;
  LocLib lib;
  int rc = loc_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  h->loc_src = nullptr;                                         // the last query is rewritten: no add until this run ends
  size_t nq = 0;
  if ((rc = loc_query(h, d_in, n, &nq, loc_qst(h), &h->d_loc_q, &h->cap_loc_q)) != TLOAM_B200_OK) return rc;
  const tloam_localize_config& c = h->loc_cfg;
  const size_t nr = h->loc_n ? nq : 0;                          // an empty map: nothing to match (EMPTY)
  const size_t passes = (size_t)c.max_iterations + 1, qb = (nr + TLOAM_LOC_THREADS - 1) / TLOAM_LOC_THREADS;
  size_t o = round_up(sizeof(tloam_loc_state), 256);
  const size_t o_sums = o;  o += round_up(qb * TLOAM_LOC_SUMS * sizeof(double), 256);
  const size_t o_idx = o;   o += round_up(passes * nr * sizeof(int), 256);
  const size_t o_d2 = o;    o += passes * nr * sizeof(double);
  if (o > h->cap_loc_run) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_loc_run); h->d_loc_run = nullptr; h->cap_loc_run = 0;
    CU_TRY(cudaMalloc(&h->d_loc_run, o + o / 2));
    h->cap_loc_run = o + o / 2;
  }
  unsigned char* base = h->d_loc_run;
  tloam_loc_state s;
  memset(&s, 0, sizeof(s));
  s.r = c.corr_dist_coarse;
  s.term = nr ? TLOAM_LOOP_VERIFY_ITERATION_LIMIT : TLOAM_LOOP_VERIFY_EMPTY;
  s.done = nr ? 0 : 1;
  if (guess) memcpy(s.guess, guess, sizeof(s.guess));
  CU_TRY(cudaMemcpyAsync(base, &s, sizeof(s), cudaMemcpyHostToDevice, h->stream));   // pageable: staged before return
  tloam_loc_args a;
  memset(&a, 0, sizeof(a));
  a.grid = h->loc_index.grid;
  a.map = h->loc_index.map; a.normal = h->loc_index.normal; a.valid = h->loc_index.valid;
  a.query = h->d_loc_q; a.nq = nr;
  a.odom = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, result));
  a.predict = guess ? 0 : 1;
  a.memory = loc_memory(h);
  a.corr_dist_coarse = c.corr_dist_coarse; a.corr_dist_fine = c.corr_dist_fine;
  a.eps_translation = c.eps_translation; a.eps_rotation = c.eps_rotation; a.max_fitness = c.max_fitness;
  a.max_iterations = c.max_iterations;
  a.state = reinterpret_cast<tloam_loc_state*>(base);
  a.sums = reinterpret_cast<double*>(base + o_sums);
  a.match_index = reinterpret_cast<int*>(base + o_idx);
  a.match_d2 = reinterpret_cast<double*>(base + o_d2);
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.run(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = loc_status(h, e, "k_loc_*")) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaMemcpyAsync(&s, a.state, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  memset(out, 0, sizeof(*out));
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) out->T[4 * j + r] = s.R[3 * r + j];
    out->T[12 + r] = s.t[r];
  }
  out->T[15] = 1.0;
  memcpy(out->T_map_odom, s.map_odom, sizeof(out->T_map_odom));
  memcpy(out->guess, s.guess, sizeof(out->guess));
  out->iterations = s.iter; out->termination = s.term; out->accepted = s.accepted;
  out->inliers = (long long)s.inliers; out->rmse = s.rmse; out->fitness = s.fitness;
  out->n_query_points = (long long)nq; out->n_map_points = (long long)h->loc_n;
  h->loc_have_prev = true;
  h->loc_ran = true; h->loc_passes = nr ? s.iter + 1 : 0; h->loc_nq = nr; h->loc_last = a;
  h->loc_serial++; h->loc_accepted = s.accepted != 0;
  h->loc_src = d_in; h->loc_src_n = n; h->loc_src_raw = d_in == h->raw_scan;
  h->loc_src_gen = h->loc_src_raw ? h->raw_gen : h->loc_in_gen;
  return TLOAM_B200_OK;
}

int tloam_b200_localize_frame(tloam_b200_handle* h, const double guess[16], tloam_localize_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || h->raw_gen != h->seg_gen) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  return loc_run(h, h->raw_scan, h->raw_n, guess, out);
}

int tloam_b200_localize(tloam_b200_handle* h, const double* xyz, size_t n, const double guess[16], tloam_localize_result* out) {
  if (!h || !out || (!xyz && n) || n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  int rc;
  if ((rc = ensure_dev(h, &h->d_loc_in, &h->cap_loc_in, n, false)) != TLOAM_B200_OK) return rc;
  h->loc_in_gen++;                                              // the host cloud of an earlier localization is replaced
  if (n && (rc = upload_host(h, h->d_loc_in, xyz, n * 24)) != TLOAM_B200_OK) return rc;
  return loc_run(h, h->d_loc_in, n, guess, out);
}

int tloam_b200_localize_matches(tloam_b200_handle* h, int pass, int* index, double* d2, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || !h->loc_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = h->loc_nq;
  if (pass < 0 || pass >= h->loc_passes || capacity < h->loc_nq) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t nq = h->loc_nq;
  const tloam_loc_args& a = h->loc_last;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (index) CU_TRY(cudaMemcpyAsync(index, a.match_index + (size_t)pass * nq, nq * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (d2) CU_TRY(cudaMemcpyAsync(d2, a.match_d2 + (size_t)pass * nq, nq * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_localize_query(tloam_b200_handle* h, double* xyz, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || !h->loc_ran) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  GMapState s;
  CU_TRY(cudaMemcpyAsync(&s, loc_qst(h), sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  *n = s.n_vox;
  if (capacity < *n || (!xyz && *n)) return TLOAM_B200_ERR_INVALID_ARG;
  if (*n) CU_TRY(cudaMemcpyAsync(xyz, h->d_loc_q, *n * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_localize_map_normals(tloam_b200_handle* h, double* normal, unsigned char* valid, int* neighbours, size_t capacity,
                                    size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || !h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  const size_t m = h->loc_n;
  *n = m;
  if (capacity < m) return TLOAM_B200_ERR_INVALID_ARG;
  if (!m) return TLOAM_B200_OK;
  const tloam_loc_index_args& a = h->loc_index;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (normal) CU_TRY(cudaMemcpyAsync(normal, a.normal, m * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (valid) CU_TRY(cudaMemcpyAsync(valid, a.valid, m, cudaMemcpyDeviceToHost, h->stream));
  if (neighbours) CU_TRY(cudaMemcpyAsync(neighbours, a.neighbours, m * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_localize_cells(tloam_b200_handle* h, unsigned* sorted_rows, unsigned long long* keys, unsigned* starts,
                              size_t capacity, size_t* n_cells) {
  if (!h || !n_cells) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || !h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  const tloam_loc_index_args& a = h->loc_index;
  CU_TRY(cudaSetDevice(h->device));
  unsigned long long nc = 0;
  if (h->loc_n) {
    CU_TRY(cudaMemcpyAsync(&nc, &a.st->n_vox, sizeof(nc), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
  }
  *n_cells = nc;
  if (capacity < h->loc_n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_n) return TLOAM_B200_OK;
  if (sorted_rows) CU_TRY(cudaMemcpyAsync(sorted_rows, a.srow, h->loc_n * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  if (keys) CU_TRY(cudaMemcpyAsync(keys, a.ckey, nc * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->stream));
  if (starts) CU_TRY(cudaMemcpyAsync(starts, a.cstart, (nc + 1) * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Relocalization in a prior map (the checks, the places, the query's descriptor and down-sample and the buffers here; the
// kernels in relocalize.cu, loaded from libtloam_b200_reloc.so by the enable call, and the descriptor's in scan_context.cu).
// ---------------------------------------------------------------------------------------------
static std::mutex g_rl_mu;
static tloam_rl_run_fn g_rl_run = nullptr;

static int rl_load(tloam_b200_handle* h, tloam_rl_run_fn* out) {
  std::lock_guard<std::mutex> lk(g_rl_mu);
  if (!g_rl_run) {
    const std::string path = sibling_path("libtloam_b200_reloc.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    tloam_rl_run_fn f = so ? reinterpret_cast<tloam_rl_run_fn>(dlsym(so, "tloam_rl_run")) : nullptr;
    if (!f) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "relocalization: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_rl_run = f;
  }
  *out = g_rl_run;
  return TLOAM_B200_OK;
}

// d_rl_small: the query's GMapState at 0, its descriptor slot at 256
static_assert(sizeof(GMapState) <= 256, "the query's GMapState must fit below its descriptor slot");

static size_t rl_slot(const tloam_relocalize_config& c) { return TLOAM_SC_SLOT_DOUBLES(c.n_ring, c.n_sector); }

void tloam_b200_relocalize_default_config(tloam_relocalize_config* c) {
  tloam_loop_config l;
  tloam_b200_loop_default_config(&l);
  c->lidar_height = l.lidar_height; c->n_ring = l.n_ring; c->n_sector = l.n_sector; c->max_radius = l.max_radius;
  c->top_k = 8; c->max_distance = 0.4;
  c->distinct_translation = 2.0; c->distinct_rotation = 10.0 * M_PI / 180.0; c->ambiguity_ratio = 1.5;
}

int tloam_b200_relocalize_enable(tloam_b200_handle* h, const tloam_relocalize_config* c) {
  if (!h || !c || c->n_ring < 1 || c->n_sector < 1 || (long long)c->n_ring * c->n_sector > 4096 || !std::isfinite(c->max_radius) ||
      !(c->max_radius > 0.0) || !std::isfinite(c->lidar_height) || c->top_k < 1 || c->top_k > TLOAM_RL_MAX_K ||
      !std::isfinite(c->max_distance) || !std::isfinite(c->distinct_translation) || !(c->distinct_translation >= 0.0) ||
      !std::isfinite(c->distinct_rotation) || !(c->distinct_rotation >= 0.0) || !std::isfinite(c->ambiguity_ratio) ||
      !(c->ambiguity_ratio >= 1.0))
    return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on) return TLOAM_B200_ERR_NOT_READY;
  tloam_rl_run_fn run;
  int rc = rl_load(h, &run);
  if (rc != TLOAM_B200_OK) return rc;
  LoopLib lib;
  if ((rc = loop_load(h, &lib)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->rl_on = false; h->rl_loaded = false; h->rl_ran = false;   // until the new configuration is in place
  if (!h->d_rl_small) CU_TRY(cudaMalloc(&h->d_rl_small, 256 + 4096 * 3 * sizeof(double)));
  cudaFree(h->d_rl_dirs); h->d_rl_dirs = nullptr;
  std::vector<double> dirs(2 * (size_t)c->n_sector);           // the loop closure's table: the same bits
  for (int k = 1; k < c->n_sector; ++k) {
    const double t = 2.0 * M_PI * k / c->n_sector;
    dirs[2 * (k - 1)] = std::cos(t);
    dirs[2 * (k - 1) + 1] = std::sin(t);
  }
  CU_TRY(cudaMalloc(&h->d_rl_dirs, dirs.size() * sizeof(double)));
  CU_TRY(cudaMemcpy(h->d_rl_dirs, dirs.data(), dirs.size() * sizeof(double), cudaMemcpyHostToDevice));
  h->rl_cfg = *c;
  h->rl_on = true;
  h->rl_loaded = false; h->rl_n = 0; h->rl_ran = false;
  return TLOAM_B200_OK;
}

// room for n places: slots, poses, each place's best distance and shift
static int rl_reserve(tloam_b200_handle* h, size_t n, size_t* o_pose, size_t* o_dist, size_t* o_shift) {
  const size_t slot = rl_slot(h->rl_cfg);
  size_t o = round_up(n * slot * sizeof(double), 256);
  *o_pose = o;  o += round_up(n * 16 * sizeof(double), 256);
  *o_dist = o;  o += round_up(n * sizeof(double), 256);
  *o_shift = o; o += n * sizeof(long long);
  if (o > h->cap_rl_places) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_rl_places); h->d_rl_places = nullptr; h->cap_rl_places = 0;
    CU_TRY(cudaMalloc(&h->d_rl_places, o ? o : 256));
    h->cap_rl_places = o ? o : 256;
  }
  return TLOAM_B200_OK;
}

static int rl_check_poses(const double* poses, size_t n) {
  for (size_t j = 0; j < 16 * n; ++j)
    if (!std::isfinite(poses[j])) return TLOAM_B200_ERR_INVALID_ARG;
  for (size_t j = 0; j < n; ++j)
    if (!pg_rigid(poses + 16 * j)) return TLOAM_B200_ERR_BAD_POSE;
  return TLOAM_B200_OK;
}

int tloam_b200_relocalize_set_places(tloam_b200_handle* h, const double* descriptors, const double* poses, size_t n) {
  if (!h || (n && (!descriptors || !poses))) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->rl_on) return TLOAM_B200_ERR_NOT_READY;
  const size_t slot = rl_slot(h->rl_cfg);
  for (size_t j = 0; j < n * slot; ++j)
    if (!std::isfinite(descriptors[j])) return TLOAM_B200_ERR_INVALID_ARG;
  int rc = rl_check_poses(poses, n);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  h->rl_loaded = false;
  size_t op, od, os;
  if ((rc = rl_reserve(h, n, &op, &od, &os)) != TLOAM_B200_OK) return rc;
  if (n && (rc = upload_host(h, h->d_rl_places, descriptors, n * slot * sizeof(double))) != TLOAM_B200_OK) return rc;
  if (n && (rc = upload_host(h, h->d_rl_places + op, poses, n * 16 * sizeof(double))) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->rl_n = n; h->rl_loaded = true;
  return TLOAM_B200_OK;
}

int tloam_b200_relocalize_set_places_loop(tloam_b200_handle* h, const double* poses, size_t n) {
  if (!h || (n && !poses)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->rl_on || !h->loop_on) return TLOAM_B200_ERR_NOT_READY;
  if (n != h->loop_frames || h->loop_cfg.n_ring != h->rl_cfg.n_ring || h->loop_cfg.n_sector != h->rl_cfg.n_sector)
    return TLOAM_B200_ERR_INVALID_ARG;
  int rc = rl_check_poses(poses, n);
  if (rc != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  h->rl_loaded = false;
  size_t op, od, os;
  if ((rc = rl_reserve(h, n, &op, &od, &os)) != TLOAM_B200_OK) return rc;
  if (n) CU_TRY(cudaMemcpyAsync(h->d_rl_places, h->d_loop_db, n * rl_slot(h->rl_cfg) * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
  if (n && (rc = upload_host(h, h->d_rl_places + op, poses, n * 16 * sizeof(double))) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->rl_n = n; h->rl_loaded = true;
  return TLOAM_B200_OK;
}

// a run's state as a tloam_localize_result (loc_run's copy home)
static void rl_result(const tloam_loc_state& s, size_t nq, size_t n_map, tloam_localize_result* out) {
  memset(out, 0, sizeof(*out));
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) out->T[4 * j + r] = s.R[3 * r + j];
    out->T[12 + r] = s.t[r];
  }
  out->T[15] = 1.0;
  memcpy(out->T_map_odom, s.map_odom, sizeof(out->T_map_odom));
  memcpy(out->guess, s.guess, sizeof(out->guess));
  out->iterations = s.iter; out->termination = s.term; out->accepted = s.accepted;
  out->inliers = (long long)s.inliers; out->rmse = s.rmse; out->fitness = s.fitness;
  out->n_query_points = (long long)nq; out->n_map_points = (long long)n_map;
}

// the query's descriptor and down-sample, the search, the guesses and the batched ICP, with one read-back of the query's
// size and one copy home
static int rl_run(tloam_b200_handle* h, const double* d_in, size_t n, tloam_relocalize_result* out) {
  if (!h->loc_loaded || !h->rl_loaded) return TLOAM_B200_ERR_NOT_READY;
  tloam_rl_run_fn run;
  int rc = rl_load(h, &run);
  if (rc != TLOAM_B200_OK) return rc;
  LoopLib lib;
  if ((rc = loop_load(h, &lib)) != TLOAM_B200_OK) return rc;
  const tloam_relocalize_config& rc_ = h->rl_cfg;
  double* qdesc = reinterpret_cast<double*>(h->d_rl_small + 256);
  tloam_sc_args sa;
  memset(&sa, 0, sizeof(sa));
  sa.n_ring = rc_.n_ring; sa.n_sector = rc_.n_sector; sa.lidar_height = rc_.lidar_height; sa.max_radius = rc_.max_radius;
  sa.dirs = h->d_rl_dirs; sa.xyz = d_in; sa.n = n; sa.db = qdesc; sa.frame = 0;
  sa.device = h->device; sa.stream = h->stream;
  int e = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.bin(&sa)));
  if (e == cudaSuccess) TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.finish(&sa)));
  if (e != cudaSuccess) {
    snprintf(h->last_error, sizeof(h->last_error), "relocalization: k_sc_bin / k_sc_finish: %s", cudaGetErrorString((cudaError_t)e));
    return TLOAM_B200_ERR_CUDA;
  }
  size_t nq = 0;
  if ((rc = loc_query(h, d_in, n, &nq, reinterpret_cast<GMapState*>(h->d_rl_small), &h->d_rl_q, &h->cap_rl_q)) != TLOAM_B200_OK)
    return rc;
  const tloam_localize_config& c = h->loc_cfg;
  const size_t nr = h->loc_n ? nq : 0;
  const size_t K = (size_t)rc_.top_k, passes = (size_t)c.max_iterations + 1, qb = (nr + TLOAM_LOC_THREADS - 1) / TLOAM_LOC_THREADS;
  const size_t home = K * sizeof(tloam_loc_state) + sizeof(tloam_rl_top);
  size_t o = round_up(home, 256);
  const size_t o_sums = o;  o += round_up(K * qb * TLOAM_LOC_SUMS * sizeof(double), 256);
  const size_t o_idx = o;   o += round_up(K * passes * nr * sizeof(int), 256);
  const size_t o_d2 = o;    o += K * passes * nr * sizeof(double);
  if (o > h->cap_rl_run) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_rl_run); h->d_rl_run = nullptr; h->cap_rl_run = 0;
    CU_TRY(cudaMalloc(&h->d_rl_run, o + o / 2));
    h->cap_rl_run = o + o / 2;
  }
  unsigned char* base = h->d_rl_run;
  std::vector<tloam_loc_state> st(K);
  for (auto& s : st) {
    memset(&s, 0, sizeof(s));
    s.r = c.corr_dist_coarse;
    s.term = nr ? TLOAM_LOOP_VERIFY_ITERATION_LIMIT : TLOAM_LOOP_VERIFY_EMPTY;
    s.done = nr ? 0 : 1;
  }
  CU_TRY(cudaMemcpyAsync(base, st.data(), K * sizeof(tloam_loc_state), cudaMemcpyHostToDevice, h->stream));   // pageable: staged
  size_t op, od, os;
  if ((rc = rl_reserve(h, h->rl_n, &op, &od, &os)) != TLOAM_B200_OK) return rc;   // the places' offsets (no growth)
  tloam_rl_args a;
  memset(&a, 0, sizeof(a));
  a.loc.grid = h->loc_index.grid;
  a.loc.map = h->loc_index.map; a.loc.normal = h->loc_index.normal; a.loc.valid = h->loc_index.valid;
  a.loc.query = h->d_rl_q; a.loc.nq = nr;
  a.loc.odom = reinterpret_cast<const double*>(reinterpret_cast<const char*>(h->d_state) + offsetof(FrameState, result));
  a.loc.memory = loc_memory(h);
  a.loc.corr_dist_coarse = c.corr_dist_coarse; a.loc.corr_dist_fine = c.corr_dist_fine;
  a.loc.eps_translation = c.eps_translation; a.loc.eps_rotation = c.eps_rotation; a.loc.max_fitness = c.max_fitness;
  a.loc.max_iterations = c.max_iterations;
  a.loc.device = h->device; a.loc.stream = h->stream;
  a.qdesc = qdesc;
  a.places = reinterpret_cast<const double*>(h->d_rl_places);
  a.poses = reinterpret_cast<const double*>(h->d_rl_places + op);
  a.n_places = h->rl_n;
  a.n_ring = rc_.n_ring; a.n_sector = rc_.n_sector; a.dirs = h->d_rl_dirs;
  a.place_distance = reinterpret_cast<double*>(h->d_rl_places + od);
  a.place_shift = reinterpret_cast<long long*>(h->d_rl_places + os);
  a.top_k = rc_.top_k; a.max_distance = rc_.max_distance; a.distinct_translation = rc_.distinct_translation;
  a.cos_distinct_rotation = std::cos(rc_.distinct_rotation); a.ambiguity_ratio = rc_.ambiguity_ratio;
  a.states = reinterpret_cast<tloam_loc_state*>(base);
  a.top = reinterpret_cast<tloam_rl_top*>(base + K * sizeof(tloam_loc_state));
  a.sums = reinterpret_cast<double*>(base + o_sums);
  a.match_index = reinterpret_cast<int*>(base + o_idx);
  a.match_d2 = reinterpret_cast<double*>(base + o_d2);
  a.device = h->device; a.stream = h->stream;
  int launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = run(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if (e != cudaSuccess) {
    snprintf(h->last_error, sizeof(h->last_error), "relocalization: k_rl_*: %s", cudaGetErrorString((cudaError_t)e));
    return TLOAM_B200_ERR_CUDA;
  }
  std::vector<unsigned char> back(home);
  CU_TRY(cudaMemcpyAsync(back.data(), base, home, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->rl_states.assign(reinterpret_cast<const tloam_loc_state*>(back.data()), reinterpret_cast<const tloam_loc_state*>(back.data()) + K);
  memcpy(&h->rl_top, back.data() + K * sizeof(tloam_loc_state), sizeof(tloam_rl_top));
  const tloam_rl_top& t = h->rl_top;
  memset(out, 0, sizeof(*out));
  out->n_hypotheses = t.n;
  out->winner = t.winner;
  if (t.n > 0 && t.winner >= 0) {
    rl_result(h->rl_states[t.winner], nq, h->loc_n, &out->result);
    out->place = t.place[t.winner]; out->shift = (int)t.shift[t.winner]; out->distance = t.distance[t.winner];
  } else {
    tloam_loc_state none;
    memset(&none, 0, sizeof(none));
    none.term = TLOAM_LOOP_VERIFY_EMPTY; none.fitness = INFINITY;
    for (int k = 0; k < 3; ++k) none.R[4 * k] = 1.0;
    for (int k = 0; k < 4; ++k) { none.guess[5 * k] = 1.0; none.odom[5 * k] = 1.0; none.map_odom[5 * k] = 1.0; }
    rl_result(none, nq, h->loc_n, &out->result);
    out->place = -1; out->shift = 0; out->distance = INFINITY; out->winner = -1;
  }
  out->ambiguous = t.ambiguous; out->accepted = t.accepted;
  if (t.accepted) h->loc_have_prev = true;                      // k_rl_select wrote the prediction's memory
  h->rl_ran = true; h->rl_nq = nr; h->rl_qn = nq; h->rl_last = a;
  return TLOAM_B200_OK;
}

int tloam_b200_relocalize_frame(tloam_b200_handle* h, tloam_relocalize_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->rl_on || h->raw_gen != h->seg_gen) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  return rl_run(h, h->raw_scan, h->raw_n, out);
}

int tloam_b200_relocalize(tloam_b200_handle* h, const double* xyz, size_t n, tloam_relocalize_result* out) {
  if (!h || !out || (!xyz && n) || n > ((size_t)1 << 30)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->rl_on) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  int rc;
  if ((rc = ensure_dev(h, &h->d_loc_in, &h->cap_loc_in, n, false)) != TLOAM_B200_OK) return rc;
  h->loc_in_gen++;                                              // the host cloud of an earlier localization is replaced
  if (n && (rc = upload_host(h, h->d_loc_in, xyz, n * 24)) != TLOAM_B200_OK) return rc;
  return rl_run(h, h->d_loc_in, n, out);
}

int tloam_b200_relocalize_hypotheses(tloam_b200_handle* h, tloam_relocalize_hypothesis* out, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->rl_on || !h->rl_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = (size_t)h->rl_top.n;
  if (capacity < *n || (!out && *n)) return TLOAM_B200_ERR_INVALID_ARG;
  for (size_t k = 0; k < *n; ++k) {
    out[k].place = h->rl_top.place[k]; out[k].shift = (int)h->rl_top.shift[k]; out[k].distance = h->rl_top.distance[k];
    rl_result(h->rl_states[k], h->rl_qn, h->loc_n, &out[k].result);
  }
  return TLOAM_B200_OK;
}

int tloam_b200_relocalize_matches(tloam_b200_handle* h, int hypothesis, int pass, int* index, double* d2, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->rl_on || !h->rl_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = h->rl_nq;
  if (hypothesis < 0 || hypothesis >= h->rl_top.n || capacity < h->rl_nq) return TLOAM_B200_ERR_INVALID_ARG;
  const int passes = h->rl_nq ? h->rl_states[hypothesis].iter + 1 : 0;
  if (pass < 0 || pass >= passes) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t nq = h->rl_nq, stride = (size_t)(h->rl_last.loc.max_iterations + 1) * nq;
  const tloam_rl_args& a = h->rl_last;
  const size_t off = (size_t)hypothesis * stride + (size_t)pass * nq;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (index) CU_TRY(cudaMemcpyAsync(index, a.match_index + off, nq * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (d2) CU_TRY(cudaMemcpyAsync(d2, a.match_d2 + off, nq * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

// ---------------------------------------------------------------------------------------------
// Updating a prior map (the checks, the state and the buffers here; the votes and the prior rows' compaction in
// map_dynamic.cu, the novelty and the additions' voxels in map_update.cu, loaded from libtloam_b200_gmd.so and
// libtloam_b200_mapu.so by the enable call).
// ---------------------------------------------------------------------------------------------
struct MuLib {
  tloam_mu_add_fn pose = nullptr, novel = nullptr;
  tloam_mu_scratch_bytes_fn scratch_bytes = nullptr;
  tloam_mu_state_of_fn state_of = nullptr;
  tloam_mu_build_fn bounds = nullptr, sort = nullptr, average = nullptr;
};
static std::mutex g_mu_mu;
static MuLib g_mu;

static int mu_load(tloam_b200_handle* h, MuLib* out) {
  std::lock_guard<std::mutex> lk(g_mu_mu);
  if (!g_mu.average) {
    const std::string path = sibling_path("libtloam_b200_mapu.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    MuLib l;
    if (so) {
      l.pose = reinterpret_cast<tloam_mu_add_fn>(dlsym(so, "tloam_mu_pose"));
      l.novel = reinterpret_cast<tloam_mu_add_fn>(dlsym(so, "tloam_mu_novel"));
      l.scratch_bytes = reinterpret_cast<tloam_mu_scratch_bytes_fn>(dlsym(so, "tloam_mu_scratch_bytes"));
      l.state_of = reinterpret_cast<tloam_mu_state_of_fn>(dlsym(so, "tloam_mu_state_of"));
      l.bounds = reinterpret_cast<tloam_mu_build_fn>(dlsym(so, "tloam_mu_bounds"));
      l.sort = reinterpret_cast<tloam_mu_build_fn>(dlsym(so, "tloam_mu_sort"));
      l.average = reinterpret_cast<tloam_mu_build_fn>(dlsym(so, "tloam_mu_average"));
    }
    if (!l.pose || !l.novel || !l.scratch_bytes || !l.state_of || !l.bounds || !l.sort || !l.average) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "map update: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_mu = l;
  }
  *out = g_mu;
  return TLOAM_B200_OK;
}

static int mu_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "map update: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

// d_mu_small: the vote pose at 0, the prior rows' count at 128, the additions' count at 136, the compaction base at 144,
// the built cloud's count at 152, the static part's block counts at 1024
constexpr size_t kMuSmall = 1024 + 4 * 1024;
static double* mu_pose(tloam_b200_handle* h) { return reinterpret_cast<double*>(h->d_mu_small); }
static unsigned long long* mu_word(tloam_b200_handle* h, int k) {
  return reinterpret_cast<unsigned long long*>(h->d_mu_small + 128 + 8 * k);
}
// the additions' arrays in d_mu_add for a capacity of cap rows
struct MuAdd { double* xyz; unsigned* frame; unsigned* through; unsigned* hits; };
static MuAdd mu_add_of(unsigned char* base, size_t cap) {
  MuAdd a;
  a.xyz = reinterpret_cast<double*>(base);
  a.frame = reinterpret_cast<unsigned*>(base + round_up(cap * 24, 256));
  a.through = reinterpret_cast<unsigned*>(base + round_up(cap * 24, 256) + round_up(cap * 4, 256));
  a.hits = reinterpret_cast<unsigned*>(base + round_up(cap * 24, 256) + 2 * round_up(cap * 4, 256));
  return a;
}
static size_t mu_add_bytes(size_t cap) { return round_up(cap * 24, 256) + 3 * round_up(cap * 4, 256); }

// after a synchronisation: the buffers adds replaced (their last readers have finished)
static void mu_free_retired(tloam_b200_handle* h) {
  for (void* p : h->mu_retired) cudaFree(p);
  h->mu_retired.clear();
}

// the prior rows' counters for the loaded map, allocated where the caller synchronises anyway (the enable, a load)
static int mu_prior_alloc(tloam_b200_handle* h) {
  const size_t n = h->loc_loaded ? h->loc_n : 0;
  if (n <= h->cap_mu_prior) return TLOAM_B200_OK;
  cudaFree(h->d_mu_prior); h->d_mu_prior = nullptr; h->cap_mu_prior = 0;
  CU_TRY(cudaMalloc(&h->d_mu_prior, 2 * n * sizeof(unsigned)));
  h->cap_mu_prior = n;
  return TLOAM_B200_OK;
}

void tloam_b200_map_update_default_config(tloam_map_update_config* c) {
  tloam_b200_global_map_dynamic_default_config(&c->image);
  c->novel_radius = 0.5;
  c->voxel = 0.5;
  c->min_frames = 3;
}

int tloam_b200_map_update_enable(tloam_b200_handle* h, const tloam_map_update_config* c) {
  if (!h || !c) return TLOAM_B200_ERR_INVALID_ARG;
  std::vector<double> tab;
  if (!gmd_config_valid(&c->image) || !gmd_tables(&c->image, &tab)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!std::isfinite(c->novel_radius) || !(c->novel_radius > 0.0) || !std::isfinite(c->voxel) || !(c->voxel > 0.0) ||
      c->min_frames < 1)
    return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on) return TLOAM_B200_ERR_NOT_READY;
  if (c->novel_radius > 3.0 * h->loc_cfg.cell) return TLOAM_B200_ERR_INVALID_ARG;   // the grid search's span
  GmdLib gmd;
  MuLib lib;
  int rc;
  if ((rc = gmd_load(h, &gmd)) != TLOAM_B200_OK || (rc = mu_load(h, &lib)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (tab.size() > h->cap_mu_tables) {
    cudaFree(h->d_mu_tables); h->d_mu_tables = nullptr; h->cap_mu_tables = 0;
    CU_TRY(cudaMalloc(&h->d_mu_tables, tab.size() * sizeof(double)));
    h->cap_mu_tables = tab.size();
  }
  CU_TRY(cudaMemcpy(h->d_mu_tables, tab.data(), tab.size() * sizeof(double), cudaMemcpyHostToDevice));
  const size_t pix = (size_t)c->image.n_rows * c->image.n_cols;
  if (pix > h->cap_mu_image) {
    cudaFree(h->d_mu_image); cudaFree(h->d_mu_window); h->d_mu_image = nullptr; h->d_mu_window = nullptr;
    h->cap_mu_image = 0;
    CU_TRY(cudaMalloc(&h->d_mu_image, pix * sizeof(unsigned long long)));
    CU_TRY(cudaMalloc(&h->d_mu_window, pix * sizeof(double)));
    h->cap_mu_image = pix;
  }
  if (!h->d_mu_small) CU_TRY(cudaMalloc(&h->d_mu_small, kMuSmall));
  mu_free_retired(h);                                           // the stream is idle
  h->mu_cfg = *c;
  h->mu_on = true;
  h->mu_fresh = true; h->mu_frames = 0; h->mu_built = false;
  h->mu_min_serial = h->loc_serial + 1;                         // the next localization is the first an add may use
  return mu_prior_alloc(h);
}

static int mu_after_load(tloam_b200_handle* h, int rc) {
  if (rc != TLOAM_B200_OK || !h->mu_on) return rc;
  mu_free_retired(h);                                           // the load synchronised
  return mu_prior_alloc(h);
}

// an empty state: the prior rows' counters (loc_n of them, sized by the enable or the load) and the additions' count
// cleared on the stream
static int mu_reset(tloam_b200_handle* h) {
  if (!h->mu_fresh) return TLOAM_B200_OK;
  const size_t n = h->loc_n;
  int rc;
  if ((rc = mu_prior_alloc(h)) != TLOAM_B200_OK) return rc;     // sized already by the enable or the load
  if (n) {
    CU_TRY(cudaMemsetAsync(h->d_mu_prior, 0, n * sizeof(unsigned), h->stream));
    CU_TRY(cudaMemsetAsync(h->d_mu_prior + h->cap_mu_prior, 0, n * sizeof(unsigned), h->stream));
  }
  CU_TRY(cudaMemsetAsync(mu_word(h, 1), 0, sizeof(unsigned long long), h->stream));
  h->mu_known = 0; h->mu_pending = 0; h->mu_fresh = false;
  return TLOAM_B200_OK;
}

// adds of the current query size the additions keep room for after a read-back of their count
constexpr size_t kMuHeadroom = 16;

// the additions hold at least `need` more rows.  The host bounds their count by the count at the last read-back plus the
// query rows of every add since; only when that bound passes the capacity is the count read back (the add's one
// synchronisation).  If the rows left then are fewer than kMuHeadroom adds of this size, the buffer grows (the rows copied
// on the stream, the old buffer freed at a later synchronisation), so a read-back comes at most once per kMuHeadroom adds.
static int mu_reserve(tloam_b200_handle* h, size_t need) {
  if (h->mu_known + h->mu_pending + need <= h->cap_mu_add) return TLOAM_B200_OK;
  if (h->mu_pending) {
    unsigned long long n = 0;
    CU_TRY(cudaMemcpyAsync(&n, mu_word(h, 1), sizeof(n), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    h->mu_known = (size_t)n; h->mu_pending = 0;
    mu_free_retired(h);
  }
  if (h->cap_mu_add - h->mu_known >= kMuHeadroom * need) return TLOAM_B200_OK;
  const size_t cap = std::max(2 * h->cap_mu_add, h->mu_known + h->mu_known / 2 + kMuHeadroom * need);
  unsigned char* p = nullptr;
  CU_TRY(cudaMalloc(&p, mu_add_bytes(cap)));
  if (h->mu_known) {
    const MuAdd o = mu_add_of(h->d_mu_add, h->cap_mu_add), q = mu_add_of(p, cap);
    const size_t k = h->mu_known;
    CU_TRY(cudaMemcpyAsync(q.xyz, o.xyz, k * 24, cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaMemcpyAsync(q.frame, o.frame, k * 4, cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaMemcpyAsync(q.through, o.through, k * 4, cudaMemcpyDeviceToDevice, h->stream));
    CU_TRY(cudaMemcpyAsync(q.hits, o.hits, k * 4, cudaMemcpyDeviceToDevice, h->stream));
  }
  if (h->d_mu_add) h->mu_retired.push_back(h->d_mu_add);
  h->d_mu_add = p; h->cap_mu_add = cap;
  return TLOAM_B200_OK;
}

int tloam_b200_map_update_add(tloam_b200_handle* h, tloam_map_update_add_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  memset(out, 0, sizeof(*out));
  out->frame = -1;
  if (!h->mu_on || !h->loc_loaded || !h->loc_ran || !h->loc_src || h->loc_serial < h->mu_min_serial ||
      h->loc_serial == h->mu_added_serial)
    return TLOAM_B200_ERR_NOT_READY;
  // the scan the localization read is still in place (tloam_b200_global_map_append_frame's rule for the raw scan)
  if (h->loc_src_raw ? (h->raw_gen != h->seg_gen || h->raw_gen != h->loc_src_gen) : h->loc_in_gen != h->loc_src_gen)
    return TLOAM_B200_ERR_NOT_READY;
  if (!h->loc_accepted) return TLOAM_B200_OK;
  GmdLib gmd;
  MuLib lib;
  int rc;
  if ((rc = gmd_load(h, &gmd)) != TLOAM_B200_OK || (rc = mu_load(h, &lib)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  if ((rc = mu_reset(h)) != TLOAM_B200_OK) return rc;
  const size_t nq = h->loc_nq;
  if ((rc = mu_reserve(h, nq)) != TLOAM_B200_OK) return rc;
  const size_t q_bytes = round_up(nq, 256) + round_up(nq * 24, 256) + TLOAM_MU_MAX_BLOCKS * 4;
  if (q_bytes > h->cap_mu_q) {                                  // the old buffer may still be read by the last add
    if (h->d_mu_q) h->mu_retired.push_back(h->d_mu_q);
    h->d_mu_q = nullptr; h->cap_mu_q = 0;
    CU_TRY(cudaMalloc(&h->d_mu_q, q_bytes + q_bytes / 2));
    h->cap_mu_q = q_bytes + q_bytes / 2;
  }
  const MuAdd ad = mu_add_of(h->d_mu_add, h->cap_mu_add);
  tloam_mu_add_args a;
  memset(&a, 0, sizeof(a));
  a.grid = h->loc_index.grid;
  a.query = h->d_loc_q; a.nq = nq;
  a.state = h->loc_last.state;
  a.radius = h->mu_cfg.novel_radius;
  a.n_prior = h->loc_n;
  a.pose = mu_pose(h); a.prior_count = mu_word(h, 0);
  a.flag = h->d_mu_q;
  a.p = reinterpret_cast<double*>(h->d_mu_q + round_up(nq, 256));
  a.block_counts = reinterpret_cast<unsigned*>(h->d_mu_q + round_up(nq, 256) + round_up(nq * 24, 256));
  a.base = mu_word(h, 2); a.count = mu_word(h, 1);
  a.add_xyz = ad.xyz; a.add_frame = ad.frame; a.add_through = ad.through; a.add_hits = ad.hits;
  a.frame = h->mu_frames;
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.pose(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = mu_status(h, e, "k_mu_pose")) != TLOAM_B200_OK) return rc;
  // the votes: the scan rows at T on the prior rows, then on the additions of the earlier adds
  const tloam_global_map_dynamic_config& c = h->mu_cfg.image;
  tloam_gmd_vote_args v;
  memset(&v, 0, sizeof(v));
  v.p.n_rows = c.n_rows; v.p.n_cols = c.n_cols; v.p.wr = c.window_rows; v.p.wc = c.window_cols;
  v.p.margin_abs = c.margin_abs; v.p.margin_rel = c.margin_rel; v.p.min_range = c.min_range; v.p.max_range = c.max_range;
  v.p.row_bounds = h->d_mu_tables; v.p.col_bounds = h->d_mu_tables + (c.n_rows + 1);
  v.scan = h->loc_src; v.n = (unsigned)h->loc_src_n; v.pose = mu_pose(h);
  v.image = h->d_mu_image; v.window = h->d_mu_window;
  v.device = h->device; v.stream = h->stream;
  for (int which = 0; which < 2; ++which) {
    v.map = which ? ad.xyz : h->loc_index.map;
    v.count = which ? mu_word(h, 1) : mu_word(h, 0);
    v.through = which ? ad.through : h->d_mu_prior;
    v.hits = which ? ad.hits : h->d_mu_prior + h->cap_mu_prior;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = gmd.vote(&v, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = gmd_status(h, e, "k_gmd_vote")) != TLOAM_B200_OK) return rc;
  }
  if (nq) {
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = lib.novel(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = mu_status(h, e, "k_mu_novel / k_mu_count / k_mu_scatter")) != TLOAM_B200_OK) return rc;
  }
  out->used = 1;
  out->frame = (long long)h->mu_frames;
  out->n_scan_points = (long long)h->loc_src_n;
  out->n_query_points = (long long)nq;
  h->mu_frames++;
  h->mu_pending += nq;
  h->mu_added_serial = h->loc_serial;
  return TLOAM_B200_OK;
}

// the additions' count (synchronises)
static int mu_count(tloam_b200_handle* h, size_t* n) {
  *n = 0;
  if (h->mu_fresh) return TLOAM_B200_OK;
  unsigned long long c = 0;
  CU_TRY(cudaMemcpyAsync(&c, mu_word(h, 1), sizeof(c), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  mu_free_retired(h);
  h->mu_known = (size_t)c; h->mu_pending = 0;
  *n = (size_t)c;
  return TLOAM_B200_OK;
}

int tloam_b200_map_update_build(tloam_b200_handle* h, tloam_map_update_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  memset(out, 0, sizeof(*out));
  if (!h->mu_on || !h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  GmdLib gmd;
  MuLib lib;
  int rc;
  if ((rc = gmd_load(h, &gmd)) != TLOAM_B200_OK || (rc = mu_load(h, &lib)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  h->mu_built = false;                                          // a refused build leaves no cloud
  if ((rc = mu_reset(h)) != TLOAM_B200_OK) return rc;
  size_t n_add = 0;
  if ((rc = mu_count(h, &n_add)) != TLOAM_B200_OK) return rc;
  const size_t n_prior = h->loc_n, rows = n_prior + n_add;
  if (rows * 3 > h->cap_mu_out) {
    cudaFree(h->d_mu_out); h->d_mu_out = nullptr; h->cap_mu_out = 0;
    CU_TRY(cudaMalloc(&h->d_mu_out, (rows + rows / 2 + 1) * 3 * sizeof(double)));
    h->cap_mu_out = (rows + rows / 2 + 1) * 3;
  }
  const size_t bytes = lib.scratch_bytes(n_add);
  if (bytes > h->cap_mu_build) {
    cudaFree(h->d_mu_build); h->d_mu_build = nullptr; h->cap_mu_build = 0;
    CU_TRY(cudaMalloc(&h->d_mu_build, bytes + bytes / 2));
    h->cap_mu_build = bytes + bytes / 2;
  }
  int e = 0, launches = 0;
  // the prior rows that are not removed, in row order, at the start of the cloud; their count in word 3
  unsigned long long* total = mu_word(h, 3);
  if (n_prior) {
    tloam_gmd_static_args s;
    memset(&s, 0, sizeof(s));
    s.map = h->loc_index.map; s.through = h->d_mu_prior; s.hits = h->d_mu_prior + h->cap_mu_prior;
    s.count = n_prior; s.min_through = (unsigned)h->mu_cfg.image.min_through;
    s.block_counts = reinterpret_cast<unsigned*>(h->d_mu_small + 1024);
    s.total = total; s.out_xyz = h->d_mu_out;
    s.device = h->device; s.stream = h->stream;
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = gmd.compact(&s, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    if ((rc = gmd_status(h, e, "k_gmd_count / k_gmd_scatter")) != TLOAM_B200_OK) return rc;
  } else {
    CU_TRY(cudaMemsetAsync(total, 0, sizeof(unsigned long long), h->stream));
  }
  const MuAdd ad = mu_add_of(h->d_mu_add, h->cap_mu_add);
  tloam_mu_build_args a;
  memset(&a, 0, sizeof(a));
  a.add_xyz = ad.xyz; a.add_frame = ad.frame; a.add_through = ad.through; a.add_hits = ad.hits;
  a.n_add = n_add;
  a.min_through = (unsigned)h->mu_cfg.image.min_through; a.min_frames = (unsigned)h->mu_cfg.min_frames;
  a.voxel = h->mu_cfg.voxel;
  a.scratch = h->d_mu_build; a.state = lib.state_of(h->d_mu_build, n_add);
  a.count = total; a.out_xyz = h->d_mu_out;
  a.device = h->device; a.stream = h->stream;
  auto run = [&](tloam_mu_build_fn f, const char* where) -> int {
    TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = f(&a, &launches)));
    h->launches += launches > 0 ? launches - 1 : 0;
    return mu_status(h, e, where);
  };
  if ((rc = run(lib.bounds, "k_mu_bounds")) != TLOAM_B200_OK) return rc;
  tloam_gmm_state gs;
  unsigned long long kept_prior = 0;
  CU_TRY(cudaMemcpyAsync(&gs, a.state, sizeof(gs), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaMemcpyAsync(&kept_prior, total, sizeof(kept_prior), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (gs.nonfinite) return TLOAM_B200_ERR_VOXEL_RANGE;
  unsigned long long n_vox = 0, n_total = kept_prior;
  if (gs.n_sel) {
    for (int d = 0; d < 3; ++d) {                               // the merge's bounds, key range and bits
      const double half = a.voxel * 0.5;
      a.mb[d] = dec_ordered(~gs.lo[d]) - half;
      const double ref = (dec_ordered(gs.hi[d]) - a.mb[d]) / a.voxel;
      if (!(ref < (double)(1u << kGMapKeyBits))) return TLOAM_B200_ERR_VOXEL_RANGE;
      const unsigned long long top = (unsigned long long)std::floor(ref);
      int bits = 0;
      while (bits < 64 && (top >> bits)) ++bits;
      a.bits[d] = bits;
    }
    a.n_sel = gs.n_sel;
    if ((rc = run(lib.sort, "k_mu_keys / k_gmm_*")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaMemcpyAsync(&n_vox, &a.state->n_vox, sizeof(n_vox), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
    a.n_vox = n_vox;
    if ((rc = run(lib.average, "k_mu_average / k_mu_count / k_mu_scatter")) != TLOAM_B200_OK) return rc;
    CU_TRY(cudaMemcpyAsync(&n_total, total, sizeof(n_total), cudaMemcpyDeviceToHost, h->stream));
    CU_TRY(cudaStreamSynchronize(h->stream));
  }
  out->n_prior = (long long)n_prior;
  out->n_prior_removed = (long long)(n_prior - kept_prior);
  out->n_additions = (long long)n_add;
  out->n_additions_removed = (long long)(n_add - gs.n_sel);
  out->n_voxels = (long long)n_vox;
  out->n_voxels_kept = (long long)(n_total - kept_prior);
  out->n_total = (long long)n_total;
  h->mu_built = true; h->mu_built_n = (size_t)n_total;
  return TLOAM_B200_OK;
}

int tloam_b200_map_update_size(tloam_b200_handle* h, size_t* n_prior, size_t* n_additions, size_t* n_built) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->mu_on || !h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  size_t n = 0;
  int rc;
  if ((rc = mu_count(h, &n)) != TLOAM_B200_OK) return rc;
  if (n_prior) *n_prior = h->loc_n;
  if (n_additions) *n_additions = n;
  if (n_built) *n_built = h->mu_built ? h->mu_built_n : 0;
  return TLOAM_B200_OK;
}

int tloam_b200_map_update_download(tloam_b200_handle* h, size_t first, size_t count, double* xyz) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->mu_on || !h->mu_built) return TLOAM_B200_ERR_NOT_READY;
  if (first > h->mu_built_n || count > h->mu_built_n - first || (count && !xyz)) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  if (count) CU_TRY(cudaMemcpyAsync(xyz, h->d_mu_out + 3 * first, count * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_map_update_votes(tloam_b200_handle* h, int which, size_t first, size_t count, unsigned* through, unsigned* hits) {
  if (!h || (which != 0 && which != 1)) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->mu_on || !h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  size_t n = 0;
  int rc;
  if ((rc = mu_count(h, &n)) != TLOAM_B200_OK) return rc;
  const size_t rows = which ? n : h->loc_n;
  if (first > rows || count > rows - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (!count) return TLOAM_B200_OK;
  if (h->mu_fresh) {                                            // nothing voted since the state was emptied
    if (through) memset(through, 0, count * sizeof(unsigned));
    if (hits) memset(hits, 0, count * sizeof(unsigned));
    return TLOAM_B200_OK;
  }
  const MuAdd ad = mu_add_of(h->d_mu_add, h->cap_mu_add);
  const unsigned* t = which ? ad.through : h->d_mu_prior;
  const unsigned* s = which ? ad.hits : h->d_mu_prior + h->cap_mu_prior;
  if (through) CU_TRY(cudaMemcpyAsync(through, t + first, count * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  if (hits) CU_TRY(cudaMemcpyAsync(hits, s + first, count * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_map_update_additions(tloam_b200_handle* h, size_t first, size_t count, double* xyz, unsigned* frame) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->mu_on || !h->loc_loaded) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  size_t n = 0;
  int rc;
  if ((rc = mu_count(h, &n)) != TLOAM_B200_OK) return rc;
  if (first > n || count > n - first) return TLOAM_B200_ERR_INVALID_ARG;
  if (!count) return TLOAM_B200_OK;
  const MuAdd ad = mu_add_of(h->d_mu_add, h->cap_mu_add);
  if (xyz) CU_TRY(cudaMemcpyAsync(xyz, ad.xyz + 3 * first, count * 24, cudaMemcpyDeviceToHost, h->stream));
  if (frame) CU_TRY(cudaMemcpyAsync(frame, ad.frame + first, count * sizeof(unsigned), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_localize_set_map_updated(tloam_b200_handle* h) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->loc_on || !h->mu_on || !h->mu_built) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  const size_t n = h->mu_built_n;
  h->loc_loaded = false; h->loc_have_prev = false; h->loc_ran = false; h->loc_passes = 0;
  h->mu_fresh = true; h->mu_frames = 0;
  int rc;
  if ((rc = loc_reserve_map(h, n)) != TLOAM_B200_OK) return rc;
  if (n) CU_TRY(cudaMemcpyAsync(h->d_loc_map, h->d_mu_out, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  return mu_after_load(h, loc_build(h, n));
}

// ---------------------------------------------------------------------------------------------
// Global registration (the checks, the keypoints' down-sample, the loader and the buffers here; each side's index and
// normals from localize.cu's tloam_loc_index, the rest in global_registration.cu, loaded from libtloam_b200_greg.so by
// the enable call).
// ---------------------------------------------------------------------------------------------
static std::mutex g_gr_mu;
static tloam_gr_run_fn g_gr_run = nullptr;

static int gr_load(tloam_b200_handle* h, tloam_gr_run_fn* out) {
  std::lock_guard<std::mutex> lk(g_gr_mu);
  if (!g_gr_run) {
    const std::string path = sibling_path("libtloam_b200_greg.so");
    void* so = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    tloam_gr_run_fn f = so ? reinterpret_cast<tloam_gr_run_fn>(dlsym(so, "tloam_gr_run")) : nullptr;
    if (!f) {
      const char* why = dlerror();
      snprintf(h->last_error, sizeof(h->last_error), "global registration: cannot load %s: %s", path.c_str(), why ? why : "missing symbol");
      if (so) dlclose(so);
      return TLOAM_B200_ERR_CUDA;
    }
    g_gr_run = f;
  }
  *out = g_gr_run;
  return TLOAM_B200_OK;
}

static int gr_status(tloam_b200_handle* h, int e, const char* where) {
  if (e == cudaSuccess) return TLOAM_B200_OK;
  snprintf(h->last_error, sizeof(h->last_error), "global registration: %s: %s", where, cudaGetErrorString((cudaError_t)e));
  return TLOAM_B200_ERR_CUDA;
}

void tloam_b200_global_registration_default_config(tloam_global_registration_config* c) {
  c->voxel = 0.5; c->cell = 1.0; c->normal_radius = 1.0; c->min_normal_neighbours = 5; c->feature_radius = 2.5;
  c->max_correspondence_distance = 0.75; c->n_hypotheses = 65536; c->seed = 0; c->edge_similarity = 0.9;
  c->min_triangle_area = 1.0; c->max_refine_iterations = 10; c->min_inliers = 30; c->min_fitness = 0.3;
}

int tloam_b200_global_registration_enable(tloam_b200_handle* h, const tloam_global_registration_config* c) {
  if (!h || !c) return TLOAM_B200_ERR_INVALID_ARG;
  const double v[7] = {c->voxel, c->cell, c->normal_radius, c->feature_radius, c->max_correspondence_distance, c->edge_similarity,
                       c->min_triangle_area};
  for (double x : v)
    if (!std::isfinite(x) || !(x > 0.0)) return TLOAM_B200_ERR_INVALID_ARG;
  if (c->min_normal_neighbours < 3 || c->normal_radius > 3.0 * c->cell || c->feature_radius > 3.0 * c->cell ||
      c->n_hypotheses < 1 || c->n_hypotheses > (1 << 20) || c->edge_similarity > 1.0 || c->max_refine_iterations < 1 ||
      c->max_refine_iterations > 100 || c->min_inliers < 0 || !(c->min_fitness >= 0.0 && c->min_fitness <= 1.0))
    return TLOAM_B200_ERR_INVALID_ARG;
  tloam_gr_run_fn run;
  int rc = gr_load(h, &run);
  if (rc != TLOAM_B200_OK) return rc;
  LocLib lib;
  if ((rc = loc_load(h, &lib)) != TLOAM_B200_OK) return rc;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!h->d_gr_small) {
    CU_TRY(cudaMalloc(&h->d_gr_small, 512));
    const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    CU_TRY(cudaMemcpy(h->d_gr_small + 256, eye, sizeof(eye), cudaMemcpyHostToDevice));
  }
  h->gr_cfg = *c;
  h->gr_on = true;
  h->gr_ran = false; h->gr_nc = 0; h->gr_nh = 0;
  return TLOAM_B200_OK;
}

// a host cloud's keypoints: the finite rows of the n rows at d_in down-sampled as loc_query does, in this feature's
// buffers, into d_gr_q; synchronises and returns their count
static int gr_query(tloam_b200_handle* h, const double* d_in, size_t n, size_t* nq) {
  return ordered_query(h, d_in, n, h->gr_cfg.voxel, reinterpret_cast<const double*>(h->d_gr_small + 256), &h->d_gr_reg,
                       &h->cap_gr_reg, &h->d_gr_fin, &h->cap_gr_fin, reinterpret_cast<GMapState*>(h->d_gr_small), &h->d_gr_q,
                       &h->cap_gr_q, nq);
}

// side k: the n keypoints at d_pts copied into its buffer and indexed with normals as a localization map is
// (loc_carve_index / loc_index_build, max_planarity 1), then the feature's arrays; synchronises after the bounds
static int gr_side(tloam_b200_handle* h, int k, const double* d_pts, size_t n, tloam_gr_side* out) {
  LocLib lib;
  int rc = loc_load(h, &lib);
  if (rc != TLOAM_B200_OK) return rc;
  const size_t base = loc_carve_index(nullptr, n, nullptr);
  const size_t need = base + round_up(n * TLOAM_GR_BINS * 4, 256) + round_up(n * 4, 256) + round_up(n * TLOAM_GR_BINS * 8, 256) +
                      round_up(n, 256) + n * 4;
  if (need > h->cap_gr_side[k]) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gr_side[k]); h->d_gr_side[k] = nullptr; h->cap_gr_side[k] = 0;
    CU_TRY(cudaMalloc(&h->d_gr_side[k], need));
    h->cap_gr_side[k] = need;
  }
  unsigned char* b = h->d_gr_side[k];
  tloam_loc_index_args a;
  memset(&a, 0, sizeof(a));
  memset(out, 0, sizeof(*out));
  size_t o = loc_carve_index(b, n, &a);
  out->spfh = reinterpret_cast<int*>(b + o);        o += round_up(n * TLOAM_GR_BINS * 4, 256);
  out->pairs = reinterpret_cast<int*>(b + o);       o += round_up(n * 4, 256);
  out->feature = reinterpret_cast<double*>(b + o);  o += round_up(n * TLOAM_GR_BINS * 8, 256);
  out->has_feature = b + o;                         o += round_up(n, 256);
  out->nn = reinterpret_cast<int*>(b + o);
  if (n) CU_TRY(cudaMemcpyAsync(const_cast<double*>(a.map), d_pts, n * 24, cudaMemcpyDeviceToDevice, h->stream));
  const tloam_global_registration_config& c = h->gr_cfg;
  if ((rc = loc_index_build(h, lib, a, n, c.cell, c.normal_radius, 1.0, c.min_normal_neighbours, &h->d_gr_scratch,
                            &h->cap_gr_scratch)) != TLOAM_B200_OK)
    return rc;
  out->grid = a.grid;
  out->xyz = a.map; out->normal = a.normal; out->valid = a.valid; out->n = n;
  return TLOAM_B200_OK;
}

// the run over the two sides built by gr_side; one copy of the state home
static int gr_run(tloam_b200_handle* h, tloam_gr_side src, tloam_gr_side tgt, tloam_global_registration_result* out) {
  tloam_gr_run_fn run;
  int rc = gr_load(h, &run);
  if (rc != TLOAM_B200_OK) return rc;
  const tloam_global_registration_config& c = h->gr_cfg;
  memset(out, 0, sizeof(*out));
  out->T[0] = out->T[5] = out->T[10] = out->T[15] = 1.0;
  out->n_source_points = (long long)src.n; out->n_target_points = (long long)tgt.n;
  out->best_hypothesis = -1;
  tloam_gr_args a;
  memset(&a, 0, sizeof(a));
  a.src = src; a.tgt = tgt;
  h->gr_last = a; h->gr_ran = true; h->gr_nc = 0; h->gr_nh = 0;
  if (!src.n || !tgt.n) {
    out->termination = TLOAM_GLOBAL_REGISTRATION_EMPTY;
    return TLOAM_B200_OK;
  }
  const size_t ns = src.n, nh = (size_t)c.n_hypotheses;
  const size_t o_corr = round_up(sizeof(tloam_gr_state), 256);
  const size_t o_hyp = o_corr + round_up(ns * 2 * sizeof(int), 256);
  const size_t o_set = o_hyp + round_up(nh * sizeof(int), 256);
  const size_t bytes = o_set + 2 * ns;
  if (bytes > h->cap_gr_run) {
    CU_TRY(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gr_run); h->d_gr_run = nullptr; h->cap_gr_run = 0;
    CU_TRY(cudaMalloc(&h->d_gr_run, bytes));
    h->cap_gr_run = bytes;
  }
  unsigned char* base = h->d_gr_run;
  a.state = reinterpret_cast<tloam_gr_state*>(base);
  a.src.n_features = &a.state->n_features[0];
  a.tgt.n_features = &a.state->n_features[1];
  a.feature_radius = c.feature_radius; a.tau = c.max_correspondence_distance;
  for (int k = 0; k < 10; ++k) {   // volatile: the boundaries' cos and sin from the C library at run time, never folded
    volatile double beta = (2.0 * (k + 1) / 11.0 - 1.0) * M_PI;
    a.theta_cs[2 * k] = std::cos(beta);
    a.theta_cs[2 * k + 1] = std::sin(beta);
  }
  a.n_hypotheses = c.n_hypotheses; a.seed = c.seed;
  a.edge_similarity = c.edge_similarity; a.min_triangle_area = c.min_triangle_area;
  a.max_refine_iterations = c.max_refine_iterations;
  a.corr = reinterpret_cast<int*>(base + o_corr);
  a.hyp_inliers = reinterpret_cast<int*>(base + o_hyp);
  a.in_set = base + o_set;
  a.device = h->device; a.stream = h->stream;
  int e = 0, launches = 0;
  TL_LAUNCH(TLOAM_B200_K_SUBMAP, (e = run(&a, &launches)));
  h->launches += launches > 0 ? launches - 1 : 0;
  if ((rc = gr_status(h, e, "k_gr_*")) != TLOAM_B200_OK) return rc;
  tloam_gr_state s;
  CU_TRY(cudaMemcpyAsync(&s, a.state, sizeof(s), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (int r = 0; r < 3; ++r) {
    for (int j = 0; j < 3; ++j) out->T[4 * j + r] = s.R[3 * r + j];
    out->T[12 + r] = s.t[r];
  }
  out->n_source_features = (long long)s.n_features[0]; out->n_target_features = (long long)s.n_features[1];
  out->n_correspondences = (long long)s.n_corr;
  out->n_valid_hypotheses = s.n_valid; out->best_hypothesis = s.best; out->best_inliers = s.best_inliers;
  out->inliers = s.inliers; out->inlier_rmse = s.rmse; out->refine_iterations = s.iterations; out->termination = s.term;
  out->fitness = (double)s.fit_count / (double)src.n;
  out->accepted = out->inliers >= c.min_inliers && out->fitness >= c.min_fitness ? 1 : 0;
  h->gr_last = a; h->gr_nc = s.n_corr; h->gr_nh = c.n_hypotheses;
  return TLOAM_B200_OK;
}

int tloam_b200_global_register(tloam_b200_handle* h, const double* src, size_t n_src, const double* tgt, size_t n_tgt,
                               tloam_global_registration_result* out) {
  if (!h || !out || (!src && n_src) || (!tgt && n_tgt) || n_src > ((size_t)1 << 30) || n_tgt > ((size_t)1 << 30))
    return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gr_on) return TLOAM_B200_ERR_NOT_READY;
  CU_TRY(cudaSetDevice(h->device));
  h->gr_ran = false;
  tloam_gr_side side[2];
  const double* cloud[2] = {src, tgt};
  const size_t n[2] = {n_src, n_tgt};
  int rc;
  for (int k = 0; k < 2; ++k) {
    if ((rc = ensure_dev(h, &h->d_gr_in, &h->cap_gr_in, n[k], false)) != TLOAM_B200_OK) return rc;
    if (n[k] && (rc = upload_host(h, h->d_gr_in, cloud[k], n[k] * 24)) != TLOAM_B200_OK) return rc;
    size_t nq = 0;
    if ((rc = gr_query(h, h->d_gr_in, n[k], &nq)) != TLOAM_B200_OK) return rc;
    if ((rc = gr_side(h, k, h->d_gr_q, nq, &side[k])) != TLOAM_B200_OK) return rc;
  }
  return gr_run(h, side[0], side[1], out);
}

int tloam_b200_global_register_loop(tloam_b200_handle* h, long long query, long long candidate,
                                    tloam_global_registration_result* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gr_on || !h->lv_on) return TLOAM_B200_ERR_NOT_READY;
  if (query < 0 || candidate < 0 || (size_t)query >= h->loop_frames || (size_t)candidate >= h->loop_frames)
    return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  h->gr_ran = false;
  tloam_gr_side side[2];
  const long long f[2] = {query, candidate};
  int rc;
  for (int k = 0; k < 2; ++k) {
    unsigned long long first = 0, cnt = 0;
    if ((rc = lv_range(h, (size_t)f[k], &first, &cnt)) != TLOAM_B200_OK) return rc;
    if ((rc = gr_side(h, k, h->d_lv_pts + 3 * first, cnt, &side[k])) != TLOAM_B200_OK) return rc;
  }
  return gr_run(h, side[0], side[1], out);
}

int tloam_b200_global_registration_side(tloam_b200_handle* h, int side, double* xyz, double* normal, unsigned char* valid,
                                        int* spfh, double* feature, unsigned char* has_feature, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gr_on || !h->gr_ran) return TLOAM_B200_ERR_NOT_READY;
  if (side != 0 && side != 1) return TLOAM_B200_ERR_INVALID_ARG;
  const tloam_gr_side& s = side ? h->gr_last.tgt : h->gr_last.src;
  const size_t m = s.n;
  *n = m;
  if (capacity < m) return TLOAM_B200_ERR_INVALID_ARG;
  if (!m) return TLOAM_B200_OK;
  const bool featured = h->gr_nh > 0;                        // an EMPTY run computed no feature
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (xyz) CU_TRY(cudaMemcpyAsync(xyz, s.xyz, m * 24, cudaMemcpyDeviceToHost, h->stream));
  if (normal) CU_TRY(cudaMemcpyAsync(normal, s.normal, m * 24, cudaMemcpyDeviceToHost, h->stream));
  if (valid) CU_TRY(cudaMemcpyAsync(valid, s.valid, m, cudaMemcpyDeviceToHost, h->stream));
  if (featured && spfh) CU_TRY(cudaMemcpyAsync(spfh, s.spfh, m * TLOAM_GR_BINS * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  if (featured && feature) CU_TRY(cudaMemcpyAsync(feature, s.feature, m * TLOAM_GR_BINS * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (featured && has_feature) CU_TRY(cudaMemcpyAsync(has_feature, s.has_feature, m, cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  if (!featured) {
    if (spfh) memset(spfh, 0, m * TLOAM_GR_BINS * sizeof(int));
    if (feature) memset(feature, 0, m * TLOAM_GR_BINS * sizeof(double));
    if (has_feature) memset(has_feature, 0, m);
  }
  return TLOAM_B200_OK;
}

int tloam_b200_global_registration_correspondences(tloam_b200_handle* h, int* pairs, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gr_on || !h->gr_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = h->gr_nc;
  if (capacity < h->gr_nc) return TLOAM_B200_ERR_INVALID_ARG;
  if (!pairs || !h->gr_nc) return TLOAM_B200_OK;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(pairs, h->gr_last.corr, h->gr_nc * 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_global_registration_hypotheses(tloam_b200_handle* h, int* inliers, size_t capacity, size_t* n) {
  if (!h || !n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!h->gr_on || !h->gr_ran) return TLOAM_B200_ERR_NOT_READY;
  *n = (size_t)h->gr_nh;
  if (capacity < *n) return TLOAM_B200_ERR_INVALID_ARG;
  if (!inliers || !*n) return TLOAM_B200_OK;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaMemcpyAsync(inliers, h->gr_last.hyp_inliers, *n * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU_TRY(cudaStreamSynchronize(h->stream));
  return TLOAM_B200_OK;
}

int tloam_b200_host_alloc(void** p, size_t bytes) {
  if (!p) return TLOAM_B200_ERR_INVALID_ARG;
  return cudaMallocHost(p, bytes) == cudaSuccess ? TLOAM_B200_OK : TLOAM_B200_ERR_CUDA;
}
int tloam_b200_host_free(void* p) { return cudaFreeHost(p) == cudaSuccess ? TLOAM_B200_OK : TLOAM_B200_ERR_CUDA; }

const char* tloam_b200_last_error(tloam_b200_handle* h) { return h ? h->last_error : ""; }

int tloam_b200_set_profiling(tloam_b200_handle* h, int on) {
  if (!h) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  h->profiling = on != 0;
  h->spans.clear(); h->ev_next = 0;
  memset(&h->prof, 0, sizeof(h->prof));
  if (on && !h->d_dbg) CU_TRY(cudaMalloc(&h->d_dbg, 16 * sizeof(unsigned long long)));
  if (h->d_dbg) {
    unsigned long long init[16];
    memset(init, 0, sizeof(init));
    init[0] = ~0ull;
    CU_TRY(cudaMemcpy(h->d_dbg, init, sizeof(init), cudaMemcpyHostToDevice));
  }
  h->ctx.dbg = on ? h->d_dbg : nullptr;
  return TLOAM_B200_OK;
}

int tloam_b200_get_profile(tloam_b200_handle* h, tloam_b200_profile* out) {
  if (!h || !out) return TLOAM_B200_ERR_INVALID_ARG;
  CU_TRY(cudaSetDevice(h->device));
  CU_TRY(cudaStreamSynchronize(h->stream));
  for (const auto& sp : h->spans) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, sp.a, sp.b) == cudaSuccess && sp.cls >= 0 && sp.cls < TLOAM_B200_K_COUNT) {
      h->prof.launches[sp.cls] += 1;
      h->prof.total_ms[sp.cls] += ms;
    }
  }
  h->spans.clear(); h->ev_next = 0;
  if (h->d_dbg) CU_TRY(cudaMemcpy(h->prof.dbg, h->d_dbg, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  *out = h->prof;
  return TLOAM_B200_OK;
}

}  // extern "C"
