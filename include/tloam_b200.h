/*
 * tloam_b200.h -- C ABI of the H100-native TLS scan-to-map registration library (libtloam_b200.so).
 *
 * This is the drop-in boundary for T-LOAM's pose-optimisation hot path.  Each entry point names the
 * reference interface it replaces ("ref:" paths are relative to the zhoupengwei/tloam tree):
 *
 *   tloam_b200_create           <- LocalRegistration::LocalRegistration(YAML::Node) + initConfig
 *                                  ref: src/models/registration/registration.cpp:182-230
 *   tloam_b200_set_source       <- RegistrationInterface::setInputSource(Frame&)
 *                                  ref: include/tloam/models/registration/registration_interface.hpp:44,
 *                                       registration.cpp:232-239
 *   tloam_b200_set_target       <- RegistrationInterface::setInputTarget(Frame&)   (+ the per-call KD-tree
 *                                  rebuild of registration.cpp:888-915, done ONCE per map here)
 *                                  ref: registration_interface.hpp:45, registration.cpp:241-248
 *   tloam_b200_scan_match       <- RegistrationInterface::scanMatching(Frame&, Isometry3d&, Isometry3d&)
 *                                  ref: registration_interface.hpp:46, registration.cpp:879-1133
 *   tloam_b200_fitness          <- RegistrationInterface::getFitnessScore()
 *                                  ref: registration_interface.hpp:47, registration.cpp:257-296
 *   tloam_b200_get_transform / _get_pose_increment <- getTransform() / getPoseIncrement()
 *                                  ref: registration.cpp:370-376
 *   tloam_b200_eval_point_to_{point,line,plane}    <- PointTo{Point,Line,Plane}Err::Evaluate
 *                                  ref: registration.cpp:19-47, 55-88, 96-117
 *
 * Conventions
 *   - clouds: contiguous AoS FP64 xyz (the layout of std::vector<Eigen::Vector3d>,
 *     ref: include/tloam/open3d/PointCloud2.hpp:396); array index 0..3 = edge, sphere, planar, ground
 *     (order of registration.cpp:233-236).
 *   - poses: 4x4 FP64 COLUMN-major (Eigen::Isometry3d::matrix().data()).
 *   - HOST inputs are copied at set_*(): caller buffers may be freed on return (unless tloam_b200_set_async_inputs).
 *     DEVICE inputs (set_*_device) are read in place by kernels on the handle's stream: keep them unchanged until
 *     that work has run, and order their producer with tloam_b200_wait_stream.
 *   - one handle = one CUDA device + one stream, single caller, not re-entrant (like the reference,
 *     ref: registration.hpp:327-329).  Distinct handles are independent.
 *   - no function aborts or throws; all return a tloam_b200_status.  There is NO CPU fallback: without a
 *     CUDA device tloam_b200_create returns TLOAM_B200_ERR_NO_DEVICE.
 */
#ifndef TLOAM_B200_H
#define TLOAM_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TLOAM_B200_MAX_OUTER 16
#define TLOAM_B200_MAX_INNER 8

typedef struct tloam_b200_handle tloam_b200_handle;

typedef enum tloam_b200_status {
  TLOAM_B200_OK = 0,
  TLOAM_B200_ERR_INVALID_ARG = 1,
  TLOAM_B200_ERR_TOO_FEW_POINTS = 2, /* a cloud has < 10 points: the reference asserts (registration.cpp:928-929) */
  TLOAM_B200_ERR_BAD_POSE = 3,       /* predict is not a rigid transform: Sophus would abort (so3.hpp:469-472) */
  TLOAM_B200_ERR_CUDA = 4,
  TLOAM_B200_ERR_NO_DEVICE = 5,
  TLOAM_B200_ERR_NOT_READY = 6,      /* scan_match before set_source / set_target */
  TLOAM_B200_ERR_NUMERIC = 7,        /* non-finite value met inside the solve */
  TLOAM_B200_ERR_MAP_DENSITY = 8,    /* a map cell (edge = search radius) holds more than 65535 points */
  TLOAM_B200_ERR_VOXEL_RANGE = 9     /* a cloud to be voxel-down-sampled spans 2^21 or more voxels on an axis (voxel too
                                        small), or a host cloud's finite rows n and voxel reach n * voxel >= 2^23 m (the
                                        headroom of the fixed-point sums; conservative): a global-map frame is not
                                        appended, the merge produces nothing, a host-input call launches nothing */
} tloam_b200_status;

/* The "TLS:" YAML block (ref: config/mapping/lidar_odometry.yaml:23-39, read at registration.cpp:212-230)
 * as a POD, same names, same defaults, plus explicit switches for reference quirks. */
typedef struct tloam_tls_config {
  int k_corr;            /* on the API surface, unused by the executed path */
  int factor_num;        /* 2 = planar+ground, 3 = +edge, 4 = +sphere (registration.hpp:144-148) */
  double edge_dist_thres, sphere_dist_thres, planar_dist_thres, ground_dist_thres;
  double edge_dir_thres;
  int edge_maxnum, sphere_maxnum, planar_maxnum, ground_maxnum;
  int max_iterations;    /* outer GNC iterations */
  double cost_threshold, gnc_factor, noise_bound, fitness_thres;
  /* extras */
  int ceres_max_num_iterations; /* options.max_num_iterations, registration.cpp:1043 */
  double reinit_dir[3];  /* replaces the unseeded Eigen::Vector3d::Random() of registration.cpp:885 */
  double initial_trust_region_radius; /* Ceres Solver::Options default 1e4 (the reference does not set it,
                          * registration.cpp:1036-1047); smaller values force the dogleg / rejected-step branches (tests) */
} tloam_tls_config;

typedef struct tloam_b200_inner_trace {
  double x_candidate[6];
  double candidate_cost, model_cost_change, relative_decrease, step_norm_scaled, radius;
  int accepted;          /* 1 accepted, 0 rejected, -1 invalid step, 2 terminated by a tolerance */
  int used_gauss_newton;
} tloam_b200_inner_trace;

typedef struct tloam_b200_outer_trace {
  double x_start[6], x_end[6];
  double initial_cost, final_cost;
  double H0[36], g0[6];  /* J^T J / J^T r (robustified) at x_start, row-major */
  double mu, th1, th2;
  double slot_sum[4];
  int n_factors[4];
  int n_inner, termination; /* 0 max-iter, 1 function tol, 2 parameter tol, 3 gradient tol, 4 radius, 5 no residuals, 6 invalid steps */
  tloam_b200_inner_trace inner[TLOAM_B200_MAX_INNER];
} tloam_b200_outer_trace;

typedef struct tloam_b200_stats {
  int n_outer, converged_early;
  double x_init[6], x_final[6];
  int gpu_launches;      /* kernels launched by this scan_match call */
  float gpu_ms;          /* device time of the call (CUDA events on the handle's stream) */
  tloam_b200_outer_trace outer[TLOAM_B200_MAX_OUTER];
} tloam_b200_stats;

void tloam_b200_default_config(tloam_tls_config* cfg);
const char* tloam_b200_status_string(int status);
const char* tloam_b200_last_error(tloam_b200_handle* h); /* text of the last CUDA failure of this handle */

/* device: CUDA ordinal. stream: a cudaStream_t to enqueue on (e.g. torch's current stream), or NULL to let
 * the handle create its own non-blocking stream. */
int tloam_b200_create(const tloam_tls_config* cfg, int device, void* stream, tloam_b200_handle** out);
int tloam_b200_destroy(tloam_b200_handle* h);

/* HOST buffers (pageable or pinned). set_target also builds the voxel-hash grids on the device.  Pinned (or registered)
 * buffers are DMA'd directly; ordinary pageable buffers -- what an unmodified front end holds, std::vector<Eigen::Vector3d>
 * -- are detected and staged by the library itself: 2 MB chunks copied by a small pool of host threads (started on first
 * use) into a ring of pinned slots while the DMA engine drains them (tloam_b200/csrc/host_stage.h; 35 GB/s instead of the
 * ~11 GB/s of cudaMemcpyAsync from pageable memory; TLOAM_B200_NO_HOST_STAGE=1 in the environment restores the latter).
 * Either way the caller's buffers have been read completely when the call returns. */
int tloam_b200_set_source(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4]);
int tloam_b200_set_target(tloam_b200_handle* h, const double* const xyz[4], const size_t n[4]);
/* DEVICE buffers (inputs already resident in HBM), same layout.  Returns without waiting: the buffers are read IN
 * PLACE (no staging copy) by kernels enqueued on the handle's stream, so they must stay unchanged until that work
 * has run (tloam_b200_synchronize, or the get_result of the frame that follows). */
int tloam_b200_set_source_device(tloam_b200_handle* h, const double* const d_xyz[4], const size_t n[4]);
int tloam_b200_set_target_device(tloam_b200_handle* h, const double* const d_xyz[4], const size_t n[4]);
/* Stream ordering of device inputs: makes the handle's stream wait (on the device) for everything enqueued so far on
 * `producer_stream` (cudaStream_t; NULL = the legacy default stream).  Call it before set_*_device when the buffers were
 * written on another stream; the handle's own stream (tloam_b200_create's `stream`) needs no call. */
int tloam_b200_wait_stream(tloam_b200_handle* h, void* producer_stream);

/* Blocking: enqueues the frame, waits, returns the pose (and optionally the trace). */
int tloam_b200_scan_match(tloam_b200_handle* h, const double predict[16], double result[16], tloam_b200_stats* stats);
/* Split form: enqueue only / wait + fetch. Lets one host thread drive several handles (one per GPU). */
int tloam_b200_scan_match_async(tloam_b200_handle* h, const double predict[16]);
int tloam_b200_get_result(tloam_b200_handle* h, double result[16], tloam_b200_stats* stats);
/* "Next" row (f)-3: constant-velocity prediction on the device (ref: src/front_end/front_end.cpp:329-330:
 * step = last^-1 * pose; predict = pose * step).  The frame is enqueued with NO host input: the prediction is computed
 * by the frame's first kernel from the two last results, which live in device memory (the pose returned by frame k
 * and the one returned by frame k-1; identity before the first frame).  set_pose_history seeds / overrides them. */
int tloam_b200_scan_match_predicted_async(tloam_b200_handle* h);
int tloam_b200_scan_match_predicted(tloam_b200_handle* h, double result[16], tloam_b200_stats* stats);
int tloam_b200_set_pose_history(tloam_b200_handle* h, const double last_pose[16], const double curr_pose[16]);
/* The per-iteration trace in tloam_b200_stats costs device time; scan_match records it iff stats != NULL, the
 * async form iff it was switched on here (default off; without it get_result fills only gpu_launches / gpu_ms). */
int tloam_b200_set_trace(tloam_b200_handle* h, int on);

/* ---- batched registration: S independent sequences (one handle each: own map, scan, pose history, submap) whose
 * frames are registered TOGETHER -- one launch sequence per batch frame instead of S.  The reference runs one
 * LocalRegistration per nodelet; this is S of them stepped in lock-step on one GPU (SURVEY.md 8(d): a single
 * 40k-feature frame cannot fill 132 SMs).  Per-sequence poses are bit-identical to the un-batched calls.
 * All sequences share `cfg`.  Feed the sequences through tloam_b200_batch_handle(b, i) (any per-handle set_* /
 * submap_* entry point) or the batch_set_* forms: xyz = S*4 pointers, n = S*4 counts, sequence-major, cloud order
 * edge, sphere, planar, ground. ---- */
typedef struct tloam_b200_batch tloam_b200_batch;
int tloam_b200_batch_create(const tloam_tls_config* cfg, int device, int S, tloam_b200_batch** out);   /* 1 <= S <= 32 */
int tloam_b200_batch_destroy(tloam_b200_batch* b);
int tloam_b200_batch_size(tloam_b200_batch* b);
tloam_b200_handle* tloam_b200_batch_handle(tloam_b200_batch* b, int i);   /* owned by the batch: do not destroy */
int tloam_b200_batch_set_target(tloam_b200_batch* b, const double* const* xyz, const size_t* n);          /* HOST */
int tloam_b200_batch_set_source(tloam_b200_batch* b, const double* const* xyz, const size_t* n);
int tloam_b200_batch_set_target_device(tloam_b200_batch* b, const double* const* d_xyz, const size_t* n); /* DEVICE */
int tloam_b200_batch_set_source_device(tloam_b200_batch* b, const double* const* d_xyz, const size_t* n);
/* predicts: S x 16 doubles (column-major 4x4 each) or NULL = constant-velocity prediction on the device per sequence
 * (front_end.cpp:329-330).  results: S x 16; statuses (optional): S tloam_b200_status values.  Returns OK iff every
 * sequence returned OK, else the first failing status. */
int tloam_b200_batch_scan_match(tloam_b200_batch* b, const double* predicts, double* results, int* statuses);
int tloam_b200_batch_scan_match_async(tloam_b200_batch* b, const double* predicts);
int tloam_b200_batch_get_results(tloam_b200_batch* b, double* results, int* statuses, float* gpu_ms /* optional */);
long long tloam_b200_batch_launch_count(tloam_b200_batch* b);   /* kernels launched by the batch and its handles */
const char* tloam_b200_batch_last_error(tloam_b200_batch* b);
/* per-kernel-class timing of the batch frame kernels (see tloam_b200_set_profiling; declared below) */
struct tloam_b200_profile;
int tloam_b200_batch_set_profiling(tloam_b200_batch* b, int on);
int tloam_b200_batch_get_profile(tloam_b200_batch* b, struct tloam_b200_profile* out);

int tloam_b200_fitness(tloam_b200_handle* h, double* fitness, double* rmse);
/* getFitnessScore as a per-frame health metric of the asynchronous flow (ref: registration.cpp:257-296; the reference
 * declares it on the interface and never calls it): when switched on, every scan_match also scores its scan against
 * the map (two kernels in the frame graph, no allocation, no extra synchronisation) and the pair comes back with the
 * frame's result. */
int tloam_b200_set_frame_fitness(tloam_b200_handle* h, int on);
int tloam_b200_get_frame_fitness(tloam_b200_handle* h, double* fitness, double* rmse);   /* of the last fetched result */
/* Pipelined use (front end one frame ahead of the GPU): set_source / submap_update return without waiting for their
 * uploads -- the HOST buffers must stay valid until the frame's result has been fetched -- and get_result waits for the
 * OLDEST un-fetched frame only (at most 2 frames in flight; no per-iteration trace in this mode). */
int tloam_b200_set_async_inputs(tloam_b200_handle* h, int on);
int tloam_b200_get_transform(tloam_b200_handle* h, double pose[16]);
int tloam_b200_get_pose_increment(tloam_b200_handle* h, double pose[16]);
/* self-check of the dense-map correspondence path (env TLOAM_B200_DENSE_CHECK=1 at create): every query it searches is
 * searched again by the plain path and compared.  out: [0] queries, [1] differing kNN lists, [2] work items, [3] TMA
 * staging passes, [4..7] details of the first mismatch, [8..11] SM cycles / 64 per phase (item total, TMA wait, fine
 * sort, search), [12] work items with <= 8 queries; accumulated since creation. */
int tloam_b200_dense_check_counters(tloam_b200_handle* h, unsigned out[16]);
int tloam_b200_synchronize(tloam_b200_handle* h);
/* total kernels launched by this handle so far */
long long tloam_b200_launch_count(tloam_b200_handle* h);

/* ---- shared-map transport (multi-GPU, config 4): the built map (cell-sorted float4 points + hash
 * tables + header) is one contiguous device blob so that a single ncclBroadcast moves it. ---- */
int tloam_b200_map_blob_size(tloam_b200_handle* h, size_t* bytes);
int tloam_b200_map_export(tloam_b200_handle* h, void* d_dst, size_t bytes);       /* D2D copy out */
int tloam_b200_map_import(tloam_b200_handle* h, const void* d_src, size_t bytes); /* D2D copy in, adopt */
int tloam_b200_get_map_origin(tloam_b200_handle* h, double origin[3]);
/* Zero-copy form (config 4: ONE collective per map epoch, no size handshake, no host synchronisation, no staging
 * copies).  The blob layout is a pure function of the configuration and the four point counts, so every rank can lay
 * the incoming blob out from n[4] alone.
 *   sender:    tloam_b200_map_send_buffer  -> the built blob itself; order the stream of the collective behind the build
 *              with tloam_b200_signal_stream(h, that_stream)
 *   receiver:  tloam_b200_map_recv_buffer  -> a SECOND blob of the handle (frames keep registering against the active map
 *              while the next one is in flight); enqueue the collective into it on any stream; then
 *              tloam_b200_map_adopt(h, that_stream): device-side wait + pointer swap, nothing else */
int tloam_b200_map_layout_bytes(tloam_b200_handle* h, const size_t n[4], size_t* bytes);
int tloam_b200_map_send_buffer(tloam_b200_handle* h, void** d_ptr, size_t* bytes);
int tloam_b200_map_recv_buffer(tloam_b200_handle* h, const size_t n[4], void** d_ptr, size_t* bytes);
int tloam_b200_map_adopt(tloam_b200_handle* h, void* producer_stream);
int tloam_b200_signal_stream(tloam_b200_handle* h, void* consumer_stream);

/* ---- piecewise entry points (parity tests; host arrays in, host arrays out, computed on the GPU) ---- */
/* Exact radius-truncated kNN on the built map of `cloud` (KDTreeFlann::SearchHybrid semantics): idx/d2 are
 * nq*k, ascending (d2, index), padded with -1 / +inf; count[i] = neighbours strictly inside the radius. */
int tloam_b200_knn(tloam_b200_handle* h, int cloud, const double* queries, size_t nq, double radius, int k,
                   int* idx, double* d2, int* count);
/* Correspondence search + primitive fit + caps for one cloud at tangent x (all weights 1):
 * valid[i] in {0,1}; prim = n*6 doubles: plane (n,d,0,0), line (a,b), point (q,0,0,0). */
int tloam_b200_build_factors(tloam_b200_handle* h, int cloud, const double x[6], int* valid, double* prim, size_t n);
/* Batched cost functors: arrays of m factors; r is m*3 (m*1 for plane), J is m*18 (m*6), cost is m. */
int tloam_b200_eval_point_to_point(tloam_b200_handle* h, const double x[6], size_t m, const double* p,
                                   const double* q, const double* w, double* r, double* J, double* cost);
int tloam_b200_eval_point_to_line(tloam_b200_handle* h, const double x[6], size_t m, const double* p,
                                  const double* a, const double* b, const double* w, double* r, double* J,
                                  double* cost);
int tloam_b200_eval_point_to_plane(tloam_b200_handle* h, const double x[6], size_t m, const double* p,
                                   const double* n, const double* d, const double* w, double* r, double* J,
                                   double* cost);
/* SE(3) helpers evaluated on the device (exp: tangent -> 4x4 col-major; log: inverse; plus: left update). */
int tloam_b200_se3_exp(tloam_b200_handle* h, const double a[6], double T[16]);
int tloam_b200_se3_log(tloam_b200_handle* h, const double T[16], double a[6]);
int tloam_b200_se3_plus(tloam_b200_handle* h, const double x[6], const double delta[6], double out[6]);
/* the 2-D trust-region boundary problem of the subspace dogleg as the device solver runs it:
 * minimise 0.5 y^T B y + g^T y on |y| = radius (B row-major 2x2) */
int tloam_b200_min_on_boundary_2d(tloam_b200_handle* h, const double B[4], const double g[2], double radius, double y[2]);

/* ---- per-kernel timing (off by default): CUDA events on the handle's stream around EVERY launch.  The
 * bracketing adds ~1-2 us of event overhead per launch, so profiled durations are upper bounds. ---- */
enum {
  TLOAM_B200_K_MAP_BBOX = 0, TLOAM_B200_K_MAP_ORIGIN, TLOAM_B200_K_MAP_INSERT, TLOAM_B200_K_MAP_OFFSETS,
  TLOAM_B200_K_MAP_SCATTER, TLOAM_B200_K_STAGE_SOURCE, TLOAM_B200_K_BEGIN_FRAME, TLOAM_B200_K_CORRESPOND,
  TLOAM_B200_K_EVAL_FIRST, TLOAM_B200_K_EVAL, TLOAM_B200_K_SUBMAP, TLOAM_B200_K_FEATURE, TLOAM_B200_K_FIRST,
  TLOAM_B200_K_DENSE_BIN, TLOAM_B200_K_DENSE, TLOAM_B200_K_FITNESS, TLOAM_B200_K_GROUND, TLOAM_B200_K_MAP_FINE,
  TLOAM_B200_K_FINE, TLOAM_B200_K_EDGE, TLOAM_B200_K_OBJECT, TLOAM_B200_K_COUNT
};
typedef struct tloam_b200_profile {
  long long launches[TLOAM_B200_K_COUNT];
  double total_ms[TLOAM_B200_K_COUNT];
  /* in-kernel timers (profiling mode): [1] ns k_eval parallel phase, [2] ns final partial sum, [3] ns solver state
   * machine, [4] number of active k_eval launches, [8] SM cycles k_correspond kNN phase summed over thread blocks,
   * [9] number of k_correspond thread blocks */
  unsigned long long dbg[16];
} tloam_b200_profile;
int tloam_b200_set_profiling(tloam_b200_handle* h, int on);   /* also clears the accumulated profile */
int tloam_b200_get_profile(tloam_b200_handle* h, tloam_b200_profile* out);

/* ---- device-side local-map maintenance ("next" row (f)-1): FrontEnd::updateSubmap on the GPU
 * (ref: src/front_end/front_end.cpp:201-267, first frame :285-305; PointCloud2 Transform / += / Crop /
 * VoxelDownSample, ref: src/open3d/PointCloud2.cpp:71-75, 96-132, 358-403, 551-559).  The map stays in HBM between
 * frames; each call ends with the same voxel-hash build as tloam_b200_set_target. ---- */
typedef struct tloam_submap_config {   /* ref: config/mapping/lidar_odometry.yaml:6-17 */
  double ground_down_sample;           /* 0.3  */
  double ground_down_sample_submap;    /* 0.45 */
  double edge_down_sample_submap;      /* 0.3  */
  int planar_frame_size;               /* 3 */
  int sphere_frame_size;               /* 3 (kept for parity; the reference builds the sphere submap from the planar buffer) */
  double edge_crop_box_length, ground_crop_box_length;   /* 100, 100 */
} tloam_submap_config;
void tloam_b200_submap_default_config(tloam_submap_config* c);
/* First frame: edge = raw edge cloud, ground_raw = raw ground cloud (voxel-down-sampled at ground_down_sample
 * inside), planar_sub / sphere_sub = the "submap index" selections of the general cloud.  HOST pointers.
 * INVALID_ARG: a crop length and submap voxel with 2 L / voxel + 1 >= 2^21 (a cropped cloud could then reach the key
 * range, which bounds every later update), or a submap voxel not > 0.  VOXEL_RANGE: ground_raw as in
 * tloam_b200_voxel_down_sample (nothing is changed).  A later update's per-voxel count is not checked against the
 * 2^23 m headroom: an accumulator would need 2^23 m / voxel rows in one voxel. */
int tloam_b200_submap_init(tloam_b200_handle* h, const tloam_submap_config* cfg, const double* edge, size_t ne,
                           const double* ground_raw, size_t ng, const double* planar_sub, size_t np,
                           const double* sphere_sub, size_t ns);
/* Later frames, after scan_match: pose = the new lidar_odom_pose (4x4 column-major).  The edge and ground
 * features appended to the map are the ones of the CURRENT SOURCE (tloam_b200_set_source), already on the device;
 * planar_sub is this frame's planar submap selection (HOST pointer, sensor frame); sphere_sub is accepted for
 * interface parity and ignored, as in the reference (front_end.cpp:220-230 iterates the planar buffer). */
int tloam_b200_submap_update(tloam_b200_handle* h, const double pose[16], const double* planar_sub, size_t np,
                             const double* sphere_sub, size_t ns);
/* Chained form: pose = the result of the frame that was just ENQUEUED on this handle (scan_match_async /
 * scan_match_predicted_async), read on the device -- no host round trip between registration and map update. */
int tloam_b200_submap_update_chained(tloam_b200_handle* h, const double* planar_sub, size_t np);
int tloam_b200_submap_sizes(tloam_b200_handle* h, size_t n[4]);   /* exact sizes (synchronises) */
/* copies map cloud `cloud` (0 edge, 1 sphere, 2 planar, 3 ground; world frame, FP64 AoS) to the host */
int tloam_b200_submap_download(tloam_b200_handle* h, int cloud, double* out, size_t capacity_points);
/* PointCloud2::VoxelDownSample on the device (HOST in / out; out must hold n points).  Rows with a non-finite coordinate
 * are left out (they do not move the min bound).  Each average is within 2^-41 + 2^-51 voxel + 1.5 ulp(max |p|) of the
 * exact mean of its voxel's rows, and bit-reproducible.  INVALID_ARG: voxel not > 0 with n > 0.  VOXEL_RANGE (checked on
 * the host, nothing launched): the finite rows span 2^21 voxels on an axis, or their count n reaches n * voxel >= 2^23 m. */
int tloam_b200_voxel_down_sample(tloam_b200_handle* h, const double* pts, size_t n, double voxel, double* out, size_t* n_out);

/* ------------------------------------------------------------------------------------------------
 * "Next" row (f)-2: PCA feature extraction on the device.  Replaces featureExtract::extractPlanarSphere /
 * calculatePCAInfo (ref: src/models/feature_extraction/feature_extract.cpp:133-197, 47-122; called from
 * FrontEnd::processCloud, src/front_end/front_end.cpp:194 and :289).  Bit-exact against oracle/feature_oracle.cpp.
 * The handle is only used for its device, stream and scratch memory: no map or scan needs to be set. */
typedef struct tloam_feature_config {   /* ref: config/mapping/feature.yaml */
  double radius;                 /* 0.2  neighbour search radius */
  int K;                         /* 20   neighbours per point (3 <= K <= 20 supported) */
  int min_neigh;                 /* 10   points with <= min_neigh neighbours are skipped */
  int planar_num, sphere_num;    /* 500, 300 */
  double cvr_scan, cvr_submap;   /* 0.25, 0.15 */
  double planar_scan_thres, planar_submap_thres, planar_vertic_thres;   /* 0.75, 0.65, 0.25 */
} tloam_feature_config;
void tloam_b200_feature_default_config(tloam_feature_config* c);
/* extractPlanarSphere: xyz = the general cloud (HOST, n x 3 FP64).  Each index buffer must hold n entries; the four
 * lists are what the reference's four std::vector<size_t> receive, INCLUDING its quirk that the two sphere lists
 * hold ranks 0..count-1 instead of point indices (feature_extract.cpp:183-188).  sphere_candidates (optional, n
 * entries) receives the point indices those ranks refer to (sphere candidates by descending flatness). */
int tloam_b200_extract_planar_sphere(tloam_b200_handle* h, const tloam_feature_config* cfg, const double* xyz, size_t n,
                                     size_t* planar_scan_index, size_t* n_planar_scan, size_t* planar_submap_index,
                                     size_t* n_planar_submap, size_t* sphere_scan_index, size_t* n_sphere_scan,
                                     size_t* sphere_submap_index, size_t* n_sphere_submap, size_t* sphere_candidates);
/* calculatePCAInfo (inspection / tests): per point cvr, flatness, sphericity, normal (n x 3), num_sum and the
 * neighbour list (n x K, ascending distance, -1 padded).  Any output pointer may be NULL. */
int tloam_b200_pca_info(tloam_b200_handle* h, const tloam_feature_config* cfg, const double* xyz, size_t n, double* cvr,
                        double* flatness, double* sphericity, double* normal, int* num_sum, int* neigh);

/* ------------------------------------------------------------------------------------------------
 * "Next" row (f)-4, first part: multi-region ground extraction of the segmentation nodelet on the device.  Replaces
 * Segmentation::groundRemove (ref: src/models/segmentation/segmentation.cpp:738-770) with everything it calls:
 * initSections / getSection (:174-238), estimateRingsAndTimes2 HDL_64E / VLP_16 (:341-443), filterByHeight (:454-470),
 * fillSectionIndex (:507-541), segmentGroundThread (:626-730), findBestPlane (:551-616).  Bit-exact against
 * oracle/segmentation_oracle.cpp.  The handle is only used for its device, stream and scratch memory. */
typedef struct tloam_ground_config {   /* ref: config/mapping/segmentation.yaml (velodyne: / groundSeg:) */
  int sensor_model;                    /* 64: HDL-64E or 16: VLP-16 (verticalRes 2.0, initAngle -15.0); others: INVALID_ARG */
  double sensor_height;                /* 1.73 */
  double vertical_res, init_angle;     /* 0.4, -24.9 */
  double sensor_min_range, sensor_max_range;   /* 1.0, 120.0 */
  int quadrant, num_sec;               /* 4, 3 */
  double plane_dis;                    /* groundSeg.dis 0.3 */
  int max_iter, ground_seed_num;       /* 3, 20 */
} tloam_ground_config;
void tloam_b200_ground_default_config(tloam_ground_config* c);
/* xyz: the scan AFTER RemoveClosedNonFinitePoints, in acquisition order (HOST, n x 3 FP64).  Index buffers hold n entries.
 * ground_index / object_index receive the indices (into xyz) of the points the reference's ground_scan / object_scan
 * receive, in that order with regions taken in (quadrant, section) order (the reference appends regions from four
 * racing threads); points of a region with <= 3 seeds reach neither list, as in the reference.  Optional outputs:
 * beam (n): (int) of the value stored in the intensity channel (HDL-64E: the beam estimate; VLP-16: beamId + correctTime,
 * see tloam_b200_ground_remove); region (n): quadrant * num_sec + section, 12 = above the height threshold, 13 = dropped;
 * height_threshold: mean z + 0.5; planes: 12 x 8 x 4 plane models [region][iteration]. */
int tloam_b200_ground_extract(tloam_b200_handle* h, const tloam_ground_config* cfg, const double* xyz, size_t n,
                              size_t* ground_index, size_t* n_ground, size_t* object_index, size_t* n_object, int* beam,
                              int* region, double* height_threshold, double* planes);
/* tloam_b200_ground_extract with the intensity channel as the reference computes it, in FP64 (optional, n values):
 * HDL-64E the beam estimate (an integer), VLP-16 beamId + correctTime (a real number; within a few ulp of libm's, the sign
 * tests of the half pass are exact).  Index lists, regions, threshold and planes are bit-exact for both sensors. */
int tloam_b200_ground_remove(tloam_b200_handle* h, const tloam_ground_config* cfg, const double* xyz, size_t n,
                             size_t* ground_index, size_t* n_ground, size_t* object_index, size_t* n_object, double* intensity,
                             int* region, double* height_threshold, double* planes);

/* ---- "next" row (f)-4, second part: LOAM-style edge extraction of the segmentation nodelet,
 * Segmentation::extractEdgePoint + extractFromSection (ref: src/models/segmentation/segmentation.cpp:1144-1304, called at
 * :64 on the clustered object points).  xyz: n AoS points; intensity: the beam id of every point (the reference keeps it in
 * the intensity channel, (int)intensity must lie in [0, sensor_model), sensor_model <= 64); beams with fewer than ring_min_num
 * points are skipped (config/mapping/segmentation.yaml: 131).  Outputs are index lists into the input, in the order in which
 * the reference appends the points: edge_index (capacity n) by (beam, sector, descending curvature), <= 20 per sector;
 * non_edge_index (capacity n) by (beam, sector, ascending curvature).  Bit-exact against oracle/segmentation_oracle.cpp.
 * A sector with more than 4096 curvature values (a beam with more than 24 586 points) is rejected: INVALID_ARG. */
int tloam_b200_extract_edge(tloam_b200_handle* h, int sensor_model, int ring_min_num, const double* xyz, const double* intensity,
                            size_t n, size_t* edge_index, size_t* n_edge, size_t* non_edge_index, size_t* n_non_edge);

/* ---- "next" row (f)-4, third part: object segmentation = Dynamic Curved-Voxel Clustering of the non-ground points,
 * Segmentation::objectSegmentation (ref: src/models/segmentation/segmentation.cpp:1085-1112) and what it calls:
 * convertToPolar (:790-837), getPolarIndex (:777-784), createHashTable (:843-874), searchKNN (:886-908), DCVC (:915-990),
 * labelAnalysis (:998-1025), colorSegmentation (:1032-1078).  The sequential labelling is replayed exactly (see
 * tloam_b200/csrc/object_segment.cuh); integer outputs are bit-exact against oracle/segmentation_oracle.cpp given the
 * same polar triples, the triples themselves agree with libm's to <= 4 ulp. */
typedef struct tloam_dcvc_config {      /* ref: config/mapping/segmentation.yaml (DCVC: / velodyne:) */
  double start_r, delta_r, delta_p, delta_a;   /* 0.35, 0.0004, 1.2, 1.2 */
  int min_seg;                                 /* 80: classes with <= min_seg points are filtered out */
  double sensor_min_range, sensor_max_range;   /* 1.0, 120.0 */
  /* the members minPitch / maxPitch / minPolar / maxPolar before the scan: resetParams() leaves 0.0
   * (segmentation.cpp:1121-1123); on the very first frame the polar pair is 5.0 (segmentation.hpp:332-333) */
  double min_pitch_init, max_pitch_init, min_polar_init, max_polar_init;
} tloam_dcvc_config;
void tloam_b200_dcvc_default_config(tloam_dcvc_config* c);
/* xyz: the object scan (HOST, n x 3 FP64, finite).  seg_index (capacity n): indices of the reference's segmented_scan,
 * cluster after cluster (size descending; equal sizes by smallest point index -- the reference leaves that to
 * unordered_map order), index order inside a cluster; sizes (capacity n) / boxes (capacity n x 6: centre xyz,
 * dimensions xyz) per cluster.  Optional outputs: root (n): smallest point index of the point's DCVC class (a canonical
 * form of label_info); cluster (n): 1-based cluster number, 0 = filtered; voxel (n): the reference's voxelIndex;
 * polar (3 n + 4): range / pitch / azimuth triples followed by minPitch, maxPitch, minPolar, maxPolar.
 * More than 4096 polar rings (the default configuration has ~500 at 120 m): INVALID_ARG. */
int tloam_b200_object_segmentation(tloam_b200_handle* h, const tloam_dcvc_config* cfg, const double* xyz, size_t n,
                                   size_t* seg_index, size_t* n_seg, int* n_clusters, int* sizes, double* boxes, int* root,
                                   int* cluster, int* voxel, double* polar);

/* The three steps of Segmentation::spinOnce (ref: src/models/segmentation/segmentation.cpp:47-66: groundRemove,
 * objectSegmentation, extractEdgePoint(segmented_scan, edge_scan, general_scan)) as ONE call: the scan crosses PCIe once,
 * every stage is fed on the device from the previous stage's index list, only the final lists come home.  All three
 * lists index the ORIGINAL scan: ground_index = the reference's ground_scan, edge_index / general_index = its edge_scan /
 * general_scan (capacity n each), in the reference's order.  sizes / boxes (capacity n / n x 6, optional): per cluster as
 * in tloam_b200_object_segmentation; beam (capacity n, optional): the beam estimate of every point of the scan (what the
 * reference keeps in the intensity channel of the object / segmented / edge / general clouds).  Identical to calling the
 * three functions one after the other with host gathers in between (tests/test_object_segmentation.py). */
int tloam_b200_segment_scan(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                            const double* xyz, size_t n, size_t* ground_index, size_t* n_ground, size_t* edge_index, size_t* n_edge,
                            size_t* general_index, size_t* n_general, int* n_clusters, int* sizes, double* boxes, int* beam);
/* Segmentation::spinOnce's compute steps :48-66 in one call: RemoveClosedNonFinitePoints(near_dis) on the device (a point
 * is kept iff it has no NaN / Inf coordinate and its norm is >= near_dis * near_dis -- a norm against a SQUARED
 * threshold, as in the reference: near_dis 3.0 removes every point closer than 9 m), then the chain of
 * tloam_b200_segment_scan on the surviving points.  xyz: the raw scan as the driver delivers it (HOST, n x 3 FP64, may
 * hold NaN / Inf rows).  All lists index the RAW scan.  intensity (optional, n values): the FP64 channel of every
 * surviving point (see tloam_b200_ground_remove), NaN for removed points.  One upload, one download. */
int tloam_b200_segment_raw_scan(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                                double near_dis, const double* xyz, size_t n, size_t* ground_index, size_t* n_ground, size_t* edge_index,
                                size_t* n_edge, size_t* general_index, size_t* n_general, int* n_clusters, int* sizes, double* boxes,
                                double* intensity);

/* ---- Raw scans in the sensor's packed layout (the reference's RosToOpen3d, ref: src/open3d/open3d_to_ros.cpp:344-374, and
 * readVelodyneToO3d, include/tloam/models/io/read_file.hpp:307-327, on the device): the records cross PCIe once, as the
 * driver delivers them, and k_unpack_scan writes (double)float of every field on the GPU -- exact, so a packed call gives the
 * bits of the FP64 call on the same values.  A sensor_msgs/PointCloud2 with FLOAT32 x / y / z (and intensity) fields, or a
 * KITTI .bin scan (16-byte records: x, y, z, reflectance).  Anything this cannot express is the caller's to refuse:
 * big-endian data, other field types, padding between rows (include/tloam_b200/packed_scan_b200.hpp does it for a
 * PointCloud2).  The kernel lives in libtloam_b200_unpack.so, loaded from this library's directory on the first packed call;
 * if it is missing these calls return ERR_CUDA (tloam_b200_last_error names the file) and nothing else is affected.
 * INVALID_ARG: data null with n > 0, point_step < 12, a field not inside the record (offset < 0 or offset + 4 >
 * point_step; intensity_offset may be -1), n > 2^26.  n == 0 is an empty scan. */
typedef struct tloam_packed_scan {
  const void* data;                   /* HOST, n records of point_step bytes, little-endian */
  size_t n, point_step;
  int x_offset, y_offset, z_offset;   /* FLOAT32 fields */
  int intensity_offset;               /* FLOAT32 field, or -1: the scan has no intensity */
} tloam_packed_scan;
/* tloam_b200_segment_raw_scan on a packed scan (its intensity field, if any, is not read: the `intensity` output is the
 * channel the segmentation computes, as there) */
int tloam_b200_segment_raw_scan_packed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                       int ring_min_num, double near_dis, const tloam_packed_scan* scan, size_t* ground_index,
                                       size_t* n_ground, size_t* edge_index, size_t* n_edge, size_t* general_index, size_t* n_general,
                                       int* n_clusters, int* sizes, double* boxes, double* intensity);

/* ---- FrontEnd::processCloud on the device (ref: src/front_end/front_end.cpp:181-199): the scan features become the
 * registration source without leaving the GPU.  VoxelDownSample(ground, ground_down_sample) and VoxelDownSample(edge,
 * edge_down_sample), extractPlanarSphere(general) with fcfg, SelectByIndex of the planar and sphere features, then
 * setInputSource: the four clouds become the handle's source exactly as if tloam_b200_set_source had been called with
 * them (staged, so tloam_b200_submap_update[_chained] can append them).  n_source[4] receives their sizes (edge, sphere,
 * planar, ground).
 *   - The down-sampled ground / edge features come out in ascending voxel index (ix, iy, iz) -- the registration caps
 *     (*_maxnum) take features in index order, so the order is part of the result -- with the averages in the fixed-point
 *     form of tloam_b200_voxel_down_sample (within 2^-41 + 2^-51 voxel + 1.5 ulp(max |p|) of the exact mean, bit-reproducible).
 *   - VOXEL_RANGE: the ground or the edge cloud fails tloam_b200_voxel_down_sample's limits at its voxel (checked on the
 *     host before anything is uploaded; the last processed frame is kept).
 *   - The sphere feature is general[0 .. n_sphere_scan): the reference's sphere lists hold ranks, not point indices
 *     (feature_extract.cpp:183-188; see tloam_b200_extract_planar_sphere), and SelectByIndex takes them literally.
 *   - The frame's raw edge and ground clouds, its planar-submap selection general[planar_submap_index] and its sphere-submap
 *     count stay on the device for tloam_b200_submap_init_frame / tloam_b200_submap_update_frame*.
 *   - Empty clouds are allowed: an empty general cloud selects nothing, an empty ground / edge cloud gives an empty feature.
 *     Voxel sizes must be > 0 even then.  A map cell of the PCA grid holding more than 65535 points: MAP_DENSITY.
 *   - Synchronises once to read the counts; no point data crosses PCIe except the three input clouds (HOST, n x 3 FP64).
 *   - All device work runs on the handle's stream, so frame k+1 may be processed as soon as frame k's submap update has
 *     been enqueued. */
int tloam_b200_process_cloud(tloam_b200_handle* h, const tloam_feature_config* fcfg, double ground_down_sample, double edge_down_sample,
                             const double* ground, size_t ng, const double* edge, size_t ne, const double* general, size_t nn,
                             size_t n_source[4]);
/* tloam_b200_segment_raw_scan followed by tloam_b200_process_cloud without the host in between: the raw scan (HOST, may hold
 * NaN / Inf rows) is uploaded once, segmented on the device, the ground / edge / general clouds are gathered from it on the
 * device, then processed as above.  An all-NaN or all-near scan gives four empty sources and OK.  VOXEL_RANGE: the scan's
 * finite rows fail tloam_b200_voxel_down_sample's limits at ground_down_sample or edge_down_sample (the ground and edge
 * clouds are subsets of them), checked on the host before the upload. */
int tloam_b200_process_raw_scan(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg, int ring_min_num,
                                double near_dis, const tloam_feature_config* fcfg, double ground_down_sample, double edge_down_sample,
                                const double* xyz, size_t n, size_t n_source[4]);
/* tloam_b200_process_raw_scan on a packed scan (validation as tloam_b200_segment_raw_scan_packed).  With an intensity field,
 * its values stay on the device with the raw scan, for tloam_b200_global_map_append_frame*. */
int tloam_b200_process_raw_scan_packed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                       int ring_min_num, double near_dis, const tloam_feature_config* fcfg, double ground_down_sample,
                                       double edge_down_sample, const tloam_packed_scan* scan, size_t n_source[4]);

/* ---- Deskewing (motion correction of a raw scan; the reference reads scanPeriod and never uses it).  Opt-in: the timed
 * forms below take per-point times; every other call behaves as before.  With t_end the largest finite time, P =
 * frame_period (the unit of the times, e.g. 0.1 s at 10 Hz) and xi = log(last^-1 . curr) (se3 log of the pose history's
 * constant-velocity increment -- the one tloam_b200_scan_match_predicted_async predicts with -- read on the device when the
 * call runs, after the previous frame's solver), every row becomes
 *     p'_i = exp(s_i . xi) . p_i,   s_i = (t_i - t_end) / P,
 * the point in the sensor frame at the end of the sweep: the pose the loop returns is the pose at t_end.  A non-finite t_i,
 * or a scan without a finite time, gives s_i = 0 (the row is copied bit for bit); non-finite rows stay non-finite.  A fresh
 * handle's history is identity, so frames 0 and 1 are not corrected unless tloam_b200_set_pose_history seeded it.
 *   - Segmentation reads the RAW scan (its ring / range-image topology is the sensor's).  The corrected scan replaces it
 *     where the ground / edge / general clouds are gathered (so the source, the submap selections and the frame are
 *     corrected) and as the raw scan tloam_b200_global_map_append_frame* and tloam_b200_registered_scan_download read.
 *   - The kernels live in libtloam_b200_deskew.so, loaded from this library's directory on the first timed call; if it is
 *     missing these calls return ERR_CUDA (tloam_b200_last_error names the file).
 *   - The key-range and headroom check (VOXEL_RANGE) reads the scan before the correction; the corrected rows' extent is
 *     not checked, and tloam_b200_submap_init_frame after a timed call does not check its ground cloud either.
 *   - INVALID_ARG, besides the untimed call's: time null with n > 0, frame_period not finite or not > 0, and for a packed
 *     time field: offset < 0 or offset + size > point_step, a datatype other than 6 / 7 / 8, unit not finite or not > 0. */
/* a time field of a tloam_packed_scan record: a record's time is the field's value times unit */
typedef struct tloam_packed_time {
  int offset;                         /* bytes into the record */
  int datatype;                       /* sensor_msgs/PointField: 6 UINT32, 7 FLOAT32, 8 FLOAT64 (little-endian) */
  double unit;                        /* e.g. 1 for seconds, 1e-9 for Ouster's nanoseconds */
} tloam_packed_time;
/* tloam_b200_process_raw_scan with time (HOST, n FP64 values, in the unit of frame_period) */
int tloam_b200_process_raw_scan_timed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                      int ring_min_num, double near_dis, const tloam_feature_config* fcfg, double ground_down_sample,
                                      double edge_down_sample, const double* xyz, const double* time, size_t n, double frame_period,
                                      size_t n_source[4]);
/* tloam_b200_process_raw_scan_packed with the time field `time` of the same records (read where they were uploaded) */
int tloam_b200_process_raw_scan_packed_timed(tloam_b200_handle* h, const tloam_ground_config* gcfg, const tloam_dcvc_config* dcfg,
                                             int ring_min_num, double near_dis, const tloam_feature_config* fcfg,
                                             double ground_down_sample, double edge_down_sample, const tloam_packed_scan* scan,
                                             const tloam_packed_time* time, double frame_period, size_t n_source[4]);

/* copies source cloud `cloud` (0 edge, 1 sphere, 2 planar, 3 ground; sensor frame, FP64 AoS) to the host (synchronises) */
int tloam_b200_source_download(tloam_b200_handle* h, int cloud, double* out, size_t capacity_points);
/* tloam_b200_submap_init from the last processed frame (front_end.cpp:285-305): edge = its raw edge cloud, ground =
 * VoxelDownSample(cfg->ground_down_sample) of its raw ground cloud, planar = general[planar_submap_index], sphere =
 * general[0 .. n_sphere_submap).  NOT_READY before any processed frame.  INVALID_ARG / VOXEL_RANGE as in
 * tloam_b200_submap_init, the ground cloud's extent being the one the processing call read on the host. */
int tloam_b200_submap_init_frame(tloam_b200_handle* h, const tloam_submap_config* cfg);
/* tloam_b200_submap_update / _chained with planar_sub = the last processed frame's planar-submap selection, read on the
 * device.  NOT_READY before any processed frame. */
int tloam_b200_submap_update_frame(tloam_b200_handle* h, const double pose[16]);
int tloam_b200_submap_update_frame_chained(tloam_b200_handle* h);

/* ---- Global map (FrontEnd::updateSubmap with mapping_flag, ref: src/front_end/front_end.cpp:269-274): every appended
 * raw scan is transformed by its pose, voxel-down-sampled ON ITS OWN and concatenated to a map kept on the device:
 *     global_map += raw.Transform(pose).VoxelDownSample(voxel)
 *   - Frames are never merged: each is down-sampled on its own grid (min bound of its transformed finite rows - voxel/2).
 *     Its voxels come out in ascending voxel index (ix, iy, iz), with the fixed-point averages of
 *     tloam_b200_voxel_down_sample; frames follow in call order.  The map is fully deterministic.
 *   - Non-finite rows are left out of the map (the reference feeds them to GetMinBound / floor: undefined behaviour).
 *   - The registered scan is T.p of every raw row, in raw order (non-finite rows stay non-finite).  The reference with
 *     mapping_flag on publishes T.T.p (Transform works in place); T.p is what it publishes with mapping_flag off.
 *   - The first frame of FrontEnd is not in the reference's map (front_end.cpp:285-305 returns before updateSubmap):
 *     append from frame 1 on to restate it.
 *   - Appends are enqueued on the handle's stream with no host round trip; the host sizes the map from an upper bound
 *     and synchronises only when the buffer has to grow (x1.5).  A frame whose finite extent reaches 2^21 voxels on an
 *     axis is refused on the device (map unchanged); the next call below that synchronises returns VOXEL_RANGE once.
 *   - Mapping is off until tloam_b200_global_map_enable; with it off none of this launches anything. */
typedef struct tloam_global_map_config {
  double voxel;                        /* VoxelDownSample size of every frame (the reference's literal 1.0) */
  size_t initial_capacity_points;      /* map buffer before the first growth */
} tloam_global_map_config;
void tloam_b200_global_map_default_config(tloam_global_map_config* c);
/* (re)starts an empty map with this configuration.  INVALID_ARG: cfg null, voxel <= 0 or not finite. */
int tloam_b200_global_map_enable(tloam_b200_handle* h, const tloam_global_map_config* cfg);
/* empties the map and forgets the registered scan (the configuration and the buffers stay).  NOT_READY if not enabled. */
int tloam_b200_global_map_reset(tloam_b200_handle* h);
/* appends a HOST raw cloud (n x 3 FP64 AoS, may hold NaN / Inf rows) with pose[16] (column-major, host) or, _chained, the
 * pose of the frame just enqueued on the handle (tloam_b200_scan_match_predicted_async).  n == 0 appends an empty frame. */
int tloam_b200_global_map_append(tloam_b200_handle* h, const double pose[16], const double* xyz, size_t n);
int tloam_b200_global_map_append_chained(tloam_b200_handle* h, const double* xyz, size_t n);
/* the same for the raw scan that the last tloam_b200_process_raw_scan uploaded (no upload).  NOT_READY when there is none,
 * or when any segmentation or process call has run since (its buffer may have been reused).
 * After tloam_b200_process_raw_scan_packed whose layout has an intensity field, the frame is appended WITH that intensity,
 * read on the device (the reference's raw cloud carries its channel into global_map += ...); without one, or after the FP64
 * tloam_b200_process_raw_scan, it is a frame without intensity.  tloam_b200_global_map_append_frame_intensity[_chained]
 * with an explicit host array takes precedence over the packed intensity.
 * After a timed process_raw_scan (see Deskewing) the frame appended is the corrected scan; after an untimed one, the raw scan. */
int tloam_b200_global_map_append_frame(tloam_b200_handle* h, const double pose[16]);
int tloam_b200_global_map_append_frame_chained(tloam_b200_handle* h);
/* exact points and frames in the map (synchronises); returns VOXEL_RANGE once after a refused frame */
int tloam_b200_global_map_size(tloam_b200_handle* h, size_t* n_points, size_t* n_frames);
/* map points [first, first + count) to out (count x 3 FP64, synchronises).  INVALID_ARG past the end. */
int tloam_b200_global_map_download(tloam_b200_handle* h, size_t first, size_t count, double* out);
/* offsets[0 .. n_frames]: the first point of every frame, then the map size (capacity >= n_frames + 1, synchronises) */
int tloam_b200_global_map_frame_offsets(tloam_b200_handle* h, size_t* offsets, size_t capacity);
/* map buffer capacity in points and the number of growths since enable (each growth synchronised once) */
int tloam_b200_global_map_capacity(tloam_b200_handle* h, size_t* capacity_points, size_t* growths);
/* T.p of every row of the last append, raw order, to out (synchronises).  *n receives the row count; NOT_READY before the
 * first append, INVALID_ARG if capacity_points < *n. */
int tloam_b200_registered_scan_download(tloam_b200_handle* h, double* out, size_t capacity_points, size_t* n);

/* ---- The map's intensity channel (the reference's map is XYZI): the same appends with the raw scan's intensity (n host
 * FP64 values, one per raw row).  Each voxel's intensity is the reference's AccumulatedPoint::GetAverageIntensity
 * (PointCloud2.cpp:253-286): a sequential FP64 sum of its rows' values in raw-row order from +0.0, divided by the count,
 * bit for bit (NaN / Inf propagate).  The rows left out of the map (non-finite xyz) are left out of the sums too.
 *   - The map has the channel under the rule of PointCloud2::operator+= (:99-100, :118-124): a frame that adds points keeps
 *     it iff (map empty || map has it) && the frame has it.  A frame that adds nothing (empty, all non-finite, refused)
 *     changes nothing; once points without intensity are in the map it has none until tloam_b200_global_map_reset.
 *   - The xyz map, the frame table and the registered scan are the bits of the same appends without intensity.
 *   - The kernels live in libtloam_b200_gmi.so, loaded from this library's directory on the first intensity call; if it is
 *     missing these calls return ERR_CUDA (tloam_b200_last_error names the file) and nothing else is affected.
 * intensity null: INVALID_ARG; mapping off: NOT_READY (and, for _frame, NOT_READY like tloam_b200_global_map_append_frame). */
int tloam_b200_global_map_append_intensity(tloam_b200_handle* h, const double pose[16], const double* xyz, const double* intensity,
                                           size_t n);
int tloam_b200_global_map_append_intensity_chained(tloam_b200_handle* h, const double* xyz, const double* intensity, size_t n);
/* the raw scan of the last tloam_b200_process_raw_scan with its intensity (as many values as that scan has rows) */
int tloam_b200_global_map_append_frame_intensity(tloam_b200_handle* h, const double pose[16], const double* intensity);
int tloam_b200_global_map_append_frame_intensity_chained(tloam_b200_handle* h, const double* intensity);
/* *has = 1 if the map has an intensity channel (non-empty, every point with one; synchronises).  Reports the sticky flags
 * as tloam_b200_global_map_size does. */
int tloam_b200_global_map_has_intensity(tloam_b200_handle* h, int* has);
/* intensities of map points [first, first + count) to out (synchronises).  NOT_READY when the map has no channel,
 * INVALID_ARG past the end. */
int tloam_b200_global_map_intensity_download(tloam_b200_handle* h, size_t first, size_t count, double* out);
/* tloam_b200_global_map_append[_chained] of a HOST packed scan (see tloam_packed_scan): one upload, unpacked on the device.
 * With an intensity field the frame is an intensity frame (as tloam_b200_global_map_append_intensity), without one a plain
 * frame.  scan null or an invalid layout: INVALID_ARG; mapping off: NOT_READY. */
int tloam_b200_global_map_append_packed(tloam_b200_handle* h, const double pose[16], const tloam_packed_scan* scan);
int tloam_b200_global_map_append_packed_chained(tloam_b200_handle* h, const tloam_packed_scan* scan);

/* ---- Loop closure (place recognition; the reference is pure odometry).  Every added frame gets a Scan Context descriptor
 * (Kim & Kim, IROS 2018) kept in a database on the device, and is compared with EVERY earlier frame at EVERY column shift.
 *   - Descriptor.  Every finite row (x, y, z) of the scan, sensor frame: r = sqrt(x*x + y*y) (separately rounded, no FMA);
 *     a row with r > max_radius is left out.  ring = clamp(ceil(r / max_radius * n_ring), 1, n_ring) - 1.  sector = the
 *     number of sector boundaries k = 1 .. n_sector - 1 the row lies strictly counter-clockwise of, where boundary k is the
 *     direction (cos, sin)(2 pi k / n_sector) computed by the C library's cos / sin on the host, a row of the upper
 *     half-plane (y > 0, or y == 0 and x >= 0) is compared with the boundaries k < n_sector / 2 and lies below the others,
 *     a row of the lower half-plane lies above those and is compared with the rest, and "counter-clockwise of (c, s)" is
 *     c*y - s*x > 0 (separately rounded): Scan Context's ceil-and-clamp sector of the azimuth in [0, 360), without atan2.
 *     Bin (ring, sector) = max of z + lidar_height over its rows; an empty bin is 0, a negative maximum stays.
 *   - Next to the n_ring x n_sector bins (row-major): the ring key (each ring's sum in sector order / n_sector) and the
 *     column norms (sqrt of the sum of squares in ring order).  Sums start from +0.0.
 *   - Distance of query A and candidate B at shift s: B_s[:, c] = B[:, (c - s) mod n_sector] (np.roll(B, s, axis=1)).  A
 *     column c counts when the norms of A[:, c] and B_s[:, c] are both non-zero; cos_c = (a . b, summed in ring order) /
 *     (|a| * |b|); distance = 1 - (sum of cos_c in ascending c) / count, or 1.0 when no column counts (Scan Context divides
 *     by zero there).  Every value is rounded as written, so the device's distances are bit-reproducible on the host.
 *   - Search.  Frame i (the i-th add since enable / reset, from 0) is compared with every frame j <= i - exclude_recent at
 *     every shift; the result is the minimum by (distance, j, s), lexicographic.  is_loop = distance < dist_threshold.
 *     yaw = -s * 2 pi / n_sector wrapped to (-pi, pi] (computed as k * (2 pi / n_sector), k = -s, or n_sector - s when
 *     2 s >= n_sector): p_candidate ~ Rz(yaw) . p_query, a coarse alignment.  No eligible frame: candidate -1, shift 0,
 *     yaw 0, distance +inf, is_loop 0.
 *   - Adds are enqueued on the handle's stream with no host round trip (the host synchronises only to grow the database,
 *     x1.5); tloam_b200_loop_result waits for the newest add only.  Nothing here touches the odometry's buffers.
 *   - The kernels live in libtloam_b200_loop.so, loaded from this library's directory on the first loop call; if it is
 *     missing these calls return ERR_CUDA (tloam_b200_last_error names the file).  Off until tloam_b200_loop_enable:
 *     every other loop call returns NOT_READY, and nothing is allocated or launched. */
typedef struct tloam_loop_config {
  double lidar_height;                 /* added to z (Scan Context's LIDAR_HEIGHT) */
  int n_ring, n_sector;                /* n_ring * n_sector <= 4096 */
  double max_radius;                   /* m */
  int exclude_recent;                  /* the newest frames a query skips: frame i sees j <= i - exclude_recent */
  double dist_threshold;               /* is_loop below this distance */
  size_t initial_capacity_frames;      /* database slots before the first growth */
} tloam_loop_config;
typedef struct tloam_loop_result {
  long long query, candidate;          /* frame indices since enable / reset; candidate -1: no eligible frame */
  int shift, is_loop;
  double yaw, distance;                /* rad; see above */
} tloam_loop_result;
/* lidar_height 2.0, n_ring 20, n_sector 60, max_radius 80 m, exclude_recent 50, dist_threshold 0.13 (Scan Context's),
 * initial_capacity_frames 1024 */
void tloam_b200_loop_default_config(tloam_loop_config* c);
/* (re)starts an empty database with this configuration.  INVALID_ARG: cfg null, n_ring or n_sector < 1, n_ring * n_sector
 * > 4096, max_radius <= 0 or not finite, exclude_recent < 0, lidar_height or dist_threshold not finite. */
int tloam_b200_loop_enable(tloam_b200_handle* h, const tloam_loop_config* cfg);
/* empties the database (the configuration and the buffers stay).  NOT_READY if not enabled. */
int tloam_b200_loop_reset(tloam_b200_handle* h);
/* adds the raw scan the last tloam_b200_process_raw_scan* uploaded (the corrected scan after a timed call) and enqueues
 * its query.  NOT_READY under tloam_b200_global_map_append_frame's rule (no such scan, or a segmentation / process call
 * since). */
int tloam_b200_loop_add_frame(tloam_b200_handle* h);
/* the same for a HOST cloud (n x 3 FP64 AoS, NaN / Inf rows allowed), uploaded */
int tloam_b200_loop_add(tloam_b200_handle* h, const double* xyz, size_t n);
/* the newest add's result (waits for that add).  NOT_READY before the first add since enable / reset. */
int tloam_b200_loop_result(tloam_b200_handle* h, tloam_loop_result* out);
/* frames in the database */
int tloam_b200_loop_size(tloam_b200_handle* h, size_t* n_frames);
/* frame's descriptor to out: n_ring * n_sector bins (row-major), n_ring ring key values, n_sector column norms
 * (synchronises).  INVALID_ARG past the last frame. */
int tloam_b200_loop_descriptor_download(tloam_b200_handle* h, size_t frame, double* out);
/* the descriptors of frames [first, first + count), one slot after another, in one copy (synchronises): what
 * tloam_b200_relocalize_set_places takes.  INVALID_ARG past the last frame. */
int tloam_b200_loop_descriptors_download(tloam_b200_handle* h, size_t first, size_t count, double* out);

/* ---- Loop verification (opt-in, on top of loop closure): a geometric check of a candidate that also gives the relative
 * pose a pose-graph edge needs.  Scan Context's yaw is one sector coarse and it gives no translation; a descriptor match
 * alone is no evidence of a loop.
 *   - Keyframes.  After tloam_b200_loop_verify_enable, every tloam_b200_loop_add_frame / tloam_b200_loop_add also stores
 *     that frame's keyframe: VoxelDownSample(voxel) of the scan's finite rows (the scan the descriptor reads), in the
 *     sensor frame, by the global map's ordered path (each voxel the fixed-point average of its rows, voxels in ascending
 *     (ix, iy, iz)).  Every add owns exactly one keyframe slot: an empty or all-non-finite scan, or one whose extent
 *     reaches 2^21 voxels on an axis (the global map's key-range refusal), gets an empty keyframe, so keyframe i is always
 *     loop frame i.  The store lives on the device; it is sized from an upper bound tightened by asynchronous read-backs
 *     and grows x1.5 with one synchronisation, so an add does not synchronise.  The global map's buffers are not used.
 *   - Verification of keyframe `query` (Q) against keyframe `candidate` (M) from the initial T = guess: T_cand_query with
 *     p_cand ~ T . p_query (tloam_loop_result's yaw convention).  Per pass, for every q in Q: p = R q + t, each component
 *     ((R[r][0] * qx + R[r][1] * qy) + R[r][2] * qz) + t[r], every operation separately rounded; its match is the nearest
 *     m in M by d2 = ((px - mx)^2 + (py - my)^2) + (pz - mz)^2 (separately rounded), the lowest index on a tie: an exact
 *     search over all of M, no grid, no radius.  The pair is an inlier iff d2 <= r * r.
 *   - Step.  Gauss-Newton on SE(3), left perturbation: e = p - m, J = [I3, -[p]x]; H = sum J^T J, g = sum J^T e over the
 *     inliers (a fixed reduction order: a run is bit-deterministic); delta = (upsilon, omega) = -H^-1 g by LDL^T; T <-
 *     exp(delta) . T with Sophus' exp.  Fewer than 6 inliers, or a pivot that is not positive and finite, stops the run.
 *   - Radius.  r starts at corr_dist_coarse.  After a step with |upsilon| < eps_translation and |omega| < eps_rotation: if
 *     r == corr_dist_fine the run has converged, else r <- max(r / 2, corr_dist_fine).  At most max_iterations steps.
 *   - Result, at the final T with one more pass at r = corr_dist_fine: inliers, rmse = sqrt(sum of their d2 / inliers) (0
 *     without inliers), fitness = the mean nearest-neighbour d2 over ALL of Q (PCL's getFitnessScore(); the ground plane
 *     matches almost anywhere, so an inlier ratio alone does not separate unrelated places), accepted = converged &&
 *     fitness <= max_fitness.  An empty keyframe: no pass, T = guess, fitness +inf, not accepted.
 *   - The kernels live in libtloam_b200_loopv.so, loaded from this library's directory on the first verification call; if
 *     it is missing these calls return ERR_CUDA (tloam_b200_last_error names the file).  Off until enabled: nothing is
 *     allocated or launched, and the loop calls give the bits and launch counts they give without it. */
typedef struct tloam_loop_verify_config {
  double voxel;                        /* keyframe down-sample, m */
  double corr_dist_coarse;             /* first correspondence radius, m */
  double corr_dist_fine;               /* last correspondence radius, m (<= corr_dist_coarse) */
  int max_iterations;                  /* Gauss-Newton steps, 1 .. 200 */
  double eps_translation;              /* m */
  double eps_rotation;                 /* rad */
  double max_fitness;                  /* m^2 */
  size_t initial_capacity_points;      /* keyframe store points before the first growth */
} tloam_loop_verify_config;
enum {
  TLOAM_LOOP_VERIFY_CONVERGED = 0,
  TLOAM_LOOP_VERIFY_ITERATION_LIMIT = 1,
  TLOAM_LOOP_VERIFY_FEW_INLIERS = 2,   /* fewer than 6 inliers in a pass */
  TLOAM_LOOP_VERIFY_SINGULAR = 3,      /* an LDL^T pivot not positive and finite */
  TLOAM_LOOP_VERIFY_EMPTY = 4          /* a keyframe without points */
};
typedef struct tloam_loop_verify_result {
  long long query, candidate;
  double T[16];                        /* T_cand_query, column-major: p_cand ~ T . p_query */
  double fitness;                      /* m^2, mean nearest-neighbour d2 over every query keyframe point */
  double rmse;                         /* m, over the inliers at corr_dist_fine */
  long long inliers;
  long long n_query_points, n_candidate_points;   /* keyframe sizes */
  int iterations;                      /* Gauss-Newton steps taken */
  int termination;                     /* TLOAM_LOOP_VERIFY_* */
  int accepted;
} tloam_loop_verify_result;
/* voxel 0.5 m, corr_dist_coarse 4 m, corr_dist_fine 1 m, max_iterations 40, eps_translation 1e-4 m, eps_rotation 1e-5 rad,
 * max_fitness 1.0 m^2, initial_capacity_points 2^21 (DESIGN.md section 4c has how they were chosen) */
void tloam_b200_loop_verify_default_config(tloam_loop_verify_config* c);
/* stores a keyframe with every later add.  Only while the loop database is empty (right after tloam_b200_loop_enable or
 * tloam_b200_loop_reset), else NOT_READY.  tloam_b200_loop_reset empties the keyframes and keeps verification on;
 * tloam_b200_loop_enable turns it off.  INVALID_ARG: cfg null; a value not finite or not > 0; corr_dist_fine >
 * corr_dist_coarse; max_iterations outside [1, 200]. */
int tloam_b200_loop_verify_enable(tloam_b200_handle* h, const tloam_loop_verify_config* cfg);
/* frame's keyframe (n x 3 FP64) to out (synchronises); *n = its size.  INVALID_ARG past the last frame or when
 * capacity_points < *n; NOT_READY when verification is off.  For tests and viewers. */
int tloam_b200_loop_keyframe_download(tloam_b200_handle* h, size_t frame, double* out, size_t capacity_points, size_t* n);
/* aligns keyframe query to keyframe candidate from guess (column-major 4 x 4; null: identity), enqueued behind every earlier
 * add, and returns once the result is home.  BAD_POSE: guess not rigid; INVALID_ARG: an index out of range; NOT_READY:
 * verification off. */
int tloam_b200_loop_verify(tloam_b200_handle* h, long long query, long long candidate, const double guess[16],
                           tloam_loop_verify_result* out);
/* the last tloam_b200_loop_verify's matches at pass k, the pass at the k-th iterate of T (0: the guess; k = iterations:
 * the final pass): per query keyframe point the candidate keyframe row (index) and its d2 (synchronises; *n = query
 * keyframe size; either output may be null).  INVALID_ARG: k outside [0, iterations], capacity < *n, or a run that made
 * no pass (an empty keyframe); NOT_READY: no verification since enable. */
int tloam_b200_loop_verify_matches(tloam_b200_handle* h, int pass, int* index, double* d2, size_t capacity, size_t* n);

/* ---- Pose graph (opt-in): the back end of loop closure.  The odometry chain and the accepted loop verifications are
 * optimised together on the device; the corrected poses and the map -> odom correction come out.  The global map, the
 * keyframes and the odometry state are not touched (tloam_b200_global_map_correct, below, moves the map).
 *   - Nodes.  Node k keeps the pose O_k it was added with for ever.  tloam_b200_pose_graph_add_node records a host pose;
 *     tloam_b200_pose_graph_add_node_chained records the device pose of the frame the handle enqueued last
 *     (tloam_b200_get_result's pose, the one tloam_b200_global_map_append_frame_chained reads; identity before the first
 *     match) by a copy on the handle's stream, without synchronising.  Calling it next to every tloam_b200_loop_add_frame
 *     keeps node i = loop frame i.  The store grows x1.5 with one synchronisation.
 *   - Edges.  Odometry (k - 1, k) for every k >= 1 with Z = O_{k-1}^-1 O_k and Omega_odom = diag(1 / sigma_odom_translation^2
 *     x 3, 1 / sigma_odom_rotation^2 x 3); loop (v->candidate, v->query) with Z = v->T and Omega_loop alike.
 *   - Cost sum_e r^T Omega r, r = log(Z^-1 T_i^-1 T_j) (se3.cuh's Sophus log, (upsilon, omega) order).
 *   - Step.  Gauss-Newton with a left perturbation T_k <- exp(delta_k) T_k; node 0 is fixed (the gauge).  First-order
 *     Jacobians J_j = Ad(T_j^-1), J_i = -J_j (the right-Jacobian inverse of r taken as I).  The normal equations
 *     H = M + B^T Omega_loop B (M the odometry chain, B the loop rows) are solved exactly by Woodbury: a block LDL^T of M
 *     along the chain, Y = M^-1 B^T, the capacitance S = Omega_loop^-1 + B Y by a dense Cholesky, delta = u - Y S^-1 B u
 *     with u = M^-1 b.  Every reduction runs in a fixed order: a run is bit-reproducible.
 *   - Every optimisation starts from the odometry poses O_k, so a result depends on the graph only.
 *   - Termination.  CONVERGED: the step's largest |upsilon| component < eps_translation and largest |omega| component
 *     < eps_rotation (the step is applied).  COST_INCREASED: the cost after a larger step is not <= the cost before; the
 *     step is reverted.  ITERATION_LIMIT after max_iterations accepted steps.  SINGULAR: an LDL^T or Cholesky pivot that
 *     is not positive and finite.  NO_LOOPS: no loop edge; nothing is launched and the poses are the O_k bit for bit.
 *   - Memory per optimisation: Y is 6 (N - 1) x (6 L + 1) doubles and S 6 L x (6 L + 1) doubles for N nodes and L loop
 *     edges (4 541 nodes, 183 loops: 240 MB; the default max_loop_edges 1 024 allows 6 GB at 20 000 nodes).
 *   - The kernels live in libtloam_b200_pg.so, loaded from this library's directory on the first optimisation; if it is
 *     missing tloam_b200_pose_graph_optimize returns ERR_CUDA (tloam_b200_last_error names the file).  Off until enabled:
 *     nothing is allocated or launched, and every other call returns NOT_READY. */
typedef struct tloam_pose_graph_config {
  double sigma_odom_translation;       /* m */
  double sigma_odom_rotation;          /* rad */
  double sigma_loop_translation;       /* m */
  double sigma_loop_rotation;          /* rad */
  int max_iterations;                  /* Gauss-Newton steps, 1 .. 100 */
  double eps_translation;              /* m */
  double eps_rotation;                 /* rad */
  size_t max_loop_edges;               /* bounds the optimisation's memory (above) */
  size_t initial_capacity_nodes;       /* node store before the first growth */
} tloam_pose_graph_config;
enum {
  TLOAM_POSE_GRAPH_CONVERGED = 0,
  TLOAM_POSE_GRAPH_ITERATION_LIMIT = 1,
  TLOAM_POSE_GRAPH_COST_INCREASED = 2,
  TLOAM_POSE_GRAPH_SINGULAR = 3,
  TLOAM_POSE_GRAPH_NO_LOOPS = 4
};
typedef struct tloam_pose_graph_result {
  long long nodes, loop_edges;
  int iterations;                      /* accepted steps */
  int termination;                     /* TLOAM_POSE_GRAPH_* */
  double initial_cost;                 /* at the odometry poses */
  double final_cost;                   /* at the returned poses */
  double step_translation;             /* the last step's largest |upsilon| component, m */
  double step_rotation;                /* the last step's largest |omega| component, rad */
} tloam_pose_graph_result;
/* sigma_odom 0.02 m / 0.001 rad, sigma_loop 0.3 m / 0.002 rad, max_iterations 20, eps_translation 1e-4 m, eps_rotation
 * 1e-6 rad, max_loop_edges 1024, initial_capacity_nodes 4096 (DESIGN.md section 4c has how they were chosen) */
void tloam_b200_pose_graph_default_config(tloam_pose_graph_config* c);
/* starts an empty graph (a graph already on is emptied).  INVALID_ARG: cfg null; a sigma or eps not finite or not > 0;
 * max_iterations outside [1, 100]; max_loop_edges 0. */
int tloam_b200_pose_graph_enable(tloam_b200_handle* h, const tloam_pose_graph_config* cfg);
/* empties the graph (nodes, loop edges, the last optimisation) and keeps the configuration */
int tloam_b200_pose_graph_reset(tloam_b200_handle* h);
/* node N = pose (column-major 4 x 4).  BAD_POSE: not rigid */
int tloam_b200_pose_graph_add_node(tloam_b200_handle* h, const double pose[16]);
/* node N = the device pose of the last enqueued frame (no synchronisation) */
int tloam_b200_pose_graph_add_node_chained(tloam_b200_handle* h);
/* loop edge (v->candidate, v->query), Z = v->T.  INVALID_ARG: v null; not v->accepted; an index outside [0, nodes);
 * candidate == query; max_loop_edges edges already.  BAD_POSE: v->T not rigid. */
int tloam_b200_pose_graph_add_loop(tloam_b200_handle* h, const tloam_loop_verify_result* v);
/* either output may be null */
int tloam_b200_pose_graph_size(tloam_b200_handle* h, size_t* nodes, size_t* loop_edges);
/* optimises the graph as it stands, enqueued behind every earlier call, and returns once the result is home */
int tloam_b200_pose_graph_optimize(tloam_b200_handle* h, tloam_pose_graph_result* out);
/* nodes first .. first + count - 1 (count x 16, column-major) to out (synchronises): the last optimisation's poses, and
 * O_k for nodes it did not cover (every node before an optimisation or after NO_LOOPS).  INVALID_ARG past the last node. */
int tloam_b200_pose_graph_download(tloam_b200_handle* h, size_t first, size_t count, double* out);
/* T = T_opt(N - 1) O_{N-1}^-1 of the last optimisation over N nodes (the map -> odom correction); identity before any
 * optimisation and after NO_LOOPS (synchronises) */
int tloam_b200_pose_graph_correction(tloam_b200_handle* h, double T[16]);

/* ---- Robust pose graph: graduated non-convexity (GNC) with a truncated-least-squares (TLS) cost over the loop edges, so
 * that a loop edge that passed verification but closes the wrong place (perceptual aliasing) is rejected instead of bending
 * the trajectory.  It optimises the graph tloam_b200_pose_graph_* built, with that graph's configuration.
 *   - Residual.  Loop edge l has the unweighted squared Mahalanobis residual rho_l = r_l^T Omega_loop r_l, r as above.
 *     Odometry edges are never robustified: they are consecutive scan matches, not place recognition.
 *   - Weights w_l in [0, 1]: cost = sum_odom r^T Omega r + sum_loop w_l r^T Omega r, and its Hessian and gradient alike
 *     (loop edge l's rows are scaled by sqrt(w_l)).
 *   - TLS rule (T-LOAM's updateWeight) with c2 = chi2_threshold, th1 = (mu + 1) / mu c2, th2 = mu / (mu + 1) c2:
 *     w = 1 at rho = 0; w = 0 at rho >= th1; w = 1 at rho <= th2; otherwise w = sqrt(c2 mu (mu + 1) / rho) - mu.
 *   - Schedule.  Every run starts from the odometry poses.
 *       1. Stage 0: all weights 1, the Gauss-Newton schedule of tloam_b200_pose_graph_optimize (max_iterations, the same
 *          accept / revert / converge rules) from the odometry poses; exactly what that call computes.
 *       2. max rho <= c2 at the accepted poses: stop, ALL_INLIERS (the result is stage 0's).
 *       3. mu_0 = c2 / (2 max rho - c2) (<= 0: 1e-10).
 *       4. Outer step: the weights from rho at the current poses; then up to inner_iterations weighted Gauss-Newton steps
 *          from the current poses with the weights fixed (each stage evaluates its start cost under its own weights, and
 *          the accept rule compares weighted costs); then mu <- gnc_factor mu.
 *       5. An update that leaves every weight exactly 0 or 1 is followed by one last stage of up to max_iterations steps at
 *          those weights: CONVERGED.  Otherwise the run stops after max_outer_iterations outer steps: OUTER_LIMIT.  A
 *          singular solve anywhere stops the run: SINGULAR.  No loop edge: NO_LOOPS, nothing is launched.
 *     A stage that ends in COST_INCREASED (its last step reverted) or its own convergence does not stop the run.
 *   - The robust run is the last optimisation: tloam_b200_pose_graph_download, _correction and
 *     tloam_b200_global_map_correct read its poses.  tloam_b200_pose_graph_loop_weights reads its weights.
 *   - Every reduction runs in a fixed order: a run is bit-reproducible.  The outer loop runs on the host, reading a few
 *     bytes of device state after every stage.  The residual and weight kernels live in libtloam_b200_pgr.so, loaded from
 *     this library's directory on the first robust optimisation (missing: ERR_CUDA, tloam_b200_last_error names it). */
typedef struct tloam_pose_graph_robust_config {
  double chi2_threshold;               /* c2, on rho (a squared Mahalanobis distance, 6 degrees of freedom) */
  double gnc_factor;                   /* mu grows by this factor per outer step, > 1 */
  int inner_iterations;                /* Gauss-Newton steps per outer step, 1 .. 100 */
  int max_outer_iterations;            /* 1 .. 1000 */
} tloam_pose_graph_robust_config;
enum {
  TLOAM_POSE_GRAPH_GNC_CONVERGED = 0,
  TLOAM_POSE_GRAPH_GNC_OUTER_LIMIT = 1,
  TLOAM_POSE_GRAPH_GNC_ALL_INLIERS = 2,
  TLOAM_POSE_GRAPH_GNC_SINGULAR = 3,
  TLOAM_POSE_GRAPH_GNC_NO_LOOPS = 4
};
typedef struct tloam_pose_graph_robust_result {
  tloam_pose_graph_result pg;          /* iterations: accepted steps over all stages; termination: the last stage's;
                                          initial_cost: stage 0's (unit weights); final_cost: the last stage's, weighted */
  int outer_iterations;                /* weight updates */
  int gnc_termination;                 /* TLOAM_POSE_GRAPH_GNC_* */
  double mu_final;                     /* the mu of the last weight update (0 when there was none) */
  long long inliers;                   /* loop edges with w == 1 */
  long long rejected;                  /* loop edges with w == 0 */
} tloam_pose_graph_robust_result;
/* chi2_threshold 16.81 (the chi-square 99 % quantile at 6 degrees of freedom), gnc_factor 1.4 (the TLS default of Yang et
 * al., RA-L 2020), inner_iterations 2, max_outer_iterations 100 */
void tloam_b200_pose_graph_robust_default_config(tloam_pose_graph_robust_config* c);
/* optimises the graph as it stands (returns once the result is home).  NOT_READY: the pose graph off.  INVALID_ARG: a null
 * argument; chi2_threshold not finite or not > 0; gnc_factor not finite or <= 1; inner_iterations outside [1, 100];
 * max_outer_iterations outside [1, 1000]. */
int tloam_b200_pose_graph_optimize_robust(tloam_b200_handle* h, const tloam_pose_graph_robust_config* cfg,
                                          tloam_pose_graph_robust_result* out);
/* loop edges first .. first + count - 1: the last optimisation's weights (1.0 for every edge after a plain optimisation,
 * before any, after NO_LOOPS, and for edges added after it).  Synchronises.  INVALID_ARG past the last edge. */
int tloam_b200_pose_graph_loop_weights(tloam_b200_handle* h, size_t first, size_t count, double* w);

/* ---- Loop-corrected global map (opt-in): every frame's block of the global map moved to its pose-graph pose.
 *   - Tracking.  tloam_b200_global_map_correction_enable is allowed only on an empty map (right after
 *     tloam_b200_global_map_enable or _reset; otherwise NOT_READY).  From then on every append records two poses at its
 *     map frame f (the index tloam_b200_global_map_frame_offsets counts; a refused frame takes no slot): O_f, the frame's
 *     odometry pose (the host pose, or for _chained appends the device pose the append reads), and P_f, the pose its block
 *     is expressed at.  P_f = M O_f, where M is the map -> odom correction of the last tloam_b200_global_map_correct
 *     (identity before one).  With M = I bit for bit, P_f is a copy of O_f and the map, the frame table, the intensity
 *     channel and the registered scan are the bits of the untracked map; otherwise the append's registered scan is P_f p.
 *     Tracking costs one extra launch per append and no synchronisation.  tloam_b200_global_map_reset empties both tables,
 *     sets M = I and keeps tracking on; tloam_b200_global_map_enable turns tracking off.
 *   - Correction.  node[f] is the pose-graph node map frame f moves with, or -1 for none (the mapping loop that appends
 *     from frame 1 and adds a node from frame 0 binds map frame f to node f + 1).  Per node k:
 *       Delta_k = T_opt(k) O_k^-1 for a node the last optimisation covered, in the operation order of
 *                 tloam_b200_pose_graph_correction (so Delta of its last node is that call's T bit for bit);
 *       Delta   = the map -> odom correction (tloam_b200_pose_graph_correction's T) for nodes added after it;
 *       Delta   = I for node -1, before any optimisation and after NO_LOOPS.
 *     C_f = Delta O_f (O_f itself when Delta is I bit for bit), so a frame bound to -1 stays at, or returns to, its
 *     odometry pose.  A frame whose C_f equals P_f bit for bit is not touched (correcting twice from one optimisation, or
 *     with Delta = I on a frame still at O_f, changes no bits); every point p of another frame becomes (C_f P_f^-1) p,
 *     and P_f = C_f.  A corrected frame is its block moved rigidly, not a new down-sampling of its scan.
 *     Then M = the map -> odom correction.
 *   - Rounding.  Every product and sum is rounded on its own (no FMA), left to right as written, poses column-major with
 *     R (r, c) = A[4c + r]:  A B: R = sum_c' R_A(r, c') R_B(c', c) over c' = 0, 1, 2, t = (R_A t_B, summed likewise) + t_A;
 *     A B^-1: R(r, c) = sum_c' R_A(r, c') R_B(c, c'), t = t_A - R t_B; the bottom row of both is (0, 0, 0, 1).  A point:
 *     x' = ((M00 x + M01 y) + M02 z) + M03.  tests/map_correct_oracle.py restates it bit for bit.
 *   - Untouched: the frame offsets and count, the intensity channel, the registered-scan buffer, the loop keyframes, the
 *     pose graph and the odometry.  The call synchronises.
 *   - The kernels live in libtloam_b200_gmc.so, loaded from this library's directory by the enable call; if it is missing
 *     the calls return ERR_CUDA (tloam_b200_last_error names the file). */
/* NOT_READY: mapping off, or the map is not empty */
int tloam_b200_global_map_correction_enable(tloam_b200_handle* h);
/* NOT_READY: mapping, tracking or the pose graph off.  INVALID_ARG: n_frames is not the map's frame count, a node[f]
 * outside [-1, nodes), or node null with frames present.  An empty map returns OK and launches nothing. */
int tloam_b200_global_map_correct(tloam_b200_handle* h, const long long* node, size_t n_frames);
/* O_f and P_f of frames first .. first + count - 1 (count x 16 each, column-major; either output may be null;
 * synchronises).  NOT_READY: mapping or tracking off.  INVALID_ARG past the last frame. */
int tloam_b200_global_map_frame_poses(tloam_b200_handle* h, size_t first, size_t count, double* odom, double* current);

/* ---- Dynamic-point removal (opt-in): free-space votes from every appended scan's range image.  A map point is dynamic
 * when later scans look through the place where it sits: the ray in its direction returns from something clearly
 * farther away.  The map itself is never edited: it stays append-only, and the map, its frame table, the intensity
 * channel, the pose tables, the registered scan and the odometry keep the bits they have with removal off.  Two counters
 * per map row, (through, hits), are kept next to it, and tloam_b200_global_map_static_download returns the map without
 * the rows judged dynamic.
 *   - Enable.  tloam_b200_global_map_dynamic_enable is allowed only on an empty map (right after
 *     tloam_b200_global_map_enable or _reset; otherwise NOT_READY).  tloam_b200_global_map_reset zeroes the counters and
 *     keeps removal on; tloam_b200_global_map_enable turns it off.  While it is off nothing is allocated or launched.
 *   - Per append.  Every tloam_b200_global_map_append* variant (host, chained, _frame, intensity, packed) votes with the
 *     sensor-frame rows it transforms (read before the transform) and the pose it places the block at: the host pose, the
 *     device pose for _chained appends, or P_f with correction tracking on.  The votes go to the map rows [0, count)
 *     present before the append; the rows the append adds start at (0, 0).  Voting adds four launches per append with at
 *     least one row and no synchronisation; an append of no rows votes nothing.  When the map grows, the counters are copied
 *     with it.
 *   - Range of a row (x, y, z): r = sqrt((x x + y y) + z z); the row is used iff min_range <= r <= max_range (a NaN or
 *     infinite row never is).
 *   - Pixel of a used row.  Column: Scan Context's sector rule with n_cols sectors (see "Loop closure"): the boundaries
 *     (cos, sin) of 2 pi k / n_cols, k = 1 .. n_cols - 1, by the C library on the host; rows with y > 0 or (y = 0 and
 *     x >= 0) count the k in 1 .. (n_cols - 1) / 2 with c_k y - s_k x > 0, the others (n_cols - 1) / 2 plus the count
 *     over the remaining k.  The sign sequence is monotone within a half-plane, so the device counts it by binary search.
 *     Row: s = z / r against b_k = sin(lo + k (hi - lo) / n_rows), k = 0 .. n_rows, lo / hi = fov_down / fov_up times
 *     (pi / 180), by the C library on the host.  The row is outside the image unless b_0 <= s <= b_n_rows; otherwise its
 *     image row is the number of k in 1 .. n_rows - 1 with s > b_k.
 *   - Range image (n_rows x n_cols, +inf = empty): the minimum r of the scan's used rows per pixel, independent of order.
 *     Window image: for pixel (i, j) the minimum over rows i - window_rows .. i + window_rows clipped to the image and
 *     columns j - window_cols .. j + window_cols wrapped around the azimuth; "unknown" if any pixel of that window is empty.
 *   - Vote of map row m at pose T (R (r, c) = T[4c + r], t = T[12 ..]): d = m - t, q_r = (R(0, r) d0 + R(1, r) d1) +
 *     R(2, r) d2, r_m its range as above.  No vote if r_m is outside [min_range, max_range] or q is outside the image.
 *     Else mg = max(margin_abs, margin_rel r_m); through += 1 iff the window value is known and > r_m + mg; hits += 1 iff
 *     the centre pixel c is not empty and |c - r_m| <= mg.
 *   - Rounding.  Every product, sum, quotient and square root is rounded on its own (no FMA), left to right as written, so
 *     tests/map_dynamic_oracle.py reproduces every counter bit for bit.
 *   - Decision.  A row is dynamic iff through >= min_through and through > hits.
 *   - With correction.  tloam_b200_global_map_correct moves blocks and leaves their counters as they are; later votes see
 *     the moved points.  Votes are not recomputed after a correction.
 *   - The kernels live in libtloam_b200_gmd.so, loaded from this library's directory by the enable call; if it is missing
 *     the calls return ERR_CUDA (tloam_b200_last_error names the file). */
typedef struct tloam_global_map_dynamic_config {
  int n_rows;                          /* range-image rows, 1 .. 1024 */
  double fov_up;                       /* degrees, <= 90 */
  double fov_down;                     /* degrees, >= -90, < fov_up */
  int n_cols;                          /* range-image columns (azimuth sectors), 1 .. 16384 */
  int window_rows;                     /* 0 .. n_rows - 1 */
  int window_cols;                     /* >= 0, 2 window_cols + 1 <= n_cols */
  double margin_abs;                   /* m, >= 0 */
  double margin_rel;                   /* fraction of the range, >= 0 */
  double min_range;                    /* m, > 0 */
  double max_range;                    /* m, >= min_range */
  int min_through;                     /* >= 1 */
} tloam_global_map_dynamic_config;
/* an HDL-64E at the map's 1 m voxel: n_rows 64, fov_up 2.0, fov_down -24.9, n_cols 1024, window_rows 1, window_cols 2,
 * margin_abs 1.0 m, margin_rel 0.02, min_range 3 m, max_range 60 m, min_through 3 (DESIGN.md section 6 has how they were
 * chosen) */
void tloam_b200_global_map_dynamic_default_config(tloam_global_map_dynamic_config* c);
/* NOT_READY: mapping off, or the map is not empty.  INVALID_ARG: cfg null, a value outside its range above, or a row
 * table that is not non-decreasing. */
int tloam_b200_global_map_dynamic_enable(tloam_b200_handle* h, const tloam_global_map_dynamic_config* cfg);
/* the counters of map rows first .. first + count - 1 (either output may be null; synchronises).  NOT_READY: mapping or
 * removal off.  INVALID_ARG past the last row. */
int tloam_b200_global_map_votes_download(tloam_b200_handle* h, size_t first, size_t count, unsigned* through, unsigned* hits);
/* the rows that are not dynamic, in map row order: xyz (*n x 3) and, when the map has an intensity channel, their intensity
 * (intensity may be null; it is not written when the map has no channel).  A count, a scan and a scatter on the device,
 * deterministic; synchronises.  *n is set first: INVALID_ARG when capacity < *n (or xyz null with *n > 0).  NOT_READY:
 * mapping or removal off.  The map's sticky refusal flag is left for the next tloam_b200_global_map_size / _download. */
int tloam_b200_global_map_static_download(tloam_b200_handle* h, double* xyz, double* intensity, size_t capacity, size_t* n);

/* ---- Merged global map: the map's frames merged into one voxel grid, the map a user publishes or saves.  The map is a
 * concatenation of per-frame down-samples, so every place several frames saw appears once per frame; the merge is
 * VoxelDownSample of the whole map (ref: src/open3d/PointCloud2.cpp:358-403), after correction and, optionally, without
 * the rows dynamic-point removal judges dynamic.
 *   - Input cloud C.  The map as it stands in stream order, after every enqueued append and correction: all rows in map
 *     row order, or with static_only the rows tloam_b200_global_map_static_download keeps (through >= min_through and
 *     through > hits is dynamic), still in map row order.
 *   - Bounds.  mb = min(C) - voxel * 0.5 per axis: voxel * 0.5 rounded on its own, then the subtraction.
 *   - Index.  floor((p - mb) / voxel) per axis, the subtraction and the division each rounded on its own (no FMA); every
 *     index is >= 0.
 *   - Key range.  If the index of the max row reaches 2^21 on an axis ((max - mb) / voxel >= 2^21, the limit the frame
 *     appends use), the merge refuses with TLOAM_B200_ERR_VOXEL_RANGE and produces nothing.  The reference's limit is
 *     INT_MAX (it logs "voxel_size is too small").  A selected row with a NaN or infinite coordinate, which no append
 *     produces, has an infinite extent and is refused the same way.
 *   - Averages (AccumulatedPoint, :246-294).  x, y, z and, when the map has a channel, the intensity are each summed with
 *     += over the voxel's rows in ascending row order, from +0.0, then divided by (double)count.  Every operation is
 *     rounded on its own; NaN and Inf intensities propagate.  tests/global_map_merge_oracle.py restates it bit for bit.
 *   - Order.  Voxels in ascending (ix, iy, iz), the order of the per-frame blocks (the reference iterates an
 *     unordered_map: its order is implementation-defined).
 *   - Intensity.  The merged cloud has a channel iff the map has one at merge time (tloam_b200_global_map_has_intensity).
 *   - Nothing else moves: the map, the frame table, the intensity channel, the vote counters, the pose tables, the
 *     registered scan, the keyframes, the pose graph and the odometry keep every bit.  The map's sticky refusal flag is
 *     left for the next tloam_b200_global_map_size / _download.
 *   - Snapshot.  The result stays on the device until the next merge (a refused merge leaves none),
 *     tloam_b200_global_map_reset or tloam_b200_global_map_enable.
 *   - Device.  A bounds pass (one small read-back), one key per row, a stable LSD radix sort on 8-bit digits
 *     (ceil((bits of ix + iy + iz, + 1 with static_only) / 8) passes), a scan of the voxel heads and one thread per voxel;
 *     three synchronisations.  Scratch: 24 B per map row (two key / row-index buffers) plus 1 KiB per 2 048 rows of
 *     radix histograms; output: 32 B per voxel (xyz and intensity).  Both are allocated by the first merge with half as
 *     much again, grow only and are freed by tloam_b200_destroy; a handle that never merges allocates and launches nothing
 *     for it.
 *   - The kernels live in libtloam_b200_gmm.so, loaded from this library's directory by the first merge; if it is missing
 *     the calls return ERR_CUDA (tloam_b200_last_error names the file). */
/* builds the merged cloud and sets *n_voxels; synchronises.  NOT_READY: mapping off, or static_only with removal off.
 * INVALID_ARG: n_voxels null, voxel <= 0 or not finite.  VOXEL_RANGE: extent >= 2^21 voxels on an axis (*n_voxels = 0).
 * An empty selection gives 0 voxels and OK. */
int tloam_b200_global_map_merge(tloam_b200_handle* h, double voxel, int static_only, size_t* n_voxels);
/* voxels [first, first + count) of the last merge: xyz (count x 3) and, when it has a channel, intensity (may be null; not
 * written without a channel).  Synchronises.  NOT_READY: no merge since enable / reset.  INVALID_ARG past the end. */
int tloam_b200_global_map_merged_download(tloam_b200_handle* h, size_t first, size_t count, double* xyz, double* intensity);

/* ---- Loop verification against a submap (opt-in, on top of loop verification): the query keyframe is aligned to the
 * keyframes of the loop frames around the candidate, moved into the candidate's sensor frame by their odometry poses, with
 * a point-to-plane residual.  One sparse keyframe leaves gaps between the sensor's rings that a point-to-point ICP locks
 * onto; the union of 2k + 1 keyframes fills them and the plane residual lets the query slide along a surface.  The
 * result is a tloam_loop_verify_result, so tloam_b200_pose_graph_add_loop takes it as it is.  tloam_b200_loop_verify is
 * not changed by any of this.
 *   - Window.  For candidate c, half window k and F loop frames: frames lo = max(0, c - k) .. hi = min(c + k, F - 1),
 *     without `query` if it lies inside.  Every window frame j has a pose O_j: with poses == NULL the pose graph's node j
 *     (node i = loop frame i), read on the device from the node store -- the odometry pose the node was added with, never
 *     an optimised one, so a verification does not depend on the optimisations before it; otherwise poses[j - lo], a host
 *     array of hi - lo + 1 column-major 4 x 4 poses (the query's entry is not read but must be rigid too).
 *   - Target.  A_j = O_c^-1 O_j, every product and sum rounded on its own, left to right, R (r, c) = O[4c + r]:
 *       R_A(r, c) = (R_c(0, r) R_j(0, c) + R_c(1, r) R_j(1, c)) + R_c(2, r) R_j(2, c)
 *       t_A(r)    = (R_c(0, r) d0 + R_c(1, r) d1) + R_c(2, r) d2,  d = t_j - t_c
 *     The target is the concatenation, in frame order then keyframe row order, of A_j p for every row p of keyframe j:
 *     x' = ((A00 x + A01 y) + A02 z) + A03.  Keyframe c's rows are copied, so k = 0 gives keyframe c bit for bit.  An empty
 *     keyframe contributes nothing; the union is not down-sampled again.
 *   - Normals.  For target row i, the rows j (i among them) with d2(i, j) <= normal_radius * normal_radius, d2 as in "Loop
 *     verification", are visited in ascending j: n_i their number; mean = (sum x_j) / n_i per axis, the sum running from
 *     0.0 in that order; C_ab = (sum (a_j - mean_a) (b_j - mean_b)) / n_i for ab = xx, xy, xz, yy, yz, zz, each product
 *     rounded and added to a sum running from 0.0 in the same order (two passes over the neighbourhood).  The eigenvalues
 *     l0 <= l1 <= l2 and the eigenvector of l0 come from a cyclic Jacobi iteration: at most 32 sweeps over the entries
 *     (0,1), (0,2), (1,2); a sweep starts only while off = (a01^2 + a02^2) + a12^2 > 1e-32 * ((a00^2 + a11^2) + a22^2) and
 *     off != 0; an entry that is 0 is skipped; theta = (a_qq - a_pp) / (2 a_pq), t = sign(theta) / (|theta| +
 *     sqrt(theta^2 + 1)), c = 1 / sqrt(t^2 + 1), s = t c; columns p, q of a, then rows p, q of a, then columns p, q of the
 *     eigenvector matrix become (c x_p - s x_q, s x_p + c x_q); the eigenvalues are sorted by the compare-exchanges (0,1),
 *     (1,2), (0,1), a tie keeping the lower axis first.  Every operation is rounded on its own.  The row's normal is that
 *     eigenvector; it is valid iff n_i >= min_normal_neighbours and l0 <= max_planarity * l1.  Its sign is whatever the
 *     iteration gives and does not enter the result (e and J change sign together).
 *   - Pass.  As in "Loop verification": p = R q + t for every row q of the query keyframe, its match the nearest target
 *     row by (d2, index) over the whole target, an inlier iff d2 <= r * r.
 *   - Step.  Over the inliers whose match m has a valid normal n (the contributing rows): e = (nx (px - mx) + ny (py - my))
 *     + nz (pz - mz), J = [n^T, (p x n)^T] for the left perturbation delta = (upsilon, omega); H = sum J^T J, g = sum J^T e
 *     in a fixed reduction order; delta = -H^-1 g by LDL^T; T <- exp(delta) . T.  Fewer than 6 contributing rows stop the
 *     run with FEW_INLIERS, a pivot that is not positive and finite with SINGULAR.  The radius schedule, the convergence
 *     test and the iteration limit are those of "Loop verification".
 *   - Result, at the final T with one more pass at r = corr_dist_fine: T = T_cand_query; fitness = the mean nearest-neighbour
 *     d2 (point to point, to the target) over ALL query rows; inliers = the contributing rows; rmse = sqrt(sum of their
 *     e^2 / inliers); n_candidate_points = the target's rows; accepted = converged && fitness <= max_fitness.  An empty
 *     query keyframe or an empty target: EMPTY, T = guess, fitness +inf, not accepted.
 *   - One verification is k_lvs_poses, k_lvs_assemble, k_lvs_normals (the normals are computed once, not per pass), then
 *     the rounds of k_lvs_match / k_lvs_reduce / k_lvs_step and the final pass, all on the handle's stream with one copy
 *     home.  The normals' neighbour search is exhaustive: its cost grows with the square of the target's rows.  The
 *     kernels live in libtloam_b200_loopvs.so, loaded from this library's directory by the enable call; if it is missing
 *     the calls return ERR_CUDA (tloam_b200_last_error names the file).  The scratch (target, normals, partials, match
 *     records) is allocated by the first run and grown when a run needs more.  Off until enabled: nothing is allocated or
 *     launched, and every other call gives the bits and launch counts it gives without it. */
typedef struct tloam_loop_verify_submap_config {
  int half_window;                     /* k, 0 .. 50 */
  double normal_radius;                /* m */
  int min_normal_neighbours;           /* >= 3 */
  double max_planarity;                /* a normal is valid iff l0 <= max_planarity * l1 */
  double corr_dist_coarse;             /* first correspondence radius, m */
  double corr_dist_fine;               /* last correspondence radius, m (<= corr_dist_coarse) */
  int max_iterations;                  /* Gauss-Newton steps, 1 .. 200 */
  double eps_translation;              /* m */
  double eps_rotation;                 /* rad */
  double max_fitness;                  /* m^2 */
} tloam_loop_verify_submap_config;
/* half_window 5, normal_radius 1 m, min_normal_neighbours 5, max_planarity 0.1, corr_dist_coarse 4 m, corr_dist_fine 1 m,
 * max_iterations 40, eps_translation 1e-4 m, eps_rotation 1e-5 rad, max_fitness 0.5 m^2 (DESIGN.md section 4c has how they
 * were chosen) */
void tloam_b200_loop_verify_submap_default_config(tloam_loop_verify_submap_config* c);
/* allowed at any database size.  NOT_READY unless loop verification is on; tloam_b200_loop_enable turns it off with loop
 * verification, tloam_b200_loop_reset keeps it on.  INVALID_ARG: cfg null; half_window outside [0, 50];
 * min_normal_neighbours < 3; another value not finite or not > 0; corr_dist_fine > corr_dist_coarse; max_iterations
 * outside [1, 200]. */
int tloam_b200_loop_verify_submap_enable(tloam_b200_handle* h, const tloam_loop_verify_submap_config* cfg);
/* aligns keyframe query to the submap around keyframe candidate from guess (column-major 4 x 4; null: identity), enqueued
 * behind every earlier add, and returns once the result is home.  NOT_READY: submap verification off, or poses null and
 * the pose graph off or with fewer than hi + 1 nodes; INVALID_ARG: an index out of range; BAD_POSE: guess or one of poses
 * not rigid. */
int tloam_b200_loop_verify_submap(tloam_b200_handle* h, long long query, long long candidate, const double guess[16],
                                  const double* poses, tloam_loop_verify_result* out);
/* the last tloam_b200_loop_verify_submap's target: per row its xyz (3), normal (3), validity and neighbour count n_i
 * (synchronises; *n = the target's rows, 0 after an EMPTY run; any output may be null).  INVALID_ARG: capacity < *n;
 * NOT_READY: no submap verification since enable.  For tests and viewers. */
int tloam_b200_loop_verify_submap_target(tloam_b200_handle* h, double* xyz, double* normal, unsigned char* valid, int* neighbours,
                                         size_t capacity, size_t* n);
/* the last tloam_b200_loop_verify_submap's matches at pass k, as tloam_b200_loop_verify_matches: per query keyframe point the
 * target row and its d2 */
int tloam_b200_loop_verify_submap_matches(tloam_b200_handle* h, int pass, int* index, double* d2, size_t capacity, size_t* n);

/* ---- Localization in a prior map (opt-in): each frame's scan is registered, point to plane, against a map loaded once --
 * for example the merged map of an earlier session -- and the pose comes out in the map's frame, with the map <- odom
 * correction.  Nothing here writes the odometry, the pose history, the submap, the global map and its tables, the loop
 * database or the pose graph; every other call keeps its bits and launch counts.
 *   - Map.  n x 3 FP64 rows, fixed after the load; row i's identity is its index.  A non-finite row is INVALID_ARG.
 *   - Index, built once per load.  mb = the rows' min per axis; a row's cell is i_d = floor((x_d - mb_d) / cell), the
 *     subtraction and the quotient each rounded; the largest index per axis must stay below 2^21 and every coordinate's
 *     unit of rounding (|x| 2^-52) below 1e-6 cell (VOXEL_RANGE otherwise);
 *     key = ix << (by + bz) | iy << bz | iz with b_d the bits of the largest index.  The rows are sorted by key by a
 *     stable LSD radix sort (a cell's rows stay in row order); the occupied cells' keys ascend and cell j holds sorted
 *     positions [start_j, start_(j+1)).
 *   - Search.  For a point p and a radius r: the nearest map row with d2 <= r * r (d2 as in "Loop verification", r * r
 *     rounded), by (d2, row index); none when no row is that close.  The cells visited on axis d run from the cell of
 *     p_d - rr rounded down to the cell of p_d + rr rounded up, rr = r (1 + 1e-7) rounded up, clipped to the map's cells;
 *     since the cell index is monotone in x, the result is that of an exhaustive scan limited to d2 <= r * r.  Both radii
 *     a search uses (corr_dist_coarse, normal_radius) must be at most 3 cells.
 *   - Normals, computed once per load for every map row: the rule of "Loop verification against a submap" (ascending row
 *     order, the two-pass covariance, the cyclic Jacobi, validity from min_normal_neighbours and max_planarity) with the
 *     neighbourhood within normal_radius taken from the grid.
 *   - Query.  VoxelDownSample(voxel) of the finite rows of the scan by the ordered path of the loop keyframes: the scan
 *     tloam_b200_process_raw_scan* left on the device (tloam_b200_localize_frame, under the NOT_READY rule of
 *     tloam_b200_global_map_append_frame) or a host cloud (tloam_b200_localize).  An extent of 2^21 voxels is VOXEL_RANGE.
 *   - Guess.  A host guess G (map <- sensor, column-major, rigid), or with guess == NULL the prediction
 *     G = L_prev . (O_prev^-1 . O_now), each product and sum rounded on its own, left to right (R (r, c) = O[4c + r]):
 *       R_D(r, c) = (R_p(0, r) R_n(0, c) + R_p(1, r) R_n(1, c)) + R_p(2, r) R_n(2, c),  t_D(r) = the same with e = t_n - t_p
 *       R_G(r, c) = (R_L(r, 0) R_D(0, c) + R_L(r, 1) R_D(1, c)) + R_L(r, 2) R_D(2, c)
 *       t_G(r)    = ((R_L(r, 0) t_D(0) + R_L(r, 1) t_D(1)) + R_L(r, 2) t_D(2)) + t_L(r)
 *     O_now is the odometry pose of the frame the handle registered last (the pose tloam_b200_pose_graph_add_node_chained
 *     records; identity before the first frame), O_prev the O_now of the previous localization, L_prev its T if it was
 *     accepted and its G otherwise.  Without a host guess, the first localization after a load is NOT_READY.
 *   - Passes, steps, radius schedule, convergence and termination: those of "Loop verification against a submap" with the
 *     map in place of the target and the grid search in place of the exhaustive one.  Pass k's match is the nearest map
 *     row within the pass's radius r_k (index -1 and d2 = +inf when none); the final pass searches within corr_dist_coarse
 *     and counts inliers within corr_dist_fine.
 *   - Result.  T (map <- sensor); T_map_odom = T . O_now^-1: R_M(r, c) = (R_T(r, 0) R_O(c, 0) + R_T(r, 1) R_O(c, 1)) +
 *     R_T(r, 2) R_O(c, 2), t_M(r) = t_T(r) - ((R_M(r, 0) t_O(0) + R_M(r, 1) t_O(1)) + R_M(r, 2) t_O(2)); inliers and rmse
 *     as in the submap verification; fitness = the mean over every query row of min(d2 of its final match,
 *     corr_dist_coarse^2) (a row without a match counts corr_dist_coarse^2); accepted = converged && fitness <= max_fitness.
 *     An empty query or an empty map: EMPTY, T = G, fitness +inf, not accepted.
 *   - Device.  A load is k_loc_bounds (one read-back), k_loc_keys, the radix sort of the merged map (k_gmm_hist /
 *     k_gmm_offsets / k_gmm_scatter per 8-bit digit, k_gmm_head_count / k_gmm_head_scatter), k_loc_cells and
 *     k_loc_normals, then one synchronisation.  A frame is the query's down-sample (one read-back of its size), then
 *     k_loc_predict, the rounds of k_loc_match / k_loc_reduce / k_loc_step, the final pass and k_loc_final, with one copy
 *     home.  Memory: 93 B per map row for the map and its index plus 24 B per row of sort scratch; the kernels live in
 *     libtloam_b200_loc.so, loaded from this library's directory by the enable call (ERR_CUDA if it is missing). */
typedef struct tloam_localize_config {
  double voxel;                        /* query down-sample, m */
  double cell;                         /* grid cell edge, m */
  double normal_radius;                /* m, <= 3 cell */
  int min_normal_neighbours;           /* >= 3 */
  double max_planarity;                /* a normal is valid iff l0 <= max_planarity * l1 */
  double corr_dist_coarse;             /* first correspondence radius, m, <= 3 cell */
  double corr_dist_fine;               /* last correspondence radius, m (<= corr_dist_coarse) */
  int max_iterations;                  /* Gauss-Newton steps, 1 .. 200 */
  double eps_translation;              /* m */
  double eps_rotation;                 /* rad */
  double max_fitness;                  /* m^2 */
} tloam_localize_config;
typedef struct tloam_localize_result {
  double T[16];                        /* map <- sensor, column-major */
  double T_map_odom[16];               /* T . O_now^-1 */
  double guess[16];                    /* the G the run started from */
  int iterations;
  int termination;                     /* TLOAM_LOOP_VERIFY_* */
  int accepted;
  long long inliers;
  double rmse, fitness;
  long long n_query_points, n_map_points;
} tloam_localize_result;
/* voxel 0.5 m, cell 1 m, normal_radius 1 m, min_normal_neighbours 5, max_planarity 0.1, corr_dist_coarse 2 m,
 * corr_dist_fine 0.5 m, max_iterations 30, eps_translation 1e-4 m, eps_rotation 1e-5 rad, max_fitness 0.5 m^2 */
void tloam_b200_localize_default_config(tloam_localize_config* c);
/* turns localization on (or re-configures it) and drops any loaded map.  INVALID_ARG: cfg null; a value not finite or
 * not > 0; min_normal_neighbours < 3; corr_dist_fine > corr_dist_coarse; max_iterations outside [1, 200];
 * corr_dist_coarse or normal_radius > 3 cell. */
int tloam_b200_localize_enable(tloam_b200_handle* h, const tloam_localize_config* cfg);
/* loads a HOST map (n x 3) and builds its index and normals; synchronises.  NOT_READY: localization off.  INVALID_ARG:
 * xyz null with n > 0, n >= 2^32, a non-finite row.  VOXEL_RANGE: an extent of 2^21 cells.  A refused load leaves no map. */
int tloam_b200_localize_set_map(tloam_b200_handle* h, const double* xyz, size_t n);
/* the same with the handle's last tloam_b200_global_map_merge, copied on the device.  NOT_READY: localization off or no
 * merge. */
int tloam_b200_localize_set_map_merged(tloam_b200_handle* h);
/* localizes the scan the last tloam_b200_process_raw_scan* left on the device from guess (NULL: the prediction) and
 * returns once the result is home.  NOT_READY: localization off, no map, no such scan, or guess NULL on the first
 * localization after a load.  BAD_POSE: guess not rigid.  VOXEL_RANGE: the query's extent. */
int tloam_b200_localize_frame(tloam_b200_handle* h, const double guess[16], tloam_localize_result* out);
/* the same for a HOST cloud (n x 3) */
int tloam_b200_localize(tloam_b200_handle* h, const double* xyz, size_t n, const double guess[16], tloam_localize_result* out);
/* the last localization's matches at pass k (0 .. iterations): per query row the map row (-1: none) and its d2 */
int tloam_b200_localize_matches(tloam_b200_handle* h, int pass, int* index, double* d2, size_t capacity, size_t* n);
/* the last localization's query (n x 3) */
int tloam_b200_localize_query(tloam_b200_handle* h, double* xyz, size_t capacity, size_t* n);
/* the loaded map's normals, validity and neighbour counts, per map row (any output may be null) */
int tloam_b200_localize_map_normals(tloam_b200_handle* h, double* normal, unsigned char* valid, int* neighbours, size_t capacity,
                                    size_t* n);
/* the loaded map's cell table: the map row at each sorted position (n), the *n_cells occupied cells' keys and their
 * starts (*n_cells + 1); capacity is that of sorted_rows and must be >= the map's rows (keys and starts need as many) */
int tloam_b200_localize_cells(tloam_b200_handle* h, unsigned* sorted_rows, unsigned long long* keys, unsigned* starts,
                              size_t capacity, size_t* n_cells);

/* ---- Relocalization in a prior map (opt-in, on top of localization): the pose of a scan in the map's frame without a
 * guess -- the first frame after a load, or after tracking is lost -- from the places of a recorded session.
 *   - Places.  Place j is a Scan Context descriptor (one slot of tloam_b200_loop_descriptor_download's layout: bins, ring
 *     key, column norms) and a pose P_j (map <- sensor, column-major, rigid): in the mapping session the loop frames'
 *     descriptors and their corrected poses (the pose graph's, or tloam_b200_global_map_frame_poses).  Loaded once, fixed
 *     after the load; place j's identity is its index.
 *   - Query descriptor.  The descriptor of the raw scan by the rule of "Loop closure", with this configuration's
 *     lidar_height, n_ring, n_sector and max_radius (they must be the ones the places were made with; only the slot size
 *     is checked).
 *   - Candidates.  Per place its best shift, the minimum of (distance, shift) over every shift, the distance exactly
 *     Scan Context's.  The places whose best distance is < max_distance, ordered by (distance, place); the first top_k are
 *     the hypotheses, rank 0 .. n_hypotheses - 1.  There is no exclude_recent.
 *   - Guess of hypothesis k (place j, shift s): G_k = P_j . Rz(yaw_s) with tloam_loop_result's yaw convention
 *     (p_place ~ Rz(yaw) p_query).  cos and sin are the sector boundary table's: direction m = (-s) mod n_sector, direction 0
 *     is (1, 0), direction m > 0 is (cos, sin)(2 pi m / n_sector) by the C library.  R_G(r, c) = (R_P(r, 0) Rz(0, c) +
 *     R_P(r, 1) Rz(1, c)) + R_P(r, 2) Rz(2, c), each product and sum rounded on its own; t_G = t_P.
 *   - Refinement.  Each hypothesis is exactly the run of "Localization in a prior map" from G_k: the same query, passes,
 *     radius schedule, termination, fitness and accepted; hypothesis k's result is tloam_b200_localize(scan, G_k) on the
 *     same map.
 *   - Selection.  The winner is the accepted hypothesis minimal by (fitness, rank); without one, the hypothesis minimal by
 *     (fitness, rank), reported but not accepted.  ambiguous: another accepted hypothesis has fitness <= ambiguity_ratio *
 *     the winner's (rounded) and a pose distinct from the winner's: |t_a - t_b| (d2 as in "Loop verification", then sqrt)
 *     > distinct_translation, or angle > distinct_rotation with angle = acos(clamp((tr - 1) * 0.5, -1, 1)), tr = the sum
 *     over the 9 entries in row-major order of R_a(i, j) R_b(i, j) (= trace(R_a^T R_b)), evaluated as clamp(...) <
 *     cos(distinct_rotation).  accepted = the winner is accepted and the result is not ambiguous.  T_map_odom = T . O_now^-1
 *     by the localization's rule.
 *   - Effect.  An accepted relocalization writes the localization's prediction memory as an accepted localization does
 *     (L = T, O = O_now), so the next tloam_b200_localize_frame(NULL) predicts from it.  A rejected one changes no
 *     localization state.  tloam_b200_localize_query / _matches keep describing the last tloam_b200_localize*.  Nothing
 *     else is written: odometry, pose history, submap, global map, loop database, pose graph, and every other call's
 *     launch counts.  No candidate: OK, n_hypotheses 0, place -1, T identity, not accepted.
 *   - Device.  k_sc_bin / k_sc_finish (libtloam_b200_loop.so) into a slot of its own, the query's down-sample (one
 *     read-back of its size), then k_rl_search, k_rl_topk, k_rl_guess and the K hypotheses' ICP in one launch sequence
 *     (k_rl_match / k_rl_reduce over query blocks x top_k, k_rl_step and k_rl_final one warp per hypothesis), k_rl_select,
 *     and one copy home.  The kernels live in libtloam_b200_reloc.so, loaded from this library's directory by the enable
 *     call (ERR_CUDA if it is missing). */
typedef struct tloam_relocalize_config {
  double lidar_height;                 /* the descriptor's, as tloam_loop_config */
  int n_ring, n_sector;
  double max_radius;                   /* m */
  int top_k;                           /* hypotheses, 1 .. 64 */
  double max_distance;                 /* a place is a candidate below this Scan Context distance */
  double distinct_translation;         /* m */
  double distinct_rotation;            /* rad */
  double ambiguity_ratio;              /* >= 1 */
} tloam_relocalize_config;
typedef struct tloam_relocalize_hypothesis {
  long long place;
  int shift;
  double distance;                     /* the place's Scan Context distance at that shift */
  tloam_localize_result result;        /* its run from G_k (result.guess) */
} tloam_relocalize_hypothesis;
typedef struct tloam_relocalize_result {
  tloam_localize_result result;        /* the winner's run */
  long long place;                     /* the winner's place, -1 without hypotheses */
  int shift;
  double distance;
  int n_hypotheses;
  int winner;                          /* its rank, -1 without hypotheses */
  int ambiguous;
  int accepted;
} tloam_relocalize_result;
/* the loop closure's descriptor shape, top_k 8, max_distance 0.4, distinct_translation 2 m, distinct_rotation 10 deg,
 * ambiguity_ratio 1.5 (DESIGN.md section 4c has how they were checked) */
void tloam_b200_relocalize_default_config(tloam_relocalize_config* c);
/* turns relocalization on (or re-configures it) and drops the places.  NOT_READY: localization off.  INVALID_ARG: cfg
 * null, the descriptor shape as tloam_b200_loop_enable refuses it, top_k outside [1, 64], a value not finite,
 * distinct_translation or distinct_rotation < 0, ambiguity_ratio < 1. */
int tloam_b200_relocalize_enable(tloam_b200_handle* h, const tloam_relocalize_config* cfg);
/* loads n places from HOST arrays: n descriptor slots and n poses (16 each, column-major).  NOT_READY: relocalization
 * off.  INVALID_ARG: a null array with n > 0, a non-finite value.  BAD_POSE: a pose not rigid.  A refused load leaves
 * no places. */
int tloam_b200_relocalize_set_places(tloam_b200_handle* h, const double* descriptors, const double* poses, size_t n);
/* the same with the handle's own loop database as the descriptors, copied on the device.  NOT_READY: relocalization or
 * loop closure off.  INVALID_ARG: n != tloam_b200_loop_size, or a descriptor shape other than the loop closure's. */
int tloam_b200_relocalize_set_places_loop(tloam_b200_handle* h, const double* poses, size_t n);
/* relocalizes the scan the last tloam_b200_process_raw_scan* left on the device and returns once the result is home.
 * NOT_READY: relocalization off, no map, no places, or no such scan (tloam_b200_localize_frame's rule).  VOXEL_RANGE: the
 * query's extent. */
int tloam_b200_relocalize_frame(tloam_b200_handle* h, tloam_relocalize_result* out);
/* the same for a HOST cloud (n x 3) */
int tloam_b200_relocalize(tloam_b200_handle* h, const double* xyz, size_t n, tloam_relocalize_result* out);
/* the last relocalization's hypotheses in rank order (*n = n_hypotheses; INVALID_ARG if capacity < *n) */
int tloam_b200_relocalize_hypotheses(tloam_b200_handle* h, tloam_relocalize_hypothesis* out, size_t capacity, size_t* n);
/* the last relocalization's matches of hypothesis k at pass p (0 .. its iterations), as tloam_b200_localize_matches */
int tloam_b200_relocalize_matches(tloam_b200_handle* h, int hypothesis, int pass, int* index, double* d2, size_t capacity,
                                  size_t* n);

/* ---- Updating a prior map (opt-in, on top of localization): the prior map of "Localization in a prior map" is kept as it
 * was loaded, and each localized frame votes on it and proposes what is new; one build gives the updated map, which
 * tloam_b200_localize_set_map_updated loads in its place.  A car parked when the map was made and gone now is seen
 * through; a wall or a street that is new finds no prior row near it.
 *   - State.  Two counters (through, hits) per prior row; the additions: rows in the map's frame, each with its frame
 *     number and its own (through, hits).  tloam_b200_map_update_enable and every map load (tloam_b200_localize_set_map,
 *     _set_map_merged, _set_map_updated) empty it; tloam_b200_localize_enable turns updating off.  While it is off nothing
 *     is allocated or launched.
 *   - Add.  tloam_b200_map_update_add uses the last tloam_b200_localize_frame or tloam_b200_localize (relocalization runs
 *     do not count).  NOT_READY when there was none since the load or the enable, when the add was already made for it, or
 *     when the scan it read has been replaced since: for _frame the raw scan under tloam_b200_global_map_append_frame's
 *     rule, for a host cloud the next tloam_b200_localize or tloam_b200_relocalize with a host cloud.  A localization that
 *     was not accepted gives OK with used = 0 and changes nothing, so a caller may add after every frame.
 *   - Votes of an add.  The scan rows the localization's query came from (the raw scan or the host cloud, sensor frame)
 *     at T = the result's T vote, by the rule of "Dynamic-point removal" with this configuration's image (range image,
 *     window image, through and hits), first on every prior row, then on every addition of the earlier adds.  The rows this
 *     add appends start at (0, 0).
 *   - Novelty of an add.  For each query row q in query order, p = T q by the localization's final pass:
 *     p_r = ((R(r, 0) q0 + R(r, 1) q1) + R(r, 2) q2) + t_r, each product and sum rounded on its own.  p is new iff no prior
 *     row (removed or not) has d2(p, m) <= novel_radius * novel_radius (d2 as in "Loop verification", the square rounded);
 *     the cells visited are those of the localization's grid search, so the answer is the exhaustive scan's.  The new p
 *     are appended to the additions in query order with frame number f = the number of used adds before this one since
 *     the state was emptied.
 *   - Removed.  A row (prior or addition) is removed iff through >= image.min_through and through > hits.
 *   - Build.  One cloud: the prior rows that are not removed, in row order (tloam_gmd_static: the rows
 *     tloam_b200_global_map_static_download's rule keeps, bit for bit), then the supported voxels.  The voxels are
 *     VoxelDownSample(voxel) of the additions that are not removed, by the rules of "Merged global map": bounds, index,
 *     VOXEL_RANGE at 2^21 voxels, sums in row order from +0.0 then / count, ascending key order.  A voxel is supported
 *     iff its rows come from at least min_frames distinct adds: the frame numbers never decrease along the additions, so
 *     within a voxel (rows in row order) the distinct count is 1 + the number of increases.  A session with no removal and
 *     no supported voxel builds the prior map bit for bit.  The cloud stays on the device until the next build, enable, or
 *     tloam_b200_localize_enable; a refused build leaves none.
 *   - Rounding.  Every product, sum, quotient and square root is rounded on its own, left to right as written, so
 *     tests/map_update_oracle.py reproduces every counter, addition and row bit for bit.
 *   - Nothing else moves.  The localization results and its prediction memory, the odometry, the pose history, the
 *     submap, the global map and its tables, the loop database and the pose graph keep their bits, and every other call
 *     its launch counts.
 *   - Device.  An add is k_mu_pose, tloam_gmd_vote twice (k_gmd_clear, k_gmd_bin, k_gmd_window, k_gmd_vote: the prior rows
 *     with a device word holding their count, then the additions with the device-side count), then k_mu_novel, k_mu_count
 *     and k_mu_scatter.  The host bounds the additions' count by the count at its last read-back plus the query rows of
 *     every add since; an add synchronises once, to read the count back, only when that bound passes the buffer's
 *     capacity, and when fewer rows than 16 adds of its size are left then, the buffer grows in the same add without a
 *     further synchronisation (the rows copied on the stream, the old buffer freed at a later synchronisation), so a
 *     read-back comes at most once per 16 adds of one size.  Every other add, the first after an enable or a load among
 *     them, enqueues its work and returns.  The prior rows' counters are allocated by the enable and by the loads.  A build is k_gmd_count / k_gmd_scatter over the prior rows, k_mu_bounds,
 *     k_mu_keys, the shared radix sort (k_gmm_hist / k_gmm_offsets / k_gmm_scatter per 8-bit digit, k_gmm_head_count /
 *     k_gmm_head_scatter), k_mu_average, k_mu_count and k_mu_scatter, with four synchronisations.
 *   - Memory.  8 B per prior row (the counters); 36 B per addition row (xyz, frame, counters); per build 24 B per row of
 *     the cloud plus 49 B per addition row of sort scratch and voxels; 25 B per query row; two range images of the
 *     configuration's size.  The kernels live in libtloam_b200_mapu.so and libtloam_b200_gmd.so, loaded from this
 *     library's directory by the enable call (ERR_CUDA if one is missing). */
typedef struct tloam_map_update_config {
  tloam_global_map_dynamic_config image;   /* the votes' range image and removal rule, as "Dynamic-point removal" */
  double novel_radius;                 /* m, > 0, <= 3 localization cells */
  double voxel;                        /* the additions' voxel, m, > 0 */
  int min_frames;                      /* distinct adds a voxel needs, >= 1 */
} tloam_map_update_config;
typedef struct tloam_map_update_add_result {
  int used;                            /* 0: the localization was not accepted, nothing changed */
  long long frame;                     /* this add's frame number, -1 when not used */
  long long n_scan_points;             /* the scan rows that voted */
  long long n_query_points;            /* the query rows tested for novelty */
} tloam_map_update_add_result;
typedef struct tloam_map_update_result {
  long long n_prior, n_prior_removed;          /* prior rows, and those removed */
  long long n_additions, n_additions_removed;  /* addition rows, and those removed */
  long long n_voxels, n_voxels_kept;           /* the additions' voxels before and after the min_frames test */
  long long n_total;                           /* the cloud's rows: n_prior - n_prior_removed + n_voxels_kept */
} tloam_map_update_result;
/* image: the dynamic removal's defaults; novel_radius 0.5 m, voxel 0.5 m, min_frames 3 (DESIGN.md section 4c has how they
 * were checked) */
void tloam_b200_map_update_default_config(tloam_map_update_config* c);
/* turns updating on (or re-configures it) and empties its state.  INVALID_ARG: cfg null, an image that
 * tloam_b200_global_map_dynamic_enable refuses, novel_radius or voxel not finite or not > 0, min_frames < 1, or (with
 * localization on) novel_radius > 3 cell.  NOT_READY: localization off. */
int tloam_b200_map_update_enable(tloam_b200_handle* h, const tloam_map_update_config* cfg);
/* votes and appends for the last localization (see Add above).  NOT_READY: updating off, no map, or the rules above. */
int tloam_b200_map_update_add(tloam_b200_handle* h, tloam_map_update_add_result* out);
/* builds the updated cloud; synchronises.  NOT_READY: updating off or no map.  VOXEL_RANGE: the kept additions' extent
 * reaches 2^21 voxels on an axis (no cloud). */
int tloam_b200_map_update_build(tloam_b200_handle* h, tloam_map_update_result* out);
/* the prior rows, the additions and the built cloud's rows (0 without a cloud); any output may be null; synchronises.
 * NOT_READY: updating off or no map. */
int tloam_b200_map_update_size(tloam_b200_handle* h, size_t* n_prior, size_t* n_additions, size_t* n_built);
/* rows [first, first + count) of the built cloud (count x 3).  NOT_READY: no cloud.  INVALID_ARG past the end. */
int tloam_b200_map_update_download(tloam_b200_handle* h, size_t first, size_t count, double* xyz);
/* the counters of rows [first, first + count) of the prior map (which 0) or of the additions (which 1); either output may
 * be null; synchronises.  NOT_READY: updating off or no map.  INVALID_ARG: which not 0 or 1, or past the end. */
int tloam_b200_map_update_votes(tloam_b200_handle* h, int which, size_t first, size_t count, unsigned* through, unsigned* hits);
/* additions [first, first + count): xyz (count x 3) and frame numbers (either may be null); as _votes */
int tloam_b200_map_update_additions(tloam_b200_handle* h, size_t first, size_t count, double* xyz, unsigned* frame);
/* tloam_b200_localize_set_map of the built cloud, copied on the device.  NOT_READY: localization or updating off, or no
 * built cloud.  Like every load it empties the update's state. */
int tloam_b200_localize_set_map_updated(tloam_b200_handle* h);

/* ---- Occupancy grid (opt-in): a 2D occupancy grid of the global map, in the layout of nav_msgs/OccupancyGrid, for a
 * planner.  Every append records a 2D scan of its rows; a build rasterises every map frame's scan at the frame's current
 * pose, so after tloam_b200_global_map_correct the next build follows the loop-corrected trajectory.  The map itself, its
 * frame table, the intensity channel, the vote counters, the pose tables, the registered scan and the odometry keep the
 * bits they have with the grid off.
 *   - Enable.  tloam_b200_occupancy_enable is allowed only on an empty map (right after tloam_b200_global_map_enable or
 *     _reset; otherwise NOT_READY).  tloam_b200_global_map_reset empties the captures and keeps the grid on;
 *     tloam_b200_global_map_enable turns it off.  While it is off nothing is allocated or launched.
 *   - Capture.  Every tloam_b200_global_map_append* variant (host, chained, _frame, intensity, packed) records, in the map
 *     frame slot it takes, the pose it places the block at (the host pose, the device pose for _chained appends, or P_f
 *     with correction tracking on) and the 2D scan of its sensor-frame rows, read before the transform.  A refused append
 *     takes no slot, so the next append overwrites its record; an append of no rows records an empty scan.  Four launches
 *     per append with rows, two without, and no synchronisation.  The records grow with the frame table.
 *   - 2D scan.  A row (x, y, z) is used iff it is finite and min_range <= rho <= max_range, rho = sqrt(x x + y y).  Its
 *     sector is Scan Context's sector rule on (x, y) with n_cols sectors ("Dynamic-point removal", Pixel of a used row).
 *     The obstacle of sector j is the used row with z_lo <= z <= z_hi of least rho, the lowest row index on a tie; its
 *     sensor-frame (x, y, z) is kept.  The floor of sector j is the largest rho of the used rows with z < z_lo.  Either may
 *     be absent (NaN).
 *   - Build pose.  P_f with correction tracking on, otherwise the recorded pose (the same bits until a correction).
 *   - Extent.  W = (max_range + max(|z_lo|, |z_hi|)) + resolution.  origin_x = resolution floor((min_f t_x - W) /
 *     resolution), width = floor(((max_f t_x + W) - origin_x) / resolution) + 1, likewise for y and height.  More than
 *     2^28 cells is VOXEL_RANGE; an empty map gives a 0 x 0 grid.
 *   - Free.  Per frame, every cell whose centre c satisfies |c - t| <= W on both axes, c_x = origin_x + ((double)i + 0.5)
 *     resolution (likewise y): d = c - t in x and y, q_r = R(0, r) d0 + R(1, r) d1 for r = 0, 1 (R(k, r) = P[4r + k]),
 *     rho_c = sqrt(q0 q0 + q1 q1), j the sector of (q0, q1).  The sector's extent e_j is its obstacle's rho, else its
 *     floor's rho.  free += 1 iff e_j exists, rho_c >= min_range and rho_c + free_margin <= e_j.
 *   - Occupied.  Each obstacle o moves to the world as w = P o with the point order of "Loop-corrected global map" (A
 *     point); its cell (floor((w_x - origin_x) / resolution), likewise y) gets occupied += 1.  A hit outside the grid is
 *     counted in dropped instead.  A cell may get both a free and a hit from one frame.
 *   - Value.  With n = occupied + free: -1 if n = 0, else (100 occupied + n / 2) / n in integer arithmetic.  Cells are
 *     row-major from cell (0, 0), i along x, with the origin at the corner of cell (0, 0): nav_msgs/OccupancyGrid's layout.
 *   - Rounding.  Every product, sum, quotient and square root is rounded on its own (no FMA), left to right as written, so
 *     tests/occupancy_oracle.py reproduces every scan, count and value bit for bit.
 *   - Device.  A capture is k_occ_clear, k_occ_bin, k_occ_pick (ties by row index) and k_occ_final into the slot the device
 *     frame count names.  A build is k_occ_extent (one read-back: it synchronises), then k_occ_free (one thread per frame
 *     and window cell, integer atomicAdd), k_occ_hits (one per frame and sector) and k_occ_value, and a read-back of
 *     dropped.  Memory: 32 B per sector and 128 B per frame slot; 9 B per cell, allocated by the first build with half as
 *     much again, grown only and freed by tloam_b200_destroy.
 *   - The kernels live in libtloam_b200_occ.so, loaded from this library's directory by the enable call; if it is missing
 *     the calls return ERR_CUDA (tloam_b200_last_error names the file). */
typedef struct tloam_occupancy_config {
  double resolution;                   /* m per cell, > 0 */
  int n_cols;                          /* sectors of the 2D scan, 1 .. 4096 */
  double z_lo;                         /* the obstacle band in the sensor frame, m, z_lo < z_hi */
  double z_hi;
  double min_range;                    /* m, > 0 */
  double max_range;                    /* m, >= min_range */
  double free_margin;                  /* m, >= 0 */
} tloam_occupancy_config;
typedef struct tloam_occupancy_info {
  double origin_x, origin_y;           /* the corner of cell (0, 0), m */
  double resolution;
  size_t width, height;                /* cells along x and y */
  size_t frames;                       /* map frames rasterised */
  unsigned long long dropped;          /* hits outside the grid */
  unsigned long long cell_tests;       /* window cells the free pass visited (frames x its window's candidates) */
} tloam_occupancy_info;
/* an HDL-64E at 1.73 m: resolution 0.1 m, n_cols 1024, z_lo -1.2 m, z_hi 0.5 m, min_range 3 m, max_range 30 m,
 * free_margin 0.1 m (DESIGN.md section 4c has how they were checked) */
void tloam_b200_occupancy_default_config(tloam_occupancy_config* c);
/* NOT_READY: mapping off, or the map is not empty.  INVALID_ARG: cfg null or a value outside its range above. */
int tloam_b200_occupancy_enable(tloam_b200_handle* h, const tloam_occupancy_config* cfg);
/* rasterises every map frame; synchronises.  NOT_READY: mapping or the grid off.  VOXEL_RANGE: more than 2^28 cells or a
 * non-finite extent (no grid).  info may be null. */
int tloam_b200_occupancy_build(tloam_b200_handle* h, tloam_occupancy_info* info);
/* the last build's values, occupied and free counts (width x height each; any output may be null); synchronises.
 * NOT_READY: the grid off, or no build since the enable or the last reset.  INVALID_ARG: capacity < width x height. */
int tloam_b200_occupancy_download(tloam_b200_handle* h, signed char* cells, unsigned* occupied, unsigned* free_count,
                                  size_t capacity);
/* the 2D scans of map frames first .. first + count - 1: scans (count x n_cols x 4: obstacle x, y, z, floor rho; NaN when
 * absent) and the recorded poses (count x 16, column-major); either may be null; synchronises.  NOT_READY: mapping or the
 * grid off.  INVALID_ARG past the last frame. */
int tloam_b200_occupancy_scans_download(tloam_b200_handle* h, size_t first, size_t count, double* scans, double* poses);

/* ---- Distance field and costmap: the distance from every cell of an occupancy grid to the nearest obstacle, for an
 * optimisation-based planner, and costmap_2d's inflated costs, for a search-based one.
 *   - Source.  tloam_b200_distance_build takes the last tloam_b200_occupancy_build's values on the device (NOT_READY when
 *     the grid is off or not built since the enable or the last reset).  tloam_b200_distance_build_grid takes a host grid
 *     in nav_msgs/OccupancyGrid's layout (int8, width x height, row-major from cell (0, 0), i along x, the origin at that
 *     cell's corner) and works on any handle, mapping on or off: a map_server PGM saved by save_occupancy_map, say.
 *   - Classes, those map_saver writes: obstacle v >= 65, free 0 <= v <= 25, unknown anything else (-1 included).  Unknown
 *     cells are not obstacles.
 *   - sq (uint32, cells^2): for a non-obstacle cell the least di^2 + dj^2 over the obstacle cells, for an obstacle cell
 *     the same over the non-obstacle cells; 0xFFFFFFFF when that set is empty.  Exact integer arithmetic.
 *   - sd (float32, m): (float)(sqrt((double)sq) * resolution), each operation rounded on its own, negated at obstacle
 *     cells; +inf / -inf when sq is 0xFFFFFFFF.
 *   - Cost (uint8, costmap_2d's codes; InflationLayer's costs at the exact distance).  An obstacle cell is 254 (LETHAL).
 *     Otherwise, with R_c = (unsigned) ceil(inflation_radius / resolution) and dist = sqrt((double)sq): c = 253 if
 *     sq <= R_c^2 and dist resolution <= inscribed_radius; (unsigned char)(252.0 exp(-cost_scaling_factor (dist
 *     resolution - inscribed_radius))) if sq <= R_c^2 otherwise; 0 if sq > R_c^2.  A free cell gets c; an unknown cell
 *     gets 253 if c = 253, else 255 (ROS 1's rule with inflate_unknown false).  The table of c by sq (R_c^2 + 1 entries)
 *     is computed per build by this library with std::sqrt / std::exp and uploaded; the device only indexes it.
 *     costmap_2d reaches cells through a wavefront from the obstacle cells, which can give a cell a farther obstacle than
 *     the nearest one; this field uses the exact nearest obstacle and does not reproduce those cells.
 *   - Values (int8): costmap_2d's Costmap2DPublisher table, 0 -> 0, 1 .. 252 -> 1 + (97 (c - 1)) / 251 in integer
 *     arithmetic, 253 -> 99, 254 -> 100, 255 -> -1, so a node publishes the costmap as a nav_msgs/OccupancyGrid with one
 *     copy.
 *   - Query.  tloam_b200_distance_query gives the bilinear interpolation of sd at the cell centres and its gradient, in
 *     FP64 with each product, sum and quotient rounded on its own (no FMA), left to right: u = (x - origin_x) / resolution
 *     - 0.5, v likewise for y; a point is valid iff width >= 2, height >= 2, 0 <= u <= width - 1, 0 <= v <= height - 1;
 *     i = min(floor(u), width - 2), j = min(floor(v), height - 2), a = u - i, b = v - j; with s_pq = sd(i + p, j + q):
 *     d = (1 - b)((1 - a) s00 + a s10) + b((1 - a) s01 + a s11), gx = ((1 - b)(s10 - s00) + b(s11 - s01)) / resolution,
 *     gy = ((1 - a)(s01 - s00) + a(s11 - s10)) / resolution.  An invalid point, and every point of a field with an infinite
 *     value (no obstacle, or only obstacles), gives NaN in all three.
 *   - Lifetime.  A field is a snapshot: a later occupancy build, a map reset or a correction leaves it alone.  The next
 *     distance build replaces it (a build refused with INVALID_ARG, NOT_READY or VOXEL_RANGE keeps it) and
 *     tloam_b200_destroy frees it.
 *   - Limits.  (width - 1)^2 + (height - 1)^2 < 2^32 - 1, otherwise VOXEL_RANGE (a 5 528 x 6 238 grid is at 6.9e7).  A host
 *     grid has 1 .. 2^28 cells, a finite origin and a finite resolution > 0; R_c <= 4096; 0 <= inscribed_radius <=
 *     inflation_radius and cost_scaling_factor >= 0, all finite; otherwise INVALID_ARG.  A 0 x 0 occupancy grid (an empty
 *     map) gives a 0 x 0 field.
 *   - Unchanged.  Nothing is hooked into appends, captures or the occupancy build: the map, its tables, the occupancy
 *     grid and the launch counts of every other call keep their bits, and nothing is allocated or loaded before the first
 *     distance call.
 *   - Device.  A build is k_dist_bands and k_dist_cols (the column pass, one thread per column and 64-row band),
 *     k_dist_rows (one thread per row and source class: the lower envelope of g^2 + (i - k)^2 with every test in 64-bit
 *     integers, cross-multiplied) and k_dist_cost (one per cell), then a read-back of the obstacle count: it synchronises.
 *     A query is k_dist_query, one thread per point.  Memory: 19 B per cell (sq 4, sd 4, the column distance 4, the row
 *     pass's stacks 4, a host grid's copy 1, cost 1, value 1), 16 B per column and band, R_c^2 + 1 B of table and 40 B per
 *     query point, allocated by the first call that needs them, grown only and freed by tloam_b200_destroy.
 *   - The kernels live in libtloam_b200_dist.so, loaded from this library's directory by the first distance call; if it
 *     is missing the calls return ERR_CUDA (tloam_b200_last_error names the file). */
typedef struct tloam_distance_config {
  double inscribed_radius;             /* m: a cell this close to an obstacle is 253 (INSCRIBED) */
  double inflation_radius;             /* m: the costs reach this far */
  double cost_scaling_factor;          /* 1/m: the decay of the cost beyond the inscribed radius */
} tloam_distance_config;
typedef struct tloam_distance_info {
  double origin_x, origin_y;           /* the corner of cell (0, 0), m */
  double resolution;
  size_t width, height;                /* cells along x and y */
  size_t obstacles;                    /* obstacle cells (v >= 65) */
} tloam_distance_info;
/* inscribed_radius 0.9 m (half of a 1.8 m-wide car), inflation_radius 3.0 m, cost_scaling_factor 3.0 (nav2's
 * inflation-layer default).  These are robot parameters, not calibrated: set them for the robot that plans. */
void tloam_b200_distance_default_config(tloam_distance_config* c);
/* from the last occupancy build; synchronises.  INVALID_ARG: cfg null or out of range.  NOT_READY: the occupancy grid off
 * or not built.  VOXEL_RANGE: the grid is too large (Limits).  info may be null. */
int tloam_b200_distance_build(tloam_b200_handle* h, const tloam_distance_config* cfg, tloam_distance_info* info);
/* from a host grid (cells: width x height int8); synchronises.  INVALID_ARG / VOXEL_RANGE as in Limits.  info may be null. */
int tloam_b200_distance_build_grid(tloam_b200_handle* h, const tloam_distance_config* cfg, const signed char* cells,
                                   size_t width, size_t height, double origin_x, double origin_y, double resolution,
                                   tloam_distance_info* info);
/* the last build's sd, sq, costs and values (width x height each, the grid's layout; any output may be null);
 * synchronises.  NOT_READY before any build.  INVALID_ARG: capacity < width x height. */
int tloam_b200_distance_download(tloam_b200_handle* h, float* sd, unsigned* sq, unsigned char* costs, signed char* values,
                                 size_t capacity);
/* n points xy (n x 2, m) -> distance (n) and gradient (n x 2, m per m), either may be null; synchronises.  NOT_READY
 * before any build.  INVALID_ARG: xy null with n > 0. */
int tloam_b200_distance_query(tloam_b200_handle* h, const double* xy, size_t n, double* distance, double* gradient);

/* ---- Path planning: the cost-to-go of every cell of the costmap to a goal (a global planner's potential), and the path
 * down it from any start.
 *   - Source.  The costs (costmap_2d's codes) of the last successful tloam_b200_distance_build or _build_grid, so a plan
 *     runs on the device's own occupancy grid or on a host grid (a localization session's saved PGM).  NOT_READY before
 *     any distance build.
 *   - Cell cost.  A cell is passable when its code c is 0 .. 252, or 255 with allow_unknown set; its traversal cost is then
 *     t = neutral_cost + cost_factor c, with c = 252 for an unknown cell, in integer arithmetic.  253 (INSCRIBED) and 254
 *     (LETHAL) are never passable, nor 255 with allow_unknown 0.  Limits: neutral_cost >= 1, neutral_cost + 252
 *     cost_factor <= 65535 (every t fits 16 bits), allow_unknown 0 or 1; otherwise INVALID_ARG.
 *   - Moves.  8-connected.  A move into a passable neighbour u costs 70 t(u) to a side neighbour and 99 t(u) to a diagonal
 *     one (99 / 70 = 1.41429); a diagonal move is allowed only when both side cells that share its corner are passable, so
 *     no path cuts a corner.  The cost is charged on the cell entered: the goal's t counts, the start's does not.
 *   - Potential P (uint64): the least total cost of a path from a cell to the goal, 0xFFFFFFFFFFFFFFFF at impassable cells
 *     and at cells that cannot reach the goal.  It is the unique solution of P(goal) = 0, P(v) = min over the allowed moves
 *     v -> u of (k t(u) + P(u)): unique because every move costs at least 70, so any order of relaxation gives the same
 *     bits.  Every finite P is below 2^53, so a float64 Dijkstra is exact on the same costs.
 *   - Cells from points: (floor((x - origin_x) / resolution), floor((y - origin_y) / resolution)), each operation rounded
 *     on its own (the occupancy build's hit rule).  A goal that is not finite, lies outside the grid or falls on an
 *     impassable cell gives INVALID_ARG.
 *   - Paths.  From a start s the path repeats one step until it reaches the goal: the next cell is the first allowed
 *     neighbour, in the order (di, dj) = (+1, 0), (0, +1), (-1, 0), (0, -1), (+1, +1), (-1, +1), (-1, -1), (+1, -1), that
 *     minimises k t(u) + P(u).  That minimum is P(v), so every step lowers P by at least 70 and the walk ends.  A path
 *     lists its cells from the start to the goal, both included (one cell for a start on the goal); its cost is P(start).
 *     Status per start: 0 reached; 1 the start is not finite or lies outside the grid; 2 the start cell is impassable; 3
 *     the goal cannot be reached.  A start with a status other than 0 has no cells and the cost 0xFFFFFFFFFFFFFFFF.  The
 *     xy of a path cell is its centre, origin + (i + 0.5) resolution, each operation rounded on its own.
 *   - Lifetime.  A build copies t into the plan's own memory, so the potential is a snapshot: a later distance build,
 *     occupancy build or map call leaves it and the kept paths alone.  The next plan build replaces it and drops the kept
 *     paths (a build refused with INVALID_ARG or NOT_READY keeps both); the next tloam_b200_plan_paths replaces the paths;
 *     tloam_b200_destroy frees them.
 *   - Unchanged.  Nothing is hooked into any other call: the distance field, the occupancy grid, the map and the launch
 *     counts of every other call keep their bits, and nothing is allocated or loaded before the first plan call.
 *   - Device.  A build is k_plan_init (one thread per cell: t, P = INF but 0 at the goal; the goal's 32 x 32-cell tile
 *     and the tiles around it as the first round's work), then rounds of k_plan_round, launched in batches of 32 with a read-back of the next round's work
 *     count after each batch.  A round's blocks each take tiles of the round's worklist, stage a tile's P and t with a
 *     one-cell halo in shared memory, relax it in place to local convergence and write back the cells that fell with a
 *     64-bit atomicMin; a tile whose halo holds a cell that fell is queued for the next round, once per round.  Then
 *     k_plan_count counts the reachable cells: it synchronises.  Paths are k_plan_length (one thread per start: the status,
 *     the cost and the path's length), a read-back of the lengths, the offsets summed on the host and k_plan_walk (one
 *     thread per start: the cells).  Memory: 10 B per cell (P 8, t 2), 12 B per tile (a stamp and two worklists), 32 B
 *     per start and 8 B per path cell, allocated by the first call that needs them, grown only and freed by
 *     tloam_b200_destroy.
 *   - The kernels live in libtloam_b200_plan.so, loaded from this library's directory by the first plan call; if it is
 *     missing the calls return ERR_CUDA (tloam_b200_last_error names the file). */
typedef struct tloam_plan_config {
  unsigned neutral_cost;               /* the cost of a free cell, per 70 of a side move */
  unsigned cost_factor;                /* the cost per costmap code */
  int allow_unknown;                   /* 1: unknown cells (255) are passable at code 252 */
} tloam_plan_config;
typedef struct tloam_plan_info {
  double origin_x, origin_y;           /* the corner of cell (0, 0), m: the distance field's */
  double resolution;
  size_t width, height;                /* cells along x and y */
  size_t goal_i, goal_j;               /* the goal's cell */
  size_t reachable;                    /* cells with a finite potential, the goal included */
  unsigned long long rounds;           /* rounds of k_plan_round that had work */
  unsigned long long tiles;            /* tiles those rounds relaxed */
} tloam_plan_info;
/* neutral_cost 50, cost_factor 3, allow_unknown 1 (global_planner's defaults) */
void tloam_b200_plan_default_config(tloam_plan_config* c);
/* the potential to the goal (goal_x, goal_y) on the last distance field's costs; synchronises.  INVALID_ARG: cfg null or
 * out of range, or a bad goal (Cells from points).  NOT_READY: no distance build yet.  info may be null. */
int tloam_b200_plan_build(tloam_b200_handle* h, const tloam_plan_config* cfg, double goal_x, double goal_y,
                          tloam_plan_info* info);
/* the last plan's P (width x height, the grid's layout; may be null); synchronises.  NOT_READY before any plan build.
 * INVALID_ARG: capacity < width x height. */
int tloam_b200_plan_download(tloam_b200_handle* h, unsigned long long* potential, size_t capacity);
/* the paths from n starts (starts_xy: n x 2, m) down the last plan, kept on the device for tloam_b200_plan_path_cells:
 * offsets (n + 1: path s is cells offsets[s] .. offsets[s + 1] - 1), statuses (n) and costs (n), each may be null;
 * synchronises.  NOT_READY before any plan build.  INVALID_ARG: starts_xy null with n > 0, or n > 2^24. */
int tloam_b200_plan_paths(tloam_b200_handle* h, const double* starts_xy, size_t n, size_t* offsets, int* statuses,
                          unsigned long long* costs);
/* the cells of the last tloam_b200_plan_paths, all paths one after the other: ij (2 ints each) and xy (the centres, 2
 * FP64 each), either may be null; synchronises.  NOT_READY before any tloam_b200_plan_paths since the last plan build.
 * INVALID_ARG: capacity < offsets[n] of that call. */
int tloam_b200_plan_path_cells(tloam_b200_handle* h, int* ij, double* xy, size_t capacity);

/* ---- Frontiers: the boundaries between known free space and unknown space on the costmap (frontier exploration,
 * Yamauchi 1997, as explore_lite finds them), each ranked by the plan's path cost to reach it.
 *   - Source.  The costs (costmap_2d's codes) of the last successful tloam_b200_distance_build or _build_grid, and the
 *     potential P of the last tloam_b200_plan_build, which must have been built on that same field.  NOT_READY when there
 *     is no distance build, no plan, or the plan is older than the field.  The plan is meant to have its goal at the
 *     robot: P(c) is then the cost of the path between c and the robot.
 *   - Frontier cell (explore_lite's isNewFrontierCell, with a threshold): a cell of code 255 (unknown, not inscribed) with
 *     at least one 4-neighbour inside the grid of code <= free_max.
 *   - Frontier: an 8-connected component of frontier cells.  Frontiers are numbered 0, 1, ... (the id) in ascending order
 *     of their least linear cell index j width + i, so the numbering does not depend on the order of any search.
 *   - Per frontier: the size n (cells), the integer sums Si, Sj of its cells' i and j, its bounding box, the centroid
 *     cx = origin_x + ((double)Si / (double)n + 0.5) resolution (likewise cy), and the approach cell: among the
 *     4-neighbours of code <= free_max of its cells, the one with the least P, ties to the lowest linear index, with its
 *     centre origin + (i + 0.5) resolution and its P.  free_max <= 252, so every approach cell is passable under any
 *     plan config.  Status 0 when that P is finite, 1 (unreachable from the plan's goal) otherwise.  Every operation in
 *     FP64 is rounded on its own (no FMA).
 *   - Filter and cost.  A frontier is kept iff (double)n resolution >= min_frontier_size.  For a reachable one
 *     distance = ((double)P / (70.0 (double)neutral_cost)) resolution, the metres of free-cell path of that cost
 *     (neutral_cost is the plan's), and cost = potential_scale distance - gain_scale ((double)n resolution):
 *     explore_lite's formula with the path cost in place of its Euclidean distance.  An unreachable frontier has distance
 *     and cost +infinity.
 *   - Order.  The kept reachable frontiers by (cost, id) ascending, then the kept unreachable ones by id.
 *   - Differences to explore_lite.  It walks free space from the robot, so it finds only the frontiers that touch the
 *     robot's free region; this finds every frontier of the grid and marks the ones the plan cannot reach.  Its distance
 *     is the Euclidean distance to the nearest frontier cell; this one is the exact path cost to the approach cell.
 *   - Limits.  free_max <= 252; min_frontier_size, potential_scale and gain_scale finite and >= 0; otherwise INVALID_ARG.
 *     The distance field's shape limit keeps width x height below 2^32 - 1, so a cell index fits 32 bits.
 *   - Lifetime.  A search is a snapshot, like a plan: later distance builds, plans and map calls leave its frontiers,
 *     cells and labels alone; the next search replaces them (a search refused with INVALID_ARG or NOT_READY keeps them)
 *     and tloam_b200_destroy frees them.
 *   - Unchanged.  Nothing is hooked into any other call: the distance field, the plan, its kept paths, the map and the
 *     launch counts of every other call keep their bits, and nothing is allocated or loaded before the first frontier
 *     call.
 *   - Device.  A search is k_fr_tile (one block per 32 x 32-cell tile: the frontier flags and a union-find of the tile
 *     in shared memory, the larger root linked under the smaller), k_fr_border (lock-free unions with atomicMin across
 *     tile edges and corners), k_fr_flatten (every label its root, which is the component's least index; the frontier
 *     cells counted), a read-back of their count, k_fr_compact (the frontier cells in index order), the stable radix sort
 *     of (root, cell) and its head scan (radix_sort.cuh), k_fr_stats (one warp per frontier over its contiguous cells; integer reductions, no
 *     atomics) and a read-back of the frontiers' statistics.  The cost, the filter and the order are computed on the
 *     host in FP64; it synchronises.  Memory: 4 B per cell, 1 B per tile and about 93 B per frontier cell (the sort's keys
 *     and rows 24 B, the heads 4 B, 64 B of statistics per frontier, sized by the cells) on the device, allocated by the
 *     first search that needs them, grown only and freed by tloam_b200_destroy.
 *   - The kernels live in libtloam_b200_frontier.so, loaded from this library's directory by the first frontier call; if
 *     it is missing the calls return ERR_CUDA (tloam_b200_last_error names the file). */
typedef struct tloam_frontier_config {
  unsigned free_max;                   /* the highest code of a free cell: 252 every cell a plan can enter, 0 explore_lite's
                                          FREE_SPACE (nothing within about 2.7 m of an obstacle at the car's inflation) */
  double min_frontier_size;            /* m: a frontier is kept when n resolution reaches it */
  double potential_scale;              /* per m of path */
  double gain_scale;                   /* per m of frontier */
} tloam_frontier_config;
typedef struct tloam_frontier {
  unsigned id;                         /* the frontier's number before the filter */
  int status;                          /* 0 reachable, 1 unreachable from the plan's goal */
  size_t size;                         /* cells */
  unsigned long long sum_i, sum_j;     /* the sums of its cells' i and j */
  size_t min_i, min_j, max_i, max_j;   /* the bounding box, cells included */
  double centroid_x, centroid_y;       /* m */
  size_t approach_i, approach_j;       /* the approach cell */
  double approach_x, approach_y;       /* its centre, m */
  unsigned long long approach_potential;   /* P there (0xFFFFFFFFFFFFFFFF when unreachable) */
  double distance;                     /* m of free-cell path (+infinity when unreachable) */
  double cost;                         /* potential_scale distance - gain_scale n resolution (+infinity when unreachable) */
} tloam_frontier;
typedef struct tloam_frontier_info {
  double origin_x, origin_y;           /* the corner of cell (0, 0), m: the distance field's */
  double resolution;
  size_t width, height;                /* cells along x and y */
  size_t goal_i, goal_j;               /* the plan's goal cell */
  size_t cells;                        /* frontier cells */
  size_t components;                   /* frontiers before the filter */
  size_t kept;                         /* frontiers after it */
  size_t reachable;                    /* kept frontiers with status 0 */
} tloam_frontier_info;
/* free_max 252, min_frontier_size 0.5 m, potential_scale 3.0, gain_scale 1.0 (explore_lite's scales; robot parameters,
 * not calibrated) */
void tloam_b200_frontier_default_config(tloam_frontier_config* c);
/* the frontiers of the last distance field, ranked by the last plan; synchronises.  INVALID_ARG: cfg null or out of
 * range.  NOT_READY: see Source.  info may be null. */
int tloam_b200_frontier_search(tloam_b200_handle* h, const tloam_frontier_config* cfg, tloam_frontier_info* info);
/* the kept frontiers of the last search in rank order (info.kept of them; out may be null); NOT_READY before any search.
 * INVALID_ARG: capacity < info.kept. */
int tloam_b200_frontier_download(tloam_b200_handle* h, tloam_frontier* out, size_t capacity);
/* the cells of the last search's kept frontiers in rank order, each frontier's cells in ascending linear index: offsets
 * (info.kept + 1: frontier k is cells offsets[k] .. offsets[k + 1] - 1), ij (2 ints each) and xy (their centres, 2 FP64
 * each), each may be null; synchronises.  NOT_READY before any search.  INVALID_ARG: capacity < offsets[info.kept]. */
int tloam_b200_frontier_cells(tloam_b200_handle* h, size_t* offsets, int* ij, double* xy, size_t capacity);
/* inspection: the last search's label of every cell (width x height, the grid's layout): the id of its frontier before
 * the filter, 0xFFFFFFFF for a cell that is not a frontier cell; synchronises.  NOT_READY before any search.
 * INVALID_ARG: capacity < width x height. */
int tloam_b200_frontier_labels(tloam_b200_handle* h, unsigned* labels, size_t capacity);

/* ---- Terrain: a 2.5D traversability map of a cloud (the elevation-map layers of grid_map / elevation_mapping): per cell
 * the ground reference, the elevation, the step, the slope and the roughness, and a nav_msgs/OccupancyGrid value, so
 * that the distance build, the planner and the frontier search see kerbs, drop-offs and steep ramps that the occupancy
 * grid's obstacle band passes over.
 *   - Source cloud C.  tloam_b200_terrain_build: the global map as it stands in stream order (after every enqueued append
 *     and correction), all rows, or with static_only the rows tloam_b200_global_map_static_download keeps (the merge's
 *     rule and counters); a correction moves the terrain with the map.  tloam_b200_terrain_build_cloud: a host cloud
 *     (n x 3 FP64, such as a saved merged map or a prior map), with mapping on or off.  Rows with a non-finite
 *     coordinate are skipped and counted.  The map's rows are per-frame voxel centroids: its voxel should be at most the
 *     terrain's resolution (the reference's 1 m map gives a 1 m-scale terrain).
 *   - Grid (the occupancy grid's conventions: nav_msgs/OccupancyGrid layout, row-major, i along x, the origin at the
 *     corner of cell (0, 0)).  Over the finite rows of C: origin = resolution floor(min / resolution) per axis (on the
 *     ordered encodings, -0.0 below +0.0), width = floor((max - origin) / resolution) + 1; a grid of more than 2^28 cells
 *     is refused (VOXEL_RANGE) and an empty selection gives a 0 x 0 grid.  With combine_occupancy the geometry (origin,
 *     resolution, width, height) is the last tloam_b200_occupancy_build's instead.  A row's cell is
 *     (floor((x - ox) / res), floor((y - oy) / res)), the subtraction and the division each rounded on its own; a row whose
 *     cell lies outside the grid is dropped and counted.
 *   - Radii.  rg, rs, rp = (unsigned) ceil(radius / resolution) of ground_radius, step_radius, slope_radius, on the host.
 *     W_r(c) is the (2r + 1)^2 window of c, clipped to the grid.
 *   - Layers, per cell c.  Every FP64 operation is rounded on its own (no FMA), left to right as written; every extremum
 *     is taken on the ordered 64-bit encoding of the doubles, so -0.0 orders below +0.0:
 *       1. zlo(c), the least z of c's rows; n(c) their count.
 *       2. G(c) = the least zlo over W_rg(c): the ground reference, +inf when the window has no row.
 *       3. The ground-side rows of c are its rows with z <= G(c) + clearance; the others are overhangs (a bridge, a
 *          canopy), left out and counted.  e(c), the elevation, is the largest z of the ground-side rows, m(c) their count.
 *          c is known iff m(c) >= min_points.
 *       4. step(c) (known c) = the largest e minus the least e over the known cells of W_rs(c).
 *       5. The plane w = a u + b v + d fitted by least squares over the known cells k of W_rp(c): u, v the integer cell
 *          offsets of k from c and w = e(k) - e(c).  The sums run over the window with dj outer and di inner, both
 *          ascending: the integer moments N, Su, Sv, Suu, Suv, Svv exactly, and from +0.0 Sw = Sw + w, Suw = Suw + u w,
 *          Svw = Svw + v w.  With the exact integer cofactors C11 = Svv N - Sv Sv, C12 = Sv Su - Suv N, C13 = Suv Sv - Svv Su,
 *          C22 = Suu N - Su Su, C23 = Suv Su - Suu Sv, C33 = Suu Svv - Suv Suv and D = Suu C11 + Suv C12 + Su C13 (each
 *          converted to FP64 exactly): a = ((C11 Suw + C12 Svw) + C13 Sw) / D, b = ((C12 Suw + C22 Svw) + C23 Sw) / D,
 *          d = ((C13 Suw + C23 Svw) + C33 Sw) / D.  slope(c) = sqrt(a a + b b) / resolution (m per m), defined iff
 *          N >= min_fit and D != 0, NaN otherwise.  roughness(c) = the largest |w - ((a u + b v) + d)| over the fit's
 *          cells (from +0.0), NaN when the slope is.
 *       6. A known cell is lethal iff step > max_step, or slope > tan(max_slope), or roughness > max_roughness (a NaN
 *          comparison is false).  The host computes tan(max_slope) with std::tan; no transcendental runs on the device.
 *       7. The value (int8): 100 lethal, 0 traversable, -1 not known.  With combine_occupancy it combines with the last
 *          occupancy build's value o of the cell: 100 if the terrain value is 100 or o >= 65; else 0 if the terrain value
 *          is 0 or 0 <= o <= 25; else -1.  The grid then knows the occupancy grid's ray-cast free space and the terrain's
 *          ground geometry.  The values are map_server's classes: tloam_b200.save_occupancy_map saves them as they are.
 *   - Costmap.  tloam_b200_distance_build_terrain runs the distance build ("Distance field and costmap") on the last
 *     terrain build's values on the device; tloam_b200_plan_build and tloam_b200_frontier_search then work on it as on any
 *     distance build.
 *   - Limits (INVALID_ARG otherwise): resolution finite and > 0; clearance, the radii and the three thresholds finite and
 *     >= 0; max_slope < pi / 2; rs, rp <= 16 and rg <= 1024 cells; min_points, min_fit >= 1; static_only only with the
 *     map source.  NOT_READY: mapping off for the map source, static_only with removal off, or combine_occupancy with no
 *     occupancy build.  VOXEL_RANGE: the grid limit.
 *   - Lifetime.  A build is a snapshot: later appends, corrections, resets and occupancy builds leave it alone; the next
 *     build replaces it (a build refused with INVALID_ARG, NOT_READY or VOXEL_RANGE keeps it) and tloam_b200_destroy
 *     frees it.
 *   - Unchanged.  Nothing is hooked into any other call: the map, its counters, the occupancy grid, the distance field
 *     (until tloam_b200_distance_build_terrain), the plan, the frontiers and the launch counts of every other call keep
 *     their bits, and nothing is allocated or loaded before the first terrain call.
 *   - Device.  A build is k_ter_bounds and a read-back of the extent (not when combining), then k_ter_low (one thread per
 *     row: atomicMax of the complemented encoding of z, and the count), k_ter_ground twice (the window max along x, then
 *     along y), k_ter_high (one thread per row: atomicMax of the ground-side rows' encodings) and k_ter_layers (one block
 *     per 32 x 32 tile with a halo of max(rs, rp) cells of the known elevations in shared memory: step, plane fit,
 *     roughness, class, value), and a read-back of the counts; it synchronises.  The result does not depend on the
 *     order of the atomics.  Memory: 65 B per cell (four 8 B encodings, two 4 B counts, three FP64 layers and the value)
 *     and, for a host cloud, 24 B per row, on the device, allocated by the first build that needs them, grown only and
 *     freed by tloam_b200_destroy.
 *   - The kernels live in libtloam_b200_terrain.so, loaded from this library's directory by the first terrain call; if
 *     it is missing the calls return ERR_CUDA (tloam_b200_last_error names the file). */
typedef struct tloam_terrain_config {
  double resolution;                   /* m per cell; with combine_occupancy the occupancy grid's is used */
  double clearance;                    /* m above G: rows higher up are overhangs */
  double ground_radius;                /* m: the window of the ground reference */
  double step_radius;                  /* m: the window of the step */
  double slope_radius;                 /* m: the window of the plane fit */
  double max_step;                     /* m */
  double max_slope;                    /* rad */
  double max_roughness;                /* m */
  unsigned min_points;                 /* ground-side rows of a known cell */
  unsigned min_fit;                    /* known cells of a defined plane fit */
  int static_only;                     /* the map source's static rows only (tloam_b200_terrain_build) */
  int combine_occupancy;               /* on the last occupancy build's grid, its values combined */
} tloam_terrain_config;
typedef struct tloam_terrain_info {
  double origin_x, origin_y;           /* the corner of cell (0, 0), m */
  double resolution;
  size_t width, height;                /* cells along x and y */
  unsigned ground_cells, step_cells, slope_cells;   /* rg, rs, rp */
  size_t rows;                         /* rows of C, selected ones for static_only */
  size_t used;                         /* finite rows in the grid */
  size_t skipped;                      /* rows with a non-finite coordinate */
  size_t dropped;                      /* finite rows outside the grid */
  size_t overhang;                     /* used rows above G + clearance */
  size_t known, lethal;                /* known cells and the lethal ones among them (before any combination) */
  int combined;                        /* the values are combined with the occupancy grid's */
} tloam_terrain_info;
/* resolution 0.2 m, clearance 2.0 m, ground_radius 1.6 m, step_radius 0.3 m, slope_radius 0.4 m, max_step 0.10 m,
 * max_slope 15 deg, max_roughness 0.10 m, min_points 1, min_fit 6, static_only 0, combine_occupancy 0: a car with an
 * HDL-64E (robot parameters, not calibrated values; DESIGN.md §4c has what was measured with them) */
void tloam_b200_terrain_default_config(tloam_terrain_config* c);
/* the terrain of the global map; synchronises.  info may be null. */
int tloam_b200_terrain_build(tloam_b200_handle* h, const tloam_terrain_config* cfg, tloam_terrain_info* info);
/* the terrain of a host cloud xyz (n x 3 FP64; null only when n == 0); synchronises.  info may be null. */
int tloam_b200_terrain_build_cloud(tloam_b200_handle* h, const tloam_terrain_config* cfg, const double* xyz, size_t n,
                                   tloam_terrain_info* info);
/* the layers of the last terrain build, width x height each in the grid's layout, each may be null: values (int8), ground
 * G (+inf: no row in the window), elevation e (NaN where m = 0), step, slope and roughness (NaN where not known or not
 * defined) and points m; synchronises.  NOT_READY before any build.  INVALID_ARG: capacity < width x height. */
int tloam_b200_terrain_download(tloam_b200_handle* h, signed char* values, double* ground, double* elevation, double* step,
                                double* slope, double* roughness, unsigned* points, size_t capacity);
/* the distance field and costmap of the last terrain build's values (see tloam_b200_distance_build); NOT_READY before
 * any terrain build. */
int tloam_b200_distance_build_terrain(tloam_b200_handle* h, const tloam_distance_config* cfg, tloam_distance_info* info);

/* ---- Global registration (opt-in): two clouds aligned with no initial guess, by FPFH features (Rusu 2009, as PCL and
 * Open3D define them), mutual matches, a RANSAC search and a truncated-least-squares refinement.  The result is meant as
 * the guess of tloam_b200_loop_verify* and tloam_b200_localize*.  Every device operation is FP64 and separately rounded
 * (no FMA, no transcendental function), so tests/global_registration_oracle.py reproduces every bit.  "Sum in order" below
 * means a running sum s = s + x_k, k ascending.
 *   - Keypoints.  A host cloud: its finite rows down-sampled as tloam_b200_localize's query is (VoxelDownSample(voxel) by
 *     the global map's ordered path at pose I), in buffers of this feature.  A loop keyframe: as stored.  Each cloud is in
 *     its sensor's frame: the viewpoint is the origin.
 *   - Index and normals.  Each side is indexed and given normals exactly as a prior map of "Localization in a prior map"
 *     is (grid of `cell`, normal_radius, min_normal_neighbours), with max_planarity = 1: every normal with enough
 *     neighbours is valid.  Then n <- -n when n . p > 0 (n . p = (nx px + ny py) + nz pz; 0 keeps the sign).
 *   - Neighbours.  Row i's neighbours are the rows v != i with a valid normal and 0 < d2 <= r^2 (d2 as the index's), in
 *     ascending sorted position of the index (cell key, then row): the walk over the cells from p - r(1 + 1e-7) to
 *     p + r(1 + 1e-7), r = feature_radius.
 *   - Pair (p1, n1) -> (p2, n2), d = p2 - p1.  When |n1 . d| < |n2 . d| the roles swap (p1 <-> p2, n1 <-> n2, d <- -d).
 *     u = n1; v = (d x u) / |d x u| per component (no pair when |d x u| = 0); w = u x v; a x b = (a1 b2 - a2 b1, ...);
 *     |x| = sqrt(x . x).  theta = atan2(w . n2, u . n2), alpha = v . n2, phi = (u . d) / sqrt(d2).
 *     Bins: theta's bin is the number of k in 1 .. 10 with theta >= beta_k = (2k / 11 - 1) pi, decided without atan2 from
 *     (x, y) = (u . n2, w . n2) and the host's (c_k, s_k) = (cos beta_k, sin beta_k): s = (c_k y - s_k x >= 0); for k <= 5
 *     the test is y >= 0 or s, for k >= 6 it is (y > 0 or (y == 0 and x < 0)) and s.  alpha and phi: floor(11 ((f + 1)
 *     0.5)) clamped to [0, 10].  Bins 0 .. 10 are theta's, 11 .. 21 alpha's, 22 .. 32 phi's.
 *   - SPFH.  Integer counts per bin over row i's pairs (i as p1), with a valid normal at i; pairs(i) = the pairs counted.
 *     SPFH_k(j) = (count * 100) / pairs(k).
 *   - FPFH.  A row with pairs(i) > 0 has a feature: over its neighbours k with pairs(k) > 0, in order, val = SPFH_k(j) / d2
 *     is summed in order into acc(j) and into sum(block of j) (11 bins per block, k then j ascending); then F(j) =
 *     (acc(j) * 100) / sum + SPFH_i(j), or acc(j) + SPFH_i(j) when that sum is 0.  A row without pairs has no feature.
 *   - Matches.  Each source feature's nearest target feature by sum over j in order of (a_j - b_j)^2, the lower row on a
 *     tie; the same from the target.  The mutual pairs (i, j) are kept in source order.  Fewer than 3: termination
 *     FEW_CORRESPONDENCES, T = I.
 *   - Hypotheses h = 0 .. n_hypotheses - 1, all evaluated.  With splitmix64(x) (Steele et al. 2014; z = x + 0x9e37..7c15,
 *     ...), r_d = splitmix64(seed ^ splitmix64((h << 2) | d)) (64-bit wrap): i0 = r_0 % n, i1 = r_1 % (n - 1) + (1 when
 *     >= i0), i2 = r_2 % (n - 2), then +1 when >= min(i0, i1), then +1 when >= max(i0, i1): three distinct pairs.  Rejected
 *     unless every edge passes Open3D's length check (ds >= dt * edge_similarity and dt >= ds * edge_similarity, d =
 *     sqrt(d2)) and both triangles' |(x1 - x0) x (x2 - x0)| >= min_triangle_area.  T_h: the frames e1 = a / |a|, b = u -
 *     (u . e1) e1, e2 = b / |b|, e3 = e1 x e2 (a = x1 - x0, u = x2 - x0) of the source (E) and target (F) triangles;
 *     R(r, c) = (F1r E1c + F2r E2c) + F3r E3c; t = c_q - R c_p with c = ((x0 + x1) + x2) / 3.  A hypothesis's inliers: the
 *     pairs with |R p + t - q|^2 < tau^2, R p + t = ((R_r0 px + R_r1 py) + R_r2 pz) + t_r.  The best has the most inliers,
 *     the lower h on a tie; none valid: NO_HYPOTHESIS, T = I.
 *   - Refinement by truncated least squares: S = the best's inliers; while fewer than max_refine_iterations fits were made
 *     and |S| >= 3 (else FEW_INLIERS): T = fit(S), S' = inliers under T, and CONVERGED when S' = S; S = S'.  ITERATION_LIMIT
 *     after max_refine_iterations fits.  Each step does not increase sum min(r^2, tau^2).  fit(S): Horn's method with
 *     every sum in pair order: c_p = sum p / |S|, c_q likewise, S_ab = sum (p_a - c_pa)(q_b - c_qb); N = [[xx+yy+zz,
 *     yz-zy, zx-xz, xy-yx], [., xx-yy-zz, xy+yx, zx+xz], [., ., yy-xx-zz, yz+zy], [., ., ., zz-xx-yy]] (left to right);
 *     nf_jacobi3's cyclic Jacobi on 4 x 4 (pairs (0,1) .. (2,3)); q = the eigenvector of the largest eigenvalue (the lower
 *     index on a tie) over sqrt(((q0^2 + q1^2) + q2^2) + q3^2); R from q = (w, x, y, z) as ((ww + xx) - yy) - zz, 2 (xy -
 *     wz), ...; t = c_q - R c_p.
 *   - Result.  inliers = |S| under the final T, inlier_rmse = sqrt(sum r^2 in order / inliers) (0 without inliers);
 *     fitness = the fraction of source keypoints with a target keypoint at d2 < tau^2 under T (the target's grid);
 *     accepted = inliers >= min_inliers and fitness >= min_fitness.  A side without keypoints: EMPTY, T = I, and no
 *     k_gr_* kernel runs (the other side has already been down-sampled and indexed; tloam_b200_global_registration_side
 *     then gives its keypoints, validity and unoriented normals, and zero counts and features).
 *   - The kernels live in libtloam_b200_greg.so, loaded from this library's directory by the enable call.  A call changes
 *     nothing else: odometry, maps, loop database and keyframes, pose graph and localization are untouched. */
typedef struct tloam_global_registration_config {
  double voxel;                        /* keypoint down-sample of a host cloud, m */
  double cell;                         /* index cell, m */
  double normal_radius;                /* m, <= 3 cell */
  int min_normal_neighbours;           /* >= 3 */
  double feature_radius;               /* m, <= 3 cell */
  double max_correspondence_distance;  /* tau, m */
  int n_hypotheses;                    /* 1 .. 2^20 */
  unsigned long long seed;
  double edge_similarity;              /* (0, 1] */
  double min_triangle_area;            /* |cross product|, m^2, > 0 */
  int max_refine_iterations;           /* 1 .. 100 */
  int min_inliers;                     /* >= 0 */
  double min_fitness;                  /* [0, 1] */
} tloam_global_registration_config;
enum {
  TLOAM_GLOBAL_REGISTRATION_CONVERGED = 0,
  TLOAM_GLOBAL_REGISTRATION_ITERATION_LIMIT = 1,
  TLOAM_GLOBAL_REGISTRATION_FEW_INLIERS = 2,          /* fewer than 3 inliers to fit */
  TLOAM_GLOBAL_REGISTRATION_FEW_CORRESPONDENCES = 3,  /* fewer than 3 mutual pairs */
  TLOAM_GLOBAL_REGISTRATION_NO_HYPOTHESIS = 4,        /* every hypothesis rejected */
  TLOAM_GLOBAL_REGISTRATION_EMPTY = 5                 /* a side without keypoints */
};
typedef struct tloam_global_registration_result {
  double T[16];                        /* target <- source, column-major (the loop call: T_cand_query) */
  long long n_source_points, n_target_points;        /* keypoints */
  long long n_source_features, n_target_features;
  long long n_correspondences;         /* mutual pairs */
  int n_valid_hypotheses, best_hypothesis, best_inliers;   /* best_hypothesis -1: none */
  int inliers;
  double inlier_rmse, fitness;
  int refine_iterations, termination, accepted;
} tloam_global_registration_result;
/* voxel 0.5 m, cell 1 m, normal_radius 1 m, min_normal_neighbours 5, feature_radius 2.5 m, tau 0.75 m, n_hypotheses
 * 65536, seed 0, edge_similarity 0.9, min_triangle_area 1 m^2, max_refine_iterations 10, min_inliers 30, min_fitness 0.3
 * (DESIGN.md section 4c has how they were chosen) */
void tloam_b200_global_registration_default_config(tloam_global_registration_config* c);
/* turns the feature on (loading libtloam_b200_greg.so and libtloam_b200_loc.so) and drops the last run.  INVALID_ARG: cfg
 * null or a value outside the ranges above. */
int tloam_b200_global_registration_enable(tloam_b200_handle* h, const tloam_global_registration_config* cfg);
/* aligns host cloud src (n_src x 3) to host cloud tgt (n_tgt x 3); synchronises.  NOT_READY: off.  INVALID_ARG: out null,
 * a null cloud with rows, or more than 2^30 rows.  VOXEL_RANGE: a cloud the down-sample's key or the index cannot hold. */
int tloam_b200_global_register(tloam_b200_handle* h, const double* src, size_t n_src, const double* tgt, size_t n_tgt,
                               tloam_global_registration_result* out);
/* aligns loop keyframe query to loop keyframe candidate (T = T_cand_query, a guess for tloam_b200_loop_verify*);
 * synchronises.  NOT_READY: this feature or loop verification off.  INVALID_ARG: an index out of range. */
int tloam_b200_global_register_loop(tloam_b200_handle* h, long long query, long long candidate,
                                    tloam_global_registration_result* out);
/* the last run's side (0 source, 1 target): keypoints (n x 3), oriented normals (n x 3; unoriented after an EMPTY run),
 * normal validity (n), SPFH counts
 * (n x 33), features (n x 33) and feature flags (n); each may be null; *n = the side's keypoints; synchronises.
 * NOT_READY: no run since enable.  INVALID_ARG: side not 0 or 1, capacity < *n. */
int tloam_b200_global_registration_side(tloam_b200_handle* h, int side, double* xyz, double* normal, unsigned char* valid,
                                        int* spfh, double* feature, unsigned char* has_feature, size_t capacity, size_t* n);
/* the last run's mutual pairs (source row, target row) in source order (n x 2, may be null); *n = their count. */
int tloam_b200_global_registration_correspondences(tloam_b200_handle* h, int* pairs, size_t capacity, size_t* n);
/* the last run's inliers per hypothesis (-1: rejected; may be null); *n = n_hypotheses, or 0 after an EMPTY run. */
int tloam_b200_global_registration_hypotheses(tloam_b200_handle* h, int* inliers, size_t capacity, size_t* n);

/* Pinned host memory helpers (optional; pinned inputs make set_* a direct DMA, no staging threads). */
int tloam_b200_host_alloc(void** p, size_t bytes);
int tloam_b200_host_free(void* p);

#ifdef __cplusplus
}
#endif
#endif
