// front_end_b200.hpp -- C++ shim: tloam::FrontEndB200, the device side of FrontEnd's per-frame glue
// (ref: src/front_end/front_end.cpp:181-199 processCloud, :201-267 updateSubmap, :285-305 the first-frame branch) on the
// C ABI of libtloam_b200.so, driving a tloam::LocalRegistrationB200 handle.  Header-only; from the host side it needs only
// CloudData::cloud_ptr->points_ (contiguous std::vector<Eigen::Vector3d>) and Eigen::Isometry3d::matrix().data().
//
// The per-frame loop of FrontEnd::updateLidarOdometry becomes three calls, each on the registration handle's stream:
//     processCloud(ground, edge, general)    replaces processCloud() + setInputSource(current_scan)
//     registration.scanMatchingPredicted(pose)  (or scanMatching with the caller's prediction)
//     updateSubmap(pose)                      replaces updateSubmap() + setInputTarget(submap)
// and on the first frame processCloud + initSubmap() replace the `!odometry_inited` branch.  The scan features, the frame's
// submap selections and the submap itself stay on the GPU; the caller reads a source cloud back only to inspect it.
// With mapping_flag (ref: front_end.cpp:57, :269-274) updateGlobalMap(raw, pose) after updateSubmap appends the frame's raw
// scan, transformed and VoxelDownSample(1.0)'d on its own, to a global map kept on the GPU (globalMap / registeredScan read
// it back); frame 0 has no append, as in the reference.  A raw scan with intensity_ gives the map its intensity channel
// (per-voxel averages, the reference's XYZI map); globalMap(points, intensity) reads it back.  updateGlobalMap also takes
// the driver's sensor_msgs/PointCloud2 as it arrived (packed_scan_b200.hpp): one upload, unpacked on the device, its
// intensity field (if any) carried into the map.  enableLoopDetection / addLoopFrame / loopResult add loop closure: a Scan
// Context descriptor per frame and an exact search over every earlier frame, on the GPU; enableLoopVerification / verifyLoop
// check a candidate by a scan-to-scan ICP of down-sampled keyframes kept on the GPU and give the relative pose;
// enableSubmapVerification / verifyLoopSubmap check it against the keyframes around the candidate, point to plane.
// enableLocalization / localizeFrame register each frame against a prior map; enableRelocalization / setPlaces /
// relocalizeFrame find the first pose in that map (or the pose after tracking is lost) from a recorded session's places;
// enableMapUpdate / addMapUpdateFrame / buildUpdatedMap keep that map up to date from the localized frames.
// enableOccupancy / occupancyGrid give a 2D occupancy grid of the map; distanceField / queryDistance its distance field
// and inflated costmap, or those of a saved grid; planPotential / planPaths plan paths on that costmap; frontiers finds
// the exploration frontiers on it, ranked by the plan.  terrainMap builds a traversability map of the map (or of a saved
// cloud) that sees kerbs and drop-offs, and distanceFieldTerrain the costmap of it.
// enableGlobalRegistration / globalRegister / globalRegisterLoop align two clouds, or two loop keyframes, with no initial
// guess: the guess for verifyLoop's ICP or for localizeFrame.
// Without the reference headers (this repository's tests) define TLOAM_B200_MOCK_HOST_TYPES and provide the host types
// (tests/mock/mock_tloam.hpp).
#ifndef TLOAM_B200_FRONT_END_B200_HPP
#define TLOAM_B200_FRONT_END_B200_HPP

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../tloam_b200.h"
#include "local_registration_b200.hpp"
#include "packed_scan_b200.hpp"

#ifndef TLOAM_B200_MOCK_HOST_TYPES
#include <yaml-cpp/yaml.h>
#include "tloam/models/utils/sensor_data.hpp"
#include "tloam/models/utils/work_space_path.h"
#endif

namespace tloam {

class FrontEndB200 {
 public:
  // reg: the registration handle the features are handed to (it must outlive this object)
  FrontEndB200(LocalRegistrationB200& reg, const tloam_feature_config& fcfg, const tloam_submap_config& scfg, double ground_down_sample,
               double edge_down_sample)
      : h_(reg.handle()), fcfg_(fcfg), scfg_(scfg), ground_down_sample_(ground_down_sample), edge_down_sample_(edge_down_sample) {}

#ifndef TLOAM_B200_MOCK_HOST_TYPES
  // Same configuration as FrontEnd::FrontEnd (ref: front_end.cpp:47-57) and featureExtract::initConfig
  // (ref: feature_extract.cpp:13-37): config/mapping/lidar_odometry.yaml and config/mapping/feature.yaml.
  explicit FrontEndB200(LocalRegistrationB200& reg) : h_(reg.handle()) {
    const YAML::Node lo = YAML::LoadFile(WORK_SPACE_PATH + "/config/mapping/lidar_odometry.yaml");
    ground_down_sample_ = lo["ground_down_sample"].as<double>();
    edge_down_sample_ = lo["edge_down_sample"].as<double>();
    tloam_b200_submap_default_config(&scfg_);
    scfg_.ground_down_sample = ground_down_sample_;
    scfg_.ground_down_sample_submap = lo["ground_down_sample_submap"].as<double>();
    scfg_.edge_down_sample_submap = lo["edge_down_sample_submap"].as<double>();
    scfg_.sphere_frame_size = lo["sphere_frame_size"].as<int>();
    scfg_.planar_frame_size = lo["planar_frame_size"].as<int>();
    scfg_.edge_crop_box_length = lo["edge_crop_box_length"].as<double>();
    scfg_.ground_crop_box_length = lo["ground_crop_box_length"].as<double>();
    const YAML::Node fe = YAML::LoadFile(WORK_SPACE_PATH + "/config/mapping/feature.yaml")["feature"];
    tloam_b200_feature_default_config(&fcfg_);
    fcfg_.radius = fe["radius"].as<double>();
    fcfg_.K = fe["K"].as<int>();
    fcfg_.planar_num = fe["planar_num"].as<int>();
    fcfg_.sphere_num = fe["sphere_num"].as<int>();
    fcfg_.min_neigh = fe["min_neigh"].as<int>();
    fcfg_.cvr_scan = fe["cvr_scan"].as<double>();
    fcfg_.cvr_submap = fe["cvr_submap"].as<double>();
    fcfg_.planar_scan_thres = fe["planar_scan_thres"].as<double>();
    fcfg_.planar_submap_thres = fe["planar_submap_thres"].as<double>();
    fcfg_.planar_vertic_thres = fe["planar_vertic_thres"].as<double>();
    if (lo["mapping_flag"].as<bool>()) enableGlobalMap();   // front_end.cpp:57
  }
#endif

  // mapping_flag on: an empty global map with VoxelDownSample(voxel) per frame (the reference's literal 1.0)
  bool enableGlobalMap(double voxel = 1.0) {
    tloam_global_map_config c;
    tloam_b200_global_map_default_config(&c);
    c.voxel = voxel;
    mapping_ = report(tloam_b200_global_map_enable(h_, &c), "enableGlobalMap");
    return mapping_;
  }
  bool mappingFlag() const { return mapping_; }
  // global_map += raw.Transform(pose).VoxelDownSample(voxel) (ref: front_end.cpp:269-274): raw = the driver's scan, NaN rows
  // allowed (left out of the map).  No-ops returning true when mapping is off, like the reference.
  // A raw cloud with intensity (PointCloud2::HasIntensity: the driver's /velodyne_points) gives each voxel the average of
  // its rows' intensity_, as VoxelDownSample does; the map keeps the channel under operator+='s rule.
  bool updateGlobalMap(const CloudData& raw, const Eigen::Isometry3d& pose) {
    if (!mapping_) return true;
    if (hasIntensity(raw))
      return report(tloam_b200_global_map_append_intensity(h_, pose.matrix().data(), data(raw), intensity(raw), size(raw)),
                    "updateGlobalMap");
    return report(tloam_b200_global_map_append(h_, pose.matrix().data(), data(raw), size(raw)), "updateGlobalMap");
  }
  // the same with the pose of the frame just enqueued on the handle (tloam_b200_scan_match_predicted_async)
  bool updateGlobalMapChained(const CloudData& raw) {
    if (!mapping_) return true;
    if (hasIntensity(raw))
      return report(tloam_b200_global_map_append_intensity_chained(h_, data(raw), intensity(raw), size(raw)), "updateGlobalMapChained");
    return report(tloam_b200_global_map_append_chained(h_, data(raw), size(raw)), "updateGlobalMapChained");
  }
  // the same from the driver's message (any sensor_msgs::PointCloud2-shaped type, see packedScanOf): no host conversion, the
  // records cross PCIe once.  A message with a FLOAT32 intensity field gives an intensity frame.  A layout packedScanOf
  // refuses returns false with lastStatus() INVALID_ARG.
  template <class Msg>
  bool updateGlobalMap(const Msg& raw, const Eigen::Isometry3d& pose) {
    if (!mapping_) return true;
    tloam_packed_scan scan;
    const int rc = packedScanOf(raw, &scan);
    if (rc != TLOAM_B200_OK) return report(rc, "updateGlobalMap");
    return report(tloam_b200_global_map_append_packed(h_, pose.matrix().data(), &scan), "updateGlobalMap");
  }
  template <class Msg>
  bool updateGlobalMapChained(const Msg& raw) {
    if (!mapping_) return true;
    tloam_packed_scan scan;
    const int rc = packedScanOf(raw, &scan);
    if (rc != TLOAM_B200_OK) return report(rc, "updateGlobalMapChained");
    return report(tloam_b200_global_map_append_packed_chained(h_, &scan), "updateGlobalMapChained");
  }
  // the whole map (synchronises) and T.p of the last appended raw scan, raw order (the reference's /raw_cloud, :84-86)
  bool globalMap(std::vector<Eigen::Vector3d>& out) {
    size_t n = 0, frames = 0;
    if (!report(tloam_b200_global_map_size(h_, &n, &frames), "globalMap")) return false;
    out.resize(n);
    return report(tloam_b200_global_map_download(h_, 0, n, reinterpret_cast<double*>(out.data())), "globalMap");
  }
  // the map with its intensity channel: `intensity` is left empty when the map has none (the reference's intensity_.clear())
  bool globalMap(std::vector<Eigen::Vector3d>& out, std::vector<double>& intensity) {
    intensity.clear();
    int has = 0;
    if (!globalMap(out) || !report(tloam_b200_global_map_has_intensity(h_, &has), "globalMap")) return false;
    if (!has) return true;
    intensity.resize(out.size());
    return report(tloam_b200_global_map_intensity_download(h_, 0, intensity.size(), intensity.data()), "globalMap");
  }
  bool registeredScan(std::vector<Eigen::Vector3d>& out) {
    size_t n = 0;
    const int rc = tloam_b200_registered_scan_download(h_, nullptr, 0, &n);
    if (rc != TLOAM_B200_OK && rc != TLOAM_B200_ERR_INVALID_ARG) return report(rc, "registeredScan");
    out.resize(n);
    return report(tloam_b200_registered_scan_download(h_, reinterpret_cast<double*>(out.data()), out.size(), &n), "registeredScan");
  }

  // loop closure (include/tloam_b200.h "Loop closure"; the reference is pure odometry): every added frame gets a Scan
  // Context descriptor on the GPU and is compared with every frame at least cfg.exclude_recent frames older.  The library
  // reports the best candidate (verifyLoop checks it); correcting the poses belongs to the caller's back end.
  bool enableLoopDetection(const tloam_loop_config& cfg) {
    loop_ = report(tloam_b200_loop_enable(h_, &cfg), "enableLoopDetection");
    return loop_;
  }
  bool enableLoopDetection() {
    tloam_loop_config c;
    tloam_b200_loop_default_config(&c);
    return enableLoopDetection(c);
  }
  bool loopDetection() const { return loop_; }
  // adds the raw scan the last tloam_b200_process_raw_scan* on this handle uploaded (deskewed when timed), read on the GPU,
  // and enqueues its query; no synchronisation
  bool addLoopFrame() { return report(tloam_b200_loop_add_frame(h_), "addLoopFrame"); }
  // the same for a host raw scan (the driver's cloud, NaN rows allowed), uploaded
  bool addLoopFrame(const CloudData& raw) { return report(tloam_b200_loop_add(h_, data(raw), size(raw)), "addLoopFrame"); }
  // the newest added frame's best earlier frame (waits for that add only); out.is_loop below cfg.dist_threshold
  bool loopResult(tloam_loop_result& out) { return report(tloam_b200_loop_result(h_, &out), "loopResult"); }

  // loop verification (include/tloam_b200.h "Loop verification"): from now on every added loop frame also keeps a
  // down-sampled keyframe on the GPU.  Call right after enableLoopDetection (an empty database).
  bool enableLoopVerification(const tloam_loop_verify_config& cfg) {
    return report(tloam_b200_loop_verify_enable(h_, &cfg), "enableLoopVerification");
  }
  bool enableLoopVerification() {
    tloam_loop_verify_config c;
    tloam_b200_loop_verify_default_config(&c);
    return enableLoopVerification(c);
  }
  // aligns the loop result's query keyframe to its candidate's from Rz(lr.yaw) by a scan-to-scan ICP on the GPU; out.T is
  // T_cand_query (column-major), to be handed to the back end when out.accepted
  bool verifyLoop(const tloam_loop_result& lr, tloam_loop_verify_result& out) {
    const double c = std::cos(lr.yaw), s = std::sin(lr.yaw);
    const double guess[16] = {c, s, 0, 0, -s, c, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    return report(tloam_b200_loop_verify(h_, lr.query, lr.candidate, guess, &out), "verifyLoop");
  }

  // loop verification against a submap (include/tloam_b200.h "Loop verification against a submap"): the query keyframe is
  // aligned, point to plane, to the keyframes of the frames around the candidate, placed by the pose graph's odometry
  // nodes.  Needs enableLoopVerification, and a pose-graph node next to every added loop frame (addPoseGraphNode).
  bool enableSubmapVerification(const tloam_loop_verify_submap_config& cfg) {
    return report(tloam_b200_loop_verify_submap_enable(h_, &cfg), "enableSubmapVerification");
  }
  bool enableSubmapVerification() {
    tloam_loop_verify_submap_config c;
    tloam_b200_loop_verify_submap_default_config(&c);
    return enableSubmapVerification(c);
  }
  // as verifyLoop, against the submap around the candidate; out.T is T_cand_query, to be handed to addLoopEdge when
  // out.accepted
  bool verifyLoopSubmap(const tloam_loop_result& lr, tloam_loop_verify_result& out) {
    const double c = std::cos(lr.yaw), s = std::sin(lr.yaw);
    const double guess[16] = {c, s, 0, 0, -s, c, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    return report(tloam_b200_loop_verify_submap(h_, lr.query, lr.candidate, guess, nullptr, &out), "verifyLoopSubmap");
  }

  // pose graph (include/tloam_b200.h "Pose graph"): the odometry chain and the accepted loop edges, optimised on the GPU.
  // The odometry is left alone; correctedPoses and the map -> odom correction are the output, and correctGlobalMap moves
  // the global map's frames to them.
  bool enablePoseGraph(const tloam_pose_graph_config& cfg) { return report(tloam_b200_pose_graph_enable(h_, &cfg), "enablePoseGraph"); }
  bool enablePoseGraph() {
    tloam_pose_graph_config c;
    tloam_b200_pose_graph_default_config(&c);
    return enablePoseGraph(c);
  }
  // a node at the pose of the frame enqueued last, copied on the device; call next to every addLoopFrame
  bool addPoseGraphNode() { return report(tloam_b200_pose_graph_add_node_chained(h_), "addPoseGraphNode"); }
  // only an accepted verification is an edge
  bool addLoopEdge(const tloam_loop_verify_result& v) { return report(tloam_b200_pose_graph_add_loop(h_, &v), "addLoopEdge"); }
  bool optimizePoseGraph(tloam_pose_graph_result& out) { return report(tloam_b200_pose_graph_optimize(h_, &out), "optimizePoseGraph"); }
  // graduated non-convexity with a truncated-least-squares cost over the loop edges (include/tloam_b200.h "Robust pose
  // graph"): a loop edge that verification accepted at the wrong place ends with weight 0; correctedPoses and
  // correctGlobalMap then read this run
  bool optimizePoseGraphRobust(const tloam_pose_graph_robust_config& cfg, tloam_pose_graph_robust_result& out) {
    return report(tloam_b200_pose_graph_optimize_robust(h_, &cfg, &out), "optimizePoseGraphRobust");
  }
  bool optimizePoseGraphRobust(tloam_pose_graph_robust_result& out) {
    tloam_pose_graph_robust_config c;
    tloam_b200_pose_graph_robust_default_config(&c);
    return optimizePoseGraphRobust(c, out);
  }
  // the last optimisation's weights of loop edges first .. first + count - 1 (1 after optimizePoseGraph)
  bool loopEdgeWeights(size_t first, size_t count, double* w) {
    return report(tloam_b200_pose_graph_loop_weights(h_, first, count, w), "loopEdgeWeights");
  }
  // nodes first .. first + count - 1 (count x 16, column-major); with `correction`, also T_opt(N-1) . O_{N-1}^-1
  bool correctedPoses(size_t first, size_t count, double* poses, double* correction = nullptr) {
    if (!report(tloam_b200_pose_graph_download(h_, first, count, poses), "correctedPoses")) return false;
    return !correction || report(tloam_b200_pose_graph_correction(h_, correction), "correctedPoses");
  }

  // loop-corrected global map (include/tloam_b200.h "Loop-corrected global map"): call right after enableGlobalMap (an
  // empty map); every later updateGlobalMap records the frame's odometry pose and the pose its block is expressed at
  bool enableGlobalMapCorrection() {
    return report(tloam_b200_global_map_correction_enable(h_), "enableGlobalMapCorrection");
  }
  // moves every map frame f to Delta_{node[f]} . O_f of the last optimizePoseGraph (node[f] = -1: left alone); with
  // updateGlobalMap from the second frame and addPoseGraphNode from the first, node[f] = f + 1.  Later frames are
  // appended at the map -> odom correction times their odometry pose.
  bool correctGlobalMap(const std::vector<long long>& node) {
    return report(tloam_b200_global_map_correct(h_, node.empty() ? nullptr : node.data(), node.size()), "correctGlobalMap");
  }
  // O_f and P_f of map frames first .. first + count - 1 (count x 16 each, column-major; either may be null)
  bool globalMapFramePoses(size_t first, size_t count, double* odom, double* current) {
    return report(tloam_b200_global_map_frame_poses(h_, first, count, odom, current), "globalMapFramePoses");
  }

  // Dynamic-point removal (include/tloam_b200.h "Dynamic-point removal"): right after enableGlobalMap, every later
  // updateGlobalMap* casts free-space votes on the map points before it; staticGlobalMap reads the map without the points
  // later scans looked through.  The map globalMap returns is not changed.
  bool enableDynamicRemoval(const tloam_global_map_dynamic_config& cfg) {
    return report(tloam_b200_global_map_dynamic_enable(h_, &cfg), "enableDynamicRemoval");
  }
  bool enableDynamicRemoval() {
    tloam_global_map_dynamic_config c;
    tloam_b200_global_map_dynamic_default_config(&c);
    return enableDynamicRemoval(c);
  }
  // the (through, hits) counters of map points first .. first + count - 1 (either may be null)
  bool globalMapVotes(size_t first, size_t count, unsigned* through, unsigned* hits) {
    return report(tloam_b200_global_map_votes_download(h_, first, count, through, hits), "globalMapVotes");
  }
  bool staticGlobalMap(std::vector<Eigen::Vector3d>& out) {
    size_t n = 0;
    const int rc = tloam_b200_global_map_static_download(h_, nullptr, nullptr, 0, &n);
    if (rc != TLOAM_B200_ERR_INVALID_ARG && !report(rc, "staticGlobalMap")) return false;
    out.resize(n);
    return report(tloam_b200_global_map_static_download(h_, reinterpret_cast<double*>(out.data()), nullptr, n, &n),
                  "staticGlobalMap");
  }
  // with the intensity of every kept point (empty when the map has no intensity channel)
  bool staticGlobalMap(std::vector<Eigen::Vector3d>& out, std::vector<double>& intensity) {
    intensity.clear();
    int has = 0;
    if (!report(tloam_b200_global_map_has_intensity(h_, &has), "staticGlobalMap")) return false;
    size_t n = 0;
    const int rc = tloam_b200_global_map_static_download(h_, nullptr, nullptr, 0, &n);
    if (rc != TLOAM_B200_ERR_INVALID_ARG && !report(rc, "staticGlobalMap")) return false;
    out.resize(n);
    if (has) intensity.resize(n);
    return report(tloam_b200_global_map_static_download(h_, reinterpret_cast<double*>(out.data()),
                                                        has ? intensity.data() : nullptr, n, &n), "staticGlobalMap");
  }

  // The occupancy grid (include/tloam_b200.h "Occupancy grid"): right after enableGlobalMap, every later updateGlobalMap*
  // records a 2D scan; occupancyGrid rasterises every map frame at its current pose.  cells is nav_msgs/OccupancyGrid's
  // data (width x height, row-major from the origin's corner), so a node fills the message with one copy.
  bool enableOccupancy(const tloam_occupancy_config& cfg) {
    return report(tloam_b200_occupancy_enable(h_, &cfg), "enableOccupancy");
  }
  bool enableOccupancy() {
    tloam_occupancy_config c;
    tloam_b200_occupancy_default_config(&c);
    return enableOccupancy(c);
  }
  bool occupancyGrid(std::vector<int8_t>& cells, tloam_occupancy_info& info) {
    if (!report(tloam_b200_occupancy_build(h_, &info), "occupancyGrid")) return false;
    cells.resize(info.width * info.height);
    return report(tloam_b200_occupancy_download(h_, reinterpret_cast<signed char*>(cells.data()), nullptr, nullptr,
                                                cells.size()), "occupancyGrid");
  }

  // The distance field and costmap (include/tloam_b200.h "Distance field and costmap") of the last occupancyGrid, or of a
  // host grid in nav_msgs/OccupancyGrid's layout (a saved map in a localization session).  sd is the signed distance in
  // m, costs costmap_2d's codes, values the costmap as nav_msgs/OccupancyGrid data (one copy into the message).
  bool distanceField(const tloam_distance_config& cfg, std::vector<float>& sd, std::vector<uint8_t>& costs,
                     std::vector<int8_t>& values, tloam_distance_info& info) {
    if (!report(tloam_b200_distance_build(h_, &cfg, &info), "distanceField")) return false;
    return downloadDistance(sd, costs, values, info);
  }
  bool distanceField(const tloam_distance_config& cfg, const std::vector<int8_t>& cells, size_t width, size_t height,
                     double origin_x, double origin_y, double resolution, std::vector<float>& sd,
                     std::vector<uint8_t>& costs, std::vector<int8_t>& values, tloam_distance_info& info) {
    if (cells.size() != width * height) return report(TLOAM_B200_ERR_INVALID_ARG, "distanceField");
    if (!report(tloam_b200_distance_build_grid(h_, &cfg, reinterpret_cast<const signed char*>(cells.data()), width, height,
                                               origin_x, origin_y, resolution, &info), "distanceField"))
      return false;
    return downloadDistance(sd, costs, values, info);
  }
  // Terrain (include/tloam_b200.h "Terrain"): the traversability map of the global map (cloud empty) or of a saved cloud
  // (n x 3, m), values in nav_msgs/OccupancyGrid's classes and the elevation (NaN without a ground-side row) and slope
  // layers in the grid's layout; distanceFieldTerrain gives the costmap of those values for planPotential.
  bool terrainMap(const tloam_terrain_config& cfg, const std::vector<double>& cloud, std::vector<int8_t>& values,
                  std::vector<double>& elevation, std::vector<double>& slope, tloam_terrain_info& info) {
    const int rc = cloud.empty() ? tloam_b200_terrain_build(h_, &cfg, &info)
                                 : tloam_b200_terrain_build_cloud(h_, &cfg, cloud.data(), cloud.size() / 3, &info);
    if (!report(rc, "terrainMap")) return false;
    const size_t n = info.width * info.height;
    values.resize(n); elevation.resize(n); slope.resize(n);
    return report(tloam_b200_terrain_download(h_, reinterpret_cast<signed char*>(values.data()), nullptr, elevation.data(),
                                              nullptr, slope.data(), nullptr, nullptr, n), "terrainMap");
  }
  bool distanceFieldTerrain(const tloam_distance_config& cfg, std::vector<float>& sd, std::vector<uint8_t>& costs,
                            std::vector<int8_t>& values, tloam_distance_info& info) {
    if (!report(tloam_b200_distance_build_terrain(h_, &cfg, &info), "distanceFieldTerrain")) return false;
    return downloadDistance(sd, costs, values, info);
  }
  // the last field's distance at the points xy (n x 2, m) and its gradient (n x 2), bilinear between the cell centres;
  // NaN outside them
  bool queryDistance(const std::vector<double>& xy, std::vector<double>& distance, std::vector<double>& gradient) {
    const size_t n = xy.size() / 2;
    distance.resize(n);
    gradient.resize(2 * n);
    return report(tloam_b200_distance_query(h_, xy.data(), n, distance.data(), gradient.data()), "queryDistance");
  }

  // Path planning (include/tloam_b200.h "Path planning") on the last distanceField's costs: the potential to the goal
  // (goal_x, goal_y), width x height in the grid's layout (0xFFFFFFFFFFFFFFFF: impassable or cut off).
  bool planPotential(const tloam_plan_config& cfg, double goal_x, double goal_y, std::vector<unsigned long long>& potential,
                     tloam_plan_info& info) {
    if (!report(tloam_b200_plan_build(h_, &cfg, goal_x, goal_y, &info), "planPotential")) return false;
    potential.resize(info.width * info.height);
    return report(tloam_b200_plan_download(h_, potential.data(), potential.size()), "planPotential");
  }
  // the paths from the starts xy (n x 2, m) down the last planPotential: per start the cell centres from the start to the
  // goal as x, y pairs (a nav_msgs/Path's poses, empty unless the status is 0), the status (0 reached, 1 start outside
  // the grid, 2 start impassable, 3 goal unreachable) and the cost
  bool planPaths(const std::vector<double>& starts_xy, std::vector<std::vector<double>>& paths_xy,
                 std::vector<int>& statuses, std::vector<unsigned long long>& costs) {
    const size_t n = starts_xy.size() / 2;
    std::vector<size_t> offsets(n + 1);
    statuses.resize(n);
    costs.resize(n);
    if (!report(tloam_b200_plan_paths(h_, starts_xy.data(), n, offsets.data(), statuses.data(), costs.data()), "planPaths"))
      return false;
    std::vector<double> xy(2 * offsets[n]);
    if (!report(tloam_b200_plan_path_cells(h_, nullptr, xy.data(), offsets[n]), "planPaths")) return false;
    paths_xy.assign(n, std::vector<double>());
    for (size_t s = 0; s < n; ++s)
      paths_xy[s].assign(xy.begin() + 2 * offsets[s], xy.begin() + 2 * offsets[s + 1]);
    return true;
  }

  // Frontiers (include/tloam_b200.h "Frontiers") of the last distanceField, ranked by the last planPotential (built with
  // its goal at the robot): the kept frontiers in rank order and each one's cell centres as x, y pairs.  The route to a
  // frontier is planPaths from its approach cell, reversed.
  bool frontiers(const tloam_frontier_config& cfg, std::vector<tloam_frontier>& out,
                 std::vector<std::vector<double>>& cells_xy, tloam_frontier_info& info) {
    if (!report(tloam_b200_frontier_search(h_, &cfg, &info), "frontiers")) return false;
    out.resize(info.kept);
    if (!report(tloam_b200_frontier_download(h_, out.data(), out.size()), "frontiers")) return false;
    size_t m = 0;
    for (const tloam_frontier& f : out) m += f.size;
    std::vector<size_t> offsets(info.kept + 1);
    std::vector<double> xy(2 * m);
    if (!report(tloam_b200_frontier_cells(h_, offsets.data(), nullptr, xy.data(), m), "frontiers")) return false;
    cells_xy.assign(info.kept, std::vector<double>());
    for (size_t k = 0; k < info.kept; ++k)
      cells_xy[k].assign(xy.begin() + 2 * offsets[k], xy.begin() + 2 * offsets[k + 1]);
    return true;
  }

  // Global registration (include/tloam_b200.h "Global registration"): two clouds aligned with no initial guess by FPFH
  // features, mutual matches, RANSAC and a truncated-least-squares refinement on the GPU.  Each cloud is in its sensor's
  // frame (normals point to the origin).  out.T is target <- source (column-major); hand it on when out.accepted.
  bool enableGlobalRegistration(const tloam_global_registration_config& cfg) {
    return report(tloam_b200_global_registration_enable(h_, &cfg), "enableGlobalRegistration");
  }
  bool enableGlobalRegistration() {
    tloam_global_registration_config c;
    tloam_b200_global_registration_default_config(&c);
    return enableGlobalRegistration(c);
  }
  bool globalRegister(const CloudData& source, const CloudData& target, tloam_global_registration_result& out) {
    return report(tloam_b200_global_register(h_, data(source), size(source), data(target), size(target), &out), "globalRegister");
  }
  // loop keyframe query to loop keyframe candidate (needs enableLoopVerification): out.T = T_cand_query, the guess that
  // tloam_b200_loop_verify takes where Scan Context's yaw would not reach
  bool globalRegisterLoop(long long query, long long candidate, tloam_global_registration_result& out) {
    return report(tloam_b200_global_register_loop(h_, query, candidate, &out), "globalRegisterLoop");
  }

  // The merged map (include/tloam_b200.h "Merged global map"): the whole map, or with static_only the points
  // staticGlobalMap keeps, merged into one voxel grid -- VoxelDownSample(voxel) of the map, the cloud to publish or save.
  bool mergedGlobalMap(double voxel, bool static_only, std::vector<Eigen::Vector3d>& out) {
    size_t n = 0;
    if (!report(tloam_b200_global_map_merge(h_, voxel, static_only ? 1 : 0, &n), "mergedGlobalMap")) return false;
    out.resize(n);
    return report(tloam_b200_global_map_merged_download(h_, 0, n, reinterpret_cast<double*>(out.data()), nullptr),
                  "mergedGlobalMap");
  }
  // with the average intensity of every voxel (empty when the map has no intensity channel)
  bool mergedGlobalMap(double voxel, bool static_only, std::vector<Eigen::Vector3d>& out, std::vector<double>& intensity) {
    intensity.clear();
    size_t n = 0;
    if (!report(tloam_b200_global_map_merge(h_, voxel, static_only ? 1 : 0, &n), "mergedGlobalMap")) return false;
    int has = 0;
    if (!report(tloam_b200_global_map_has_intensity(h_, &has), "mergedGlobalMap")) return false;
    out.resize(n);
    if (has) intensity.resize(n);
    return report(tloam_b200_global_map_merged_download(h_, 0, n, reinterpret_cast<double*>(out.data()),
                                                        has ? intensity.data() : nullptr), "mergedGlobalMap");
  }

  // Localization in a prior map (include/tloam_b200.h "Localization in a prior map"): a map from an earlier session (for
  // example its mergedGlobalMap, saved by the caller) is loaded once; each frame is then registered against it and comes
  // out in the map's frame, with the map <- odom correction.  The odometry and the maps above are not touched.
  bool enableLocalization(const tloam_localize_config& cfg) { return report(tloam_b200_localize_enable(h_, &cfg), "enableLocalization"); }
  bool enableLocalization() {
    tloam_localize_config c;
    tloam_b200_localize_default_config(&c);
    return enableLocalization(c);
  }
  bool setPriorMap(const std::vector<Eigen::Vector3d>& map) {
    return report(tloam_b200_localize_set_map(h_, map.empty() ? nullptr : reinterpret_cast<const double*>(map.data()), map.size()),
                  "setPriorMap");
  }
  // the handle's last mergedGlobalMap, on the device
  bool setPriorMapMerged() { return report(tloam_b200_localize_set_map_merged(h_), "setPriorMapMerged"); }
  // the scan the handle processed last; guess null: the prediction from the previous localization and the odometry
  bool localizeFrame(tloam_localize_result& out, const Eigen::Isometry3d* guess = nullptr) {
    return report(tloam_b200_localize_frame(h_, guess ? guess->matrix().data() : nullptr, &out), "localizeFrame");
  }
  // a host cloud
  bool localize(const CloudData& scan, tloam_localize_result& out, const Eigen::Isometry3d* guess = nullptr) {
    return report(tloam_b200_localize(h_, data(scan), size(scan), guess ? guess->matrix().data() : nullptr, &out), "localize");
  }

  // Relocalization in a prior map (include/tloam_b200.h "Relocalization in a prior map"): the places of a recorded session
  // (its loop frames' descriptors, as loopDescriptors returns them, and their poses) are loaded once; relocalizeFrame then
  // finds the pose of the processed scan in the map without a guess, and an accepted result seeds the next
  // localizeFrame(out, nullptr).  Needs enableLocalization and a prior map.
  bool enableRelocalization(const tloam_relocalize_config& cfg) {
    const bool ok = report(tloam_b200_relocalize_enable(h_, &cfg), "enableRelocalization");
    if (ok) place_slot_ = (size_t)cfg.n_ring * cfg.n_sector + cfg.n_ring + cfg.n_sector;
    return ok;
  }
  bool enableRelocalization() {
    tloam_relocalize_config c;
    tloam_b200_relocalize_default_config(&c);
    return enableRelocalization(c);
  }
  // the loop database's descriptors, one slot after another (what setPlaces takes); the slot is enableRelocalization's,
  // which must have the loop detection's shape
  bool loopDescriptors(std::vector<double>& out) {
    if (!place_slot_) return report(TLOAM_B200_ERR_NOT_READY, "loopDescriptors");
    size_t n = 0;
    if (!report(tloam_b200_loop_size(h_, &n), "loopDescriptors")) return false;
    out.resize(n * place_slot_);
    return report(tloam_b200_loop_descriptors_download(h_, 0, n, n ? out.data() : nullptr), "loopDescriptors");
  }
  // descriptors: poses.size() slots of enableRelocalization's shape; poses: map <- sensor
  bool setPlaces(const std::vector<double>& descriptors, const std::vector<Eigen::Isometry3d>& poses) {
    if (descriptors.size() != poses.size() * place_slot_) return report(TLOAM_B200_ERR_INVALID_ARG, "setPlaces");
    const std::vector<double> p = columnMajor(poses);
    return report(tloam_b200_relocalize_set_places(h_, descriptors.empty() ? nullptr : descriptors.data(), p.empty() ? nullptr : p.data(),
                                                    poses.size()),
                  "setPlaces");
  }
  // the handle's own loop database as the descriptors, one pose per loop frame
  bool setPlacesFromLoop(const std::vector<Eigen::Isometry3d>& poses) {
    const std::vector<double> p = columnMajor(poses);
    return report(tloam_b200_relocalize_set_places_loop(h_, p.empty() ? nullptr : p.data(), poses.size()), "setPlacesFromLoop");
  }
  // the scan the handle processed last
  bool relocalizeFrame(tloam_relocalize_result& out) { return report(tloam_b200_relocalize_frame(h_, &out), "relocalizeFrame"); }
  // a host cloud
  bool relocalize(const CloudData& scan, tloam_relocalize_result& out) {
    return report(tloam_b200_relocalize(h_, data(scan), size(scan), &out), "relocalize");
  }

  // Updating a prior map (include/tloam_b200.h "Updating a prior map"): after each localizeFrame / localize,
  // addMapUpdateFrame lets that frame's scan vote on the prior map's points and keeps its points no prior point is near
  // (out.used = 0 when the localization was not accepted, and nothing changes); buildUpdatedMap gives the prior points not
  // seen through, then the new voxels enough frames agree on; updatedMap reads it back and setPriorMapUpdated loads it in
  // place of the prior map.  Needs enableLocalization and a prior map; enableLocalization turns it off.
  bool enableMapUpdate(const tloam_map_update_config& cfg) { return report(tloam_b200_map_update_enable(h_, &cfg), "enableMapUpdate"); }
  bool enableMapUpdate() {
    tloam_map_update_config c;
    tloam_b200_map_update_default_config(&c);
    return enableMapUpdate(c);
  }
  bool addMapUpdateFrame(tloam_map_update_add_result& out) { return report(tloam_b200_map_update_add(h_, &out), "addMapUpdateFrame"); }
  bool addMapUpdateFrame() {
    tloam_map_update_add_result r;
    return addMapUpdateFrame(r);
  }
  bool buildUpdatedMap(tloam_map_update_result& out) { return report(tloam_b200_map_update_build(h_, &out), "buildUpdatedMap"); }
  // the last buildUpdatedMap's points
  bool updatedMap(std::vector<Eigen::Vector3d>& out) {
    size_t n = 0;
    if (!report(tloam_b200_map_update_size(h_, nullptr, nullptr, &n), "updatedMap")) return false;
    out.resize(n);
    return report(tloam_b200_map_update_download(h_, 0, n, n ? reinterpret_cast<double*>(out.data()) : nullptr), "updatedMap");
  }
  bool setPriorMapUpdated() { return report(tloam_b200_localize_set_map_updated(h_), "setPriorMapUpdated"); }

  // processCloud + setInputSource (ref: front_end.cpp:181-199, :313): the three clouds the segmentation nodelet publishes
  bool processCloud(CloudData& ground, CloudData& edge, CloudData& general) {
    return report(tloam_b200_process_cloud(h_, &fcfg_, ground_down_sample_, edge_down_sample_, data(ground), size(ground), data(edge),
                                           size(edge), data(general), size(general), n_source_),
                  "processCloud");
  }
  // the `!odometry_inited` branch (ref: front_end.cpp:285-305) from the frame processCloud saw last
  bool initSubmap() { return report(tloam_b200_submap_init_frame(h_, &scfg_), "initSubmap"); }
  // updateSubmap + setInputTarget (ref: front_end.cpp:201-267, :333): pose = the new lidar_odom_pose
  bool updateSubmap(const Eigen::Isometry3d& pose) {
    return report(tloam_b200_submap_update_frame(h_, pose.matrix().data()), "updateSubmap");
  }
  // the same with the pose of the frame just enqueued on the handle (tloam_b200_scan_match_predicted_async): no host round trip
  bool updateSubmapChained() { return report(tloam_b200_submap_update_frame_chained(h_), "updateSubmapChained"); }

  // sizes of the current source (edge, sphere, planar, ground) and a copy of one of its clouds (inspection)
  const size_t* sourceSizes() const { return n_source_; }
  bool sourceCloud(int cloud, std::vector<Eigen::Vector3d>& out) {
    if (cloud < 0 || cloud > 3) return report(TLOAM_B200_ERR_INVALID_ARG, "sourceCloud");
    out.resize(n_source_[cloud]);
    return report(tloam_b200_source_download(h_, cloud, reinterpret_cast<double*>(out.data()), out.size()), "sourceCloud");
  }
  int lastStatus() const { return last_status_; }

 private:
  static const double* data(const CloudData& c) {
    return c.cloud_ptr->points_.empty() ? nullptr : reinterpret_cast<const double*>(c.cloud_ptr->points_.data());
  }
  static size_t size(const CloudData& c) { return c.cloud_ptr->points_.size(); }
  static std::vector<double> columnMajor(const std::vector<Eigen::Isometry3d>& poses) {
    std::vector<double> out(16 * poses.size());
    for (size_t j = 0; j < poses.size(); ++j)
      for (int i = 0; i < 16; ++i) out[16 * j + i] = poses[j].matrix().data()[i];
    return out;
  }
  static bool hasIntensity(const CloudData& c) {                     // PointCloud2::HasIntensity (PointCloud2.hpp:108-110)
    return !c.cloud_ptr->intensity_.empty() && c.cloud_ptr->intensity_.size() == c.cloud_ptr->points_.size();
  }
  static const double* intensity(const CloudData& c) { return c.cloud_ptr->intensity_.data(); }
  bool downloadDistance(std::vector<float>& sd, std::vector<uint8_t>& costs, std::vector<int8_t>& values,
                        const tloam_distance_info& info) {
    const size_t n = info.width * info.height;
    sd.resize(n);
    costs.resize(n);
    values.resize(n);
    return report(tloam_b200_distance_download(h_, sd.data(), nullptr, costs.data(), reinterpret_cast<signed char*>(values.data()),
                                               n), "distanceField");
  }
  bool report(int rc, const char* where) {
    last_status_ = rc;
    if (rc != TLOAM_B200_OK)
      std::fprintf(stderr, "[tloam_b200] %s: %s %s\n", where, tloam_b200_status_string(rc), tloam_b200_last_error(h_));
    return rc == TLOAM_B200_OK;
  }
  tloam_b200_handle* h_ = nullptr;
  tloam_feature_config fcfg_;
  tloam_submap_config scfg_;
  double ground_down_sample_ = 0.3, edge_down_sample_ = 0.1;
  size_t n_source_[4] = {0, 0, 0, 0};
  bool mapping_ = false;
  bool loop_ = false;
  size_t place_slot_ = 0;               // descriptor slot of enableRelocalization's shape
  int last_status_ = TLOAM_B200_OK;
};

}  // namespace tloam
#endif
