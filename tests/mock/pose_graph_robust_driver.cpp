// Drives tloam::FrontEndB200's robust pose graph the way a back end would: every raw scan of the file is added to the loop
// database and, through addPoseGraphNode, to the graph; a candidate that verifyLoop accepts becomes a loop edge, and a
// second copy of it with its translation moved by `shift` metres models a false loop; then one robust optimisation.
//     pose_graph_robust_driver raw.bin exclude_recent shift
// raw.bin: uint64 scan count, then per scan a count and the points (FP64 x, y, z).  Prints per scan "query candidate
// accepted", then "nodes loop_edges iterations termination initial_cost final_cost outer_iterations gnc_termination mu_final
// inliers rejected", then every loop edge's weight, then the 16 entries of every corrected pose and of the correction.
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: pose_graph_robust_driver raw.bin exclude_recent shift\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint64_t count = 0;
  if (std::fread(&count, sizeof(count), 1, f) != 1) return 2;
  std::vector<tloam::CloudData> raw(count);
  for (auto& c : raw) {
    uint64_t n = 0;
    if (std::fread(&n, sizeof(n), 1, f) != 1) return 2;
    c.cloud_ptr->points_.resize(n);
    if (n && std::fread(c.cloud_ptr->points_.data(), sizeof(Eigen::Vector3d), n, f) != n) return 2;
  }
  std::fclose(f);
  tloam_tls_config cfg;
  tloam_b200_default_config(&cfg);
  tloam_feature_config fcfg;
  tloam_b200_feature_default_config(&fcfg);
  tloam_submap_config scfg;
  tloam_b200_submap_default_config(&scfg);
  std::unique_ptr<tloam::LocalRegistrationB200> reg;
  try {
    reg.reset(new tloam::LocalRegistrationB200(cfg));
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  tloam::FrontEndB200 fe(*reg, fcfg, scfg, scfg.ground_down_sample, 0.1);
  tloam_loop_config lcfg;
  tloam_b200_loop_default_config(&lcfg);
  lcfg.exclude_recent = std::atoi(argv[2]);
  if (!fe.enableLoopDetection(lcfg) || !fe.enableLoopVerification() || !fe.enablePoseGraph()) return 4;
  size_t edges = 0;
  for (size_t k = 0; k < raw.size(); ++k) {
    if (!fe.addLoopFrame(raw[k]) || !fe.addPoseGraphNode()) return 6;
    tloam_loop_result r;
    if (!fe.loopResult(r)) return 7;
    int accepted = 0;
    if (r.candidate >= 0) {
      tloam_loop_verify_result v;
      if (!fe.verifyLoop(r, v)) return 8;
      accepted = v.accepted;
      if (v.accepted) {
        if (!fe.addLoopEdge(v)) return 9;
        v.T[12] += std::atof(argv[3]);
        if (!fe.addLoopEdge(v)) return 9;
        edges += 2;
      }
    }
    std::printf("%lld %lld %d\n", r.query, r.candidate, accepted);
  }
  tloam_pose_graph_robust_result rr;
  if (!fe.optimizePoseGraphRobust(rr)) return 10;
  const tloam_pose_graph_result& pr = rr.pg;
  std::printf("%lld %lld %d %d %.17g %.17g %d %d %.17g %lld %lld\n", pr.nodes, pr.loop_edges, pr.iterations, pr.termination,
              pr.initial_cost, pr.final_cost, rr.outer_iterations, rr.gnc_termination, rr.mu_final, rr.inliers, rr.rejected);
  std::vector<double> w(edges);
  if (!fe.loopEdgeWeights(0, edges, w.data())) return 12;
  for (size_t l = 0; l < edges; ++l) std::printf(l ? " %.17g" : "%.17g", w[l]);
  std::printf("\n");
  std::vector<double> poses(16 * raw.size());
  double corr[16];
  if (!fe.correctedPoses(0, raw.size(), poses.data(), corr)) return 11;
  for (size_t k = 0; k <= raw.size(); ++k) {
    const double* T = k < raw.size() ? poses.data() + 16 * k : corr;
    for (int i = 0; i < 16; ++i) std::printf(i ? " %.17g" : "%.17g", T[i]);
    std::printf("\n");
  }
  return 0;
}
