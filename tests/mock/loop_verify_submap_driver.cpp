// Drives tloam::FrontEndB200's loop verification against a submap the way a back end would: every raw scan of the file is
// added to the loop database with a keyframe and a pose-graph node at pose k = (step * k, 0, 0); a frame with a candidate is
// verified by verifyLoopSubmap from the loop result's yaw, and an accepted result becomes a loop edge.
//     loop_verify_submap_driver raw.bin exclude_recent half_window step
// raw.bin: uint64 scan count, then per scan a count and the points (FP64 x, y, z).  Prints per scan "query candidate" and,
// when there is a candidate, "iterations termination inliers accepted n_candidate_points fitness rmse" and the 16 entries
// of T; then "edges n".
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 5) { std::fprintf(stderr, "usage: loop_verify_submap_driver raw.bin exclude_recent half_window step\n"); return 2; }
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
  tloam_loop_verify_submap_config vcfg;
  tloam_b200_loop_verify_submap_default_config(&vcfg);
  vcfg.half_window = std::atoi(argv[3]);
  const double step = std::atof(argv[4]);
  if (!fe.enableLoopDetection(lcfg) || !fe.enableLoopVerification() || !fe.enableSubmapVerification(vcfg) || !fe.enablePoseGraph())
    return 4;
  for (size_t k = 0; k < raw.size(); ++k) {
    if (!fe.addLoopFrame(raw[k])) return 6;
    const double pose[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, step * static_cast<double>(k), 0, 0, 1};
    if (tloam_b200_pose_graph_add_node(reg->handle(), pose) != TLOAM_B200_OK) return 5;
    tloam_loop_result r;
    if (!fe.loopResult(r)) return 7;
    std::printf("%lld %lld", r.query, r.candidate);
    if (r.candidate >= 0) {
      tloam_loop_verify_result v;
      if (!fe.verifyLoopSubmap(r, v)) return 8;
      std::printf(" %d %d %lld %d %lld %.17g %.17g", v.iterations, v.termination, v.inliers, v.accepted, v.n_candidate_points,
                  v.fitness, v.rmse);
      for (int i = 0; i < 16; ++i) std::printf(" %.17g", v.T[i]);
      if (v.accepted && !fe.addLoopEdge(v)) return 9;
    }
    std::printf("\n");
  }
  size_t nodes = 0, edges = 0;
  if (tloam_b200_pose_graph_size(reg->handle(), &nodes, &edges) != TLOAM_B200_OK) return 10;
  std::printf("edges %zu\n", edges);
  return 0;
}
