// Drives tloam::FrontEndB200's loop-corrected global map the way a back end would: every raw scan of the file is added to
// the loop database and the pose graph, every scan after the first to the global map (updateGlobalMapChained, so map frame
// f is node f + 1); a candidate that verifyLoop accepts becomes a loop edge; then one optimisation and correctGlobalMap.
//     map_correct_driver raw.bin exclude_recent
// raw.bin: uint64 scan count, then per scan a count and the points (FP64 x, y, z).  Prints "points frames termination",
// then per map frame the 16 entries of O_f and of P_f on one line, then every map point.
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: map_correct_driver raw.bin exclude_recent\n"); return 2; }
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
  if (!fe.enableGlobalMap() || !fe.enableGlobalMapCorrection()) return 4;
  if (!fe.enableLoopDetection(lcfg) || !fe.enableLoopVerification() || !fe.enablePoseGraph()) return 4;
  for (size_t k = 0; k < raw.size(); ++k) {
    if (k && !fe.updateGlobalMapChained(raw[k])) return 5;
    if (!fe.addLoopFrame(raw[k]) || !fe.addPoseGraphNode()) return 6;
    tloam_loop_result r;
    if (!fe.loopResult(r)) return 7;
    if (r.candidate >= 0) {
      tloam_loop_verify_result v;
      if (!fe.verifyLoop(r, v)) return 8;
      if (v.accepted && !fe.addLoopEdge(v)) return 9;
    }
  }
  tloam_pose_graph_result pr;
  if (!fe.optimizePoseGraph(pr)) return 10;
  std::vector<long long> node;
  for (size_t k = 1; k < raw.size(); ++k) node.push_back((long long)k);
  if (!fe.correctGlobalMap(node)) return 11;
  std::vector<Eigen::Vector3d> map;
  if (!fe.globalMap(map)) return 12;
  std::vector<double> O(16 * node.size()), P(16 * node.size());
  if (!fe.globalMapFramePoses(0, node.size(), O.data(), P.data())) return 13;
  std::printf("%zu %zu %d\n", map.size(), node.size(), pr.termination);
  for (size_t k = 0; k < node.size(); ++k) {
    for (int i = 0; i < 16; ++i) std::printf(i ? " %.17g" : "%.17g", O[16 * k + i]);
    for (int i = 0; i < 16; ++i) std::printf(" %.17g", P[16 * k + i]);
    std::printf("\n");
  }
  for (const auto& p : map) std::printf("%.17g %.17g %.17g\n", p[0], p[1], p[2]);
  return 0;
}
