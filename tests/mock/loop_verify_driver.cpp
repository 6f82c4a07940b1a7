// Drives tloam::FrontEndB200's loop verification the way a front end would: every raw scan of the file is added to the
// loop database with a keyframe (even scans through tloam_b200_process_raw_scan and addLoopFrame(), odd ones through
// addLoopFrame(CloudData)); a frame with a candidate is verified by verifyLoop from the loop result's yaw.
//     loop_verify_driver raw.bin exclude_recent
// raw.bin: uint64 scan count, then per scan a count and the points (FP64 x, y, z).  Prints per scan "query candidate" and,
// when there is a candidate, "iterations termination inliers accepted fitness rmse" and the 16 entries of T.
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: loop_verify_driver raw.bin exclude_recent\n"); return 2; }
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
  fcfg.cvr_submap = 0.005; fcfg.cvr_scan = 0.01;             // the synthetic street scene has few curvature maxima
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
  if (!fe.enableLoopDetection(lcfg) || !fe.enableLoopVerification()) return 4;
  tloam_ground_config gcfg;
  tloam_dcvc_config dcfg;
  tloam_b200_ground_default_config(&gcfg);
  tloam_b200_dcvc_default_config(&dcfg);
  for (size_t k = 0; k < raw.size(); ++k) {
    const std::vector<Eigen::Vector3d>& p = raw[k].cloud_ptr->points_;
    if (k % 2 == 0) {
      size_t ns[4];
      if (tloam_b200_process_raw_scan(reg->handle(), &gcfg, &dcfg, 131, 3.0, &fcfg, 0.3, 0.1,
                                      p.empty() ? nullptr : reinterpret_cast<const double*>(p.data()), p.size(), ns) != TLOAM_B200_OK)
        return 5;
      if (!fe.addLoopFrame()) return 6;
    } else if (!fe.addLoopFrame(raw[k])) {
      return 6;
    }
    tloam_loop_result r;
    if (!fe.loopResult(r)) return 7;
    std::printf("%lld %lld", r.query, r.candidate);
    if (r.candidate >= 0) {
      tloam_loop_verify_result v;
      if (!fe.verifyLoop(r, v)) return 8;
      std::printf(" %d %d %lld %d %.17g %.17g", v.iterations, v.termination, v.inliers, v.accepted, v.fitness, v.rmse);
      for (int i = 0; i < 16; ++i) std::printf(" %.17g", v.T[i]);
    }
    std::printf("\n");
  }
  return 0;
}
