// Drives tloam::GlobalRegistrationB200 (the RegistrationInterface drop-in) and tloam::FrontEndB200's global registration the
// way a loop-closure or relocalization node would: two scans in, the transform between them out, with no guess.
//     global_registration_driver in.bin out.bin
// in.bin: uint64 n, the source (n x 3 FP64), uint64 m, the target (m x 3 FP64).  Both calls use the default
// configuration.  Prints "termination accepted inliers".  out.bin receives, for the drop-in then for FrontEndB200, T (16
// FP64, column-major), fitness and inlier rmse (FP64), and inliers, correspondences, best hypothesis (int64).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"
#include "../../include/tloam_b200/global_registration_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

static bool read_cloud(FILE* g, std::vector<Eigen::Vector3d>& out) {
  uint64_t n = 0;
  if (std::fread(&n, sizeof(n), 1, g) != 1) return false;
  out.resize(n);
  return n == 0 || std::fread(out.data(), sizeof(Eigen::Vector3d), n, g) == n;
}

static void write_result(FILE* fo, const double T[16], double fitness, double rmse, const tloam_global_registration_result& r) {
  const double f[2] = {fitness, rmse};
  const int64_t k[3] = {r.inliers, r.n_correspondences, r.best_hypothesis};
  std::fwrite(T, sizeof(double), 16, fo);
  std::fwrite(f, sizeof(double), 2, fo);
  std::fwrite(k, sizeof(int64_t), 3, fo);
}

int main(int argc, char** argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: global_registration_driver in.bin out.bin\n");
    return 2;
  }
  FILE* g = std::fopen(argv[1], "rb");
  if (!g) return 2;
  tloam::Frame src, tgt;
  if (!read_cloud(g, src.scan_cloud->points_) || !read_cloud(g, tgt.scan_cloud->points_)) return 2;
  std::fclose(g);

  std::unique_ptr<tloam::GlobalRegistrationB200> global;
  try {
    global.reset(new tloam::GlobalRegistrationB200());
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  global->setInputSource(src);
  global->setInputTarget(tgt);
  Eigen::Isometry3d predict, T;
  if (!global->scanMatching(src, predict, T)) return 4;
  const std::pair<double, double> fs = global->getFitnessScore();

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
  if (!fe.enableGlobalRegistration()) return 5;
  tloam::CloudData s, t;
  s.cloud_ptr = src.scan_cloud;
  t.cloud_ptr = tgt.scan_cloud;
  tloam_global_registration_result r;
  if (!fe.globalRegister(s, t, r)) return 6;

  const tloam_global_registration_result& a = global->result();
  std::printf("%d %d %d\n", a.termination, a.accepted, a.inliers);
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  write_result(fo, T.matrix().data(), fs.first, fs.second, a);
  write_result(fo, r.T, r.fitness, r.inlier_rmse, r);
  std::fclose(fo);
  return 0;
}
