// Drives tloam::FrontEndB200's localization the way a node that drives a mapped area again would: a prior map is loaded
// (setPriorMap), the first scan is localized from a guess and every later one from the prediction (a null guess).
//     localize_driver map.bin scans.bin gx gy gyaw
// map.bin: uint64 count, then the points (FP64 x, y, z).  scans.bin: uint64 scan count, then per scan a count and its
// points.  The guess of the first scan is Rz(gyaw) with translation (gx, gy, 0).  Prints one line per scan: iterations,
// termination, accepted, inliers, fitness, rmse, then T and T_map_odom (column-major, %.17g).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

static bool read_points(FILE* f, std::vector<Eigen::Vector3d>& out) {
  uint64_t n = 0;
  if (std::fread(&n, sizeof(n), 1, f) != 1) return false;
  out.resize(n);
  return !n || std::fread(out.data(), sizeof(Eigen::Vector3d), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc < 6) {
    std::fprintf(stderr, "usage: localize_driver map.bin scans.bin gx gy gyaw\n");
    return 2;
  }
  std::vector<Eigen::Vector3d> map;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f || !read_points(f, map)) return 2;
  std::fclose(f);
  f = std::fopen(argv[2], "rb");
  if (!f) return 2;
  uint64_t count = 0;
  if (std::fread(&count, sizeof(count), 1, f) != 1) return 2;
  std::vector<tloam::CloudData> scans(count);
  for (size_t k = 0; k < count; ++k)
    if (!read_points(f, scans[k].cloud_ptr->points_)) return 2;
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
  if (!fe.enableLocalization() || !fe.setPriorMap(map)) return 4;
  const double yaw = std::atof(argv[5]);
  Eigen::Isometry3d guess;
  double* g = guess.matrix().data();                               // column-major: (r, c) at 4 c + r
  for (int i = 0; i < 16; ++i) g[i] = i % 5 == 0 ? 1.0 : 0.0;
  g[0] = std::cos(yaw); g[4] = -std::sin(yaw);
  g[1] = std::sin(yaw); g[5] = std::cos(yaw);
  g[12] = std::atof(argv[3]);
  g[13] = std::atof(argv[4]);
  for (size_t k = 0; k < scans.size(); ++k) {
    tloam_localize_result r;
    if (!fe.localize(scans[k], r, k == 0 ? &guess : nullptr)) return 5;
    std::printf("%d %d %d %lld %.17g %.17g", r.iterations, r.termination, r.accepted, r.inliers, r.fitness, r.rmse);
    for (int i = 0; i < 16; ++i) std::printf(" %.17g", r.T[i]);
    for (int i = 0; i < 16; ++i) std::printf(" %.17g", r.T_map_odom[i]);
    std::printf("\n");
  }
  return 0;
}
