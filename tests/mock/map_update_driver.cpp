// Drives tloam::FrontEndB200's map update the way a node that localizes in a saved map and keeps it current would: a prior
// map is loaded (setPriorMap) and updating enabled, every scan is localized (the first from a guess, every later one from
// the prediction) and added (addMapUpdateFrame); then one build, the updated map read back and loaded in place of the prior
// map (setPriorMapUpdated), and the first scan localized against it from the guess.
//     map_update_driver map.bin scans.bin gx gy gyaw min_frames
// map.bin: uint64 count, then the points (FP64 x, y, z).  scans.bin: uint64 scan count, then per scan a count and its
// points.  The guess is Rz(gyaw) with translation (gx, gy, 0).  Prints one line per scan (accepted, used, frame), one line
// of build counts (n_prior, n_prior_removed, n_additions, n_additions_removed, n_voxels, n_voxels_kept, n_total), one line
// per point of the updated map, and the last localization (iterations, termination, accepted, fitness, then T
// column-major), every double as %.17g.
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
  if (argc < 7) {
    std::fprintf(stderr, "usage: map_update_driver map.bin scans.bin gx gy gyaw min_frames\n");
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
  tloam_map_update_config ucfg;
  tloam_b200_map_update_default_config(&ucfg);
  ucfg.min_frames = std::atoi(argv[6]);
  if (!fe.enableLocalization() || !fe.setPriorMap(map) || !fe.enableMapUpdate(ucfg)) return 4;
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
    tloam_map_update_add_result a;
    if (!fe.localize(scans[k], r, k == 0 ? &guess : nullptr) || !fe.addMapUpdateFrame(a)) return 5;
    std::printf("%d %d %lld\n", r.accepted, a.used, a.frame);
  }
  tloam_map_update_result b;
  std::vector<Eigen::Vector3d> updated;
  if (!fe.buildUpdatedMap(b) || !fe.updatedMap(updated) || !fe.setPriorMapUpdated()) return 6;
  std::printf("%lld %lld %lld %lld %lld %lld %lld\n", b.n_prior, b.n_prior_removed, b.n_additions, b.n_additions_removed,
              b.n_voxels, b.n_voxels_kept, b.n_total);
  for (const Eigen::Vector3d& p : updated) std::printf("%.17g %.17g %.17g\n", p[0], p[1], p[2]);
  tloam_localize_result r;
  if (scans.empty() || !fe.localize(scans[0], r, &guess)) return 7;
  std::printf("%d %d %d %.17g", r.iterations, r.termination, r.accepted, r.fitness);
  for (int i = 0; i < 16; ++i) std::printf(" %.17g", r.T[i]);
  std::printf("\n");
  return 0;
}
