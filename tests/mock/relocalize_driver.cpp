// Drives tloam::FrontEndB200's relocalization the way a node that starts in a mapped area would: the prior map and the
// places of the recorded session are loaded (setPriorMap, setPlaces), each scan is relocalized without a guess, and after
// an accepted relocalization the same scan is localized from the prediction (a null guess).
//     relocalize_driver map.bin places.bin scans.bin
// map.bin: uint64 count, then the points (FP64 x, y, z).  places.bin: uint64 count, uint64 slot, then count descriptor
// slots and count poses (16 FP64, column-major).  scans.bin: uint64 scan count, then per scan a count and its points.
// Prints one line per scan: n_hypotheses, winner, place, shift, ambiguous, accepted, fitness, then T (column-major,
// %.17g), then the guess of the localization that follows an accepted relocalization (16 zeros otherwise).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

static bool read_points(FILE* f, std::vector<Eigen::Vector3d>& out) {
  uint64_t n = 0;
  if (std::fread(&n, sizeof(n), 1, f) != 1) return false;
  out.resize(n);
  return !n || std::fread(out.data(), sizeof(Eigen::Vector3d), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc < 4) {
    std::fprintf(stderr, "usage: relocalize_driver map.bin places.bin scans.bin\n");
    return 2;
  }
  std::vector<Eigen::Vector3d> map;
  FILE* f = std::fopen(argv[1], "rb");
  if (!f || !read_points(f, map)) return 2;
  std::fclose(f);
  f = std::fopen(argv[2], "rb");
  if (!f) return 2;
  uint64_t n = 0, slot = 0;
  if (std::fread(&n, sizeof(n), 1, f) != 1 || std::fread(&slot, sizeof(slot), 1, f) != 1) return 2;
  std::vector<double> desc(n * slot);
  std::vector<Eigen::Isometry3d> poses(n);
  if (n && std::fread(desc.data(), sizeof(double), desc.size(), f) != desc.size()) return 2;
  for (auto& P : poses)
    if (std::fread(P.matrix().data(), sizeof(double), 16, f) != 16) return 2;
  std::fclose(f);
  f = std::fopen(argv[3], "rb");
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
  if (!fe.enableLocalization() || !fe.setPriorMap(map) || !fe.enableRelocalization() || !fe.setPlaces(desc, poses)) return 4;
  for (size_t k = 0; k < scans.size(); ++k) {
    tloam_relocalize_result r;
    if (!fe.relocalize(scans[k], r)) return 5;
    std::printf("%d %d %lld %d %d %d %.17g", r.n_hypotheses, r.winner, r.place, r.shift, r.ambiguous, r.accepted, r.result.fitness);
    for (int i = 0; i < 16; ++i) std::printf(" %.17g", r.result.T[i]);
    tloam_localize_result l;
    for (int i = 0; i < 16; ++i) l.guess[i] = 0.0;
    if (r.accepted && !fe.localize(scans[k], l, nullptr)) return 6;
    for (int i = 0; i < 16; ++i) std::printf(" %.17g", l.guess[i]);
    std::printf("\n");
  }
  return 0;
}
