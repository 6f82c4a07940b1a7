// Drives tloam::FrontEndB200's dynamic-point removal the way a mapping node would: removal is enabled right after the map,
// every raw scan of the file is appended with its pose (updateGlobalMap, with intensity), then the counters and the static
// map are read back.
//     map_dynamic_driver raw.bin out.bin n_rows n_cols fov_down fov_up
// raw.bin: uint64 scan count, then per scan its pose (16 FP64, column-major), a count, the points (FP64 x, y, z) and their
// intensities.  Prints "points static".  out.bin receives the counters (points x 2 uint32: through, then hits), the static
// map (count + points) and its intensity (count + values).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 7) {
    std::fprintf(stderr, "usage: map_dynamic_driver raw.bin out.bin n_rows n_cols fov_down fov_up\n");
    return 2;
  }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  uint64_t count = 0;
  if (std::fread(&count, sizeof(count), 1, f) != 1) return 2;
  std::vector<tloam::CloudData> raw(count);
  std::vector<Eigen::Isometry3d> pose(count);
  for (size_t k = 0; k < count; ++k) {
    if (std::fread(pose[k].matrix().data(), sizeof(double), 16, f) != 16) return 2;
    uint64_t n = 0;
    if (std::fread(&n, sizeof(n), 1, f) != 1) return 2;
    raw[k].cloud_ptr->points_.resize(n);
    raw[k].cloud_ptr->intensity_.resize(n);
    if (n && std::fread(raw[k].cloud_ptr->points_.data(), sizeof(Eigen::Vector3d), n, f) != n) return 2;
    if (n && std::fread(raw[k].cloud_ptr->intensity_.data(), sizeof(double), n, f) != n) return 2;
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
  tloam_global_map_dynamic_config dcfg;
  tloam_b200_global_map_dynamic_default_config(&dcfg);
  dcfg.n_rows = std::atoi(argv[3]);
  dcfg.n_cols = std::atoi(argv[4]);
  dcfg.fov_down = std::atof(argv[5]);
  dcfg.fov_up = std::atof(argv[6]);
  if (!fe.enableGlobalMap() || !fe.enableDynamicRemoval(dcfg)) return 4;
  for (size_t k = 0; k < raw.size(); ++k)
    if (!fe.updateGlobalMap(raw[k], pose[k])) return 5;
  std::vector<Eigen::Vector3d> map, kept;
  std::vector<double> intensity;
  if (!fe.globalMap(map) || !fe.staticGlobalMap(kept, intensity)) return 6;
  std::vector<unsigned> through(map.size()), hits(map.size());
  if (!fe.globalMapVotes(0, map.size(), through.data(), hits.data())) return 7;
  std::printf("%zu %zu\n", map.size(), kept.size());
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  if (!map.empty()) {
    std::fwrite(through.data(), sizeof(unsigned), through.size(), fo);
    std::fwrite(hits.data(), sizeof(unsigned), hits.size(), fo);
  }
  uint64_t n = kept.size();
  std::fwrite(&n, sizeof(n), 1, fo);
  if (n) std::fwrite(kept.data(), sizeof(Eigen::Vector3d), n, fo);
  n = intensity.size();
  std::fwrite(&n, sizeof(n), 1, fo);
  if (n) std::fwrite(intensity.data(), sizeof(double), n, fo);
  std::fclose(fo);
  return 0;
}
