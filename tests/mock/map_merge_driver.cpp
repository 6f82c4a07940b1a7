// Drives tloam::FrontEndB200's merged global map the way a mapping node that saves its map would: the map and dynamic-point
// removal are enabled, every raw scan of the file is appended with its pose (updateGlobalMap, with intensity), then the
// map is merged into one voxel grid twice: whole, and without the points judged dynamic.
//     map_merge_driver raw.bin out.bin voxel n_rows n_cols fov_down fov_up
// raw.bin: uint64 scan count, then per scan its pose (16 FP64, column-major), a count, the points (FP64 x, y, z) and their
// intensities.  Prints "merged merged_static".  out.bin receives, for the whole map and then the static one, the merged
// cloud (count + points) and its intensity (count + values).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

static void write_cloud(FILE* fo, const std::vector<Eigen::Vector3d>& pts, const std::vector<double>& intensity) {
  uint64_t n = pts.size();
  std::fwrite(&n, sizeof(n), 1, fo);
  if (n) std::fwrite(pts.data(), sizeof(Eigen::Vector3d), n, fo);
  n = intensity.size();
  std::fwrite(&n, sizeof(n), 1, fo);
  if (n) std::fwrite(intensity.data(), sizeof(double), n, fo);
}

int main(int argc, char** argv) {
  if (argc < 8) {
    std::fprintf(stderr, "usage: map_merge_driver raw.bin out.bin voxel n_rows n_cols fov_down fov_up\n");
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
  const double voxel = std::atof(argv[3]);
  dcfg.n_rows = std::atoi(argv[4]);
  dcfg.n_cols = std::atoi(argv[5]);
  dcfg.fov_down = std::atof(argv[6]);
  dcfg.fov_up = std::atof(argv[7]);
  if (!fe.enableGlobalMap() || !fe.enableDynamicRemoval(dcfg)) return 4;
  for (size_t k = 0; k < raw.size(); ++k)
    if (!fe.updateGlobalMap(raw[k], pose[k])) return 5;
  std::vector<Eigen::Vector3d> merged, merged_static;
  std::vector<double> intensity, intensity_static;
  if (!fe.mergedGlobalMap(voxel, false, merged, intensity) ||
      !fe.mergedGlobalMap(voxel, true, merged_static, intensity_static))
    return 6;
  std::printf("%zu %zu\n", merged.size(), merged_static.size());
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  write_cloud(fo, merged, intensity);
  write_cloud(fo, merged_static, intensity_static);
  std::fclose(fo);
  return 0;
}
