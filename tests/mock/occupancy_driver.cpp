// Drives tloam::FrontEndB200's occupancy grid the way a mapping node would: the grid is enabled right after the map, every
// raw scan of the file is appended with its pose (updateGlobalMap), then the grid is built and read back.
//     occupancy_driver raw.bin out.bin resolution n_cols max_range
// raw.bin: uint64 scan count, then per scan its pose (16 FP64, column-major), a count and the points (FP64 x, y, z).
// Prints "width height".  out.bin receives origin_x, origin_y, resolution (FP64), dropped (uint64) and the cells (int8).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 6) {
    std::fprintf(stderr, "usage: occupancy_driver raw.bin out.bin resolution n_cols max_range\n");
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
    if (n && std::fread(raw[k].cloud_ptr->points_.data(), sizeof(Eigen::Vector3d), n, f) != n) return 2;
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
  tloam_occupancy_config ocfg;
  tloam_b200_occupancy_default_config(&ocfg);
  ocfg.resolution = std::atof(argv[3]);
  ocfg.n_cols = std::atoi(argv[4]);
  ocfg.max_range = std::atof(argv[5]);
  if (!fe.enableGlobalMap() || !fe.enableOccupancy(ocfg)) return 4;
  for (size_t k = 0; k < raw.size(); ++k)
    if (!fe.updateGlobalMap(raw[k], pose[k])) return 5;
  std::vector<int8_t> cells;
  tloam_occupancy_info info;
  if (!fe.occupancyGrid(cells, info)) return 6;
  std::printf("%zu %zu\n", info.width, info.height);
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  const double head[3] = {info.origin_x, info.origin_y, info.resolution};
  std::fwrite(head, sizeof(double), 3, fo);
  const uint64_t dropped = info.dropped;
  std::fwrite(&dropped, sizeof(dropped), 1, fo);
  if (!cells.empty()) std::fwrite(cells.data(), 1, cells.size(), fo);
  std::fclose(fo);
  return 0;
}
