// Drives tloam::FrontEndB200's distance field the way a planning node would: the occupancy grid of the mapped scans gives
// one field, then a saved grid (a localization session's map) gives another, and the second is queried at points.
//     distance_driver raw.bin grid.bin out.bin resolution n_cols max_range
// raw.bin: uint64 scan count, then per scan its pose (16 FP64, column-major), a count and the points (FP64 x, y, z).
// grid.bin: uint64 width, height, FP64 origin_x, origin_y, resolution, the cells (int8), uint64 n, the points (n x 2 FP64).
// Prints "width height obstacles" of each field.  out.bin receives, per field, sd (float32), costs (uint8) and values
// (int8), then the query's distances (n FP64) and gradients (n x 2 FP64).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <vector>

static void put(FILE* f, const tloam_distance_info& info, const std::vector<float>& sd, const std::vector<uint8_t>& costs,
                const std::vector<int8_t>& values) {
  std::printf("%zu %zu %zu\n", info.width, info.height, info.obstacles);
  if (sd.empty()) return;
  std::fwrite(sd.data(), sizeof(float), sd.size(), f);
  std::fwrite(costs.data(), 1, costs.size(), f);
  std::fwrite(values.data(), 1, values.size(), f);
}

int main(int argc, char** argv) {
  if (argc < 7) {
    std::fprintf(stderr, "usage: distance_driver raw.bin grid.bin out.bin resolution n_cols max_range\n");
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
  FILE* g = std::fopen(argv[2], "rb");
  if (!g) return 2;
  uint64_t wh[2] = {0, 0};
  double head[3] = {0.0, 0.0, 0.0};
  if (std::fread(wh, sizeof(uint64_t), 2, g) != 2 || std::fread(head, sizeof(double), 3, g) != 3) return 2;
  std::vector<int8_t> cells(wh[0] * wh[1]);
  if (!cells.empty() && std::fread(cells.data(), 1, cells.size(), g) != cells.size()) return 2;
  uint64_t nq = 0;
  if (std::fread(&nq, sizeof(nq), 1, g) != 1) return 2;
  std::vector<double> xy(2 * nq);
  if (nq && std::fread(xy.data(), sizeof(double), xy.size(), g) != xy.size()) return 2;
  std::fclose(g);

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
  ocfg.resolution = std::atof(argv[4]);
  ocfg.n_cols = std::atoi(argv[5]);
  ocfg.max_range = std::atof(argv[6]);
  if (!fe.enableGlobalMap() || !fe.enableOccupancy(ocfg)) return 4;
  for (size_t k = 0; k < raw.size(); ++k)
    if (!fe.updateGlobalMap(raw[k], pose[k])) return 5;
  std::vector<int8_t> grid;
  tloam_occupancy_info oinfo;
  if (!fe.occupancyGrid(grid, oinfo)) return 6;
  tloam_distance_config dcfg;
  tloam_b200_distance_default_config(&dcfg);
  std::vector<float> sd;
  std::vector<uint8_t> costs;
  std::vector<int8_t> values;
  tloam_distance_info info;
  FILE* fo = std::fopen(argv[3], "wb");
  if (!fo) return 2;
  if (!fe.distanceField(dcfg, sd, costs, values, info)) return 7;
  put(fo, info, sd, costs, values);
  if (!fe.distanceField(dcfg, cells, wh[0], wh[1], head[0], head[1], head[2], sd, costs, values, info)) return 8;
  put(fo, info, sd, costs, values);
  std::vector<double> distance, gradient;
  if (!fe.queryDistance(xy, distance, gradient)) return 9;
  if (nq) {
    std::fwrite(distance.data(), sizeof(double), distance.size(), fo);
    std::fwrite(gradient.data(), sizeof(double), gradient.size(), fo);
  }
  std::fclose(fo);
  return 0;
}
