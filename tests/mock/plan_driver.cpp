// Drives tloam::FrontEndB200's path planning the way a planning node would: a saved grid (a localization session's map)
// gives a costmap, a goal gives a potential, and the starts give paths ready to publish as nav_msgs/Path.
//     plan_driver in.bin out.bin
// in.bin: uint64 width, height, FP64 origin_x, origin_y, resolution, the cells (int8), FP64 goal x, y, uint64 n, the
// starts (n x 2 FP64).  The costmap uses the distance defaults but inscribed 0.3 m and inflation 1.0 m.
// Prints "width height reachable".  out.bin receives the potential (uint64), then per start its status (int64), cost
// (uint64), cell count m (uint64) and path xy (m x 2 FP64).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: plan_driver in.bin out.bin\n");
    return 2;
  }
  FILE* g = std::fopen(argv[1], "rb");
  if (!g) return 2;
  uint64_t wh[2] = {0, 0};
  double head[3] = {0.0, 0.0, 0.0};
  if (std::fread(wh, sizeof(uint64_t), 2, g) != 2 || std::fread(head, sizeof(double), 3, g) != 3) return 2;
  std::vector<int8_t> cells(wh[0] * wh[1]);
  if (!cells.empty() && std::fread(cells.data(), 1, cells.size(), g) != cells.size()) return 2;
  double goal[2] = {0.0, 0.0};
  uint64_t n = 0;
  if (std::fread(goal, sizeof(double), 2, g) != 2 || std::fread(&n, sizeof(n), 1, g) != 1) return 2;
  std::vector<double> starts(2 * n);
  if (n && std::fread(starts.data(), sizeof(double), starts.size(), g) != starts.size()) return 2;
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
  tloam_distance_config dcfg;
  tloam_b200_distance_default_config(&dcfg);
  dcfg.inscribed_radius = 0.3;
  dcfg.inflation_radius = 1.0;
  std::vector<float> sd;
  std::vector<uint8_t> costs;
  std::vector<int8_t> values;
  tloam_distance_info dinfo;
  if (!fe.distanceField(dcfg, cells, wh[0], wh[1], head[0], head[1], head[2], sd, costs, values, dinfo)) return 4;
  tloam_plan_config pcfg;
  tloam_b200_plan_default_config(&pcfg);
  std::vector<unsigned long long> potential;
  tloam_plan_info info;
  if (!fe.planPotential(pcfg, goal[0], goal[1], potential, info)) return 5;
  std::vector<std::vector<double>> paths;
  std::vector<int> statuses;
  std::vector<unsigned long long> path_costs;
  if (!fe.planPaths(starts, paths, statuses, path_costs)) return 6;
  std::printf("%zu %zu %zu\n", info.width, info.height, info.reachable);
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  std::fwrite(potential.data(), sizeof(unsigned long long), potential.size(), fo);
  for (size_t s = 0; s < paths.size(); ++s) {
    const int64_t status = statuses[s];
    const uint64_t head_out[2] = {path_costs[s], paths[s].size() / 2};
    std::fwrite(&status, sizeof(status), 1, fo);
    std::fwrite(head_out, sizeof(uint64_t), 2, fo);
    if (!paths[s].empty()) std::fwrite(paths[s].data(), sizeof(double), paths[s].size(), fo);
  }
  std::fclose(fo);
  return 0;
}
