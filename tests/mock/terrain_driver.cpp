// Drives tloam::FrontEndB200's terrain map the way a navigation node would with a saved map: the cloud gives a terrain
// map, its values a costmap, and the costmap a plan to a goal.
//     terrain_driver in.bin out.bin
// in.bin: uint64 n, the cloud (n x 3 FP64), FP64 goal x, y.  The terrain uses its defaults, the costmap the distance
// defaults, the plan its defaults.  Prints "width height known lethal reachable".  out.bin receives FP64 origin_x,
// origin_y, the values (int8), the elevation and the slope (FP64 each), then the costs (uint8).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: terrain_driver in.bin out.bin\n");
    return 2;
  }
  FILE* g = std::fopen(argv[1], "rb");
  if (!g) return 2;
  uint64_t n = 0;
  if (std::fread(&n, sizeof(n), 1, g) != 1) return 2;
  std::vector<double> cloud(3 * n);
  if (n && std::fread(cloud.data(), sizeof(double), cloud.size(), g) != cloud.size()) return 2;
  double goal[2] = {0.0, 0.0};
  if (std::fread(goal, sizeof(double), 2, g) != 2) return 2;
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
  tloam_terrain_config tcfg;
  tloam_b200_terrain_default_config(&tcfg);
  std::vector<int8_t> values;
  std::vector<double> elevation, slope;
  tloam_terrain_info info;
  if (!fe.terrainMap(tcfg, cloud, values, elevation, slope, info)) return 4;
  tloam_distance_config dcfg;
  tloam_b200_distance_default_config(&dcfg);
  std::vector<float> sd;
  std::vector<uint8_t> costs;
  std::vector<int8_t> cost_values;
  tloam_distance_info dinfo;
  if (!fe.distanceFieldTerrain(dcfg, sd, costs, cost_values, dinfo)) return 5;
  tloam_plan_config pcfg;
  tloam_b200_plan_default_config(&pcfg);
  std::vector<unsigned long long> potential;
  tloam_plan_info pinfo;
  if (!fe.planPotential(pcfg, goal[0], goal[1], potential, pinfo)) return 6;
  std::printf("%zu %zu %zu %zu %zu\n", info.width, info.height, info.known, info.lethal, pinfo.reachable);
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  const double origin[2] = {info.origin_x, info.origin_y};
  std::fwrite(origin, sizeof(double), 2, fo);
  if (!values.empty()) {
    std::fwrite(values.data(), 1, values.size(), fo);
    std::fwrite(elevation.data(), sizeof(double), elevation.size(), fo);
    std::fwrite(slope.data(), sizeof(double), slope.size(), fo);
    std::fwrite(costs.data(), 1, costs.size(), fo);
  }
  std::fclose(fo);
  return 0;
}
