// Drives tloam::FrontEndB200's frontier search the way an exploration node would: a saved grid gives a costmap, the
// robot's position gives a plan, and the frontiers ranked by that plan give the next goal and its route.
//     frontier_driver in.bin out.bin
// in.bin: uint64 width, height, FP64 origin_x, origin_y, resolution, the cells (int8), FP64 robot x, y.  The costmap uses
// the distance defaults but inscribed 0.3 m and inflation 1.0 m; the plan and the search use their defaults.
// Prints "cells components kept reachable".  out.bin receives per kept frontier, in rank order, its id (uint64), status
// (int64), size (uint64), approach potential (uint64), cost, distance, centroid x, y and approach x, y (FP64), then its
// cells' centres (size x 2 FP64); then the route to the first reachable frontier (uint64 m, m x 2 FP64: the reversed
// path from its approach cell, from the robot to the approach), m = 0 when none is reachable.
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

int main(int argc, char** argv) {
  if (argc < 3) {
    std::fprintf(stderr, "usage: frontier_driver in.bin out.bin\n");
    return 2;
  }
  FILE* g = std::fopen(argv[1], "rb");
  if (!g) return 2;
  uint64_t wh[2] = {0, 0};
  double head[3] = {0.0, 0.0, 0.0};
  if (std::fread(wh, sizeof(uint64_t), 2, g) != 2 || std::fread(head, sizeof(double), 3, g) != 3) return 2;
  std::vector<int8_t> cells(wh[0] * wh[1]);
  if (!cells.empty() && std::fread(cells.data(), 1, cells.size(), g) != cells.size()) return 2;
  double robot[2] = {0.0, 0.0};
  if (std::fread(robot, sizeof(double), 2, g) != 2) return 2;
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
  tloam_plan_info pinfo;
  if (!fe.planPotential(pcfg, robot[0], robot[1], potential, pinfo)) return 5;
  tloam_frontier_config frcfg;
  tloam_b200_frontier_default_config(&frcfg);
  std::vector<tloam_frontier> found;
  std::vector<std::vector<double>> found_xy;
  tloam_frontier_info info;
  if (!fe.frontiers(frcfg, found, found_xy, info)) return 6;
  std::vector<double> route;
  if (!found.empty() && found[0].status == 0) {
    std::vector<std::vector<double>> paths;
    std::vector<int> statuses;
    std::vector<unsigned long long> path_costs;
    if (!fe.planPaths(std::vector<double>{found[0].approach_x, found[0].approach_y}, paths, statuses, path_costs)) return 7;
    for (size_t k = paths[0].size() / 2; k-- > 0;) {
      route.push_back(paths[0][2 * k]);
      route.push_back(paths[0][2 * k + 1]);
    }
  }
  std::printf("%zu %zu %zu %zu\n", info.cells, info.components, info.kept, info.reachable);
  FILE* fo = std::fopen(argv[2], "wb");
  if (!fo) return 2;
  for (size_t k = 0; k < found.size(); ++k) {
    const tloam_frontier& f = found[k];
    const uint64_t ids[4] = {f.id, (uint64_t)(int64_t)f.status, f.size, f.approach_potential};
    const double v[6] = {f.cost, f.distance, f.centroid_x, f.centroid_y, f.approach_x, f.approach_y};
    std::fwrite(ids, sizeof(uint64_t), 4, fo);
    std::fwrite(v, sizeof(double), 6, fo);
    if (!found_xy[k].empty()) std::fwrite(found_xy[k].data(), sizeof(double), found_xy[k].size(), fo);
  }
  const uint64_t m = route.size() / 2;
  std::fwrite(&m, sizeof(m), 1, fo);
  if (m) std::fwrite(route.data(), sizeof(double), route.size(), fo);
  std::fclose(fo);
  return 0;
}
