// Drives tloam::FrontEndB200 + tloam::LocalRegistrationB200 like front_end_map_driver.cpp, with raw scans that carry
// intensity_ (the driver's XYZI cloud, ref: src/open3d/open3d_to_ros.cpp:361-373): frame 0 seeds the submap and is not
// mapped; frames 1 and 2 are registered from the predictions in the file and appended to the global map with their poses,
// frame 1 by updateGlobalMap and frame 2 by updateGlobalMapChained.
//     front_end_map_intensity_driver frames.bin raw.bin out.bin
// frames.bin: as front_end_map_driver; raw.bin: the 3 raw scans as count + points + count intensities.  Prints, per registered
// frame, the 16 values of its pose (column-major); out.bin receives the global map (count + points) and its intensity
// channel (count + values; count 0 when the map has none).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

static bool read_cloud(FILE* f, tloam::CloudData& c, bool with_intensity) {
  uint64_t n = 0;
  if (fread(&n, sizeof(n), 1, f) != 1) return false;
  c.cloud_ptr->points_.resize(n);
  if (n && fread(c.cloud_ptr->points_.data(), sizeof(Eigen::Vector3d), n, f) != n) return false;
  if (!with_intensity) return true;
  c.cloud_ptr->intensity_.resize(n);
  return !n || fread(c.cloud_ptr->intensity_.data(), sizeof(double), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: front_end_map_intensity_driver frames.bin raw.bin out.bin\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  tloam::CloudData ground[3], edge[3], general[3], raw[3];
  for (int k = 0; k < 3; ++k)
    if (!read_cloud(f, ground[k], false) || !read_cloud(f, edge[k], false) || !read_cloud(f, general[k], false)) return 2;
  Eigen::Isometry3d predict[2];
  for (int k = 0; k < 2; ++k)
    if (fread(predict[k].matrix().data(), sizeof(double), 16, f) != 16) return 2;
  std::fclose(f);
  FILE* fr = std::fopen(argv[2], "rb");
  if (!fr) return 2;
  for (int k = 0; k < 3; ++k)
    if (!read_cloud(fr, raw[k], true)) return 2;
  std::fclose(fr);
  tloam_tls_config cfg;
  tloam_b200_default_config(&cfg);
  tloam_feature_config fcfg;
  tloam_b200_feature_default_config(&fcfg);
  fcfg.cvr_submap = 0.005; fcfg.cvr_scan = 0.01;             // the synthetic street scene has few curvature maxima
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
  if (!fe.enableGlobalMap()) return 8;                          // mapping_flag: true
  if (!fe.processCloud(ground[0], edge[0], general[0]) || !fe.initSubmap()) return 4;
  for (int k = 1; k < 3; ++k) {
    if (!fe.processCloud(ground[k], edge[k], general[k])) return 5;
    tloam::Frame result;
    Eigen::Isometry3d pose;
    if (!reg->scanMatching(result, predict[k - 1], pose)) return 6;
    if (!fe.updateSubmap(pose)) return 7;
    if (!(k == 1 ? fe.updateGlobalMap(raw[k], pose) : fe.updateGlobalMapChained(raw[k]))) return 9;
    for (int i = 0; i < 16; ++i) std::printf("%.17g%c", pose.matrix().data()[i], i == 15 ? '\n' : ' ');
  }
  std::vector<Eigen::Vector3d> map;
  std::vector<double> intensity;
  if (!fe.globalMap(map, intensity)) return 10;
  FILE* fo = std::fopen(argv[3], "wb");
  if (!fo) return 2;
  uint64_t n = map.size();
  std::fwrite(&n, sizeof(n), 1, fo);
  if (n) std::fwrite(map.data(), sizeof(Eigen::Vector3d), n, fo);
  n = intensity.size();
  std::fwrite(&n, sizeof(n), 1, fo);
  if (n) std::fwrite(intensity.data(), sizeof(double), n, fo);
  std::fclose(fo);
  return 0;
}
