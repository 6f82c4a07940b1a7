// Drives tloam::FrontEndB200 + tloam::LocalRegistrationB200 the way FrontEnd::updateLidarOdometry does with mapping_flag set
// (ref: src/front_end/front_end.cpp:269-274, :278-337) for three frames: frame 0 seeds the submap (processCloud + initSubmap)
// and is not mapped; frames 1 and 2 are processed, registered from the prediction in the file, appended to the submap and
// appended to the global map with their poses.
//     front_end_map_driver frames.bin raw.bin out.bin
// frames.bin: for each of the 3 frames the ground, edge and general clouds as count + points, then 2 predictions (4x4
// column-major); raw.bin: the 3 raw scans as count + points.  Prints, per registered frame, its four source sizes and the
// 16 values of the pose (column-major); out.bin receives the global map and the last registered scan (each count + points).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

static bool read_cloud(FILE* f, tloam::CloudData& c) {
  uint64_t n = 0;
  if (fread(&n, sizeof(n), 1, f) != 1) return false;
  c.cloud_ptr->points_.resize(n);
  return !n || fread(c.cloud_ptr->points_.data(), sizeof(Eigen::Vector3d), n, f) == n;
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: front_end_map_driver frames.bin raw.bin out.bin\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  tloam::CloudData ground[3], edge[3], general[3], raw[3];
  for (int k = 0; k < 3; ++k)
    if (!read_cloud(f, ground[k]) || !read_cloud(f, edge[k]) || !read_cloud(f, general[k])) return 2;
  Eigen::Isometry3d predict[2];
  for (int k = 0; k < 2; ++k)
    if (fread(predict[k].matrix().data(), sizeof(double), 16, f) != 16) return 2;
  std::fclose(f);
  FILE* fr = std::fopen(argv[2], "rb");
  if (!fr) return 2;
  for (int k = 0; k < 3; ++k)
    if (!read_cloud(fr, raw[k])) return 2;
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
    if (!fe.updateGlobalMap(raw[k], pose)) return 9;
    const size_t* n = fe.sourceSizes();
    std::printf("%zu %zu %zu %zu\n", n[0], n[1], n[2], n[3]);
    for (int i = 0; i < 16; ++i) std::printf("%.17g%c", pose.matrix().data()[i], i == 15 ? '\n' : ' ');
  }
  std::vector<Eigen::Vector3d> map, scan;
  if (!fe.globalMap(map) || !fe.registeredScan(scan)) return 10;
  FILE* fo = std::fopen(argv[3], "wb");
  if (!fo) return 2;
  for (const std::vector<Eigen::Vector3d>* v : {&map, &scan}) {
    const uint64_t n = v->size();
    std::fwrite(&n, sizeof(n), 1, fo);
    if (n) std::fwrite(v->data(), sizeof(Eigen::Vector3d), n, fo);
  }
  std::fclose(fo);
  return 0;
}
