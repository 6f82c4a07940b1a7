// Drives tloam::FrontEndB200 + tloam::LocalRegistrationB200 like front_end_map_intensity_driver.cpp, with the raw scans
// handed over as the driver's sensor_msgs/PointCloud2 (a mock of its members below): frame 0 seeds the submap and is not
// mapped; frames 1 and 2 are registered from the predictions in the file and appended to the global map from their
// messages, frame 1 by updateGlobalMap(msg, pose) and frame 2 by updateGlobalMapChained(msg).  A big-endian message is then
// refused with INVALID_ARG and leaves the map alone.
//     packed_scan_driver frames.bin raw.bin out.bin
// frames.bin: as front_end_map_driver; raw.bin: per scan, uint64 width, height, point_step, int32 x / y / z / intensity
// offsets (intensity -1: no such field), then width * height * point_step bytes.  Prints, per registered frame, the 16
// values of its pose (column-major); out.bin receives the global map (count + points) and its intensity channel (count +
// values; count 0 when the map has none).
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/front_end_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

namespace mock_msgs {                       // the members of sensor_msgs::PointField / PointCloud2 the shim reads
struct PointField {
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 0;
};
struct PointCloud2 {
  uint32_t height = 0, width = 0;
  std::vector<PointField> fields;
  uint8_t is_bigendian = 0;
  uint32_t point_step = 0, row_step = 0;
  std::vector<uint8_t> data;
  uint8_t is_dense = 0;
};
}  // namespace mock_msgs

// compiles only if a CloudData argument still selects the CloudData overloads (the message template would read .fields)
bool mapCloudData(tloam::FrontEndB200& fe, const tloam::CloudData& raw, const Eigen::Isometry3d& pose) {
  return fe.updateGlobalMap(raw, pose) && fe.updateGlobalMapChained(raw);
}

static bool read_cloud(FILE* f, tloam::CloudData& c) {
  uint64_t n = 0;
  if (fread(&n, sizeof(n), 1, f) != 1) return false;
  c.cloud_ptr->points_.resize(n);
  return !n || fread(c.cloud_ptr->points_.data(), sizeof(Eigen::Vector3d), n, f) == n;
}

static bool read_msg(FILE* f, mock_msgs::PointCloud2& m) {
  uint64_t dims[3];
  int32_t off[4];
  if (fread(dims, sizeof(uint64_t), 3, f) != 3 || fread(off, sizeof(int32_t), 4, f) != 4) return false;
  m.width = (uint32_t)dims[0]; m.height = (uint32_t)dims[1]; m.point_step = (uint32_t)dims[2];
  m.row_step = m.width * m.point_step;
  static const char* const names[4] = {"x", "y", "z", "intensity"};
  for (int k = 0; k < 4; ++k) {
    if (off[k] < 0) continue;
    mock_msgs::PointField pf;
    pf.name = names[k]; pf.offset = (uint32_t)off[k]; pf.datatype = 7; pf.count = 1;
    m.fields.push_back(pf);
  }
  mock_msgs::PointField ring;                // a field the shim does not read
  ring.name = "ring"; ring.offset = 0; ring.datatype = 4; ring.count = 1;
  m.fields.push_back(ring);
  m.data.resize((size_t)m.height * m.row_step);
  return m.data.empty() || fread(m.data.data(), 1, m.data.size(), f) == m.data.size();
}

int main(int argc, char** argv) {
  if (argc < 4) { std::fprintf(stderr, "usage: packed_scan_driver frames.bin raw.bin out.bin\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  tloam::CloudData ground[3], edge[3], general[3];
  for (int k = 0; k < 3; ++k)
    if (!read_cloud(f, ground[k]) || !read_cloud(f, edge[k]) || !read_cloud(f, general[k])) return 2;
  Eigen::Isometry3d predict[2];
  for (int k = 0; k < 2; ++k)
    if (fread(predict[k].matrix().data(), sizeof(double), 16, f) != 16) return 2;
  std::fclose(f);
  FILE* fr = std::fopen(argv[2], "rb");
  if (!fr) return 2;
  mock_msgs::PointCloud2 raw[3];
  for (int k = 0; k < 3; ++k)
    if (!read_msg(fr, raw[k])) return 2;
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
  Eigen::Isometry3d pose;
  for (int k = 1; k < 3; ++k) {
    if (!fe.processCloud(ground[k], edge[k], general[k])) return 5;
    tloam::Frame result;
    if (!reg->scanMatching(result, predict[k - 1], pose)) return 6;
    if (!fe.updateSubmap(pose)) return 7;
    if (!(k == 1 ? fe.updateGlobalMap(raw[k], pose) : fe.updateGlobalMapChained(raw[k]))) return 9;
    for (int i = 0; i < 16; ++i) std::printf("%.17g%c", pose.matrix().data()[i], i == 15 ? '\n' : ' ');
  }
  mock_msgs::PointCloud2 big = raw[1];
  big.is_bigendian = 1;
  if (fe.updateGlobalMap(big, pose) || fe.lastStatus() != TLOAM_B200_ERR_INVALID_ARG) return 11;
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
