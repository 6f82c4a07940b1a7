// Drives tloam::SegmentationB200 on VLP-16 scans the way Segmentation::spinOnce does (ref: src/models/segmentation/
// segmentation.cpp:47-66).  Reads a file written by the Python test (binary: count, raw points, count, points of the raw
// scan after RemoveClosedNonFinitePoints).  Prints, for two consecutive frames of segmentRawScan(raw): "ng nb ne nn", the
// boxes, then one line per ground / edge / general point; then for groundRemove(filtered): "ng no ncur" and one line per
// ground / object / current_scan point.  A point line is the bit pattern of its first coordinate and its intensity.
#define TLOAM_B200_MOCK_HOST_TYPES
#include "mock_tloam.hpp"
#include "../../include/tloam_b200/segmentation_b200.hpp"

#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>

static bool read_cloud(FILE* f, std::vector<Eigen::Vector3d>& pts) {
  uint64_t n = 0;
  if (fread(&n, sizeof(n), 1, f) != 1) return false;
  pts.resize(n);
  return !n || fread(pts.data(), sizeof(Eigen::Vector3d), n, f) == n;
}

static void dump(const tloam::CloudData& c) {
  for (size_t i = 0; i < c.cloud_ptr->points_.size(); ++i) {
    uint64_t bits;
    std::memcpy(&bits, &c.cloud_ptr->points_[i].v[0], 8);
    std::printf("%llu %.17g\n", (unsigned long long)bits, c.cloud_ptr->intensity_[i]);
  }
}

int main(int argc, char** argv) {
  if (argc < 2) { std::fprintf(stderr, "usage: vlp16_driver scans.bin\n"); return 2; }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<Eigen::Vector3d> raw, filtered;
  if (!read_cloud(f, raw) || !read_cloud(f, filtered)) return 2;
  std::fclose(f);
  tloam_ground_config gcfg;
  tloam_b200_ground_default_config(&gcfg);
  gcfg.sensor_model = 16; gcfg.vertical_res = 2.0; gcfg.init_angle = -15.0;   // the VLP-16 settings (INTEGRATION.md)
  tloam_dcvc_config dcfg;
  tloam_b200_dcvc_default_config(&dcfg);
  dcfg.min_polar_init = dcfg.max_polar_init = 5.0;             // first frame (segmentation.hpp:332-333)
  std::unique_ptr<tloam::SegmentationB200> seg;
  try {
    seg.reset(new tloam::SegmentationB200(gcfg, dcfg, 131));
  } catch (const std::exception& e) {
    std::fprintf(stderr, "%s\n", e.what());
    return 3;
  }
  for (int frame = 0; frame < 2; ++frame) {
    tloam::CloudData scan, ground, edge, general;
    scan.cloud_ptr->points_ = raw;
    std::vector<tloam::BoxB200> boxes;
    if (!seg->segmentRawScan(scan, ground, edge, general, &boxes)) return 4;
    std::printf("%zu %zu %zu %zu\n", ground.cloud_ptr->points_.size(), boxes.size(), edge.cloud_ptr->points_.size(),
                general.cloud_ptr->points_.size());
    for (const tloam::BoxB200& b : boxes)
      std::printf("%d %d %.17g %.17g %.17g %.17g %.17g %.17g\n", b.label, b.points, b.position[0], b.position[1], b.position[2],
                  b.dimensions[0], b.dimensions[1], b.dimensions[2]);
    dump(ground);
    dump(edge);
    dump(general);
  }
  tloam::CloudData current, ground, object;
  current.cloud_ptr->points_ = filtered;
  if (!seg->groundRemove(current, ground, object)) return 5;
  std::printf("%zu %zu %zu\n", ground.cloud_ptr->points_.size(), object.cloud_ptr->points_.size(), current.cloud_ptr->points_.size());
  dump(ground);
  dump(object);
  dump(current);
  return 0;
}
