// Hands the driver's sensor_msgs/PointCloud2 (a mock of its members below) to the timed packed call, as a deskewing front
// end would: packedScanOf + packedTimeOf, then tloam_b200_process_raw_scan_packed_timed with a seeded pose history, and the
// corrected scan read back through global_map_append_frame(I) + registered_scan_download.
//     deskew_driver describe in.bin           prints, per message, "rc_scan rc_time offset datatype unit" (no GPU needed)
//     deskew_driver run in.bin out.bin        also processes every message whose descriptors are valid
// in.bin: double last_pose[16], curr_pose[16] (column-major), frame_period, uint32 message count, then per message: uint32
// field count, per field uint8 name length, name, uint32 offset, uint8 datatype, uint32 count; uint8 is_bigendian, uint32
// width, height, point_step, then width * height * point_step bytes.  out.bin: per processed message, uint64 rows, then its
// corrected scan (rows x 3 FP64).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/tloam_b200/packed_scan_b200.hpp"

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

template <class T>
static bool get(FILE* f, T* v, size_t n = 1) { return std::fread(v, sizeof(T), n, f) == n; }

static bool read_msg(FILE* f, mock_msgs::PointCloud2& m) {
  uint32_t nf = 0;
  if (!get(f, &nf)) return false;
  for (uint32_t k = 0; k < nf; ++k) {
    mock_msgs::PointField pf;
    uint8_t len = 0;
    if (!get(f, &len)) return false;
    pf.name.resize(len);
    if (len && std::fread(&pf.name[0], 1, len, f) != len) return false;
    if (!get(f, &pf.offset) || !get(f, &pf.datatype) || !get(f, &pf.count)) return false;
    m.fields.push_back(pf);
  }
  if (!get(f, &m.is_bigendian) || !get(f, &m.width) || !get(f, &m.height) || !get(f, &m.point_step)) return false;
  m.row_step = m.width * m.point_step;
  m.data.resize(static_cast<size_t>(m.height) * m.row_step);
  return m.data.empty() || std::fread(m.data.data(), 1, m.data.size(), f) == m.data.size();
}

int main(int argc, char** argv) {
  if (argc < 3 || (std::strcmp(argv[1], "run") == 0 && argc < 4)) {
    std::fprintf(stderr, "usage: deskew_driver describe|run in.bin [out.bin]\n");
    return 2;
  }
  const bool run = std::strcmp(argv[1], "run") == 0;
  FILE* f = std::fopen(argv[2], "rb");
  if (!f) return 2;
  double last[16], curr[16], period = 0.0;
  uint32_t count = 0;
  if (!get(f, last, 16) || !get(f, curr, 16) || !get(f, &period) || !get(f, &count)) return 2;
  std::vector<mock_msgs::PointCloud2> msgs(count);
  for (auto& m : msgs)
    if (!read_msg(f, m)) return 2;
  std::fclose(f);
  tloam_b200_handle* h = nullptr;
  tloam_ground_config gcfg;
  tloam_dcvc_config dcfg;
  tloam_feature_config fcfg;
  FILE* fo = nullptr;
  const double eye[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  if (run) {
    tloam_tls_config cfg;
    tloam_b200_default_config(&cfg);
    int rc = tloam_b200_create(&cfg, 0, nullptr, &h);
    if (rc != TLOAM_B200_OK) { std::fprintf(stderr, "create: %s\n", tloam_b200_status_string(rc)); return 3; }
    tloam_b200_ground_default_config(&gcfg);
    tloam_b200_dcvc_default_config(&dcfg);
    tloam_b200_feature_default_config(&fcfg);
    fcfg.cvr_submap = 0.005; fcfg.cvr_scan = 0.01;             // the synthetic street scene has few curvature maxima
    tloam_global_map_config mcfg;
    mcfg.voxel = 1.0; mcfg.initial_capacity_points = 1 << 20;
    if (tloam_b200_global_map_enable(h, &mcfg) != TLOAM_B200_OK) return 4;
    fo = std::fopen(argv[3], "wb");
    if (!fo) return 2;
  }
  for (const auto& m : msgs) {
    tloam_packed_scan scan;
    tloam_packed_time time;
    const int rs = tloam::packedScanOf(m, &scan), rt = tloam::packedTimeOf(m, &time);
    if (rt == TLOAM_B200_OK) std::printf("%d %d %d %d %.17g\n", rs, rt, time.offset, time.datatype, time.unit);
    else std::printf("%d %d\n", rs, rt);
    if (!run || rs != TLOAM_B200_OK || rt != TLOAM_B200_OK) continue;
    size_t ns[4];
    if (tloam_b200_set_pose_history(h, last, curr) != TLOAM_B200_OK) return 5;
    int rc = tloam_b200_process_raw_scan_packed_timed(h, &gcfg, &dcfg, 131, 3.0, &fcfg, 0.3, 0.1, &scan, &time, period, ns);
    if (rc != TLOAM_B200_OK) { std::fprintf(stderr, "process: %s %s\n", tloam_b200_status_string(rc), tloam_b200_last_error(h)); return 6; }
    if (tloam_b200_global_map_append_frame(h, eye) != TLOAM_B200_OK) return 7;
    size_t n = 0;
    std::vector<double> out(3 * scan.n + 3);
    if (tloam_b200_registered_scan_download(h, out.data(), scan.n, &n) != TLOAM_B200_OK) return 8;
    const uint64_t rows = n;
    std::fwrite(&rows, sizeof(rows), 1, fo);
    if (n) std::fwrite(out.data(), sizeof(double), 3 * n, fo);
  }
  if (fo) std::fclose(fo);
  if (h) tloam_b200_destroy(h);
  return 0;
}
