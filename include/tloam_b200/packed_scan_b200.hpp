// packed_scan_b200.hpp -- C++ shim: the tloam_packed_scan of a sensor_msgs/PointCloud2, so that the driver's message is
// handed to the packed entry points of libtloam_b200.so as it arrived (one upload, unpacked on the device) instead of being
// converted point by point on the host (ref: src/open3d/open3d_to_ros.cpp:344-374, RosToOpen3d).  Header-only; it reads
// only the members every PointCloud2-shaped type has: fields[].name / offset / datatype / count, point_step, row_step,
// width, height, is_bigendian and data.
//
// Deliberately stricter than RosToOpen3d, which reads any field named "intensity" as a float whatever its datatype: x, y, z
// and intensity must be FLOAT32 (datatype 7) with count 1.  Big-endian data and rows with padding (row_step != width *
// point_step) are refused too.  A message without an intensity field is a scan without intensity.  packedTimeOf describes
// the message's per-point time field for the timed (deskewing) call.
#ifndef TLOAM_B200_PACKED_SCAN_B200_HPP
#define TLOAM_B200_PACKED_SCAN_B200_HPP

#include <climits>
#include <cstddef>

#include "../tloam_b200.h"

namespace tloam {

// fills *out from msg (out->data points into msg.data: the message must outlive the call it is passed to).  Returns
// TLOAM_B200_OK, or TLOAM_B200_ERR_INVALID_ARG for a layout the packed calls cannot take.
template <class Msg>
int packedScanOf(const Msg& msg, tloam_packed_scan* out) {
  if (!out || msg.is_bigendian) return TLOAM_B200_ERR_INVALID_ARG;
  const size_t n = static_cast<size_t>(msg.width) * static_cast<size_t>(msg.height);
  if (static_cast<size_t>(msg.row_step) != static_cast<size_t>(msg.width) * static_cast<size_t>(msg.point_step))
    return TLOAM_B200_ERR_INVALID_ARG;
  if (msg.data.size() < n * static_cast<size_t>(msg.point_step)) return TLOAM_B200_ERR_INVALID_ARG;
  static const char* const kNames[4] = {"x", "y", "z", "intensity"};
  int off[4] = {-1, -1, -1, -1};
  for (const auto& f : msg.fields) {
    for (int k = 0; k < 4; ++k) {
      if (f.name != kNames[k]) continue;
      if (f.datatype != 7 || f.count != 1 || f.offset > static_cast<unsigned>(INT_MAX)) return TLOAM_B200_ERR_INVALID_ARG;   // FLOAT32
      off[k] = static_cast<int>(f.offset);
    }
  }
  if (off[0] < 0 || off[1] < 0 || off[2] < 0) return TLOAM_B200_ERR_INVALID_ARG;
  out->data = msg.data.empty() ? nullptr : msg.data.data();
  out->n = n;
  out->point_step = msg.point_step;
  out->x_offset = off[0]; out->y_offset = off[1]; out->z_offset = off[2]; out->intensity_offset = off[3];
  return TLOAM_B200_OK;
}

// fills *out with the per-point time field of msg, for tloam_b200_process_raw_scan_packed_timed: the first of "time"
// (FLOAT32, seconds: velodyne_pointcloud), "t" (UINT32, nanoseconds: Ouster) and "timestamp" (FLOAT64, seconds: Hesai) the
// message has, which must have that datatype with count 1.  Returns TLOAM_B200_OK, or TLOAM_B200_ERR_INVALID_ARG for a
// big-endian message, a message without any of the three fields, or one of another type (tloam_b200.packed_time's rules).
template <class Msg>
int packedTimeOf(const Msg& msg, tloam_packed_time* out) {
  if (!out || msg.is_bigendian) return TLOAM_B200_ERR_INVALID_ARG;
  static const char* const kNames[3] = {"time", "t", "timestamp"};
  static const int kTypes[3] = {7, 6, 8};                 // FLOAT32, UINT32, FLOAT64
  static const double kUnits[3] = {1.0, 1e-9, 1.0};
  for (int k = 0; k < 3; ++k) {
    for (const auto& f : msg.fields) {
      if (f.name != kNames[k]) continue;
      if (f.datatype != kTypes[k] || f.count != 1 || f.offset > static_cast<unsigned>(INT_MAX)) return TLOAM_B200_ERR_INVALID_ARG;
      out->offset = static_cast<int>(f.offset);
      out->datatype = kTypes[k];
      out->unit = kUnits[k];
      return TLOAM_B200_OK;
    }
  }
  return TLOAM_B200_ERR_INVALID_ARG;
}

}  // namespace tloam
#endif
