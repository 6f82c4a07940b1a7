// ground_extract_b200.hpp -- C++ shim: tloam::GroundExtractB200, the device replacement of the ground-removal step of
// the segmentation nodelet, Segmentation::groundRemove (ref: src/models/segmentation/segmentation.cpp:738-770; members
// current_scan / ground_scan / object_scan, ref: include/tloam/models/segmentation/segmentation.hpp), implemented on
// the C ABI of libtloam_b200.so ("next" row 8(f)-4, first part).  Header-only; from the host side it needs only
// CloudData::cloud_ptr->points_ / intensity_ (ref: include/tloam/models/utils/sensor_data.hpp:17-43).
//
// In the reference tree, Segmentation::groundRemove() becomes:
//     return ground_extract_b200_->groundRemove(current_scan, ground_scan, object_scan);
// Without the reference headers (this repository's tests) define TLOAM_B200_MOCK_HOST_TYPES and provide tloam::CloudData
// with the same members (tests/mock/mock_tloam.hpp).
#ifndef TLOAM_B200_GROUND_EXTRACT_B200_HPP
#define TLOAM_B200_GROUND_EXTRACT_B200_HPP

#include <cstdio>
#include <stdexcept>
#include <string>
#include <vector>

#include "../tloam_b200.h"

#ifndef TLOAM_B200_MOCK_HOST_TYPES
#include <yaml-cpp/yaml.h>
#include "tloam/models/utils/sensor_data.hpp"
#endif

namespace tloam {

class GroundExtractB200 {
 public:
  // `shared` = a handle that already exists (e.g. LocalRegistrationB200::handle()); nullptr = own handle on `device`.
  explicit GroundExtractB200(const tloam_ground_config& cfg, tloam_b200_handle* shared = nullptr, int device = 0) : cfg_(cfg) {
    attach(shared, device);
  }

#ifndef TLOAM_B200_MOCK_HOST_TYPES
  // Reads the keys Segmentation::initVeldyneConfig / initGroundSegConfig read (ref: segmentation.cpp:114-133;
  // config/mapping/segmentation.yaml "velodyne:" and "groundSeg:").
  GroundExtractB200(const YAML::Node& velodyne, const YAML::Node& ground_seg, tloam_b200_handle* shared = nullptr, int device = 0) {
    tloam_b200_ground_default_config(&cfg_);
    cfg_.sensor_model = velodyne["sensorModel"].as<int>();
    cfg_.sensor_height = velodyne["sensorHeight"].as<double>();
    cfg_.vertical_res = velodyne["verticalRes"].as<double>();
    cfg_.init_angle = velodyne["initAngle"].as<double>();
    cfg_.sensor_min_range = velodyne["sensorMinRange"].as<double>();
    cfg_.sensor_max_range = velodyne["sensorMaxRange"].as<double>();
    cfg_.quadrant = ground_seg["quadrant"].as<int>();
    cfg_.num_sec = ground_seg["numSec"].as<int>();
    cfg_.plane_dis = ground_seg["dis"].as<double>();
    cfg_.max_iter = ground_seg["maxIter"].as<int>();
    cfg_.ground_seed_num = ground_seg["ground_seed_num"].as<int>();
    attach(shared, device);
  }
#endif

  ~GroundExtractB200() { if (own_) tloam_b200_destroy(h_); }
  GroundExtractB200(const GroundExtractB200&) = delete;
  GroundExtractB200& operator=(const GroundExtractB200&) = delete;

  // ref: segmentation.cpp:738-770.  current_scan: the scan after RemoveClosedNonFinitePoints (:472-505).  On return
  // ground_scan / object_scan have received (+=, like the reference) the ground / non-ground points; the ground
  // intensities are the fractional part of the channel (0 for the HDL-64E branch, :692-695), the object intensities the
  // channel (:707-709); current_scan keeps the points at or below the height threshold with the channel as intensity
  // (filterByHeight, :454-470).  The channel: HDL-64E the beam estimate, VLP-16 beamId + correctTime (:386-429).
  bool groundRemove(CloudData& current_scan, CloudData& ground_scan, CloudData& object_scan) {
    const auto pts = current_scan.cloud_ptr->points_;          // copy: current_scan is rewritten below
    const size_t n = pts.size();
    gi_.resize(n); oi_.resize(n); intensity_.resize(n); region_.resize(n);
    size_t ng = 0, no = 0;
    last_status_ = tloam_b200_ground_remove(h_, &cfg_, n ? reinterpret_cast<const double*>(pts.data()) : nullptr, n, gi_.data(), &ng,
                                            oi_.data(), &no, intensity_.data(), region_.data(), &height_threshold_, nullptr);
    if (last_status_ != TLOAM_B200_OK) {
      std::fprintf(stderr, "[tloam_b200] groundRemove: %s %s\n", tloam_b200_status_string(last_status_), tloam_b200_last_error(h_));
      return false;
    }
    for (size_t k = 0; k < ng; ++k) {
      const double c = intensity_[gi_[k]];
      ground_scan.cloud_ptr->points_.push_back(pts[gi_[k]]);
      ground_scan.cloud_ptr->intensity_.push_back(c - static_cast<int>(c));
    }
    for (size_t k = 0; k < no; ++k) {
      object_scan.cloud_ptr->points_.push_back(pts[oi_[k]]);
      object_scan.cloud_ptr->intensity_.push_back(intensity_[oi_[k]]);
    }
    current_scan.cloud_ptr->points_.clear();
    current_scan.cloud_ptr->intensity_.clear();
    for (size_t i = 0; i < n; ++i)
      if (region_[i] != 12) {                                   // 12 = above the height threshold (moved to non_ground_scan)
        current_scan.cloud_ptr->points_.push_back(pts[i]);
        current_scan.cloud_ptr->intensity_.push_back(intensity_[i]);
      }
    return true;
  }

  double heightThreshold() const { return height_threshold_; }
  int lastStatus() const { return last_status_; }
  tloam_b200_handle* handle() const { return h_; }
  const tloam_ground_config& config() const { return cfg_; }

 private:
  void attach(tloam_b200_handle* shared, int device) {
    if (shared) { h_ = shared; own_ = false; return; }
    tloam_tls_config c;
    tloam_b200_default_config(&c);
    const int rc = tloam_b200_create(&c, device, nullptr, &h_);
    if (rc != TLOAM_B200_OK) throw std::runtime_error(std::string("tloam_b200_create: ") + tloam_b200_status_string(rc));
    own_ = true;
  }
  tloam_ground_config cfg_;
  tloam_b200_handle* h_ = nullptr;
  bool own_ = false;
  int last_status_ = TLOAM_B200_OK;
  double height_threshold_ = 0.0;
  std::vector<size_t> gi_, oi_;
  std::vector<double> intensity_;
  std::vector<int> region_;
};

}  // namespace tloam
#endif
