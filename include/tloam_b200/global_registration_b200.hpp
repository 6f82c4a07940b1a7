// global_registration_b200.hpp -- C++ shim: tloam::GlobalRegistrationB200, a RegistrationInterface
// (ref: include/tloam/models/registration/registration_interface.hpp:40-48) that aligns two scans with no initial guess on
// the C ABI of libtloam_b200.so (include/tloam_b200.h "Global registration").  It fills the place of the reference's
// GlobalRegistration (ref: registration.hpp:368), whose scanMatching is a stub (ref: registration.cpp:1135-1161).
// Header-only; from the host side it needs only Frame::scan_cloud->points_ (contiguous std::vector<Eigen::Vector3d>) and
// Eigen::Isometry3d::matrix().data().
//
//     GlobalRegistrationB200 global;                   // its own handle, default configuration
//     global.setInputSource(current);                  // scan_cloud of each frame, in its sensor's frame
//     global.setInputTarget(candidate);
//     global.scanMatching(current, ignored, T);         // T: target <- source; the guess for LocalRegistrationB200 or
//     auto fs = global.getFitnessScore();               //    verifyLoop; fs = (fitness, inlier rmse); accepted() says
//                                                       //    whether T passed min_inliers and min_fitness
// Without the reference headers (this repository's tests) define TLOAM_B200_MOCK_HOST_TYPES and provide the host types
// (tests/mock/mock_tloam.hpp).
#ifndef TLOAM_B200_GLOBAL_REGISTRATION_B200_HPP
#define TLOAM_B200_GLOBAL_REGISTRATION_B200_HPP

#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../tloam_b200.h"

#ifndef TLOAM_B200_MOCK_HOST_TYPES
#include "tloam/models/registration/registration_interface.hpp"
#endif

namespace tloam {

class GlobalRegistrationB200 : public RegistrationInterface {
 public:
  explicit GlobalRegistrationB200(int device = 0, void* stream = nullptr) {
    tloam_global_registration_config c;
    tloam_b200_global_registration_default_config(&c);
    create(c, device, stream);
  }
  explicit GlobalRegistrationB200(const tloam_global_registration_config& cfg, int device = 0, void* stream = nullptr) {
    create(cfg, device, stream);
  }
  ~GlobalRegistrationB200() override { tloam_b200_destroy(h_); }
  GlobalRegistrationB200(const GlobalRegistrationB200&) = delete;
  GlobalRegistrationB200& operator=(const GlobalRegistrationB200&) = delete;

  // the scan clouds are copied on the host; the registration runs in scanMatching
  bool setInputSource(Frame& f) override { return keep(f, source_); }
  bool setInputTarget(Frame& f) override { return keep(f, target_); }

  // there is no prediction to use: predict_pose_ is ignored.  result_pose_ = T (target <- source); false on an error
  // status (an empty side is not an error: T = I, termination EMPTY, not accepted)
  bool scanMatching(Frame&, Eigen::Isometry3d&, Eigen::Isometry3d& result_pose_) override {
    const double* s = source_.empty() ? nullptr : source_.data();
    const double* t = target_.empty() ? nullptr : target_.data();
    if (!report(tloam_b200_global_register(h_, s, source_.size() / 3, t, target_.size() / 3, &result_), "scanMatching")) return false;
    for (int i = 0; i < 16; ++i) result_pose_.matrix().data()[i] = result_.T[i];
    return true;
  }

  // (fitness, inlier rmse) of the last scanMatching: the fraction of source keypoints with a target keypoint within
  // max_correspondence_distance under T, and the rmse of the final inliers
  std::pair<double, double> getFitnessScore() override { return std::make_pair(result_.fitness, result_.inlier_rmse); }

  bool accepted() const { return result_.accepted != 0; }
  const tloam_global_registration_result& result() const { return result_; }
  int lastStatus() const { return last_status_; }
  tloam_b200_handle* handle() { return h_; }

 private:
  void create(const tloam_global_registration_config& cfg, int device, void* stream) {
    tloam_tls_config tls;
    tloam_b200_default_config(&tls);
    int rc = tloam_b200_create(&tls, device, stream, &h_);
    if (rc != TLOAM_B200_OK) throw std::runtime_error(std::string("tloam_b200_create: ") + tloam_b200_status_string(rc));
    rc = tloam_b200_global_registration_enable(h_, &cfg);
    if (rc != TLOAM_B200_OK) {
      const std::string why = std::string("tloam_b200_global_registration_enable: ") + tloam_b200_status_string(rc) + " " +
                              tloam_b200_last_error(h_);
      tloam_b200_destroy(h_);
      h_ = nullptr;
      throw std::runtime_error(why);
    }
    std::memset(&result_, 0, sizeof(result_));
    result_.T[0] = result_.T[5] = result_.T[10] = result_.T[15] = 1.0;
    result_.best_hypothesis = -1;
    result_.termination = TLOAM_GLOBAL_REGISTRATION_EMPTY;
  }
  static bool keep(Frame& f, std::vector<double>& out) {
    out.clear();
    if (f.scan_cloud && !f.scan_cloud->points_.empty()) {
      const double* p = reinterpret_cast<const double*>(f.scan_cloud->points_.data());
      out.assign(p, p + 3 * f.scan_cloud->points_.size());
    }
    return true;
  }
  bool report(int rc, const char* where) {
    last_status_ = rc;
    if (rc != TLOAM_B200_OK)
      std::fprintf(stderr, "[tloam_b200] %s: %s %s\n", where, tloam_b200_status_string(rc), tloam_b200_last_error(h_));
    return rc == TLOAM_B200_OK;
  }
  tloam_b200_handle* h_ = nullptr;
  std::vector<double> source_, target_;
  tloam_global_registration_result result_;
  int last_status_ = TLOAM_B200_OK;
};

}  // namespace tloam
#endif
