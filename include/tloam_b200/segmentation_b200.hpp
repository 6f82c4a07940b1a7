// segmentation_b200.hpp -- C++ shim: tloam::SegmentationB200, the device replacement of the three compute steps of the
// segmentation nodelet's spinOnce (ref: src/models/segmentation/segmentation.cpp:47-66):
//     groundRemove()                                            -> GroundExtractB200::groundRemove      (:738-770)
//     objectSegmentation()                                      -> SegmentationB200::objectSegmentation (:1085-1112)
//     extractEdgePoint(segmented_scan, edge_scan, general_scan) -> SegmentationB200::extractEdgePoint   (:1211-1304)
// implemented on the C ABI of libtloam_b200.so ("next" row 8(f)-4).  Header-only; from the host side it needs only
// CloudData::cloud_ptr->points_ / intensity_ (ref: include/tloam/models/utils/sensor_data.hpp:17-43).
//
// In the reference tree the three member functions become one-line forwards, e.g.
//     bool Segmentation::objectSegmentation() { return seg_b200_->objectSegmentation(object_scan, segmented_scan, &boxes_); }
// (publishing jsk BoundingBox messages from `boxes_` stays on the host: it is ROS, out of scope here).
// Without the reference headers (this repository's tests) define TLOAM_B200_MOCK_HOST_TYPES (tests/mock/mock_tloam.hpp).
#ifndef TLOAM_B200_SEGMENTATION_B200_HPP
#define TLOAM_B200_SEGMENTATION_B200_HPP

#include "ground_extract_b200.hpp"

namespace tloam {

struct BoxB200 {                 // what colorSegmentation puts into a jsk BoundingBox (:1058-1073)
  int label;                     // 1-based position in labelRecords
  double position[3];            // centre
  double dimensions[3];
  int points;                    // cluster size
};

class SegmentationB200 {
 public:
  SegmentationB200(const tloam_ground_config& ground, const tloam_dcvc_config& dcvc, int ring_min_num, tloam_b200_handle* shared = nullptr,
                   int device = 0)
      : ground_(ground, shared, device), dcvc_(dcvc), sensor_model_(ground.sensor_model), ring_min_num_(ring_min_num) {
    h_ = ground_.handle();
  }

#ifndef TLOAM_B200_MOCK_HOST_TYPES
  // Reads the keys Segmentation::initWithConfig reads (ref: segmentation.cpp:95-141; config/mapping/segmentation.yaml).
  explicit SegmentationB200(const YAML::Node& config_node, tloam_b200_handle* shared = nullptr, int device = 0)
      : ground_(config_node["velodyne"], config_node["groundSeg"], shared, device) {
    tloam_b200_dcvc_default_config(&dcvc_);
    dcvc_.start_r = config_node["DCVC"]["startR"].as<double>();
    dcvc_.delta_r = config_node["DCVC"]["deltaR"].as<double>();
    dcvc_.delta_p = config_node["DCVC"]["deltaP"].as<double>();
    dcvc_.delta_a = config_node["DCVC"]["deltaA"].as<double>();
    dcvc_.min_seg = config_node["DCVC"]["minSeg"].as<int>();
    dcvc_.sensor_min_range = config_node["velodyne"]["sensorMinRange"].as<double>();
    dcvc_.sensor_max_range = config_node["velodyne"]["sensorMaxRange"].as<double>();
    dcvc_.min_polar_init = dcvc_.max_polar_init = 5.0;        // the members' initial values (segmentation.hpp:332-333), first frame only
    sensor_model_ = config_node["velodyne"]["sensorModel"].as<int>();
    near_dis_ = config_node["velodyne"]["near_dis"].as<double>();
    ring_min_num_ = config_node["groundSeg"]["ringMinNum"].as<int>();
    h_ = ground_.handle();
  }
#endif

  bool groundRemove(CloudData& current_scan, CloudData& ground_scan, CloudData& object_scan) {
    return ground_.groundRemove(current_scan, ground_scan, object_scan);
  }

  // ref: :1085-1112.  segmented_scan receives (emplace_back, like colorSegmentation) the points of every class with more
  // than minSeg points, class after class; boxes (optional) one entry per class.
  bool objectSegmentation(const CloudData& object_scan, CloudData& segmented_scan, std::vector<BoxB200>* boxes = nullptr) {
    const auto& pts = object_scan.cloud_ptr->points_;
    const auto& inten = object_scan.cloud_ptr->intensity_;
    const size_t n = pts.size();
    if (n == 0) { std::fprintf(stderr, "[tloam_b200] objectSegmentation: not enough point to convert\n"); return false; }   // :1092-1093
    seg_.resize(n); sizes_.resize(n); boxes_.resize(6 * n);
    size_t ns = 0;
    int nc = 0;
    last_status_ = tloam_b200_object_segmentation(h_, &dcvc_, reinterpret_cast<const double*>(pts.data()), n, seg_.data(), &ns, &nc,
                                                  sizes_.data(), boxes_.data(), nullptr, nullptr, nullptr, nullptr);
    if (last_status_ != TLOAM_B200_OK) {
      std::fprintf(stderr, "[tloam_b200] objectSegmentation: %s %s\n", tloam_b200_status_string(last_status_), tloam_b200_last_error(h_));
      return false;
    }
    for (size_t k = 0; k < ns; ++k) {
      segmented_scan.cloud_ptr->points_.push_back(pts[seg_[k]]);
      segmented_scan.cloud_ptr->intensity_.push_back(seg_[k] < inten.size() ? inten[seg_[k]] : 0.0);
    }
    if (boxes)
      for (int c = 0; c < nc; ++c) {
        BoxB200 b;
        b.label = c + 1; b.points = sizes_[c];
        for (int d = 0; d < 3; ++d) { b.position[d] = boxes_[6 * c + d]; b.dimensions[d] = boxes_[6 * c + 3 + d]; }
        boxes->push_back(b);
      }
    dcvc_.min_polar_init = dcvc_.max_polar_init = 0.0;         // resetParams() (:1121-1123) leaves zeros for the next frame
    dcvc_.min_pitch_init = dcvc_.max_pitch_init = 0.0;
    return true;
  }

  // ref: :1211-1304.  cloud_in: points whose intensity is the beam id.  Returns false on an empty input like the reference.
  bool extractEdgePoint(const CloudData& cloud_in, CloudData& out_edge_point, CloudData& non_edge_point) {
    const auto& pts = cloud_in.cloud_ptr->points_;
    const auto& inten = cloud_in.cloud_ptr->intensity_;
    const size_t n = pts.size();
    if (n == 0 || inten.size() != n) { std::fprintf(stderr, "[tloam_b200] extractEdgePoint: not enough points.\n"); return false; }
    edge_.resize(n); non_.resize(n);
    size_t ne = 0, nn = 0;
    last_status_ = tloam_b200_extract_edge(h_, sensor_model_, ring_min_num_, reinterpret_cast<const double*>(pts.data()), inten.data(), n,
                                           edge_.data(), &ne, non_.data(), &nn);
    if (last_status_ != TLOAM_B200_OK) {
      std::fprintf(stderr, "[tloam_b200] extractEdgePoint: %s %s\n", tloam_b200_status_string(last_status_), tloam_b200_last_error(h_));
      return false;
    }
    for (size_t k = 0; k < ne; ++k) {
      out_edge_point.cloud_ptr->points_.push_back(pts[edge_[k]]);
      out_edge_point.cloud_ptr->intensity_.push_back(inten[edge_[k]]);
    }
    for (size_t k = 0; k < nn; ++k) {
      non_edge_point.cloud_ptr->points_.push_back(pts[non_[k]]);
      non_edge_point.cloud_ptr->intensity_.push_back(inten[non_[k]]);
    }
    return true;
  }

  // The three steps above as ONE device pass: the scan crosses PCIe once.  ground_scan / edge_scan / general_scan receive
  // the points the three separate calls would have produced (same order, same intensities: the fractional part of the
  // channel for ground points, the channel for the others); `scan` (finite points) is left untouched.
  bool segmentScan(const CloudData& scan, CloudData& ground_scan, CloudData& edge_scan, CloudData& general_scan,
                   std::vector<BoxB200>* boxes = nullptr) {
    return chain(scan, 0.0, ground_scan, edge_scan, general_scan, boxes);   // near_dis 0 keeps every finite point
  }

  // Segmentation::spinOnce's compute steps (:48-66) in one device pass: RemoveClosedNonFinitePoints(near_dis) -- every
  // point without NaN / Inf and with a norm >= near_dis * near_dis survives, as in the reference -- then segmentScan.
  // raw_scan: the scan as the driver delivers it; it is left untouched (the reference compacts current_scan in place).
  bool segmentRawScan(const CloudData& raw_scan, CloudData& ground_scan, CloudData& edge_scan, CloudData& general_scan,
                      std::vector<BoxB200>* boxes = nullptr) {
    return chain(raw_scan, near_dis_, ground_scan, edge_scan, general_scan, boxes);
  }

  double nearDis() const { return near_dis_; }
  void setNearDis(double d) { near_dis_ = d; }
  int lastStatus() const { return last_status_; }
  tloam_b200_handle* handle() const { return h_; }

 private:
  bool chain(const CloudData& scan, double near_dis, CloudData& ground_scan, CloudData& edge_scan, CloudData& general_scan,
             std::vector<BoxB200>* boxes) {
    const auto& pts = scan.cloud_ptr->points_;
    const size_t n = pts.size();
    if (n == 0) return false;
    seg_.resize(n); edge_.resize(n); non_.resize(n); sizes_.resize(n); boxes_.resize(6 * n); intensity_.resize(n);
    size_t ng = 0, ne = 0, nn = 0;
    int nc = 0;
    last_status_ = tloam_b200_segment_raw_scan(h_, &ground_.config(), &dcvc_, ring_min_num_, near_dis, reinterpret_cast<const double*>(pts.data()),
                                               n, seg_.data(), &ng, edge_.data(), &ne, non_.data(), &nn, &nc, sizes_.data(), boxes_.data(),
                                               intensity_.data());
    if (last_status_ != TLOAM_B200_OK) {
      std::fprintf(stderr, "[tloam_b200] segmentScan: %s %s\n", tloam_b200_status_string(last_status_), tloam_b200_last_error(h_));
      return false;
    }
    auto append = [&](CloudData& out, const std::vector<size_t>& idx, size_t cnt, bool ground) {
      for (size_t k = 0; k < cnt; ++k) {
        const double c = intensity_[idx[k]];
        out.cloud_ptr->points_.push_back(pts[idx[k]]);
        out.cloud_ptr->intensity_.push_back(ground ? c - static_cast<int>(c) : c);   // ground: :692-693
      }
    };
    append(ground_scan, seg_, ng, true);
    append(edge_scan, edge_, ne, false);
    append(general_scan, non_, nn, false);
    if (boxes)
      for (int c = 0; c < nc; ++c) {
        BoxB200 b;
        b.label = c + 1; b.points = sizes_[c];
        for (int d = 0; d < 3; ++d) { b.position[d] = boxes_[6 * c + d]; b.dimensions[d] = boxes_[6 * c + 3 + d]; }
        boxes->push_back(b);
      }
    dcvc_.min_polar_init = dcvc_.max_polar_init = 0.0;         // resetParams() (:1121-1123)
    dcvc_.min_pitch_init = dcvc_.max_pitch_init = 0.0;
    return true;
  }

  GroundExtractB200 ground_;
  tloam_dcvc_config dcvc_;
  int sensor_model_ = 64, ring_min_num_ = 131;
  double near_dis_ = 3.0;                                      // velodyne.near_dis (config/mapping/segmentation.yaml)
  tloam_b200_handle* h_ = nullptr;
  int last_status_ = TLOAM_B200_OK;
  std::vector<size_t> seg_, edge_, non_;
  std::vector<int> sizes_;
  std::vector<double> boxes_, intensity_;
};

}  // namespace tloam
#endif
