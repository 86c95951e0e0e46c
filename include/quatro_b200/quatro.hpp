// quatro.hpp -- source-compatible replacement of the reference's include/quatro.hpp for the hot path:
//   voxelize<T>()                                        (reference include/quatro.hpp:49-68)
//   template<PS,PT,Scalar> class Quatro : pcl::Registration  (reference include/quatro.hpp:70-1061)
// implemented as thin callers of the C-ABI (include/quatro_b200.h).  Same names, argument meaning and
// error behaviour as the reference, so examples/run_global_registration.cpp:103-108,206-207,243-246,
// 290-292 compile unchanged against this header.  No computation happens on the host.
#pragma once

#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../quatro_b200.h"
#include "pcl_compat.hpp"

namespace qb200 {

struct HandleDeleter {
  void operator()(qb200_handle* h) const { qb200_destroy(h); }
};
using HandlePtr = std::unique_ptr<qb200_handle, HandleDeleter>;

constexpr int kDefaultRawPoints = 262144;  // the example's loader reads at most 250 k points (run_global_registration.cpp:384-388)
constexpr int kMaxCorr = QB200_MAX_CORR;    // qb200_config::max_corr limit

inline HandlePtr make_handle(int device = 0, int slots = 1, int max_voxel_points = 16384, int max_raw_points = kDefaultRawPoints,
                             int max_corr = 4096) {
  qb200_config cfg;
  qb200_default_config(&cfg);
  cfg.device = device;
  cfg.max_batch_slots = slots;
  cfg.max_voxel_points = max_voxel_points;
  cfg.max_raw_points = max_raw_points;
  cfg.max_corr = max_corr;
  qb200_handle* h = nullptr;
  const int st = qb200_create(&cfg, &h);
  if (st != QB200_OK) throw std::runtime_error("qb200_create failed (status " + std::to_string(st) + "): no usable CUDA device; there is no CPU fallback");
  return HandlePtr(h);
}

// One handle shared by the free functions / FPFHManager of a process, like the reference's
// function-local static filter and FPFH objects (quatro.hpp:53, fpfh_manager.hpp:110): not thread-safe.
struct SharedHandle {
  HandlePtr h;
  int raw_points = kDefaultRawPoints;  // capacities h was created with
  bool grown = false;                  // voxel / correspondence capacities at their maxima
};
inline SharedHandle& shared_state() {
  static SharedHandle s{make_handle()};
  return s;
}
inline qb200_handle* shared_handle() { return shared_state().h.get(); }
inline bool shared_handle_grown() { return shared_state().grown; }
// pcl::VoxelGrid / FLANN have no capacity: when a scan or a match overflows the handle's capacities, the shared handle is rebuilt
// with the largest ones (QB200_MAX_VOXEL_POINTS per cloud, QB200_MAX_CORR correspondences) instead of handing truncated data to the next
// stage.  max_raw_points grows to n_raw (rounded up to a multiple of 65536) when a scan holds more points than the handle takes.
inline qb200_handle* grow_shared_handle(size_t n_raw = 0) {
  SharedHandle& s = shared_state();
  if (n_raw > (size_t)s.raw_points) {
    const size_t r = (n_raw + 65535) / 65536 * 65536;
    if (r > (size_t)INT32_MAX) throw std::runtime_error("voxelize: scan of " + std::to_string(n_raw) + " points exceeds the device capacity");
    s.raw_points = (int)r;
  }
  s.h.reset();  // release the old workspaces before allocating the larger ones
  s.h = make_handle(0, 1, QB200_MAX_VOXEL_POINTS, s.raw_points, kMaxCorr);
  s.grown = true;
  return s.h.get();
}

template <class PointT>
inline const float* as_float4(const pcl::PointCloud<PointT>& c) {
  static_assert(sizeof(PointT) == 16, "point type must be a 16-byte xyz+pad record");
  return c.points.empty() ? nullptr : reinterpret_cast<const float*>(c.points.data());
}

}  // namespace qb200

// ---- voxelize (reference include/quatro.hpp:49-68) ---------------------------------------------------
// Pointer types are left generic so that boost::shared_ptr (PCL < 1.11) and std::shared_ptr clouds both bind.
template <typename T>
void voxelize_impl(const pcl::PointCloud<T>& src, pcl::PointCloud<T>& dst, double voxelSize) {
  qb200_handle* h = qb200::shared_handle();
  if (src.points.size() > (size_t)qb200::shared_state().raw_points) h = qb200::grow_shared_handle(src.points.size());
  std::vector<T> out(src.points.size());
  int32_t n_out = 0;
  // PCL's VoxelGrid keeps every finite point: flagged-point dropping (skip_flagged) is a batch-pipeline option only
  int st = qb200_voxelize(h, qb200::as_float4(src), (int32_t)src.points.size(), (float)voxelSize, 0,
                          out.empty() ? nullptr : reinterpret_cast<float*>(out.data()), (int32_t)out.size(), &n_out);
  if (st == QB200_CAPACITY_EXCEEDED && !qb200::shared_handle_grown()) {  // more occupied voxels than the handle holds: never return
    h = qb200::grow_shared_handle();                                      // the truncated (lowest-z) subset
    st = qb200_voxelize(h, qb200::as_float4(src), (int32_t)src.points.size(), (float)voxelSize, 0,
                        out.empty() ? nullptr : reinterpret_cast<float*>(out.data()), (int32_t)out.size(), &n_out);
  }
  if (st == QB200_CAPACITY_EXCEEDED)
    throw std::runtime_error("voxelize: more than " + std::to_string(QB200_MAX_VOXEL_POINTS) + " occupied voxels in one cloud exceed the device capacity");
  if (st < 0 && st != QB200_ERR_VOXEL_OVERFLOW) throw std::runtime_error(std::string("qb200_voxelize: ") + qb200_last_error(h));
  out.resize((size_t)n_out);
  dst.points.assign(out.begin(), out.end());
  dst.width = (unsigned)dst.points.size();
  dst.height = 1;
}
template <typename T, typename PtrOut>
void voxelize(pcl::PointCloud<T>& src, PtrOut dstPtr, double voxelSize) {
  voxelize_impl(src, *dstPtr, voxelSize);
}
template <typename PtrIn, typename PtrOut, typename = decltype(*std::declval<PtrIn>())>
void voxelize(const PtrIn srcPtr, PtrOut dstPtr, double voxelSize) {
  voxelize_impl(*srcPtr, *dstPtr, voxelSize);
}

// ---- Quatro (reference include/quatro.hpp:70-1061) -----------------------------------------------------
template <typename PointSource, typename PointTarget, typename Scalar = double>
class Quatro : public pcl::Registration<PointSource, PointTarget, Scalar> {
  using Base = pcl::Registration<PointSource, PointTarget, Scalar>;

 public:
  using PointCloudSource = typename Base::PointCloudSource;
  using PointCloudSourceConstPtr = typename PointCloudSource::ConstPtr;
  using PointCloudTarget = typename Base::PointCloudTarget;
  using PointCloudTargetConstPtr = typename PointCloudTarget::ConstPtr;
  using Matrix4 = typename Base::Matrix4;
  using Base::input_;
  using Base::reg_name_;
  using Base::target_;

  Quatro() : noise_bound_(0.3), handle_(qb200::make_handle()) { reg_name_ = "Quatro"; }
  Quatro(const Quatro&) = delete;
  Quatro(Quatro&&) = delete;
  Quatro& operator=(const Quatro&) = delete;
  Quatro& operator=(Quatro&&) = delete;
  ~Quatro() {}

  bool using_pre_estimated_RyRx_ = false;
  Eigen::Matrix3d estimated_RyRx_ = Eigen::Matrix3d::Identity();

  struct RegistrationSolution {
    bool valid = true;
    double scale = 1.0;
    Eigen::Vector3d translation{{0, 0, 0}};
    Eigen::Matrix3d rotation = Eigen::Matrix3d::Identity();
  };
  RegistrationSolution solution_;

  enum class ROTATION_ESTIMATION_ALGORITHM { GNC_TLS = 0, FGR = 1 };
  enum class INLIER_SELECTION_MODE { PMC_EXACT = 0, PMC_HEU = 1, KCORE_HEU = 2, NONE = 3 };
  enum class INLIER_GRAPH_FORMULATION { CHAIN = 0, COMPLETE = 1 };

  struct Params {  // field-for-field the reference's struct (quatro.hpp:202-268), same defaults
    std::string reg_name = "Quatro";
    std::string cote_mode = "median";
    bool using_rot_inliers_when_estimating_cote = false;
    double noise_bound = 0.3;
    double cbar2 = 1;
    bool estimate_scaling = true;  // ignored by the reference as well (scale is hard-wired to 1, quatro.hpp:361)
    ROTATION_ESTIMATION_ALGORITHM rotation_estimation_algorithm = ROTATION_ESTIMATION_ALGORITHM::GNC_TLS;
    double rotation_gnc_factor = 1.4;
    size_t rotation_max_iterations = 100;
    double rotation_cost_threshold = 1e-6;
    INLIER_GRAPH_FORMULATION rotation_tim_graph = INLIER_GRAPH_FORMULATION::CHAIN;
    INLIER_SELECTION_MODE inlier_selection_mode = INLIER_SELECTION_MODE::PMC_HEU;
    double kcore_heuristic_threshold = 0.5;
    bool use_max_clique = true;
    bool max_clique_exact_solution = true;
    double max_clique_time_limit = 3600;
  };
  double noise_bound_;  // translation (COTE) bound: ctor constant 0.3, independent of Params (quatro.hpp:115,601)
  double cost_ = 0.0;

  Params getParams() { return params_; }
  void setParams(Params params) { params_ = params; }

  void setPreEstaimatedRyRx(Eigen::Matrix4d& estimated_RyRx) {  // (sic) quatro.hpp:276-279
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) estimated_RyRx_(r, c) = estimated_RyRx(r, c);
    using_pre_estimated_RyRx_ = true;
  }

  void setInputSource(const PointCloudSourceConstPtr& cloud) override { Base::setInputSource(cloud); }
  void setInputTarget(const PointCloudTargetConstPtr& cloud) override {
    if (cloud->points.empty()) {  // quatro.hpp:298-302
      PCL_ERROR("[pcl::%s::setInputSource] Invalid or empty point cloud dataset given!\n", this->getClassName().c_str());
      return;
    }
    Base::setInputTarget(cloud);
  }

  void reset(const Params& params) {  // quatro.hpp:755-765
    reg_name_ = params.reg_name;
    params_ = params;
    max_clique_.clear();
    final_inliers_.clear();
    num_rot_inliers_ = num_maxclique_ = 0;
  }

  inline void setMaximumIterations(int nr_iterations) { this->max_iterations_ = nr_iterations; }

  // what pcl::Registration::align() would call: an empty override in the reference too (quatro.hpp:767)
  void computeTransformation(PointCloudSource&, const Matrix4&) override {}

  // the real entry point (quatro.hpp:769-936)
  void computeTransformation(Eigen::Matrix4d& output) {
    if (!input_ || !target_) throw std::invalid_argument("[Quatro] input source / target not set");
    if (input_->points.size() != target_->points.size())
      throw std::invalid_argument("[Quatro] source and target must hold the same number of matched points");
    if (reg_name_ != "Quatro") throw std::invalid_argument("[solveForRotation] The param is wrong! It should be 'TEASER' or 'Quatro'");
    if (params_.cote_mode != "median" && params_.cote_mode != "weighted_mean") throw std::invalid_argument("[COTE]: Wrong parameter comes!");
    qb200_params p = to_c_params();
    const int32_t L = (int32_t)input_->points.size();
    src_matched_ = input_->points;
    tgt_matched_ = target_->points;
    if (L > handle_corr_ && L <= qb200::kMaxCorr) {  // a larger matched set than the handle holds: rebuild it once
      handle_.reset();
      handle_ = qb200::make_handle(0, 1, 16384, qb200::kDefaultRawPoints, qb200::kMaxCorr);
      handle_corr_ = qb200::kMaxCorr;
    }
    qb200_result res;
    const int st = qb200_solve_correspondences(handle_.get(), qb200::as_float4(*input_), qb200::as_float4(*target_), L, &p, &res);
    if (st < 0) throw std::runtime_error(std::string("qb200_solve_correspondences: ") + qb200_last_error(handle_.get()));
    fetch_ints(&qb200_get_last_clique, max_clique_);
    num_maxclique_ = res.clique_size;
    if (!res.valid) {  // clique size <= 1: solution invalid, output left untouched (quatro.hpp:809-813)
      solution_.valid = false;
      return;
    }
    // the reference doubles params_.noise_bound on every call (quatro.hpp:850-852); reset() restores it
    params_.noise_bound *= (2 / solution_.scale);
    fetch_ints(&qb200_get_last_final_inliers, final_inliers_);
    num_rot_inliers_ = res.n_rot_inliers;
    cost_ = res.cost;
    solution_.valid = true;
    solution_.scale = 1.0;
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) solution_.rotation(r, c) = res.T[4 * c + r];
      solution_.translation(r) = res.T[12 + r];
    }
    std::memcpy(output.data(), res.T, sizeof(res.T));
  }

  void getMaxCliques(pcl::PointCloud<PointType>& source_max_clique, pcl::PointCloud<PointType>& target_max_clique) {
    set_inliers(src_matched_, source_max_clique, max_clique_);
    set_inliers(tgt_matched_, target_max_clique, max_clique_);
  }
  void getFinalInliers(pcl::PointCloud<PointType>& source_inliers, pcl::PointCloud<PointType>& target_inliers) {
    set_inliers(src_matched_, source_inliers, final_inliers_);
    set_inliers(tgt_matched_, target_inliers, final_inliers_);
  }
  std::vector<int> getFinalInliersIndices() { return final_inliers_; }
  int getNumRotaionInliers() { return num_rot_inliers_; }  // (sic)
  int getNumMaxCliqueInliers() { return num_maxclique_; }

 private:
  qb200_params to_c_params() const {
    qb200_params p;
    qb200_default_params(&p);
    p.noise_bound = params_.noise_bound;
    p.cbar2 = params_.cbar2;
    p.rotation_gnc_factor = params_.rotation_gnc_factor;
    p.rotation_max_iterations = (int32_t)params_.rotation_max_iterations;
    p.rotation_cost_threshold = params_.rotation_cost_threshold;
    p.kcore_heuristic_threshold = params_.kcore_heuristic_threshold;
    p.inlier_selection_mode = (int32_t)params_.inlier_selection_mode;
    p.cote_mode = params_.cote_mode == "median" ? QB200_COTE_MEDIAN : QB200_COTE_WEIGHTED_MEAN;
    p.using_rot_inliers_when_estimating_cote = params_.using_rot_inliers_when_estimating_cote ? 1 : 0;
    p.cote_noise_bound = noise_bound_;
    // function-local static of the reference (quatro.hpp:469-470): latched once per process and template
    // instantiation at the first solve, = params_.noise_bound after its doubling
    static double rot_noise_bound = 2.0 * params_.noise_bound;
    p.rot_noise_bound = rot_noise_bound;
    p.use_pre_estimated_RyRx = using_pre_estimated_RyRx_ ? 1 : 0;
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) p.RyRx[3 * r + c] = estimated_RyRx_(r, c);
    return p;
  }
  template <class F>
  void fetch_ints(F getter, std::vector<int>& out) {
    int32_t n = 0;
    out.assign(input_ ? input_->points.size() : 0, 0);
    getter(handle_.get(), out.empty() ? nullptr : out.data(), (int32_t)out.size(), &n);
    out.resize((size_t)n);
  }
  static void set_inliers(const std::vector<PointSource>& raw, pcl::PointCloud<PointType>& inliers, const std::vector<int>& idx) {
    inliers.clear();
    inliers.reserve(idx.size());
    for (const int i : idx) inliers.push_back(PointType(raw[i].x, raw[i].y, raw[i].z));
  }

  Params params_;
  qb200::HandlePtr handle_;
  int handle_corr_ = 4096;  // max_corr of handle_
  int num_rot_inliers_ = 0, num_maxclique_ = 0;
  std::vector<int> max_clique_, final_inliers_;
  std::vector<PointSource> src_matched_, tgt_matched_;
};
