// fpfh_manager.hpp -- source-compatible replacement of the reference's include/fpfh_manager.hpp:
// normals + FPFH-33 for both clouds, mutual-NN matching with the tuple test, packing of the matched
// pairs -- one C-ABI call (qb200_match_and_pack) -- plus the descriptor / normal getters (:161-177), the odometry
// mode that reuses the previous target as the next source (swapTgt2Src, :74-77, :111-118) and the matched-pair PCD
// cache (save/loadFeaturePair, :179-232).  No computation happens on the host.
#pragma once

#include <algorithm>
#include <cstdio>
#include <iostream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "quatro.hpp"

class FPFHManager {
 public:
  std::vector<std::pair<int, int>> corr;
  Eigen::Matrix3Xd src_matched, tgt_matched;
  Eigen::Matrix3Xd src_normals, tgt_normals;  // src_normals: "not in use" in the reference as well
  pcl::PointCloud<PointType> src_matched_pcl, tgt_matched_pcl;

  FPFHManager(double normal_radius, double fpfh_radius, int interval = 1)
      : normal_radius_(normal_radius), fpfh_radius_(fpfh_radius), interval_(interval) {}
  FPFHManager() {}

  void flushAllFeatures() { is_initial_ = true; }
  // fpfh_manager.hpp:74-77: the previous target becomes the source.  The descriptors of a cloud are a pure function of the cloud,
  // so handing the kept target cloud to the device again reproduces the reference's reuse exactly; pipelines that start from raw
  // scans keep the descriptors resident on the device instead (qb200_cache_scans / qb200_register_cached).
  void swapTgt2Src() {
    src_cloud_ = tgt_cloud_;
    obj_descriptors_ = scene_descriptors_;
  }
  void setOdometryTest(bool on) { is_odometry_test_ = on; }  // the reference's is_odometry_test_ flag (:36), which it never sets
  void setParams(float normal_radius, float fpfh_radius, int interval) {
    normal_radius_ = normal_radius; fpfh_radius_ = fpfh_radius; interval_ = interval;
  }
  void clearInputs() {
    is_initial_ = true;
    corr.clear();
    src_cloud_.clear(); tgt_cloud_.clear();
    obj_descriptors_.clear(); scene_descriptors_.clear();
  }
  void setLoadDir(std::string loaddir) { loaddir_ = loaddir; }
  void setSaveDir(std::string savedir) { savedir_ = savedir; }
  // lattice cell of the neighbour search (only fixes the accumulation order); 0 = library default ((1 + 2^-9) fpfh_radius)
  void setGridCell(float cell) { grid_cell_ = cell; }
  void setSeed(uint64_t seed) { seed_ = seed; }  // tuple-test RNG (the reference seeds with time(NULL))

  void setFeaturePair(pcl::PointCloud<PointType>::Ptr src, pcl::PointCloud<PointType>::Ptr target) {
    if (normal_radius_ > fpfh_radius_) {  // fpfh_manager.hpp:99-102
      std::cout << normal_radius_ << " <-> " << fpfh_radius_ << std::endl;
      throw std::invalid_argument("[FPFHManager]: Normal should be lower than fpfh_radius!!!!");
    }
    if (is_initial_ && !is_odometry_test_) {
      src_cloud_ = *src;
      is_initial_ = false;
    } else {
      swapTgt2Src();  // to reduce computational cost on odometry test (fpfh_manager.hpp:115-118): the given src is ignored
    }
    tgt_cloud_ = *target;
    qb200_params p;
    qb200_default_params(&p);
    p.normal_radius = (float)normal_radius_;
    p.fpfh_radius = (float)fpfh_radius_;
    p.grid_cell = grid_cell_;
    p.seed = seed_;
    const int32_t ns = (int32_t)src_cloud_.points.size(), nt = (int32_t)tgt_cloud_.points.size();
    const int32_t cap = std::min(ns, nt);
    std::vector<int32_t> c(2 * (size_t)std::max(cap, 1));
    std::vector<PointType> sm((size_t)std::max(cap, 1)), tm((size_t)std::max(cap, 1));
    int32_t n = 0;
    qb200_handle* h = qb200::shared_handle();
    int st = qb200_match_and_pack(h, qb200::as_float4(src_cloud_), ns, qb200::as_float4(tgt_cloud_), nt, &p, c.data(),
                                  reinterpret_cast<float*>(sm.data()), reinterpret_cast<float*>(tm.data()), cap, &n);
    // a cloud beyond the default voxel capacity, or more correspondences than the default max_corr: grow once, never truncate
    if (!qb200::shared_handle_grown() && ((st == QB200_ERR_BAD_ARG && (ns > 16384 || nt > 16384)) || st == QB200_CAPACITY_EXCEEDED)) {
      h = qb200::grow_shared_handle();
      st = qb200_match_and_pack(h, qb200::as_float4(src_cloud_), ns, qb200::as_float4(tgt_cloud_), nt, &p, c.data(),
                                reinterpret_cast<float*>(sm.data()), reinterpret_cast<float*>(tm.data()), cap, &n);
    }
    if (st == QB200_CAPACITY_EXCEEDED) throw std::runtime_error("[FPFHManager]: more correspondences than the device capacity (max_corr)");
    if (st < 0) throw std::runtime_error(std::string("qb200_match_and_pack: ") + qb200_last_error(h));
    // descriptors and normals stay on the device until asked for; fetch them once per pair like the reference keeps them
    fetch_features(h, 0, ns, obj_descriptors_, nullptr);
    std::vector<pcl::Normal> tgt_normals_raw;
    fetch_features(h, 1, nt, scene_descriptors_, &tgt_normals_raw);
    corr.resize((size_t)n);
    src_matched.resize(3, n);
    tgt_matched.resize(3, n);
    tgt_normals.resize(3, n);
    src_matched_pcl.clear();
    tgt_matched_pcl.clear();
    for (int i = 0; i < n; ++i) {
      corr[i] = {c[2 * i], c[2 * i + 1]};
      src_matched(0, i) = sm[i].x; src_matched(1, i) = sm[i].y; src_matched(2, i) = sm[i].z;
      tgt_matched(0, i) = tm[i].x; tgt_matched(1, i) = tm[i].y; tgt_matched(2, i) = tm[i].z;
      const pcl::Normal& nn = tgt_normals_raw[(size_t)c[2 * i + 1]];
      tgt_normals(0, i) = (double)nn.normal_x; tgt_normals(1, i) = (double)nn.normal_y; tgt_normals(2, i) = (double)nn.normal_z;
      src_matched_pcl.push_back(PointType(sm[i].x, sm[i].y, sm[i].z));
      tgt_matched_pcl.push_back(PointType(tm[i].x, tm[i].y, tm[i].z));
    }
  }
  Eigen::Matrix3Xd getSrcMatched() { return src_matched; }
  Eigen::Matrix3Xd getTgtMatched() { return tgt_matched; }
  Eigen::Matrix3Xd getTgtNormals() { return tgt_normals; }
  pcl::PointCloud<pcl::FPFHSignature33> getObjDescriptor() { return obj_descriptors_; }
  pcl::PointCloud<pcl::FPFHSignature33> getSceneDescriptor() { return scene_descriptors_; }
  pcl::PointCloud<PointType> getSrcKps() { return src_matched_pcl; }
  pcl::PointCloud<PointType> getTgtKps() { return tgt_matched_pcl; }
  std::vector<std::pair<int, int>> getCorrespondences() { return corr; }

  // matched-pair cache: "<dir>/%06d_to_%06d.pcd", the source half first (fpfh_manager.hpp:179-232)
  void saveFeaturePair(int src_idx, int tgt_idx, bool verbose = false) {
    if (savedir_.empty()) throw std::invalid_argument("Save dir. is not set");
    const std::string pcdname = pair_file(savedir_, src_idx, tgt_idx);
    if (verbose) {
      std::cout << "[SAVER]: " << pcdname << std::endl;
      std::cout << src_matched_pcl.points.size() << " + " << tgt_matched_pcl.points.size() << std::endl;
    }
    if (pcl::io::savePCDFile(pcdname, src_matched_pcl + tgt_matched_pcl) != 0) throw std::runtime_error("[FPFHManager]: cannot write " + pcdname);
  }
  void loadFeaturePair(int src_idx, int tgt_idx, bool verbose = false) {
    if (loaddir_.empty()) throw std::invalid_argument("Load dir. is not set");
    const std::string pcdname = pair_file(loaddir_, src_idx, tgt_idx);
    pcl::PointCloud<PointType> merge;
    if (pcl::io::loadPCDFile(pcdname, merge) == -1) throw std::invalid_argument("[FPFHManager]: Load feature set failed.");
    if (verbose) std::cout << "[LOADER]: Loaded data from " << pcdname << "..." << std::endl << merge.points.size();
    src_matched_pcl.clear();
    tgt_matched_pcl.clear();
    const size_t half = merge.points.size() / 2;
    for (size_t i = 0; i < merge.points.size(); ++i) (i < half ? src_matched_pcl : tgt_matched_pcl).push_back(merge.points[i]);
    if (verbose) std::cout << "=>" << src_matched_pcl.points.size() << " " << tgt_matched_pcl.points.size() << std::endl;
  }

 private:
  static std::string pair_file(const std::string& dir, int a, int b) {
    char name[64];
    std::snprintf(name, sizeof(name), "/%06d_to_%06d.pcd", a, b);
    return dir + name;
  }
  static void fetch_features(qb200_handle* h, int which, int32_t n_points, pcl::PointCloud<pcl::FPFHSignature33>& desc, std::vector<pcl::Normal>* normals) {
    desc.clear();
    desc.resize((size_t)n_points);
    if (normals) normals->assign((size_t)n_points, pcl::Normal());
    if (n_points == 0) return;
    int32_t n = 0;
    const int st = qb200_get_last_features(h, which, normals ? reinterpret_cast<float*>(normals->data()) : nullptr,
                                           reinterpret_cast<float*>(desc.points.data()), n_points, &n);
    if (st < 0 || n != n_points) throw std::runtime_error(std::string("qb200_get_last_features: ") + qb200_last_error(h));
  }

  double normal_radius_ = 0.5, fpfh_radius_ = 0.75;
  int interval_ = 1;
  float grid_cell_ = 0.f;
  uint64_t seed_ = 0x5EED;
  bool is_initial_ = true, is_odometry_test_ = false;
  std::string savedir_, loaddir_;
  pcl::PointCloud<PointType> src_cloud_, tgt_cloud_;
  pcl::PointCloud<pcl::FPFHSignature33> obj_descriptors_, scene_descriptors_;
};
