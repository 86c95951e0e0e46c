// The example's step after computeTransformation (examples/run_global_registration.cpp:253-288) on the host, through
// pcl_compat.hpp's transformPointCloud: the source keypoints transformed, the matched ones in correspondence order, and the good-match
// loop, with pow(d, 2) written d * d (the convention qb200_align_batch_each documents).
//   align_example in.bin out.bin
// in.bin:  int32 n_src, n_tgt, n_corr; float64 T[16] (column-major); float64 voxel_size; float32 src[n_src][3], tgt[n_tgt][3];
//          int32 corr[n_corr][2]
// out.bin: float32 transformed_src[n_src][3]; float32 matched[n_corr][3]; int32 n_good; int32 good_ids[n_good];
//          float32 good_matched[n_good][3]
#include <math.h>
#include <stdint.h>

#include <fstream>
#include <iostream>
#include <vector>

#include "quatro_b200/pcl_compat.hpp"

template <class T>
static void get(std::ifstream& in, T* v, size_t n) {
  in.read(reinterpret_cast<char*>(v), (std::streamsize)(n * sizeof(T)));
}

template <class T>
static void put(std::ofstream& out, const T* v, size_t n) {
  out.write(reinterpret_cast<const char*>(v), (std::streamsize)(n * sizeof(T)));
}

static void put_xyz(std::ofstream& out, const pcl::PointXYZ& p) {
  const float v[3] = {p.x, p.y, p.z};
  put(out, v, 3);
}

int main(int argc, char** argv) {
  if (argc != 3) {
    std::cerr << "usage: align_example in.bin out.bin" << std::endl;
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  int32_t n[3];
  get(in, n, 3);
  Eigen::Matrix4d T;
  get(in, T.data(), 16);
  double voxel_size;
  get(in, &voxel_size, 1);
  pcl::PointCloud<pcl::PointXYZ> srcFeat, tgtFeat;
  for (int side = 0; side < 2; ++side) {
    for (int32_t i = 0; i < n[side]; ++i) {
      float v[3];
      get(in, v, 3);
      (side ? tgtFeat : srcFeat).push_back(pcl::PointXYZ(v[0], v[1], v[2]));
    }
  }
  std::vector<int32_t> corr(2 * (size_t)n[2]);
  get(in, corr.data(), corr.size());
  if (!in) {
    std::cerr << "short input" << std::endl;
    return 1;
  }

  pcl::PointCloud<pcl::PointXYZ> srcMatched;
  for (int32_t k = 0; k < n[2]; ++k) srcMatched.push_back(srcFeat[corr[2 * k]]);
  pcl::PointCloud<pcl::PointXYZ> transformed_srcMatched, transformed_src, good_matched_pcl;
  pcl::transformPointCloud(srcMatched, transformed_srcMatched, T);
  pcl::transformPointCloud(srcFeat, transformed_src, T);
  std::vector<int32_t> good_ids;
  for (int32_t k = 0; k < n[2]; ++k) {
    const int src_idx = corr[2 * k], dst_idx = corr[2 * k + 1];
    const double dx = double(transformed_src[src_idx].x) - double(tgtFeat.points[dst_idx].x);
    const double dy = double(transformed_src[src_idx].y) - double(tgtFeat.points[dst_idx].y);
    const double dz = double(transformed_src[src_idx].z) - double(tgtFeat.points[dst_idx].z);
    const double distance = sqrt(dx * dx + dy * dy + dz * dz);
    if (distance < voxel_size * 3.0) {
      good_ids.push_back(k);
      good_matched_pcl.push_back(transformed_src[src_idx]);
    }
  }

  std::ofstream out(argv[2], std::ios::binary);
  for (const pcl::PointXYZ& p : transformed_src) put_xyz(out, p);
  for (const pcl::PointXYZ& p : transformed_srcMatched) put_xyz(out, p);
  const int32_t n_good = (int32_t)good_ids.size();
  put(out, &n_good, 1);
  put(out, good_ids.data(), good_ids.size());
  for (const pcl::PointXYZ& p : good_matched_pcl) put_xyz(out, p);
  return out ? 0 : 1;
}
