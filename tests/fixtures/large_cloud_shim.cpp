// GPU check of the C++ drop-in layer on clouds beyond the default capacities: a dense indoor pair whose scans hold ~500 k points and
// whose clouds keep more than 65536 voxel points at a 0.05 m voxel.  voxelize, FPFHManager::setFeaturePair and
// Quatro::computeTransformation must grow their handles (raw points, voxel points, correspondences) instead of throwing.
//   large_cloud_shim src.bin tgt.bin      (float32 xyzw records, every record is read)
#include <fstream>
#include <iomanip>
#include <iostream>

#include "quatro_b200/fpfh_manager.hpp"

static pcl::PointCloud<PointType>::Ptr load(const char* path) {
  std::ifstream in(path, std::ios::binary | std::ios::ate);
  const size_t bytes = (size_t)in.tellg();
  in.seekg(0);
  std::vector<float> v(bytes / 4);
  in.read(reinterpret_cast<char*>(v.data()), (std::streamsize)bytes);
  auto c = std::make_shared<pcl::PointCloud<PointType>>();
  for (size_t i = 0; i + 3 < v.size(); i += 4) c->push_back(PointType(v[i], v[i + 1], v[i + 2]));
  return c;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  // the indoor configuration: 0.05 m voxel, 0.10 / 0.15 m normal / FPFH radii, 0.05 m noise bounds; the rest as config/params.yaml
  const double voxel_size = 0.05, normal_radius = 0.10, fpfh_radius = 0.15, noise_bound = 0.05;
  pcl::PointCloud<PointType>::Ptr src_raw = load(argv[1]), tgt_raw = load(argv[2]);
  pcl::PointCloud<PointType>::Ptr src_vox(new pcl::PointCloud<PointType>), tgt_vox(new pcl::PointCloud<PointType>);
  try {
    voxelize(src_raw, src_vox, voxel_size);
    voxelize(tgt_raw, tgt_vox, voxel_size);
    FPFHManager fpfh(normal_radius, fpfh_radius);
    fpfh.flushAllFeatures();
    fpfh.setFeaturePair(src_vox, tgt_vox);
    pcl::PointCloud<PointType>::Ptr src_kps(new pcl::PointCloud<PointType>), tgt_kps(new pcl::PointCloud<PointType>);
    *src_kps = fpfh.getSrcKps();
    *tgt_kps = fpfh.getTgtKps();

    Quatro<PointType, PointType> quatro;
    Quatro<PointType, PointType>::Params params;
    params.noise_bound = noise_bound;
    params.rotation_max_iterations = 50;
    params.rotation_cost_threshold = 0.00011;
    quatro.reset(params);
    quatro.noise_bound_ = noise_bound;
    quatro.setInputSource(src_kps);
    quatro.setInputTarget(tgt_kps);
    Eigen::Matrix4d output = Eigen::Matrix4d::Identity();
    quatro.computeTransformation(output);

    std::cout << "raw " << src_raw->size() << " " << tgt_raw->size() << "\n";
    std::cout << "voxels " << src_vox->size() << " " << tgt_vox->size() << "\n";
    std::cout << "corr " << fpfh.getCorrespondences().size() << "\n";
    std::cout << "clique " << quatro.getNumMaxCliqueInliers() << "\n";
    std::cout << std::setprecision(17);
    for (int r = 0; r < 4; ++r) std::cout << "T " << output(r, 0) << " " << output(r, 1) << " " << output(r, 2) << " " << output(r, 3) << "\n";
  } catch (const std::exception& e) {
    std::cerr << "exception: " << e.what() << std::endl;
    return 1;
  }
  std::cout << "LARGE_CLOUD_SHIM_OK" << std::endl;
  return 0;
}
