// GPU check of Quatro::computeTransformation on a matched set larger than 8192 correspondences: the shim must grow its handle to
// QB200_MAX_CORR correspondences and solve, not throw.
//   wide_corr_shim src.bin tgt.bin      (float32 xyzw records of the matched points, same count in both files)
#include <fstream>
#include <iomanip>
#include <iostream>

#include "quatro_b200/quatro.hpp"

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
  pcl::PointCloud<PointType>::Ptr src = load(argv[1]), tgt = load(argv[2]);
  try {
    Quatro<PointType, PointType> quatro;
    Quatro<PointType, PointType>::Params params;
    params.noise_bound = 0.3;
    params.rotation_max_iterations = 50;
    params.rotation_cost_threshold = 0.00011;
    quatro.reset(params);
    quatro.setInputSource(src);
    quatro.setInputTarget(tgt);
    Eigen::Matrix4d output = Eigen::Matrix4d::Identity();
    quatro.computeTransformation(output);
    std::cout << "corr " << src->size() << "\n";
    std::cout << "clique " << quatro.getNumMaxCliqueInliers() << "\n";
    std::cout << std::setprecision(17);
    for (int r = 0; r < 4; ++r) std::cout << "T " << output(r, 0) << " " << output(r, 1) << " " << output(r, 2) << " " << output(r, 3) << "\n";
  } catch (const std::exception& e) {
    std::cerr << "exception: " << e.what() << std::endl;
    return 1;
  }
  std::cout << "WIDE_CORR_SHIM_OK" << std::endl;
  return 0;
}
