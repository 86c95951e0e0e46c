// Learned descriptors through the C-ABI: two keypoint clouds with 32-float descriptor rows (stored 40 floats apart, as a feature
// store with per-point metadata would keep them) are matched and then registered by the descriptor batch calls.
//   descriptor_batch_shim
// Prints "match <status> <n_mutual> <n_corr>" and "register <status> <n_corr> <clique_size> <valid>".
#include <stdint.h>

#include <cmath>
#include <iostream>
#include <vector>

#include "quatro_b200.h"

int main() {
  const int n = 400, dim = 32, stride = 40;
  std::vector<float> src(4 * n), tgt(4 * n), sd((size_t)n * stride), td((size_t)n * stride);
  uint32_t s = 12345u;
  auto rnd = [&]() { s = s * 1664525u + 1013904223u; return (float)(s >> 8) / 16777216.0f; };
  for (int i = 0; i < n; ++i) {
    for (int k = 0; k < 3; ++k) src[4 * i + k] = 40.0f * rnd() - 20.0f;
    src[4 * i + 3] = 1.0f;
    tgt[4 * i] = src[4 * i] + 1.0f; tgt[4 * i + 1] = src[4 * i + 1] - 0.5f; tgt[4 * i + 2] = src[4 * i + 2]; tgt[4 * i + 3] = 1.0f;
    for (int d = 0; d < stride; ++d) {
      sd[(size_t)i * stride + d] = d < dim ? rnd() : NAN;  // the metadata past dim is never read
      td[(size_t)i * stride + d] = d < dim ? sd[(size_t)i * stride + d] + 0.001f * rnd() : NAN;
    }
  }
  qb200_handle* h = nullptr;
  qb200_config cfg;
  qb200_default_config(&cfg);
  cfg.max_batch_slots = 2;
  cfg.max_voxel_points = 512;
  if (int rc = qb200_create(&cfg, &h)) {
    std::cerr << "qb200_create: " << rc << std::endl;
    return 1;
  }
  qb200_params p;
  qb200_default_params(&p);
  const qb200_descriptor_pair pair = {src.data(), sd.data(), tgt.data(), td.data(), n, n, dim, stride};
  qb200_result r;
  int rc = qb200_match_descriptors_each(h, &pair, 1, &p, QB200_MEM_HOST, &r, nullptr);
  std::cout << "match " << rc << " " << r.status << " " << r.n_mutual << " " << r.n_corr << std::endl;
  rc = qb200_register_descriptors_each(h, &pair, 1, &p, QB200_MEM_HOST, &r, nullptr);
  std::cout << "register " << rc << " " << r.status << " " << r.n_corr << " " << r.clique_size << " " << r.valid << std::endl;
  qb200_destroy(h);
  return rc;
}
