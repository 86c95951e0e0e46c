// Raw LiDAR scans through the example's pre-processing in one call: qb200_preprocess_batch removes the ground (Patchwork) and the
// small sub-clusters (range-image segmentation) of every scan and hands back the valid segments.
//   preprocess_batch_shim scan1.bin [scan2.bin ...]      (float32 xyzw records)
// Prints one line per scan: "scan <i> <status> <ground> <non-ground> <valid> <outlier> <x of the first valid point>".
#include <stdint.h>

#include <fstream>
#include <iostream>
#include <vector>

#include "quatro_b200.h"

static std::vector<float> load(const char* path) {
  std::ifstream in(path, std::ios::binary | std::ios::ate);
  const size_t bytes = (size_t)in.tellg();
  in.seekg(0);
  std::vector<float> v(bytes / 4);
  in.read(reinterpret_cast<char*>(v.data()), (std::streamsize)bytes);
  return v;
}

int main(int argc, char** argv) {
  if (argc < 2) {
    std::cerr << "usage: preprocess_batch_shim scan1.bin [scan2.bin ...]" << std::endl;
    return 2;
  }
  std::vector<std::vector<float>> scans;
  for (int i = 1; i < argc; ++i) scans.push_back(load(argv[i]));
  const int n = (int)scans.size();

  qb200_config cfg;
  qb200_default_config(&cfg);
  cfg.max_batch_slots = 4;
  qb200_handle* h = nullptr;
  if (qb200_create(&cfg, &h) != QB200_OK) {
    std::cerr << "qb200_create failed" << std::endl;
    return 1;
  }
  qb200_patchwork_params pp;
  qb200_default_patchwork_params(&pp);
  qb200_segment_params sp;
  qb200_default_segment_params(&sp);
  std::vector<const float*> ptrs(n);
  std::vector<int32_t> sizes(n);
  for (int i = 0; i < n; ++i) {
    ptrs[i] = scans[i].data();
    sizes[i] = (int32_t)(scans[i].size() / 4);
  }
  const int cap = sp.n_scan * sp.horizon_scan;  // every valid segment of a scan fits
  std::vector<float> valid((size_t)n * cap * 4);
  std::vector<int32_t> counts((size_t)n * 4), status(n);
  qb200_preprocess_out out = {};
  out.cap_per_scan = cap;
  out.kind = QB200_MEM_HOST;
  out.valid4 = valid.data();
  out.counts = counts.data();
  out.status = status.data();
  const int rc = qb200_preprocess_batch(h, ptrs.data(), sizes.data(), n, QB200_MEM_HOST, &pp, &sp, &out);
  if (rc != QB200_OK) {
    std::cerr << "qb200_preprocess_batch: " << rc << " " << qb200_last_error(h) << std::endl;
    qb200_destroy(h);
    return 1;
  }
  for (int i = 0; i < n; ++i) {
    const int32_t* c = &counts[(size_t)i * 4];
    std::cout << "scan " << i << " " << status[i] << " " << c[0] << " " << c[1] << " " << c[2] << " " << c[3];
    if (c[2] > 0) std::cout << " " << valid[(size_t)i * cap * 4];
    std::cout << "\n";
  }
  qb200_destroy(h);
  std::cout << "PREPROCESS_BATCH_SHIM_OK" << std::endl;
  return 0;
}
