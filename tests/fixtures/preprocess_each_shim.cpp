// A mixed fleet's raw scans through pre-processing and registration, as INTEGRATION.md shows it: one qb200_preprocess_batch_each
// call with every scan's own lidar model and mounting height, its valid segments left on the device and registered from there.
//   preprocess_each_shim <model> <sensor_height> scan.bin  [<model> <sensor_height> scan.bin ...]   (float32 xyzw records)
// model: 0 = Velodyne-64-HDE, 1 = VLP-16.  Scans (0, 1), (2, 3), ... are registered as pairs.
// Prints one line per scan ("scan <i> <status> <ground> <non-ground> <valid> <outlier>") and one per pair ("pair <k> <valid> <status>
// <n_corr> <clique_size>").
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

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
  if (argc < 4 || (argc - 1) % 3 != 0) {
    std::cerr << "usage: preprocess_each_shim <model> <sensor_height> scan.bin [<model> <sensor_height> scan.bin ...]" << std::endl;
    return 2;
  }
  const int N = (argc - 1) / 3, P = N / 2;
  std::vector<int> model(N);
  std::vector<double> height(N);
  std::vector<std::vector<float>> data(N);
  std::vector<const float*> scans(N);
  std::vector<int32_t> n(N);
  for (int i = 0; i < N; ++i) {
    model[i] = atoi(argv[1 + 3 * i]);
    height[i] = atof(argv[2 + 3 * i]);
    data[i] = load(argv[3 + 3 * i]);
    scans[i] = data[i].data();
    n[i] = (int32_t)(data[i].size() / 4);
  }
  qb200_config cfg;
  qb200_default_config(&cfg);
  cfg.max_batch_slots = 4;
  qb200_handle* h = nullptr;
  if (qb200_create(&cfg, &h) != QB200_OK) {
    std::cerr << "qb200_create failed" << std::endl;
    return 1;
  }
  qb200_params p;
  qb200_default_params(&p);

  // ---- the INTEGRATION.md snippet ----
  // scans[i]: n[i] x {x,y,z,w} host records of N raw scans; model[i] 0 = HDL-64E, 1 = VLP-16; height[i] its mounting height
  std::vector<qb200_patchwork_params> pw(N);
  std::vector<qb200_segment_params> sg(N);
  for (int i = 0; i < N; ++i) {
    qb200_default_patchwork_params(&pw[i]);
    pw[i].sensor_height = height[i];                        // the -1.8 h cut and the seed margin follow it
    qb200_default_segment_params(&sg[i]);                   // "Velodyne-64-HDE"
    if (model[i] == 1) {                                    // "VLP-16" (imageProjection.hpp:93-100)
      sg[i].n_scan = 16;  sg[i].horizon_scan = 1800;
      sg[i].ang_res_x = 0.2f;  sg[i].ang_res_y = 2.0f;  sg[i].ang_bottom = (float)(15.0 + 0.1);
    }
  }
  const int32_t cap = 64 * 1800;                            // the fleet's largest image: every valid segment fits
  float* valid_dev = nullptr;
  cudaMalloc(&valid_dev, (size_t)N * cap * 4 * sizeof(float));
  std::vector<int32_t> counts(N * 4), status(N);
  qb200_preprocess_out out = {};
  out.cap_per_scan = cap;  out.kind = QB200_MEM_DEVICE;  out.valid4 = valid_dev;
  out.counts = counts.data();  out.status = status.data();
  int rc = qb200_preprocess_batch_each(h, scans.data(), n.data(), N, QB200_MEM_HOST, pw.data(), sg.data(), &out);
  std::vector<qb200_pair> pairs(P);
  std::vector<qb200_result> results(P);
  for (int k = 0; k < P; ++k) {
    pairs[k].src = valid_dev + (size_t)(2 * k) * cap * 4;      pairs[k].n_src = counts[4 * (2 * k) + 2];
    pairs[k].tgt = valid_dev + (size_t)(2 * k + 1) * cap * 4;  pairs[k].n_tgt = counts[4 * (2 * k + 1) + 2];
  }
  p.skip_flagged = 0;                                       // ground is gone already
  if (rc == QB200_OK) rc = qb200_register_batch(h, pairs.data(), P, &p, QB200_MEM_DEVICE, results.data());
  // ---- end of the snippet ----

  if (rc != QB200_OK) {
    std::cerr << "pre-processing / registration: " << rc << " " << qb200_last_error(h) << std::endl;
    cudaFree(valid_dev);
    qb200_destroy(h);
    return 1;
  }
  for (int i = 0; i < N; ++i) {
    const int32_t* c = &counts[(size_t)i * 4];
    std::cout << "scan " << i << " " << status[i] << " " << c[0] << " " << c[1] << " " << c[2] << " " << c[3] << "\n";
  }
  for (int k = 0; k < P; ++k)
    std::cout << "pair " << k << " " << results[k].valid << " " << results[k].status << " " << results[k].n_corr << " "
              << results[k].clique_size << "\n";
  cudaFree(valid_dev);
  qb200_destroy(h);
  std::cout << "PREPROCESS_EACH_SHIM_OK" << std::endl;
  return 0;
}
