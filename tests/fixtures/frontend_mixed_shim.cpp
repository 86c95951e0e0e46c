// A sweep mixing presets, as INTEGRATION.md shows it: one qb200_register_batch_mixed call registers pairs of street and dense
// configurations together, and one more call retries the pairs that came back invalid or with few inliers at a finer voxel with the
// tuple test off.
//   frontend_mixed_shim src0.bin tgt0.bin [src1.bin tgt1.bin ...]   (float32 xyzw records)
// Even pairs use the street preset (qb200_default_params), odd pairs the dense one (voxel 0.22 m, tuple test off).  Prints one line
// per pair ("pair <k> <valid> <status> <n_corr> <clique_size>") and one per retried pair ("retry <k> <valid> <status> <n_final>").
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
  if (argc < 3 || (argc - 1) % 2 != 0) {
    std::cerr << "usage: frontend_mixed_shim src0.bin tgt0.bin [src1.bin tgt1.bin ...]" << std::endl;
    return 2;
  }
  const int P = (argc - 1) / 2;
  std::vector<std::vector<float>> data(2 * P);
  std::vector<qb200_pair> pairs(P);
  std::vector<int> dense(P);
  for (int k = 0; k < P; ++k) {
    data[2 * k] = load(argv[1 + 2 * k]);
    data[2 * k + 1] = load(argv[2 + 2 * k]);
    pairs[k].src = data[2 * k].data();      pairs[k].n_src = (int32_t)(data[2 * k].size() / 4);
    pairs[k].tgt = data[2 * k + 1].data();  pairs[k].n_tgt = (int32_t)(data[2 * k + 1].size() / 4);
    dense[k] = k % 2;
  }
  qb200_config cfg;
  qb200_default_config(&cfg);
  cfg.max_batch_slots = 4;
  qb200_handle* h = nullptr;
  if (qb200_create(&cfg, &h) != QB200_OK) {
    std::cerr << "qb200_create failed" << std::endl;
    return 1;
  }

  // ---- the INTEGRATION.md snippet ----
  // pairs[k]: P scan pairs on the host; dense[k] != 0 for the pairs that use the dense preset
  std::vector<qb200_params> params(P);
  std::vector<qb200_result> results(P);
  for (int k = 0; k < P; ++k) {
    qb200_default_params(&params[k]);                     // street: voxel 0.3 m, radii 0.5 / 0.75 m, tuple test on
    if (dense[k]) {
      params[k].voxel_size = 0.22f;                       // dense: finer voxel, every mutual nearest neighbour kept
      params[k].use_tuple_test = 0;
    }
  }
  int rc = qb200_register_batch_mixed(h, pairs.data(), P, params.data(), QB200_MEM_HOST, results.data(), NULL);
  // the pairs that failed, or kept fewer than 10 final inliers, again in one call: finer voxel, tuple test off
  std::vector<qb200_pair> retry;
  std::vector<qb200_params> retry_params;
  std::vector<int> retried;
  for (int k = 0; rc == QB200_OK && k < P; ++k) {
    if (results[k].valid && results[k].n_final_inliers >= 10) continue;
    qb200_params q = params[k];
    q.voxel_size *= 0.75f;
    q.use_tuple_test = 0;
    retry.push_back(pairs[k]);
    retry_params.push_back(q);
    retried.push_back(k);
  }
  std::vector<qb200_result> retry_results(retry.size());
  if (rc == QB200_OK && !retry.empty())
    rc = qb200_register_batch_mixed(h, retry.data(), (int32_t)retry.size(), retry_params.data(), QB200_MEM_HOST, retry_results.data(),
                                    NULL);
  // ---- end of the snippet ----

  if (rc != QB200_OK) {
    std::cerr << "qb200_register_batch_mixed: " << rc << " " << qb200_last_error(h) << std::endl;
    qb200_destroy(h);
    return 1;
  }
  for (int k = 0; k < P; ++k)
    std::cout << "pair " << k << " " << results[k].valid << " " << results[k].status << " " << results[k].n_corr << " "
              << results[k].clique_size << "\n";
  for (size_t r = 0; r < retried.size(); ++r)
    std::cout << "retry " << retried[r] << " " << retry_results[r].valid << " " << retry_results[r].status << " "
              << retry_results[r].n_final_inliers << "\n";
  qb200_destroy(h);
  std::cout << "FRONTEND_MIXED_SHIM_OK" << std::endl;
  return 0;
}
