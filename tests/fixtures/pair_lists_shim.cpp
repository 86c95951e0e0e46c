// A loop-closure sweep through the C-ABI that keeps every pair's lists: qb200_register_batch_ex registers the query scan against each
// candidate and hands back, per pair, the final inliers as (source voxel, target voxel) index pairs.
//   pair_lists_shim query.bin cand1.bin [cand2.bin ...]      (float32 xyzw records)
// Prints one line per candidate: "pair <i> <status> <n_corr> <clique_size> <n_final_inliers> <flags> <first inlier src> <tgt>".
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
  if (argc < 3) {
    std::cerr << "usage: pair_lists_shim query.bin cand1.bin [cand2.bin ...]" << std::endl;
    return 2;
  }
  const std::vector<float> query = load(argv[1]);
  std::vector<std::vector<float>> cands;
  for (int i = 2; i < argc; ++i) cands.push_back(load(argv[i]));
  const int n = (int)cands.size();

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
  std::vector<qb200_pair> pairs(n);
  for (int i = 0; i < n; ++i) {
    pairs[i].src = query.data();
    pairs[i].n_src = (int32_t)(query.size() / 4);
    pairs[i].tgt = cands[i].data();
    pairs[i].n_tgt = (int32_t)(cands[i].size() / 4);
  }
  const int cap = cfg.max_corr;
  std::vector<int32_t> corr((size_t)n * cap * 2), inl((size_t)n * cap);
  qb200_pair_lists lists = {};
  lists.cap_per_pair = cap;
  lists.kind = QB200_MEM_HOST;
  lists.corr = corr.data();
  lists.final_inliers = inl.data();
  std::vector<qb200_result> res(n);
  const int rc = qb200_register_batch_ex(h, pairs.data(), n, &p, QB200_MEM_HOST, res.data(), &lists);
  if (rc != QB200_OK) {
    std::cerr << "qb200_register_batch_ex: " << rc << " " << qb200_last_error(h) << std::endl;
    qb200_destroy(h);
    return 1;
  }
  for (int i = 0; i < n; ++i) {
    const qb200_result& r = res[i];
    std::cout << "pair " << i << " " << r.status << " " << r.n_corr << " " << r.clique_size << " " << r.n_final_inliers << " " << r.flags;
    if (r.n_final_inliers > 0) {
      const int32_t k = inl[(size_t)i * cap];  // a final inlier is a correspondence id of this pair
      std::cout << " " << corr[((size_t)i * cap + k) * 2] << " " << corr[((size_t)i * cap + k) * 2 + 1];
    }
    std::cout << "\n";
  }
  qb200_destroy(h);
  std::cout << "PAIR_LISTS_SHIM_OK" << std::endl;
  return 0;
}
