// lists.cu -- the per-pair lists of the batch entry points (qb200_pair_lists): correspondences, matched points, max clique, final
// inliers and the two inlier masks of every pair of a wave, packed at the caller's fixed per-pair stride.
//
// The lists already lie in the lane's [S * Lc] buffers when the wave's pose is done; pack_lists_kernel copies each pair's live
// prefix to its destination and marks the record when a list had to be clipped, so it runs after finalize_status_kernel and before
// the D2H of the records (api.cu: wave_submit).  In a match wave it runs after match_records_kernel instead: the clique and mask arrays
// are absent from its ListDst and clique_size is 0, so it packs the correspondences and matched points only.  The destination is the caller's device arrays, or the lane's pinned staging block
// written through its mapped address, so that only live entries cross PCIe; wave_collect copies them on to the caller's host arrays.
#include "handle.cuh"

namespace qb {

namespace {

constexpr int kPackThreads = 256;

// One CTA per pair of the wave.
__global__ void __launch_bounds__(kPackThreads) pack_lists_kernel(qb200_result* __restrict__ results, int Lc, const int* __restrict__ corr_src,
                                                                  const int* __restrict__ corr_tgt, const float4* __restrict__ ma,
                                                                  const float4* __restrict__ mb, const int* __restrict__ clique,
                                                                  const int* __restrict__ final_inl, const unsigned char* __restrict__ rot_mask,
                                                                  const unsigned char* __restrict__ trans_mask, ListDst d) {
  const int pair = blockIdx.x, tid = threadIdx.x;
  qb200_result* r = results + pair;
  if (r->status == QB200_CAPACITY_EXCEEDED) return;
  const int nc = r->n_corr, nq = r->clique_size, nf = r->n_final_inliers;
  const int mc = list_entries(nc, Lc, d.cap), mq = list_entries(nq, Lc, d.cap), mf = list_entries(nf, Lc, d.cap);
  const size_t so = (size_t)pair * Lc, o = (size_t)pair * d.stride;
  for (int i = tid; i < mc; i += kPackThreads) {
    if (d.corr) d.corr[o + i] = make_int2(corr_src[so + i], corr_tgt[so + i]);
    if (d.sm) d.sm[o + i] = ma[so + i];
    if (d.tm) d.tm[o + i] = mb[so + i];
  }
  // a clique of at most one member is not solved (pose.cu): no mask was written for it, its entries are 0
  const bool solved = nq > 1;
  for (int i = tid; i < mq; i += kPackThreads) {
    if (d.clique) d.clique[o + i] = clique[so + i];
    if (d.rm) d.rm[o + i] = solved ? rot_mask[so + i] : 0;
    if (d.tmask) d.tmask[o + i] = solved ? trans_mask[so + i] : 0;
  }
  if (d.fin)
    for (int i = tid; i < mf; i += kPackThreads) d.fin[o + i] = final_inl[so + i];
  if (tid == 0) {
    const bool clipped = (nc > d.cap && (d.corr || d.sm || d.tm)) || (nq > d.cap && (d.clique || d.rm || d.tmask)) || (nf > d.cap && d.fin);
    if (clipped) r->flags |= QB200_FLAG_LISTS_TRUNCATED;
  }
}

}  // namespace

ListDst ListDst::caller(const qb200_pair_lists& l, long long first) {
  const long long c = l.cap_per_pair, o = first * c;
  ListDst d;
  d.corr = l.corr ? reinterpret_cast<int2*>(l.corr) + o : nullptr;
  d.sm = l.src_matched4 ? reinterpret_cast<float4*>(l.src_matched4) + o : nullptr;
  d.tm = l.tgt_matched4 ? reinterpret_cast<float4*>(l.tgt_matched4) + o : nullptr;
  d.clique = l.clique ? l.clique + o : nullptr;
  d.fin = l.final_inliers ? l.final_inliers + o : nullptr;
  d.rm = l.rot_inlier_mask ? l.rot_inlier_mask + o : nullptr;
  d.tmask = l.trans_inlier_mask ? l.trans_inlier_mask + o : nullptr;
  d.stride = c;
  d.cap = l.cap_per_pair;
  return d;
}

size_t ListDst::carve(unsigned char* base, int S, int cap, const qb200_pair_lists& l, ListDst* d) {
  const size_t n = (size_t)S * cap;
  size_t off = 0;
  auto take = [&](size_t bytes, bool want) -> unsigned char* {
    unsigned char* p = base && want ? base + off : nullptr;
    off += (bytes + 15) & ~(size_t)15;
    return p;
  };
  // every list has its place whichever are asked for, so the block's size depends on S and cap only
  d->sm = reinterpret_cast<float4*>(take(n * sizeof(float4), l.src_matched4));
  d->tm = reinterpret_cast<float4*>(take(n * sizeof(float4), l.tgt_matched4));
  d->corr = reinterpret_cast<int2*>(take(n * sizeof(int2), l.corr));
  d->clique = reinterpret_cast<int*>(take(n * sizeof(int), l.clique));
  d->fin = reinterpret_cast<int*>(take(n * sizeof(int), l.final_inliers));
  d->rm = take(n, l.rot_inlier_mask);
  d->tmask = take(n, l.trans_inlier_mask);
  d->stride = cap;
  d->cap = cap < l.cap_per_pair ? cap : l.cap_per_pair;
  return off;
}

int launch_pack_lists(Lane* h, int n_pairs, const ListDst& dst) {
  if (n_pairs <= 0) return QB200_OK;
  pack_lists_kernel<<<n_pairs, kPackThreads, 0, h->stream>>>(h->d_results, h->Lc, h->corr_src, h->corr_tgt, h->ma, h->mb, h->clique, h->final_inl,
                                                             h->rot_mask, h->trans_mask, dst);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
