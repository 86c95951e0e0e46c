// match.cu -- K6 (33-D all-pairs nearest neighbour, both directions; nn_dim_kernel for other lengths) + K7 (mutual check, tuple
// test, dedupe/sort, packing of the matched point pairs).   sm_90a
//
// Replaces Matcher::calculateCorrespondences / normalizePoints / advancedMatching
// (include/teaser_utils/feature_matcher.h:42-74, src/teaser_utils/feature_matcher.cc:18-265, which
// builds two FLANN kd-trees) and the packing loop of FPFHManager::setFeaturePair
// (include/fpfh_manager.hpp:130-152).
//
// The two exact 1-NN searches are the row- and column-argmin of one N_src x N_tgt distance matrix
// that is never materialised: a CTA owns a 128-row stripe of source descriptors (staged once in
// shared memory, dimension-major), streams 128-column target tiles through a cp.async double
// buffer, keeps row minima in registers and folds each tile's column minima into colbest with
// one 64-bit atomicMin per column.  Distances are the fused-multiply-add chain over d = 0..32 of
// (a_d - b_d)^2 and minima carry the candidate index in the low word, so ties resolve to the
// lowest index whatever order the stripes arrive in -- exactly the CPU oracle's arithmetic, hence
// bit-identical argmins.  The scratch is colbest itself: linear in max_voxel_points.
#include <stdlib.h>

#include "handle.cuh"
#include "qb_math.cuh"

namespace qb {

constexpr int kMT = kMatchTile;      // 128 x 128 tile
constexpr int kMatchThreads = 256;   // 16 x 16 threads, 8 x 8 distances each

__device__ __forceinline__ unsigned long long pack_dist(float d, int idx) {
  return ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)idx;
}
__device__ __forceinline__ unsigned long long umin64(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
__device__ __forceinline__ unsigned long long shfl_xor_u64(unsigned long long v, int m) {
  const unsigned lo = __shfl_xor_sync(0xffffffffu, (unsigned)v, m), hi = __shfl_xor_sync(0xffffffffu, (unsigned)(v >> 32), m);
  return ((unsigned long long)hi << 32) | lo;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
// src_bytes < 16: the rest of the 16 bytes is zero-filled (0: nothing is read)
__device__ __forceinline__ void cp_async16_zfill(void* smem, const void* gmem, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// load rows d = 0..32 of a 128-wide column window [c0, c0+128) of a dimension-major matrix
__device__ __forceinline__ void load_tile_async(float (*dst)[kMT], const float* __restrict__ src, int V, int c0) {
  for (int ch = threadIdx.x; ch < kDescDim * (kMT / 4); ch += kMatchThreads) {
    const int d = ch / (kMT / 4), c4 = (ch % (kMT / 4)) * 4;
    cp_async16(&dst[d][c4], src + (size_t)d * V + c0 + c4);
  }
}

__global__ void __launch_bounds__(kMatchThreads, 2)
match_stripe_kernel(const float* __restrict__ desc_t, const int* __restrict__ n_vox, int V, const int* __restrict__ only,
                    unsigned long long* __restrict__ rowbest, unsigned long long* __restrict__ colbest) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float(*As)[kMT] = reinterpret_cast<float(*)[kMT]>(smem_raw);                                    // [33][128]
  float(*Bs0)[kMT] = reinterpret_cast<float(*)[kMT]>(smem_raw + sizeof(float) * kDescDim * kMT);  // [33][128]
  float(*Bs1)[kMT] = reinterpret_cast<float(*)[kMT]>(smem_raw + 2 * sizeof(float) * kDescDim * kMT);
  unsigned long long(*colred)[kMT] =
      reinterpret_cast<unsigned long long(*)[kMT]>(smem_raw + 3 * sizeof(float) * kDescDim * kMT);  // [8][128]

  const int pair = blockIdx.y, stripe = blockIdx.x;
  if (only != nullptr && only[pair] == 0) return;  // fallback mode: only the pairs whose tensor-core queue overflowed
  const int nA = n_vox[2 * pair], nB = n_vox[2 * pair + 1];
  const int r0 = stripe * kMT;
  if (r0 >= nA || nB <= 0) return;
  const float* __restrict__ A = desc_t + (size_t)(2 * pair) * kDescK * V;
  const float* __restrict__ B = desc_t + (size_t)(2 * pair + 1) * kDescK * V;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, warp = threadIdx.x >> 5;

  load_tile_async(As, A, V, r0);
  load_tile_async(Bs0, B, V, 0);
  cp_async_commit();

  unsigned long long rbest[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) rbest[r] = ~0ull;

  const int n_tiles = (nB + kMT - 1) / kMT;
  for (int jt = 0; jt < n_tiles; ++jt) {
    float(*Bs)[kMT] = (jt & 1) ? Bs1 : Bs0;
    if (jt + 1 < n_tiles) {
      load_tile_async((jt & 1) ? Bs0 : Bs1, B, V, (jt + 1) * kMT);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    float acc[8][8];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[r][c] = 0.0f;
#pragma unroll 3
    for (int d = 0; d < kDescDim; ++d) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[d][ty * 8]), a1 = *reinterpret_cast<const float4*>(&As[d][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[d][tx * 8]), b1 = *reinterpret_cast<const float4*>(&Bs[d][tx * 8 + 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = desc_dist_step(acc[r][c], a[r], b[c]);
    }
    // epilogue: fold into row minima (registers) and this tile's column minima
    const int cbase = jt * kMT + tx * 8, rbase = r0 + ty * 8;
    unsigned long long cbest[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) cbest[c] = ~0ull;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const bool rv = rbase + r < nA;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float dd = acc[r][c];
        const bool ok = rv && (cbase + c < nB) && (dd == dd);  // NaN never wins
        const unsigned long long pr = ok ? pack_dist(dd, cbase + c) : ~0ull;
        const unsigned long long pc = ok ? pack_dist(dd, rbase + r) : ~0ull;
        rbest[r] = umin64(rbest[r], pr);
        cbest[c] = umin64(cbest[c], pc);
      }
    }
    // columns: the two ty rows of a warp, then the 8 warps through shared memory
#pragma unroll
    for (int c = 0; c < 8; ++c) cbest[c] = umin64(cbest[c], shfl_xor_u64(cbest[c], 16));
    if ((threadIdx.x & 31) < 16) {
#pragma unroll
      for (int c = 0; c < 8; ++c) colred[warp][tx * 8 + c] = cbest[c];
    }
    __syncthreads();
    if (threadIdx.x < kMT) {
      unsigned long long m = colred[0][threadIdx.x];
#pragma unroll
      for (int w = 1; w < 8; ++w) m = umin64(m, colred[w][threadIdx.x]);
      const int col = jt * kMT + threadIdx.x;
      if (col < nB && m != ~0ull) atomicMin(colbest + (size_t)pair * V + col, m);  // the minimum does not depend on stripe order
    }
    // the next iteration's first __syncthreads orders the colred reads above before its writes,
    // and the B buffer being overwritten next was last read two barriers ago.
  }
  // rows: fold the 16 tx lanes that share a row group
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    unsigned long long m = rbest[r];
    m = umin64(m, shfl_xor_u64(m, 1));
    m = umin64(m, shfl_xor_u64(m, 2));
    m = umin64(m, shfl_xor_u64(m, 4));
    m = umin64(m, shfl_xor_u64(m, 8));
    if (tx == 0 && r0 + ty * 8 + r < nA) rowbest[(size_t)pair * V + r0 + ty * 8 + r] = m;
  }
}

// ---- K6 for descriptors of any other length than 33 (a descriptor wave's pairs whose d_feat entries say so) ----
// The structure of match_stripe_kernel with the K extent streamed: a CTA owns a 128-row stripe of the source and walks 128-column
// tiles of the target; for each tile, chunks of kDimChunk dimensions of the stripe and of the tile arrive through one cp.async double
// buffer, and every thread keeps its 8 x 8 distances in registers across the chunks.  So each distance is still one chain of
// desc_dist_step over d = 0 .. dim - 1 in ascending order.  The rows past dim of the last chunk are zero-filled on both sides and add
// fmaf(0, 0, acc) = acc (acc is +0, positive, +inf or NaN: never -0), so the chain is the reference's bit for bit.  Row and column
// minima are folded as in match_stripe_kernel: packed (distance bits, index) u64, ties to the lowest index, NaN never wins.
constexpr int kDimChunk = 32;

// rows k0 .. k0 + 31 of a 128-wide column window [c0, c0 + 128) of a cloud's dimension-major rows (row d at src + d * ld, ld a
// multiple of 4); rows >= dim and columns >= ld are zero-filled without a read
__device__ __forceinline__ void load_chunk_async(float (*dst)[kMT], const float* __restrict__ src, int ld, int dim, int k0, int c0) {
  for (int ch = threadIdx.x; ch < kDimChunk * (kMT / 4); ch += kMatchThreads) {
    const int d = ch / (kMT / 4), c4 = (ch % (kMT / 4)) * 4;
    const bool ok = k0 + d < dim && c0 + c4 < ld;
    cp_async16_zfill(&dst[d][c4], ok ? src + (size_t)(k0 + d) * ld + c0 + c4 : src, ok ? 16 : 0);
  }
}

__global__ void __launch_bounds__(kMatchThreads, 2)
nn_dim_kernel(const FeatureSrc* __restrict__ table, int V, unsigned long long* __restrict__ rowbest, unsigned long long* __restrict__ colbest) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float(*As)[kDimChunk][kMT] = reinterpret_cast<float(*)[kDimChunk][kMT]>(smem_raw);                                        // [2][32][128]
  float(*Bs)[kDimChunk][kMT] = reinterpret_cast<float(*)[kDimChunk][kMT]>(smem_raw + 2 * sizeof(float) * kDimChunk * kMT);  // [2][32][128]
  unsigned long long(*colred)[kMT] =
      reinterpret_cast<unsigned long long(*)[kMT]>(smem_raw + 4 * sizeof(float) * kDimChunk * kMT);                          // [8][128]

  const int pair = blockIdx.y, stripe = blockIdx.x;
  const FeatureSrc fa = table[2 * pair], fb = table[2 * pair + 1];
  if (fa.dim == kDescDim) return;  // an FPFH-33 pair: the tensor-core matcher's
  const int nA = fa.n, nB = fb.n, dim = fa.dim;
  const int r0 = stripe * kMT;
  if (r0 >= nA || nB <= 0) return;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4, warp = threadIdx.x >> 5;
  const int n_chunks = (dim + kDimChunk - 1) / kDimChunk, n_tiles = (nB + kMT - 1) / kMT, n_steps = n_chunks * n_tiles;

  // step s: chunk s % n_chunks of column tile s / n_chunks
  load_chunk_async(As[0], fa.out, fa.ld, dim, 0, r0);
  load_chunk_async(Bs[0], fb.out, fb.ld, dim, 0, 0);
  cp_async_commit();

  unsigned long long rbest[8];
#pragma unroll
  for (int r = 0; r < 8; ++r) rbest[r] = ~0ull;
  float acc[8][8];
  for (int st = 0, jt = 0, kc = 0; st < n_steps; ++st) {
    const int buf = st & 1;
    __syncthreads();  // every thread is done with the buffer the next load overwrites (read in step st - 1)
    if (st + 1 < n_steps) {
      const int kn = kc + 1 == n_chunks ? 0 : kc + 1, jn = kc + 1 == n_chunks ? jt + 1 : jt;
      load_chunk_async(As[buf ^ 1], fa.out, fa.ld, dim, kn * kDimChunk, r0);
      load_chunk_async(Bs[buf ^ 1], fb.out, fb.ld, dim, kn * kDimChunk, jn * kMT);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kc == 0) {
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = 0.0f;
    }
#pragma unroll 4
    for (int d = 0; d < kDimChunk; ++d) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][d][ty * 8]), a1 = *reinterpret_cast<const float4*>(&As[buf][d][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][d][tx * 8]), b1 = *reinterpret_cast<const float4*>(&Bs[buf][d][tx * 8 + 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int r = 0; r < 8; ++r)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[r][c] = desc_dist_step(acc[r][c], a[r], b[c]);
    }
    if (++kc < n_chunks) continue;
    // the tile's distances are complete: fold them into row minima (registers) and the tile's column minima
    kc = 0;
    const int cbase = jt * kMT + tx * 8, rbase = r0 + ty * 8;
    unsigned long long cbest[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) cbest[c] = ~0ull;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const bool rv = rbase + r < nA;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float dd = acc[r][c];
        const bool ok = rv && (cbase + c < nB) && (dd == dd);  // NaN never wins
        const unsigned long long pr = ok ? pack_dist(dd, cbase + c) : ~0ull;
        const unsigned long long pc = ok ? pack_dist(dd, rbase + r) : ~0ull;
        rbest[r] = umin64(rbest[r], pr);
        cbest[c] = umin64(cbest[c], pc);
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) cbest[c] = umin64(cbest[c], shfl_xor_u64(cbest[c], 16));
    if ((threadIdx.x & 31) < 16) {
#pragma unroll
      for (int c = 0; c < 8; ++c) colred[warp][tx * 8 + c] = cbest[c];
    }
    __syncthreads();
    if (threadIdx.x < kMT) {
      unsigned long long m = colred[0][threadIdx.x];
#pragma unroll
      for (int w = 1; w < 8; ++w) m = umin64(m, colred[w][threadIdx.x]);
      const int col = jt * kMT + threadIdx.x;
      if (col < nB && m != ~0ull) atomicMin(colbest + (size_t)pair * V + col, m);
    }
    ++jt;
    // colred is written again only after the next tile's steps, each of which opens with a __syncthreads
  }
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    unsigned long long m = rbest[r];
    m = umin64(m, shfl_xor_u64(m, 1));
    m = umin64(m, shfl_xor_u64(m, 2));
    m = umin64(m, shfl_xor_u64(m, 4));
    m = umin64(m, shfl_xor_u64(m, 8));
    if (tx == 0 && r0 + ty * 8 + r < nA) rowbest[(size_t)pair * V + r0 + ty * 8 + r] = m;
  }
}

// column minima of nn_dim_kernel's pairs start at "none" (~0)
__global__ void __launch_bounds__(256) nn_dim_colreset_kernel(const FeatureSrc* __restrict__ table, int V, unsigned long long* __restrict__ colbest) {
  const int pair = blockIdx.y, col = blockIdx.x * blockDim.x + threadIdx.x;
  const FeatureSrc fb = table[2 * pair + 1];
  if (fb.dim == kDescDim || col >= fb.n) return;
  colbest[(size_t)pair * V + col] = ~0ull;
}

constexpr size_t kDimSmem = 4 * sizeof(float) * kDimChunk * kMT + 8 * kMT * sizeof(unsigned long long);

int launch_match_dim(Lane* h, int n_pairs) {
  const int V = h->V;
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)nn_dim_kernel, kDimSmem));
  nn_dim_colreset_kernel<<<dim3((V + 255) / 256, n_pairs), 256, 0, h->stream>>>(h->d_feat, V, h->colbest);
  nn_dim_kernel<<<dim3(h->NS, n_pairs), kMatchThreads, kDimSmem, h->stream>>>(h->d_feat, V, h->rowbest, h->colbest);
  h->launches += 2;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

// column minima of the pairs being (re)done start at "none" (~0); match_stripe_kernel then atomicMins every stripe's minima into them
__global__ void __launch_bounds__(256) match_colreset_kernel(const int* __restrict__ n_vox, int V, const int* __restrict__ only,
                                                             unsigned long long* __restrict__ colbest) {
  const int pair = blockIdx.y;
  if (only != nullptr && only[pair] == 0) return;
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= n_vox[2 * pair + 1]) return;
  colbest[(size_t)pair * V + col] = ~0ull;
}

// mutual nearest neighbours, listed by ascending index in the LARGER cloud (feature_matcher.cc:84-89,146-177).
// One CTA per pair: ordered compaction with a carried block scan.
__global__ void __launch_bounds__(1024) match_mutual_kernel(const unsigned long long* __restrict__ rowbest, const unsigned long long* __restrict__ colbest,
                                                            const int* __restrict__ n_vox, int V, int* __restrict__ mut_i, int* __restrict__ mut_j,
                                                            int* __restrict__ n_mutual, int* __restrict__ swapped_out, unsigned char* __restrict__ mark,
                                                            int* __restrict__ partner) {
  __shared__ int sm[33];
  const int pair = blockIdx.x;
  const int nA = n_vox[2 * pair], nB = n_vox[2 * pair + 1];
  const bool swapped = nB > nA;
  const unsigned long long* __restrict__ rb = rowbest + (size_t)pair * V;
  const unsigned long long* __restrict__ cb = colbest + (size_t)pair * V;
  const int nI = swapped ? nB : nA;
  int carry = 0;
  for (int base = 0; base < nI; base += blockDim.x) {
    const int i = base + threadIdx.x;
    int j = -1, keep = 0;
    if (i < nI && nA > 0 && nB > 0) {
      const unsigned long long bi = swapped ? cb[i] : rb[i];
      if (bi != ~0ull) {
        j = (int)(unsigned)bi;
        const unsigned long long bj = swapped ? rb[j] : cb[j];
        keep = (bj != ~0ull && (int)(unsigned)bj == i) ? 1 : 0;
      }
    }
    int tot;
    const int ex = block_excl_scan(keep, sm, &tot);
    if (keep) {
      mut_i[(size_t)pair * V + carry + ex] = i;
      mut_j[(size_t)pair * V + carry + ex] = j;
    }
    carry += tot;
  }
  for (int t = threadIdx.x; t < V; t += blockDim.x) {
    mark[(size_t)pair * V + t] = 0;
    partner[(size_t)pair * V + t] = -1;
  }
  if (threadIdx.x == 0) {
    n_mutual[pair] = carry;
    swapped_out[pair] = swapped ? 1 : 0;
  }
}

// Matcher::normalizePoints: float mean accumulated in index order.  One warp per cloud: chunks of 32 points are staged in
// shared memory with coalesced loads (two chunks ahead); lanes 0..2 each own one coordinate and run its serial addition
// chain from shared memory (a 4-cycle dependent add per point instead of a shuffle round trip).  Only the clouds of pairs that run
// the tuple test, its only reader.
__global__ void __launch_bounds__(32) cloud_mean_kernel(const float4* __restrict__ pts, const int* __restrict__ n_pts, int V,
                                                        const PairSolve* __restrict__ solve, float* __restrict__ mean) {
  constexpr int kChunk = 4;                 // 32-point rows per round: 4 loads per lane in flight cover the L2 / DRAM latency
  __shared__ float buf[2][3][32 * kChunk];
  const int cloud = blockIdx.x, lane = (int)lane_id();
  if (!solve[cloud >> 1].use_tuple) return;
  const int n = n_pts[cloud];
  const float4* __restrict__ p = pts + (size_t)cloud * V;
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  float acc = 0.f;
  float4 nxt[kChunk];
#pragma unroll
  for (int c = 0; c < kChunk; ++c) nxt[c] = 32 * c + lane < n ? p[32 * c + lane] : zero;
  for (int base = 0, it = 0; base < n; base += 32 * kChunk, ++it) {
    const int b = it & 1;
#pragma unroll
    for (int c = 0; c < kChunk; ++c) {
      buf[b][0][32 * c + lane] = nxt[c].x; buf[b][1][32 * c + lane] = nxt[c].y; buf[b][2][32 * c + lane] = nxt[c].z;
      const int i = base + 32 * kChunk + 32 * c + lane;
      nxt[c] = i < n ? p[i] : zero;          // in flight while this round is summed
    }
    __syncwarp();
    const int lim = min(32 * kChunk, n - base);
    if (lane < 3) {
      const float* __restrict__ src = buf[b][lane];
      if (lim == 32 * kChunk) {
#pragma unroll
        for (int l = 0; l < 32 * kChunk; ++l) acc = acc + src[l];
      } else {
        for (int l = 0; l < lim; ++l) acc = acc + src[l];
      }
    }
    // the other buffer is rewritten next iteration; this one only after another __syncwarp
  }
  if (lane < 3 && n > 0) mean[cloud * 4 + lane] = acc / (float)n;
  if (lane == 3 && n > 0) mean[cloud * 4 + 3] = 0.f;
}

__device__ __forceinline__ void philox4x32_10(unsigned long long seed, unsigned long long ctr, unsigned out[4]) {
  unsigned c0 = (unsigned)ctr, c1 = (unsigned)(ctr >> 32), c2 = 0, c3 = 0;
  unsigned k0 = (unsigned)seed, k1 = (unsigned)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const unsigned hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const unsigned hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const unsigned n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ float tri_side(const float4 a, const float4 b, const float* __restrict__ m) {
  // points are mean-centred copies: (a - mean) - (b - mean), every step rounded to float
  const float dx = (a.x - m[0]) - (b.x - m[0]), dy = (a.y - m[1]) - (b.y - m[1]), dz = (a.z - m[2]) - (b.z - m[2]);
  return sqrtf((dx * dx + dy * dy) + dz * dz);
}

// tuple (triangle side-ratio) test, feature_matcher.cc:187-247: one thread per trial, counter-based RNG.  Every trial reads six
// random matched points: a CTA first stages the pair's matched points (both clouds, xyz) in shared memory when they fit
// (<= kTupleStage mutual pairs: a street pair has 1.2-2.3 k), so the random reads stay on chip instead of chasing mut_i / mut_j and
// then the point through L2 for each of the six points of a trial.  Scale, trials and seed are the pair's own
// (solve[pair]); the CTAs of a pair that does not run the test leave at once.
//
// The mark is a conjunction over the three sides, and most random triples already fail side 0 (r0, r1).  So a warp tests side 0
// of 32 trials, queues the ones that pass in shared memory (r0, r1 and the raw third draw), and tests sides 1 and 2 once 32 are
// queued: the square roots and divisions of the other two sides run in full warps and only for the triples that need them.
// Which trials mark a point does not change, nor does a mark (a trial sets it to 1 or leaves it).  r % ncorr is qb_fastmod.
constexpr int kTupleStage = 4096;          // 96 KB of staged points
// 512 threads at 55 registers and 108 KB of shared memory: a tuple CTA fits on an SM beside a tc_nn_kernel CTA of another lane
constexpr int kTupleThreads = 512;
constexpr int kTupleWarps = kTupleThreads / 32;
constexpr int kTupleQueue = 64;             // < 32 entries left over + one warp's 32 pushes
constexpr int kTupleCtasPerPair = 16;
constexpr size_t kTupleSmem = sizeof(float) * 2 * kTupleStage * 3 + sizeof(unsigned) * kTupleWarps * 3 * kTupleQueue;
__global__ void __launch_bounds__(kTupleThreads) tuple_test_kernel(const float4* __restrict__ vox_pts, int V, const int* __restrict__ mut_i,
                                                                   const int* __restrict__ mut_j, const int* __restrict__ n_mutual,
                                                                   const int* __restrict__ swapped, const float* __restrict__ mean,
                                                                   const PairSolve* __restrict__ solve, unsigned char* __restrict__ mark) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float(*sp)[kTupleStage][3] = reinterpret_cast<float(*)[kTupleStage][3]>(smem_raw);                                // [2][kTupleStage][3]
  unsigned(*sq)[3][kTupleQueue] = reinterpret_cast<unsigned(*)[3][kTupleQueue]>(smem_raw + sizeof(float) * 2 * kTupleStage * 3);
  const int pair = blockIdx.y;
  if (!solve[pair].use_tuple) return;
  const int ncorr = n_mutual[pair];
  if (ncorr <= 0) return;
  const float scale = solve[pair].tuple_scale;
  const unsigned long long seed = solve[pair].seed;
  const long long trials = (long long)ncorr * solve[pair].tuple_trials;
  const unsigned nc = (unsigned)ncorr;
  const uint64_t magic = qb_fastmod_magic(nc);
  const bool sw = swapped[pair] != 0;
  // fi = larger cloud, fj = smaller
  const int ci = sw ? 2 * pair + 1 : 2 * pair, cj = sw ? 2 * pair : 2 * pair + 1;
  const float4* __restrict__ pi = vox_pts + (size_t)ci * V;
  const float4* __restrict__ pj = vox_pts + (size_t)cj * V;
  const float* __restrict__ mi = mean + ci * 4;
  const float* __restrict__ mj = mean + cj * 4;
  const int* __restrict__ li = mut_i + (size_t)pair * V;
  const int* __restrict__ lj = mut_j + (size_t)pair * V;
  unsigned char* __restrict__ mk = mark + (size_t)pair * V;
  const bool staged = ncorr <= kTupleStage;  // uniform for the CTA
  if (staged) {
    for (int e = threadIdx.x; e < ncorr; e += blockDim.x) {
      const float4 a = pi[li[e]], b = pj[lj[e]];
      sp[0][e][0] = a.x; sp[0][e][1] = a.y; sp[0][e][2] = a.z;
      sp[1][e][0] = b.x; sp[1][e][1] = b.y; sp[1][e][2] = b.z;
    }
    __syncthreads();
  }
  auto point = [&](int side, int r) -> float4 {
    if (staged) return make_float4(sp[side][r][0], sp[side][r][1], sp[side][r][2], 0.f);
    return side == 0 ? pi[li[r]] : pj[lj[r]];
  };
  const int lane = (int)lane_id();
  unsigned* __restrict__ q0 = sq[threadIdx.x >> 5][0];
  unsigned* __restrict__ q1 = sq[threadIdx.x >> 5][1];
  unsigned* __restrict__ q2 = sq[threadIdx.x >> 5][2];
  auto finish = [&](int e) {  // sides 1 and 2 of a queued trial
    const int r0 = (int)q0[e], r1 = (int)q1[e], r2 = (int)qb_fastmod(q2[e], magic, nc);
    const float4 a0 = point(0, r0), a1 = point(0, r1), a2 = point(0, r2);
    const float4 b0 = point(1, r0), b1 = point(1, r1), b2 = point(1, r2);
    const float li1 = tri_side(a1, a2, mi), li2 = tri_side(a2, a0, mi);
    const float lj1 = tri_side(b1, b2, mj), lj2 = tri_side(b2, b0, mj);
    if ((li1 * scale < lj1) && (lj1 < li1 / scale) && (li2 * scale < lj2) && (lj2 < li2 / scale)) {
      mk[r0] = 1; mk[r1] = 1; mk[r2] = 1;
    }
  };
  int queued = 0;  // warp-uniform
  for (long long t0 = (long long)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); t0 < trials; t0 += (long long)gridDim.x * blockDim.x) {
    const long long t = t0 + lane;
    bool pass = false;
    unsigned r[4] = {0u, 0u, 0u, 0u};
    if (t < trials) {
      philox4x32_10(seed, (unsigned long long)t, r);
      r[0] = qb_fastmod(r[0], magic, nc);
      r[1] = qb_fastmod(r[1], magic, nc);
      const float li0 = tri_side(point(0, (int)r[0]), point(0, (int)r[1]), mi);
      const float lj0 = tri_side(point(1, (int)r[0]), point(1, (int)r[1]), mj);
      pass = (li0 * scale < lj0) && (lj0 < li0 / scale);
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, pass);
    if (pass) {
      const int e = queued + __popc(ballot & ((1u << lane) - 1u));
      q0[e] = r[0]; q1[e] = r[1]; q2[e] = r[2];
    }
    queued += __popc(ballot);
    __syncwarp();
    if (queued >= 32) {
      queued -= 32;
      finish(queued + lane);
      __syncwarp();  // the next pushes overwrite these entries
    }
  }
  if (lane < queued) finish(lane);
}

// survivors -> partner[src] = tgt  (mutual NN is a bijection, so sorting by (src,tgt) = sorting by src)
__global__ void __launch_bounds__(256) scatter_partner_kernel(const int* __restrict__ mut_i, const int* __restrict__ mut_j,
                                                              const int* __restrict__ n_mutual, const int* __restrict__ swapped,
                                                              const unsigned char* __restrict__ mark, const PairSolve* __restrict__ solve,
                                                              int V, int* __restrict__ partner) {
  const int pair = blockIdx.y;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_mutual[pair]) return;
  if (solve[pair].use_tuple && !mark[(size_t)pair * V + e]) return;
  const int i = mut_i[(size_t)pair * V + e], j = mut_j[(size_t)pair * V + e];
  const bool sw = swapped[pair] != 0;
  const int s = sw ? j : i, t = sw ? i : j;
  partner[(size_t)pair * V + s] = t;
}

// ordered compaction over source index -> correspondence list + matched point copies
__global__ void __launch_bounds__(1024) pack_corr_kernel(const int* __restrict__ partner, const float4* __restrict__ vox_pts, const int* __restrict__ n_vox,
                                                         int V, int Lc, int* __restrict__ corr_src, int* __restrict__ corr_tgt,
                                                         float4* __restrict__ ma, float4* __restrict__ mb, int* __restrict__ n_corr,
                                                         int* __restrict__ cloud_status, int keep_w) {
  __shared__ int sm[33];
  const int pair = blockIdx.x;
  const int nA = n_vox[2 * pair];
  const float4* __restrict__ ps = vox_pts + (size_t)(2 * pair) * V;
  const float4* __restrict__ pt = vox_pts + (size_t)(2 * pair + 1) * V;
  int carry = 0;
  for (int base = 0; base < nA; base += blockDim.x) {
    const int s = base + threadIdx.x;
    const int t = s < nA ? partner[(size_t)pair * V + s] : -1;
    const int keep = t >= 0 ? 1 : 0;
    int tot;
    const int ex = block_excl_scan(keep, sm, &tot);
    const int o = carry + ex;
    if (keep && o < Lc) {
      corr_src[(size_t)pair * Lc + o] = s;
      corr_tgt[(size_t)pair * Lc + o] = t;
      const float4 a = ps[s], b = pt[t];
      ma[(size_t)pair * Lc + o] = make_float4(a.x, a.y, a.z, keep_w ? a.w : 1.0f);
      mb[(size_t)pair * Lc + o] = make_float4(b.x, b.y, b.z, keep_w ? b.w : 1.0f);
    }
    carry += tot;
  }
  if (threadIdx.x == 0) {
    if (carry > Lc) {
      carry = Lc;
      cloud_status[2 * pair] = QB200_CAPACITY_EXCEEDED;
    }
    n_corr[pair] = carry;
  }
}

size_t match_smem_bytes() { return 3 * sizeof(float) * kDescDim * kMT + 8 * kMT * sizeof(unsigned long long); }

// exact fp32 CUDA-core nearest neighbours (both directions).  only == nullptr: every pair; otherwise just the
// pairs flagged in only[] (the tensor-core filter's overflow fallback).
int launch_match_exact(Lane* h, int n_pairs, const int* only, const int* n_pts) {
  const int V = h->V;
  const size_t smem = match_smem_bytes();
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)match_stripe_kernel, smem));
  const dim3 gf((V + 255) / 256, n_pairs);
  match_colreset_kernel<<<gf, 256, 0, h->stream>>>(n_pts, V, only, h->colbest);
  const dim3 gs(h->NS, n_pairs);
  if (only == nullptr) cudaEventRecord(h->kev[0], h->stream);
  match_stripe_kernel<<<gs, kMatchThreads, smem, h->stream>>>(h->desc_t, n_pts, V, only, h->rowbest, h->colbest);
  if (only == nullptr) {
    cudaEventRecord(h->kev[1], h->stream);
    h->kev_armed[0] = 1;
  }
  h->launches += 2;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

// QB200_TC_VERIFY: count nearest-neighbour entries whose packed (distance bits, index) differ between the two K6 implementations
__global__ void match_verify_kernel(const unsigned long long* __restrict__ rb_tc, const unsigned long long* __restrict__ cb_tc,
                                    const unsigned long long* __restrict__ rb_ex, const unsigned long long* __restrict__ cb_ex,
                                    const int* __restrict__ n_vox, int V, unsigned long long* __restrict__ stats) {
  const int pair = blockIdx.y, i = blockIdx.x * blockDim.x + threadIdx.x;
  const int ns = n_vox[2 * pair], nt = n_vox[2 * pair + 1];
  if (ns <= 0 || nt <= 0) return;
  const int nr = ns, ncol = nt;  // rowbest: best target of every source point; colbest: best source of every target point
  unsigned bad = 0, cnt = 0;
  if (i < nr) { ++cnt; bad += rb_tc[(size_t)pair * V + i] != rb_ex[(size_t)pair * V + i]; }
  if (i < ncol) { ++cnt; bad += cb_tc[(size_t)pair * V + i] != cb_ex[(size_t)pair * V + i]; }
  cnt = __reduce_add_sync(0xffffffffu, cnt);
  bad = __reduce_add_sync(0xffffffffu, bad);
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicAdd(stats + 4, (unsigned long long)cnt);
    if (bad) atomicAdd(stats + 5, (unsigned long long)bad);
  }
}

// One thread per pair of a match wave: the record a register call would hold after its matcher (fill_counters_kernel's counters,
// finalize_status_kernel's front-end status), with the solver fields of a pair that was not solved.  An empty side is
// QB200_DEGENERATE_INPUT; any other pair is QB200_OK, whatever its correspondence count.
__global__ void match_records_kernel(qb200_result* __restrict__ results, int n_pairs, WaveCounters c) {
  const int pair = blockIdx.x * blockDim.x + threadIdx.x;
  if (pair >= n_pairs) return;
  qb200_result* r = results + pair;
  const int ns = c.n_vox[2 * pair], nt = c.n_vox[2 * pair + 1];
  const int s0 = c.cloud_status[2 * pair], s1 = c.cloud_status[2 * pair + 1];
  r->valid = 0;
  r->status = s0 != 0 ? s0 : s1 != 0 ? s1 : (ns <= 0 || nt <= 0) ? QB200_DEGENERATE_INPUT : QB200_OK;
  r->n_src_vox = ns;
  r->n_tgt_vox = nt;
  r->n_mutual = c.n_mutual[pair];
  r->n_corr = c.n_corr[pair];
  r->max_core = 0;
  r->clique_size = 0;
  r->gnc_iters = 0;
  r->n_rot_inliers = 0;
  r->n_final_inliers = 0;
  r->flags = c.flags[pair];
  r->n_edges = 0;
  r->cost = 0.0;
  for (int i = 0; i < 16; ++i) r->T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

int launch_match_records(Lane* h, int n_pairs) {
  if (n_pairs <= 0) return QB200_OK;
  match_records_kernel<<<(n_pairs + 127) / 128, 128, 0, h->stream>>>(h->d_results, n_pairs, h->ctr);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

void match_fields(PairSolve* e, const qb200_params& p) {
  e->use_tuple = (p.use_tuple_test && p.tuple_scale != 0.0f) ? 1 : 0;
  e->tuple_scale = p.tuple_scale;
  e->tuple_trials = p.tuple_trials_per_corr;
  e->seed = p.seed;
}

int launch_match(Lane* h, int n_pairs, int keep_w, int dims) {
  if (n_pairs <= 0) return QB200_OK;
  const int V = h->V;
  const int* n_pts = dims ? h->ctr.n_fpfh : h->ctr.n_vox;
  const bool fpfh = dims == 0 || (dims & kDimsFpfh);
  int rc = !fpfh ? QB200_OK : h->force_exact_match ? launch_match_exact(h, n_pairs, nullptr, n_pts) : launch_match_nn(h, n_pairs, n_pts);
  if (rc) return rc;
  if (fpfh && h->tc_verify && !h->force_exact_match) {
    // whole-batch self-check: keep the tensor-core results, redo every pair with the exact CUDA-core kernel, compare
    unsigned long long* rb_tc = reinterpret_cast<unsigned long long*>(h->key_b.get());                   // the sort workspace is idle here
    unsigned long long* cb_tc = rb_tc + (size_t)h->S * V;
    QB_CUDA_TRY(h, cudaMemcpyAsync(rb_tc, h->rowbest, (size_t)n_pairs * V * 8, cudaMemcpyDeviceToDevice, h->stream));
    QB_CUDA_TRY(h, cudaMemcpyAsync(cb_tc, h->colbest, (size_t)n_pairs * V * 8, cudaMemcpyDeviceToDevice, h->stream));
    if ((rc = launch_match_exact(h, n_pairs, nullptr, n_pts))) return rc;
    const dim3 gv((V + 255) / 256, n_pairs);
    match_verify_kernel<<<gv, 256, 0, h->stream>>>(rb_tc, cb_tc, h->rowbest, h->colbest, n_pts, V, h->tc_stats);
    h->launches += 1;
  }
  // after the FPFH-33 K6, whose clearing of rowbest / colbest covers every pair of the wave
  if ((dims & kDimsOther) && (rc = launch_match_dim(h, n_pairs))) return rc;
  match_mutual_kernel<<<n_pairs, 1024, 0, h->stream>>>(h->rowbest, h->colbest, h->ctr.n_vox, V, h->mut_i, h->mut_j, h->ctr.n_mutual,
                                                       h->ctr.swapped, h->mark, h->partner);
  h->launches += 1;
  bool any_tuple = false;  // the host's copy of the pairs' table (h_solve) decides whether the tuple test is launched at all
  for (int s = 0; s < n_pairs; ++s) any_tuple |= h->h_solve[s].use_tuple != 0;
  if (any_tuple) {
    cloud_mean_kernel<<<2 * n_pairs, 32, 0, h->stream>>>(h->vox_pts, h->ctr.n_vox, V, h->d_solve, h->mean);
    QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)tuple_test_kernel, kTupleSmem));
    const dim3 gt(kTupleCtasPerPair, n_pairs);
    tuple_test_kernel<<<gt, kTupleThreads, kTupleSmem, h->stream>>>(h->vox_pts, V, h->mut_i, h->mut_j, h->ctr.n_mutual, h->ctr.swapped, h->mean, h->d_solve,
                                                           h->mark);
    h->launches += 2;
  }
  const dim3 gsc((V + 255) / 256, n_pairs);
  scatter_partner_kernel<<<gsc, 256, 0, h->stream>>>(h->mut_i, h->mut_j, h->ctr.n_mutual, h->ctr.swapped, h->mark, h->d_solve, V, h->partner);
  pack_corr_kernel<<<n_pairs, 1024, 0, h->stream>>>(h->partner, h->vox_pts, h->ctr.n_vox, V, h->Lc, h->corr_src, h->corr_tgt, h->ma, h->mb,
                                                    h->ctr.n_corr, h->ctr.cloud_status, keep_w);
  h->launches += 2;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
