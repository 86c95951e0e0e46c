// sort.cu -- per-cloud stable radix sort in shared memory (sm_90a): the lattice-cell sort of K2 and the descriptor-norm sort of K6.
//
// Both sorts order at most max_voxel_points (key, point index) pairs PER CLOUD, and only the first n_vox of them carry live keys.  A
// device-wide radix sort (round 1: cub::DeviceRadixSort over n_clouds * V items, 6-9 launches of 25-30 us per wave each) moves every
// item through HBM once per 8-bit pass; here one CTA per cloud never moves the keys and permutes a 16-bit index array in shared
// memory with 4-bit LSD passes -- only over the digits in which the cloud's keys actually differ (a street scan's lattice keys vary
// in ~8 of 13 digits).  Stable like the device-wide sort, so the output is identical: equal keys keep ascending point index.
//
// Layout in: key_in[cloud * V + q] for q < V (values are the point indices q themselves); out: key_out / val_out[cloud * V + r].
//
// Shared memory holds the two index arrays, the count table and ONE BYTE per point: the two digits of the next two passes, packed
// from key_in (L2-resident after the first read) every other varying digit.  That is 5 V + 16 KB (96 KB at V = 16384), so a sort
// CTA fits on an SM beside a tc_nn_kernel CTA (100 KB) instead of closing the SM to the matcher of the other lanes.
#include "handle.cuh"

namespace qb {

constexpr int kSortThreads = 512;
// Larger clouds go through the device-wide sort (sort_pairs).  Not a hardware limit: 17920 is the largest V (a multiple of 128) whose
// keys, two index arrays and count table fitted the 227 KB of an SM when the keys lived in shared memory; it is kept so that the
// same handles take the same sort as before (both sorts are stable, so the output does not depend on it).  The byte-digit layout
// below would fit V up to about 43 000.
constexpr int kCloudSortMaxV = 17920;

size_t cloud_sort_smem_bytes(int V) { return (size_t)2 * V * 2 + (size_t)16 * kSortThreads * 2 + (size_t)V; }

// f1, f2: bit offsets that split the low 52 key bits into up to three fields [0,f1) [f1,f2) [f2,52) (lattice keys: i | j | k at 0 / 18 /
// 36; norm keys: one field).  Every field is sorted relative to its minimum inside the cloud: the cell coordinates carry offsets of
// 2^17 / 2^15, so neighbouring cells on either side of an axis differ in ALL bits of a field (0x1FFFF vs 0x20000) although their
// difference is 1; relative fields vary in 2-3 digits instead of 4-5.  The order is unchanged (no borrow crosses a field).
__global__ void __launch_bounds__(kSortThreads) cloud_sort_kernel(const uint64_t* __restrict__ key_in, const int* __restrict__ n_items, int V,
                                                                  int f1, int f2, uint64_t* __restrict__ key_out, uint32_t* __restrict__ val_out) {
  constexpr int NT = kSortThreads;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned short* idx_a = reinterpret_cast<unsigned short*>(smem_raw);    // [V] current order
  unsigned short* idx_b = idx_a + V;                                      // [V] next order
  unsigned short* counts = idx_b + V;                                     // [16][NT] per-(digit value, thread) counts -> start offsets
  unsigned char* digits = reinterpret_cast<unsigned char*>(counts + 16 * NT);  // [V] by point index: this pass's digit | the next one's
  __shared__ int s_scan[33];
  __shared__ unsigned long long s_vary;
  __shared__ unsigned int s_min[3];
  const int cloud = blockIdx.x, tid = threadIdx.x;
  const size_t base = (size_t)cloud * V;
  const uint64_t* __restrict__ kin = key_in + base;
  int n = n_items[cloud];
  n = n < 0 ? 0 : (n > V ? V : n);
  if (tid == 0) { s_vary = 0ull; s_min[0] = s_min[1] = s_min[2] = 0xFFFFFFFFu; }
  __syncthreads();
  const unsigned long long m0 = (1ull << f1) - 1ull, m1 = (1ull << (f2 - f1)) - 1ull, m2 = (1ull << (52 - f2)) - 1ull;
  {
    unsigned int a0 = 0xFFFFFFFFu, a1 = 0xFFFFFFFFu, a2 = 0xFFFFFFFFu;
    for (int q = tid; q < n; q += NT) {
      const unsigned long long k = kin[q];
      idx_a[q] = (unsigned short)q;
      a0 = min(a0, (unsigned int)(k & m0)); a1 = min(a1, (unsigned int)((k >> f1) & m1)); a2 = min(a2, (unsigned int)((k >> f2) & m2));
    }
    a0 = __reduce_min_sync(0xffffffffu, a0); a1 = __reduce_min_sync(0xffffffffu, a1); a2 = __reduce_min_sync(0xffffffffu, a2);
    if ((tid & 31) == 0) { atomicMin(&s_min[0], a0); atomicMin(&s_min[1], a1); atomicMin(&s_min[2], a2); }
  }
  __syncthreads();
  // field-wise relative keys k - kmin: every field is >= its minimum, no borrow
  const unsigned long long kmin = (unsigned long long)s_min[0] | ((unsigned long long)s_min[1] << f1) | ((unsigned long long)s_min[2] << f2);
  {  // which key bits differ inside this cloud?
    unsigned long long v = 0ull;
    const unsigned long long k0 = n > 0 ? kin[0] - kmin : 0ull;
    for (int q = tid; q < n; q += NT) v |= (kin[q] - kmin) ^ k0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v |= __shfl_xor_sync(0xffffffffu, v, o);
    if ((tid & 31) == 0 && v) atomicOr(&s_vary, v);
  }
  __syncthreads();
  const unsigned long long vary = s_vary;
  const int ipt = (n + NT - 1) / NT;                       // consecutive positions per thread (<= 35 for V <= kCloudSortMaxV)
  const int p0 = tid * ipt, p1 = min(n, p0 + ipt);
  unsigned short* cur = idx_a;
  unsigned short* nxt = idx_b;
  int nib = 0;                                             // which nibble of digits[] holds this pass's digit (block-uniform)
  for (int s = 0; s < 64; s += 4) {
    if (((vary >> s) & 15ull) == 0ull) continue;           // every key has the same digit here (block-uniform)
    if (nib == 0) {  // pack this digit and the next varying one; the previous pass's last reads of digits[] are behind its barrier
      const unsigned long long above = s + 4 < 64 ? vary >> (s + 4) : 0ull;
      const int s2 = above ? s + 4 + 4 * ((__ffsll((long long)above) - 1) >> 2) : s;
      for (int q = tid; q < n; q += NT) {
        const unsigned long long k = kin[q] - kmin;
        digits[q] = (unsigned char)(((k >> s) & 15ull) | (((k >> s2) & 15ull) << 4));
      }
      __syncthreads();
    }
    const int sd = 4 * nib;
    nib ^= 1;
    // ---- count the digit values of this thread's run of positions (8-bit fields: value d lives in c[d >> 3], byte d & 7)
    unsigned long long c0 = 0ull, c1 = 0ull;
    for (int p = p0; p < p1; ++p) {
      const int d = (digits[cur[p]] >> sd) & 15;
      const unsigned long long one = 1ull << (8 * (d & 7));
      if (d < 8) c0 += one; else c1 += one;
    }
#pragma unroll
    for (int b = 0; b < 8; ++b) {
      counts[b * NT + tid] = (unsigned short)((c0 >> (8 * b)) & 255ull);
      counts[(b + 8) * NT + tid] = (unsigned short)((c1 >> (8 * b)) & 255ull);
    }
    __syncthreads();
    // ---- exclusive scan of the flattened [digit value][thread] table: thread t owns entries 16 t .. 16 t + 15
    {
      unsigned short loc[16];
      int sum = 0;
#pragma unroll
      for (int e = 0; e < 16; ++e) {
        const int c = counts[16 * tid + e];
        loc[e] = (unsigned short)sum;
        sum += c;
      }
      int total;
      const int ex = block_excl_scan(sum, s_scan, &total);
#pragma unroll
      for (int e = 0; e < 16; ++e) counts[16 * tid + e] = (unsigned short)(ex + loc[e]);
    }
    __syncthreads();
    // ---- stable scatter: the same walk, each value's running offset starts at this thread's table entry
    c0 = 0ull; c1 = 0ull;
    for (int p = p0; p < p1; ++p) {
      const unsigned short i = cur[p];
      const int d = (digits[i] >> sd) & 15;
      const int sh = 8 * (d & 7);
      const int run = (int)(((d < 8 ? c0 : c1) >> sh) & 255ull);
      nxt[counts[d * NT + tid] + run] = i;
      const unsigned long long one = 1ull << sh;
      if (d < 8) c0 += one; else c1 += one;
    }
    __syncthreads();
    unsigned short* t = cur; cur = nxt; nxt = t;
  }
  for (int r = tid; r < V; r += NT) {
    if (r < n) {
      const unsigned short i = cur[r];
      key_out[base + r] = kin[i];
      val_out[base + r] = (uint32_t)i;
    } else {  // dead items keep their place behind the live ones (their keys compare above every live key)
      key_out[base + r] = kin[r];
      val_out[base + r] = (uint32_t)r;
    }
  }
}

// Sort the first n_items[c] keys of every cloud c (key_a -> key_b, val_b = source index).  Returns QB200_ERR_UNSUPPORTED when
// max_voxel_points is too large for the shared-memory layout (the caller then uses the device-wide sort).
int launch_cloud_sort(Lane* h, int n_clouds, const int* n_items, int f1, int f2) {
  if (n_clouds <= 0) return QB200_OK;
  if (h->V > kCloudSortMaxV) return QB200_ERR_UNSUPPORTED;
  const size_t smem = cloud_sort_smem_bytes(h->V);
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)cloud_sort_kernel, smem));
  cloud_sort_kernel<<<n_clouds, kSortThreads, smem, h->stream>>>(h->key_a, n_items, h->V, f1, f2, h->key_b, h->val_b);
  h->launches += 1;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
