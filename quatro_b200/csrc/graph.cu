// graph.cu -- K8: translation-invariant-measurement (TIM) consistency graph.   sm_90a
//
// Replaces Quatro::computeTIMs + solveForScale + the inlier_graph_.addEdge loop
// (include/quatro.hpp:307-386, 784-789; include/teaser/graph.h:96-104).  The reference
// materialises 2 x 3 x M doubles of TIMs, M index pairs and an M-byte mask (M = L(L-1)/2, ~65 B per
// pair, SURVEY.md 8d) and then inserts edges one by one; here a pair (i,j) is tested straight from
// the two matched point sets and only the bit-packed symmetric adjacency matrix is written.
//
// Arithmetic.  The reference's mask is abs(db/da - 1) <= beta/da && abs(da/db - 1) <= beta/db in fp64
// (quatro.hpp:363-385), i.e. |da - db| <= beta up to rounding.  With A = da^2, B = db^2, s' = A + B - beta^2,
// D = A - B, g = beta^2 (2 s' + beta^2) and t = D^2 - g (= (A + B - beta^2)^2 - 4AB):
//        edge  <=>  t <= 0  or  s' <= 0.
// The kernel evaluates this in fp32 with A, B in Gram form (|a_i|^2 + |a_j|^2 - 2 a_i.a_j: 4 instead of 6 operations per
// distance) -- ~18 instructions per pair test -- together with a RIGOROUS bound of its own rounding error:
//        |t_c - t| <= 36u M |D_c| + 1500 u^2 M^2 + 46 u beta^2 M =: q,   u = 2^-24,  M >= |a_i|^2+|b_i|^2+|a_j|^2+|b_j|^2 + 2 beta^2
// (derivation in DESIGN.md 5.2).  Each lane evaluates its columns with scalar IEEE-rn operations (explicit
// __fmaf_rn / __fadd_rn: no contraction decides the rounding).  Only pairs with |t_c| <= q -- a band of ~1e-4 relative width around the threshold --
// or with both distances ~0 (the literal expression is NaN -> false for coincident duplicates) evaluate the literal fp64
// expression, and so does every test whose M exceeds 2^62 (the bound needs D^2, 2 beta^2 s' and q finite), so the adjacency is
// bit-identical to the fp64 reference for any input.
//
// The same file imports caller graphs for qb200_max_clique_batch_each (edge lists or adjacency rows into the lane's adj, with the
// validity checks of DESIGN.md 5.4) in place of K8.
//
// Work decomposition.  A WARP work item is 64 rows x 128 columns of the upper triangle (any pair of the launch: one global item
// list); the warp stages its 64 row points in shared memory as (-2a, |a|^2 - beta^2/4 | -2b, |b|^2 - beta^2/4) -- read back as
// broadcast operands of the FMAs -- and each lane keeps FOUR columns in registers.  No CTA barrier in
// the item loop.  Result bits are shifted in from the SIGN BITS of t, s' and |t| - q with funnel shifts (no compare / select per
// test); a warp shuffle transpose turns the per-column words into the row-major half, so both halves of the symmetric matrix come
// out of one evaluation of the M pair tests.  (Timing experiment, round 2: without the two 4-byte row-strided stores and the
// transpose per 32 x 32 block the kernel runs 0.144 instead of 0.174 ms at 32 x L = 3000.)
#include "handle.cuh"

namespace qb {

constexpr int kGW = 4;    // warps per CTA
constexpr int kGC = 4;    // columns per lane (a warp covers kGC x 32 columns)
constexpr int kGRB = 2;   // 32-row blocks per work item (a WARP's work item: 64 rows x kGC x 32 columns)

// the literal reference expression (fp64, no FMA contraction: library is built with -fmad=false)
__device__ __noinline__ bool tim_consistent_fp64(const float4 ai, const float4 aj, const float4 bi, const float4 bj, double beta) {
  const double ax = (double)aj.x - (double)ai.x, ay = (double)aj.y - (double)ai.y, az = (double)aj.z - (double)ai.z;
  const double bx = (double)bj.x - (double)bi.x, by = (double)bj.y - (double)bi.y, bz = (double)bj.z - (double)bi.z;
  const double v1 = sqrt(ax * ax + ay * ay + az * az);
  const double v2 = sqrt(bx * bx + by * by + bz * bz);
  const double alpha_f = beta * (1.0 / v1);
  const double raw_f = v2 / v1;
  const bool in_f = fabs(raw_f - 1.0) <= alpha_f;
  const double alpha_r = beta * (1.0 / v2);
  const double raw_r = v1 / v2;
  const bool in_r = fabs(raw_r - 1.0) <= alpha_r;
  return in_f && in_r;
}

// 32 x 32 bit transpose across a warp: lane l holds row l; afterwards lane l holds column l
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x) {
  const int lane = lane_id();
#pragma unroll
  for (int s = 16; s >= 1; s >>= 1) {
    const uint32_t mask = s == 16 ? 0x0000FFFFu : s == 8 ? 0x00FF00FFu : s == 4 ? 0x0F0F0F0Fu : s == 2 ? 0x33333333u : 0x55555555u;
    const uint32_t y = __shfl_xor_sync(0xffffffffu, x, s);
    x = (lane & s) ? (((y >> s) & mask) | (x & ~mask)) : ((x & mask) | ((y & mask) << s));
  }
  return x;
}

// WARP work items (64 rows x kGC*32 columns) of the upper triangle of one pair: row group rg meets the column groups q >= rg*kGRB/kGC
// (the first group that is not entirely below the diagonal).  Round 2, first version: a CTA item of 256 rows x 512 columns with the
// rows staged once per CTA -- 29 % of the items of an L = 3000 pair touch the diagonal, where one of the four warps has half the work,
// and the barrier around the staging was the top stall reason (1.5 warps per issue).  Every warp now stages its own 64 rows
// (~1 % of the item's instructions) and no barrier is left in the item loop.
__device__ __forceinline__ int graph_items(int L) {
  if (L <= 0) return 0;
  const int nb = (L + 31) >> 5, ncq = (nb + kGC - 1) / kGC, nrg = (nb + kGRB - 1) / kGRB;
  int t = 0;
  for (int rg = 0; rg < nrg; ++rg) t += max(0, ncq - rg * kGRB / kGC);
  return t;
}

constexpr int kGraphMaxPairs = 2048;  // = the largest max_batch_slots qb200_create accepts

__global__ void __launch_bounds__(kGW * 32, 4) tim_graph_kernel(const float4* __restrict__ ma, const float4* __restrict__ mb,
                                                                const int* __restrict__ n_corr, int n_pairs, int Lc, int W,
                                                                const PairSolve* __restrict__ solve, uint32_t* __restrict__ adj) {
  __shared__ float4 s_row[kGW][kGRB * 32][2];  // per warp and row: (-2a, |a|^2 - beta^2/4) | (-2b, |b|^2 - beta^2/4)
  __shared__ int s_pref[kGraphMaxPairs + 1];   // exclusive prefix of the pairs' item counts: the warps stride over ALL pairs' items,
  __shared__ int s_scan[33];                   // so a pair with many correspondences is spread over the whole grid
  __shared__ GraphConst s_gc[kGW];             // per warp: the constants of its item's pair (read at their uses, like launch constants)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  {
    int carry = 0;
    for (int base = 0; base < n_pairs; base += kGW * 32) {
      const int p = base + tid;
      const int c = (p < n_pairs && solve[p].mode != QB200_INLIER_NONE) ? graph_items(n_corr[p]) : 0;  // INLIER_NONE: no graph
      int tot;
      const int ex = block_excl_scan(c, s_scan, &tot);
      if (p < n_pairs) s_pref[p] = carry + ex;
      carry += tot;
    }
    if (tid == 0) s_pref[n_pairs] = carry;
    __syncthreads();
  }
  const int total_items = s_pref[n_pairs];
  float4(* __restrict__ row_w)[2] = s_row[warp];

  for (int g = blockIdx.x * kGW + warp; g < total_items; g += gridDim.x * kGW) {
    int lo = 0, hi = n_pairs - 1;  // the pair that owns item g (warp-uniform binary search)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_pref[mid] <= g) lo = mid; else hi = mid - 1;
    }
    const int pair = lo;
    const int L = n_corr[pair];
    const int nb = (L + 31) >> 5;                  // 32-wide blocks per side
    const int ncq = (nb + kGC - 1) / kGC;          // column groups of kGC blocks
    int item = g - s_pref[pair], rg = 0;
    for (;; ++rg) {
      const int cnt = max(0, ncq - rg * kGRB / kGC);
      if (item < cnt) break;
      item -= cnt;
    }
    const int cb0 = (rg * kGRB / kGC + item) * kGC;  // first column block of this item
    const float4* __restrict__ A = ma + (size_t)pair * Lc;
    const float4* __restrict__ B = mb + (size_t)pair * Lc;
    uint32_t* __restrict__ G = adj + (size_t)pair * Lc * W;
    // ---- this warp's rows
    float mmr[kGRB];
    __syncwarp();
    if (lane == 0) s_gc[warp] = solve[pair].gc;  // the pair's own beta
    __syncwarp();
    const volatile GraphConst& gc = s_gc[warp];  // volatile: loaded at every use, no register held across the item
#pragma unroll
    for (int rb = 0; rb < kGRB; ++rb) {
      const int i = (rg * kGRB + rb) * 32 + lane;
      const bool v = i < L;
      const float4 pa = v ? A[i] : zero4, pb = v ? B[i] : zero4;
      const float na = fmaf(pa.z, pa.z, fmaf(pa.y, pa.y, pa.x * pa.x));
      const float nbn = fmaf(pb.z, pb.z, fmaf(pb.y, pb.y, pb.x * pb.x));
      row_w[rb * 32 + lane][0] = make_float4(-2.0f * pa.x, -2.0f * pa.y, -2.0f * pa.z, na - gc.hb2q);
      row_w[rb * 32 + lane][1] = make_float4(-2.0f * pb.x, -2.0f * pb.y, -2.0f * pb.z, nbn - gc.hb2q);
      float m = na + nbn;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      mmr[rb] = m;
    }
    __syncwarp();
    // ---- this lane's columns
    float4 ca[kGC], cb[kGC];
    float cm[kGC];
    bool cv[kGC];
#pragma unroll
    for (int c = 0; c < kGC; ++c) {
      const int j = (cb0 + c) * 32 + lane;
      cv[c] = j < L;
      const float4 pa = cv[c] ? A[j] : zero4, pb = cv[c] ? B[j] : zero4;
      const float na = fmaf(pa.z, pa.z, fmaf(pa.y, pa.y, pa.x * pa.x));
      const float nbn = fmaf(pb.z, pb.z, fmaf(pb.y, pb.y, pb.x * pb.x));
      ca[c] = make_float4(pa.x, pa.y, pa.z, na - gc.hb2q);
      cb[c] = make_float4(pb.x, pb.y, pb.z, nbn - gc.hb2q);
      cm[c] = na + nbn;
    }
    const float ntwob2 = -gc.twob2, nb4 = -gc.b4;
#pragma unroll
    for (int rbl = 0; rbl < kGRB; ++rbl) {
      const int bi = rg * kGRB + rbl;
      if (bi >= nb) break;
      if (cb0 + kGC - 1 < bi) continue;  // all column blocks below the diagonal (warp-uniform)
      const float mm = mmr[rbl];
      float qa[kGC], qk[kGC], Mj[kGC];
#pragma unroll
      for (int c = 0; c < kGC; ++c) {
        Mj[c] = (mm + cm[c] + gc.two_b2_slack) * 1.00001f;
        qa[c] = gc.c1 * Mj[c];
        qk[c] = (gc.c2 * Mj[c] + gc.c3) * Mj[c];
      }
      uint32_t wt[kGC], ws[kGC], wa[kGC];
      float smin[kGC];
#pragma unroll
      for (int c = 0; c < kGC; ++c) { wt[c] = ws[c] = wa[c] = 0u; smin[c] = 3.0e38f; }
      const float4(* __restrict__ row_p)[2] = row_w + rbl * 32;
#pragma unroll 8
      for (int r = 0; r < 32; ++r) {
        const float4 r0 = row_p[r][0], r1 = row_p[r][1];
#pragma unroll
        for (int c = 0; c < kGC; ++c) {
          const float Ap = __fmaf_rn(r0.x, ca[c].x, __fmaf_rn(r0.y, ca[c].y, __fmaf_rn(r0.z, ca[c].z, __fadd_rn(r0.w, ca[c].w))));
          const float Bp = __fmaf_rn(r1.x, cb[c].x, __fmaf_rn(r1.y, cb[c].y, __fmaf_rn(r1.z, cb[c].z, __fadd_rn(r1.w, cb[c].w))));
          const float D = __fsub_rn(Ap, Bp), sp = __fadd_rn(Ap, Bp);
          const float ng = __fmaf_rn(ntwob2, sp, nb4);           // -g = -(2 beta^2 s' + beta^4)
          const float t = __fmaf_rn(D, D, ng);
          // |t| - q, q = |D| c1 M + K (|.| is an operand modifier)
          const float w = fabsf(t) - fmaf(fabsf(D), qa[c], qk[c]);
          wt[c] = __funnelshift_l(__float_as_uint(t), wt[c], 1);    // sign(t):  t < 0
          ws[c] = __funnelshift_l(__float_as_uint(sp), ws[c], 1);   // sign(s'): s' < 0
          wa[c] = __funnelshift_l(__float_as_uint(w), wa[c], 1);    // |t| inside the error band
          smin[c] = fminf(smin[c], sp);
        }
      }
      const int nvalid = L - bi * 32;
      const uint32_t rows_ok = nvalid >= 32 ? ~0u : ((1u << nvalid) - 1u);
#pragma unroll
      for (int c = 0; c < kGC; ++c) {
        const int cbk = cb0 + c;
        if (cbk < bi || cbk >= nb) continue;  // warp-uniform
        uint32_t e = __brev(wt[c] | ws[c]);   // row 0 was shifted in first
        uint32_t am = __brev(wa[c]);
        uint32_t live = cv[c] ? rows_ok : 0u;
        if (cbk == bi) live &= ~(1u << lane);  // i == j
        // both squared distances ~0 (s' ~ -beta^2): the literal expression is 0/0 for coincident duplicates -> ask it
        float sm = smin[c];
        if (cbk == bi) {  // the diagonal pairs (i == j) sit at s' = -beta^2 themselves: redo the minimum without them
          sm = 3.0e38f;
#pragma unroll 1
          for (int r = 0; r < 32; ++r) {
            const float4 r0 = row_p[r][0], r1 = row_p[r][1];
            const float Ap = fmaf(r0.x, ca[c].x, fmaf(r0.y, ca[c].y, fmaf(r0.z, ca[c].z, r0.w + ca[c].w)));
            const float Bp = fmaf(r1.x, cb[c].x, fmaf(r1.y, cb[c].y, fmaf(r1.z, cb[c].z, r1.w + cb[c].w)));
            if (r != lane) sm = fminf(sm, Ap + Bp);
          }
        }
        // M beyond 2^62 (or inf / NaN): D^2, 2 beta^2 s' or q may overflow, and the band no longer bounds the error (DESIGN 5.2)
        if (sm <= fmaf(64.0f * 5.9604645e-8f, Mj[c], -gc.b2) || !(Mj[c] <= 0x1p62f)) am = ~0u;
        am &= live;
        if (am) {
          const int j = cbk * 32 + lane;
          const float4 aj = A[j], bj = B[j];
          while (am) {
            const int r = __ffs(am) - 1;
            am &= am - 1;
            const int i = bi * 32 + r;
            const bool ok = tim_consistent_fp64(A[i], aj, B[i], bj, gc.beta);
            e = ok ? (e | (1u << r)) : (e & ~(1u << r));
          }
        }
        e &= live;
        // transposed half: row j, word bi.   row-major half: row (bi*32 + lane), word cbk.
        if (cv[c]) G[(size_t)(cbk * 32 + lane) * W + bi] = e;
        if (cbk != bi) {
          const uint32_t tr = warp_transpose32(e);
          const int irow = bi * 32 + lane;
          if (irow < L) G[(size_t)irow * W + cbk] = tr;
        }
      }
    }
  }
}

// degrees + edge count (one warp per row)
__global__ void __launch_bounds__(256) degree_kernel(uint32_t* __restrict__ adj, const int* __restrict__ n_corr, int Lc, int W,
                                                     const PairSolve* __restrict__ solve, int* __restrict__ deg, long long* __restrict__ n_edges) {
  const int pair = blockIdx.y;
  if (solve[pair].mode == QB200_INLIER_NONE) return;  // n_edges stays 0, as when the whole wave skips K8
  const int L = n_corr[pair];
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= L) return;
  const int nb = (L + 31) >> 5;
  uint32_t* __restrict__ G = adj + ((size_t)pair * Lc + row) * W;
  int d = 0;
  for (int w = lane_id(); w < nb; w += 32) d += __popc(G[w]);  // words beyond ceil(L/32) are never read by any consumer: leaving them
                                                               // untouched keeps the wave's adjacency footprint (L * nb words per pair) inside the L2
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if (lane_id() == 0) {
    deg[(size_t)pair * Lc + row] = d;
    atomicAdd((unsigned long long*)(n_edges + pair), (unsigned long long)d);  // 2E; halved by the reader
  }
}

int launch_degree(Lane* h, int n_pairs) {
  if (n_pairs <= 0) return QB200_OK;
  const dim3 gd((h->Lc + 7) / 8, n_pairs);
  degree_kernel<<<gd, 256, 0, h->stream>>>(h->adj, h->ctr.n_corr, h->Lc, h->W, h->d_solve, h->deg, h->ctr.n_edges);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

// ---- caller graphs (qb200_max_clique_batch_each): the adjacency of a graph wave from the caller's edge lists or rows ----------------
// Every kernel finds graph g's entry in the wave's table (GraphSrc) and writes only the L rows, ceil(L / 32) words each, that K9 reads.

// a graph is invalid: its status, and a mode that every K9 kernel skips (degree_kernel leaves its n_edges 0)
__device__ __forceinline__ void refuse_graph(int g, PairSolve* __restrict__ solve, int* __restrict__ status) {
  status[g] = QB200_ERR_BAD_ARG;
  solve[g].mode = QB200_INLIER_NONE;
}

constexpr int kImportThreads = 256;

// blockIdx.y = graph: its rows into its slot, the bits at columns >= L cleared; an edge-list graph (rows == nullptr) gets zeros, which
// edge_import_kernel then fills.  Host rows were copied into the slot beforehand and are masked in place.
__global__ void __launch_bounds__(kImportThreads) row_import_kernel(const GraphSrc* __restrict__ table, int Lc, int W, uint32_t* __restrict__ adj) {
  const int g = blockIdx.y;
  const GraphSrc s = table[g];
  const int nb = (s.L + 31) >> 5;
  const long long words = (long long)s.L * nb;
  const uint32_t last = (s.L & 31) ? (1u << (s.L & 31)) - 1u : ~0u;
  uint32_t* __restrict__ G = adj + (size_t)g * Lc * W;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / nb), w = (int)(i % nb);
    uint32_t x = 0u;
    if (s.rows) {
      x = s.rows[(size_t)r * s.stride + w];
      if (w == nb - 1) x &= last;
    }
    G[(size_t)r * W + w] = x;
  }
}

// Grid over (edge chunk, graph): both bits of every edge (u, v) with 0 <= u, v < L and u != v; any other edge refuses the graph.
// only < 0: blockIdx.y = graph, its edges from its table entry (nullptr: none in this launch); only >= 0: graph `only`, n edges at e.
// atomicOr makes repeated edges and both orientations of one edge set the same two bits, so neither order nor chunking matters.
__global__ void __launch_bounds__(kImportThreads) edge_import_kernel(const GraphSrc* __restrict__ table, int only, const int2* __restrict__ e,
                                                                     long long n, int Lc, int W, uint32_t* __restrict__ adj,
                                                                     PairSolve* __restrict__ solve, int* __restrict__ status) {
  const int g = only >= 0 ? only : blockIdx.y;
  if (only < 0) {
    e = table[g].edges;
    n = table[g].n_edges;
  }
  if (!e) return;
  const int L = table[g].L;
  uint32_t* __restrict__ G = adj + (size_t)g * Lc * W;
  bool bad = false;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int2 uv = e[i];
    if ((unsigned)uv.x >= (unsigned)L || (unsigned)uv.y >= (unsigned)L || uv.x == uv.y) {
      bad = true;
      continue;
    }
    atomicOr(&G[(size_t)uv.x * W + (uv.y >> 5)], 1u << (uv.y & 31));
    atomicOr(&G[(size_t)uv.y * W + (uv.x >> 5)], 1u << (uv.x & 31));
  }
  if (bad) refuse_graph(g, solve, status);
}

// One warp per 32 x 32 tile (bi, bj >= bi) of a row graph: lane l holds row bi*32 + l of tile (bi, bj) and row bj*32 + l of tile
// (bj, bi); the transpose of the first (warp_transpose32) must equal the second, and a diagonal tile must have no bit (i, i).  Rows
// at or past L count as empty (row_import_kernel cleared their columns in the rows below L).
constexpr int kCheckWarps = 8;
__global__ void __launch_bounds__(kCheckWarps * 32) symmetry_check_kernel(const GraphSrc* __restrict__ table, int Lc, int W,
                                                                          const uint32_t* __restrict__ adj, PairSolve* __restrict__ solve,
                                                                          int* __restrict__ status) {
  const int g = blockIdx.y, lane = lane_id();
  const GraphSrc s = table[g];
  if (!s.rows) return;  // edge lists are symmetric and loop-free by construction
  const int L = s.L, nb = (L + 31) >> 5;
  const uint32_t* __restrict__ G = adj + (size_t)g * Lc * W;
  bool fault = false;
  for (long long t = (long long)blockIdx.x * kCheckWarps + (threadIdx.x >> 5); t < (long long)nb * nb; t += (long long)gridDim.x * kCheckWarps) {
    const int bi = (int)(t / nb), bj = (int)(t % nb);
    if (bj < bi) continue;  // warp-uniform: the lower tiles are the transposes of the upper ones
    const int ri = bi * 32 + lane, rj = bj * 32 + lane;
    const uint32_t a = ri < L ? G[(size_t)ri * W + bj] : 0u;
    const uint32_t b = rj < L ? G[(size_t)rj * W + bi] : 0u;
    fault |= warp_transpose32(a) != b;
    if (bi == bj) fault |= ((a >> lane) & 1u) != 0u;
  }
  if (__any_sync(0xffffffffu, fault) && lane == 0) refuse_graph(g, solve, status);
}

// One thread per graph: the record of a graph wave.  A refused graph keeps its status and zero counters (K9 skipped it).
__global__ void clique_records_kernel(qb200_result* __restrict__ results, int n_graphs, WaveCounters c) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_graphs) return;
  qb200_result* r = results + g;
  r->valid = 0;
  r->status = c.cloud_status[g];
  r->n_src_vox = 0;
  r->n_tgt_vox = 0;
  r->n_mutual = 0;
  r->n_corr = c.n_corr[g];
  r->max_core = c.max_core[g];
  r->clique_size = c.n_clique[g];
  r->gnc_iters = 0;
  r->n_rot_inliers = 0;
  r->n_final_inliers = 0;
  r->flags = c.flags[g];
  r->n_edges = c.n_edges[g] / 2;
  r->cost = 0.0;
  for (int i = 0; i < 16; ++i) r->T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

// enough CTAs to cover `items` per graph at one item per thread, at most 4096 (the kernels stride)
static unsigned import_ctas(long long items) {
  const long long b = (items + kImportThreads - 1) / kImportThreads;
  return (unsigned)(b < 1 ? 1 : b > 4096 ? 4096 : b);
}

int launch_row_import(Lane* h, int n_graphs, int max_L) {
  if (n_graphs <= 0) return QB200_OK;
  const long long nb = (max_L + 31) / 32;
  row_import_kernel<<<dim3(import_ctas((long long)max_L * nb), n_graphs), kImportThreads, 0, h->stream>>>(h->d_graph, h->Lc, h->W, h->adj);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_edge_import(Lane* h, int n_graphs, long long max_edges, int only, const int2* edges) {
  if (n_graphs <= 0 || max_edges <= 0) return QB200_OK;
  const dim3 grid(import_ctas(max_edges), only >= 0 ? 1 : n_graphs);
  edge_import_kernel<<<grid, kImportThreads, 0, h->stream>>>(h->d_graph, only, edges, max_edges, h->Lc, h->W, h->adj, h->d_solve,
                                                             h->ctr.cloud_status);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_symmetry_check(Lane* h, int n_graphs, int max_L) {
  if (n_graphs <= 0 || max_L <= 0) return QB200_OK;
  const long long nb = (max_L + 31) / 32, warps_ctas = (nb * nb + kCheckWarps - 1) / kCheckWarps;
  const unsigned ctas = (unsigned)(warps_ctas > 8192 ? 8192 : warps_ctas);
  symmetry_check_kernel<<<dim3(ctas, n_graphs), kCheckWarps * 32, 0, h->stream>>>(h->d_graph, h->Lc, h->W, h->adj, h->d_solve,
                                                                                   h->ctr.cloud_status);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_clique_records(Lane* h, int n_graphs) {
  if (n_graphs <= 0) return QB200_OK;
  clique_records_kernel<<<(n_graphs + 127) / 128, 128, 0, h->stream>>>(h->d_results, n_graphs, h->ctr);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

// ---- TIM graphs handed out (qb200_build_graph_batch_each): K8's rows, degrees and edge lists into caller layouts ------------------
// K8 writes words 0 .. ceil(L / 32) - 1 of a set's L rows and degree_kernel reads only those: the words past them hold whatever an
// earlier wave left there, so every kernel below reads the first ceil(L / 32) words of a row and nothing else.

constexpr int kExportThreads = 256;

// Grid over (chunk, set): set g's L rows with words_per_row words each (the words from ceil(L / 32) on as zero) and its L degrees
__global__ void __launch_bounds__(kExportThreads) graph_export_kernel(const int* __restrict__ n_corr, int Lc, int W,
                                                                      const uint32_t* __restrict__ adj, const int* __restrict__ deg,
                                                                      GraphDst d) {
  const int g = blockIdx.y, L = n_corr[g], nb = (L + 31) >> 5, wpr = d.words_per_row;
  const uint32_t* __restrict__ G = adj + (size_t)g * Lc * W;
  const long long t0 = (long long)blockIdx.x * blockDim.x + threadIdx.x, step = (long long)gridDim.x * blockDim.x;
  if (d.adj) {
    uint32_t* __restrict__ out = d.adj + (size_t)g * d.rows_per_set * wpr;
    for (long long i = t0; i < (long long)L * wpr; i += step) {
      const int r = (int)(i / wpr), w = (int)(i % wpr);
      out[i] = w < nb ? G[(size_t)r * W + w] : 0u;
    }
  }
  if (d.degree)
    for (long long r = t0; r < L; r += step) d.degree[(size_t)g * d.rows_per_set + r] = deg[(size_t)g * Lc + r];
}

// the bits j > i of word w of row i
__device__ __forceinline__ uint32_t upper_bits(int i, int w, uint32_t x) {
  const int wi = i >> 5, b = i & 31;
  return w > wi ? x : w < wi || b == 31 ? 0u : x & (~0u << (b + 1));
}

// One CTA per set (blockIdx.x): off[i] = the edges (u, v), u < v, of the rows before i, and off[L] = all of them, at g * off_stride.
// A warp per row counts its upper bits; the CTA then scans the counts in place, kEdgeScanThreads rows at a time.
constexpr int kEdgeScanThreads = 1024;
__global__ void __launch_bounds__(kEdgeScanThreads) edge_offsets_kernel(const int* __restrict__ n_corr, int Lc, int W,
                                                                        const uint32_t* __restrict__ adj, int* __restrict__ off,
                                                                        int off_stride) {
  __shared__ int s_scan[33];
  const int g = blockIdx.x, L = n_corr[g], nb = (L + 31) >> 5, lane = lane_id(), warp = threadIdx.x >> 5;
  const uint32_t* __restrict__ G = adj + (size_t)g * Lc * W;
  int* __restrict__ o = off + (size_t)g * off_stride;
  for (int i = warp; i < L; i += kEdgeScanThreads / 32) {
    int c = 0;
    for (int w = (i >> 5) + lane; w < nb; w += 32) c += __popc(upper_bits(i, w, G[(size_t)i * W + w]));
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) c += __shfl_xor_sync(0xffffffffu, c, s);
    if (lane == 0) o[i] = c;
  }
  __syncthreads();
  int carry = 0;
  for (int base = 0; base < L; base += kEdgeScanThreads) {
    const int i = base + threadIdx.x;
    int tot;
    const int ex = block_excl_scan(i < L ? o[i] : 0, s_scan, &tot);
    if (i < L) o[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) o[L] = carry;
}

// Grid over (row chunk, set), a warp per row: row i's edges (i, j), j > i, in ascending j, at their indices off[i] .. off[i + 1] - 1 of
// the set's list; only the indices in [e0, e1) are written, at out + index - e0.  only < 0: blockIdx.y = set g, whose window starts at
// out + g * out_stride; only >= 0: set `only` alone.  A lane takes one word of 32 and finds where its edges start from a warp prefix
// of the words' popcounts.
constexpr int kEmitWarps = 8;
__global__ void __launch_bounds__(kEmitWarps * 32) edge_emit_kernel(const int* __restrict__ n_corr, int Lc, int W,
                                                                    const uint32_t* __restrict__ adj, const int* __restrict__ off,
                                                                    int off_stride, int only, long long e0, long long e1,
                                                                    int2* __restrict__ out, long long out_stride) {
  const int g = only >= 0 ? only : blockIdx.y, L = n_corr[g], nb = (L + 31) >> 5, lane = lane_id();
  const uint32_t* __restrict__ G = adj + (size_t)g * Lc * W;
  const int* __restrict__ o = off + (size_t)g * off_stride;
  if (only < 0) out += (size_t)g * out_stride;
  for (int i = blockIdx.x * kEmitWarps + (threadIdx.x >> 5); i < L; i += gridDim.x * kEmitWarps) {
    long long idx = o[i];
    if (idx >= e1 || o[i + 1] <= e0 || o[i + 1] == idx) continue;  // warp-uniform: no edge of this row falls in the window
    for (int w0 = i >> 5; w0 < nb && idx < e1; w0 += 32) {
      const int w = w0 + lane;
      uint32_t x = w < nb ? upper_bits(i, w, G[(size_t)i * W + w]) : 0u;
      const int c = __popc(x);
      int tot;
      long long k = idx + warp_excl_scan(c, &tot);
      for (; x; x &= x - 1, ++k)
        if (k >= e0 && k < e1) out[k - e0] = make_int2(i, w * 32 + __ffs(x) - 1);
      idx += tot;
    }
  }
}

// One thread per set: the record of a graph wave.  cap_edges > 0: the set's edge list holds cap_edges entries.
__global__ void graph_records_kernel(qb200_result* __restrict__ results, int n_sets, WaveCounters c, long long cap_edges) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_sets) return;
  qb200_result* r = results + g;
  const long long e = c.n_edges[g] / 2;
  memset(r, 0, sizeof(*r));
  r->status = QB200_OK;
  r->n_corr = c.n_corr[g];
  r->n_edges = e;
  r->flags = cap_edges > 0 && e > cap_edges ? QB200_FLAG_LISTS_TRUNCATED : 0;
  for (int i = 0; i < 16; ++i) r->T[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

int launch_graph_export(Lane* h, int n_sets, const GraphDst& d) {
  if (n_sets <= 0 || (!d.adj && !d.degree)) return QB200_OK;
  const long long words = (long long)h->Lc * (d.adj ? d.words_per_row : 1);
  const long long b = (words + kExportThreads - 1) / kExportThreads;
  const unsigned ctas = (unsigned)(b < 1 ? 1 : b > 2048 ? 2048 : b);
  graph_export_kernel<<<dim3(ctas, n_sets), kExportThreads, 0, h->stream>>>(h->ctr.n_corr, h->Lc, h->W, h->adj, h->deg, d);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_edge_offsets(Lane* h, int n_sets) {
  if (n_sets <= 0) return QB200_OK;
  edge_offsets_kernel<<<n_sets, kEdgeScanThreads, 0, h->stream>>>(h->ctr.n_corr, h->Lc, h->W, h->adj, h->korder, h->Lc + 2);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_edge_emit(Lane* h, int n_sets, int only, long long e0, long long e1, int2* out, long long out_stride) {
  if (n_sets <= 0 || e1 <= e0) return QB200_OK;
  const unsigned ctas = (unsigned)((h->Lc + kEmitWarps - 1) / kEmitWarps);
  edge_emit_kernel<<<dim3(ctas, only >= 0 ? 1 : n_sets), kEmitWarps * 32, 0, h->stream>>>(h->ctr.n_corr, h->Lc, h->W, h->adj, h->korder,
                                                                                          h->Lc + 2, only, e0, e1, out, out_stride);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

int launch_graph_records(Lane* h, int n_sets, long long cap_edges) {
  if (n_sets <= 0) return QB200_OK;
  graph_records_kernel<<<(n_sets + 127) / 128, 128, 0, h->stream>>>(h->d_results, n_sets, h->ctr, cap_edges);
  h->launches++;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

GraphConst graph_const(double noise_bound, double cbar2) {
  const double beta = 2 * noise_bound * sqrt(cbar2);  // quatro.hpp:367
  const double u = 5.9604644775390625e-8;             // 2^-24
  GraphConst gc;
  gc.beta = beta;
  gc.b2 = (float)(beta * beta);
  gc.hb2q = 0.25f * gc.b2;
  gc.twob2 = 2.0f * gc.b2;
  gc.b4 = gc.b2 * gc.b2;
  gc.c1 = (float)(36.0 * u * 1.02);
  gc.c2 = (float)(1500.0 * u * u * 1.02);
  gc.c3 = (float)(46.0 * u * beta * beta * 1.02);
  gc.two_b2_slack = (float)(2.0 * beta * beta * 1.00001);
  return gc;
}

int launch_graph(Lane* h, int n_pairs) {
  if (n_pairs <= 0) return QB200_OK;
  // one wave of resident CTAs whose warps stride over every pair's work items (64 rows x 128 columns each)
  cudaEventRecord(h->kev[2], h->stream);
  tim_graph_kernel<<<dim3(h->n_sm * 4), kGW * 32, 0, h->stream>>>(h->ma, h->mb, h->ctr.n_corr, n_pairs, h->Lc, h->W, h->d_solve, h->adj);
  cudaEventRecord(h->kev[3], h->stream);
  h->kev_armed[1] = 1;
  const dim3 gd((h->Lc + 7) / 8, n_pairs);
  degree_kernel<<<gd, 256, 0, h->stream>>>(h->adj, h->ctr.n_corr, h->Lc, h->W, h->d_solve, h->deg, h->ctr.n_edges);
  h->launches += 2;
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
