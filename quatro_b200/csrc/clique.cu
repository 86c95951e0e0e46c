// clique.cu -- K9: k-core decomposition + PMC heuristic maximum clique on the bit adjacency.  sm_90a
//
// Replaces teaser::MaxCliqueSolver::findMaxClique (src/graph.cc:12-130) and the pmc routines it
// calls ([EXT] pmc_graph::compute_cores, pmc_heu::search with heu_strat = "kcore").  pmc is
// downloaded by the reference's build and absent here; the semantics restated are:
//   * Batagelj-Zaversnik peeling with pmc's bucket mechanics (vertices in id order inside a bin;
//     a decremented vertex is swapped with the first vertex of its bin) -> kcore[v] = core(v)+1 and
//     the peel order;
//   * for start vertices in reverse peel order: P = {u in adj(v): kcore[u] > mc}; if |P| > mc the
//     greedy descent pops the candidate with the largest (kcore, id) and intersects P with its
//     neighbourhood until P is empty; a longer chain replaces the incumbent; stop at mc >= max_core+1.
// The reference runs the start vertices on 12 racy OpenMP threads; like the CPU oracle these kernels
// reproduce the SEQUENTIAL semantics (SURVEY.md 8c) bit for bit.  One CTA per registration pair:
//
//   kcore_kernel  The peel stays a sequence of L steps (the order is the output); a step is parallel inside: `above` (bitset of
//     vertices whose current degree exceeds the current level) turns "neighbour with deg[u] > deg[v]" into one AND; the surviving
//     neighbours are expanded to an ascending list with one warp scan and every neighbour's bucket move is done by its own lane.
//     Moves into different buckets commute; the members of one bucket (same current degree) must be applied in id order: their
//     ranks come from __match_any_sync, and with the ranks known the moves of a group have a closed form (member t lands on slot
//     bin+t; the non-members displaced from the target slots take the old slots of the members that sat outside, found by a short
//     chain walk) -- no serial replay.  Small graphs (L up to ~700) run on ONE warp with the whole adjacency in shared memory and
//     no block barrier; large graphs split the degree buckets over four warps by residue class (one block barrier per step) and
//     stream rows through a cp.async ring.  (A variant with thread-per-word ownership and five block barriers per step measured
//     3000 cycles per step -- barrier-bound -- and was dropped, DESIGN.md 10.)
//   clique_cta_kernel  The start vertices are tried SPECULATIVELY, one per warp, against the current incumbent size
//     mc; results are committed in sequential order (the first warp that beats mc wins, later warps are discarded and
//     redone), which is exactly the sequential outcome because a descent only depends on mc at its start.  Vertices
//     are renumbered by (kcore, id) rank (permute_adj_kernel), so "largest (kcore,id) candidate" is the highest set
//     bit of P and a descent step is one multi-word AND.
#include "handle.cuh"
#include "kcore_cutoff.cuh"

namespace qb {

__device__ __forceinline__ int warp_max(int v) { return __reduce_max_sync(0xffffffffu, v); }
__device__ __forceinline__ int warp_sum(int v) { return __reduce_add_sync(0xffffffffu, v); }

// stable counting sort of vertices by key[v] (ids ascending inside a bucket); bin[d] ends up as the
// START of bucket d (d = 0..maxkey), bin[maxkey+1] = n.  One warp.
__device__ void warp_bucket_sort(const unsigned short* __restrict__ key, int n, int maxkey, int* __restrict__ bin,
                                 unsigned short* __restrict__ pos, unsigned short* __restrict__ vert) {
  const int lane = lane_id();
  for (int d = lane; d <= maxkey + 1; d += 32) bin[d] = 0;
  __syncwarp();
  for (int v = lane; v < n; v += 32) atomicAdd(&bin[key[v]], 1);
  __syncwarp();
  int carry = 0;
  for (int base = 0; base <= maxkey + 1; base += 32) {  // exclusive scan
    const int d = base + lane;
    const int c = d <= maxkey + 1 ? bin[d] : 0;
    int tot;
    const int ex = warp_excl_scan(c, &tot);
    if (d <= maxkey + 1) bin[d] = carry + ex;
    carry += tot;
  }
  __syncwarp();
  for (int base = 0; base < n; base += 32) {  // placement, ids ascending inside a bucket
    const int v = base + lane;
    const bool act = v < n;
    const int d = act ? key[v] : -1 - lane;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & ((1u << lane) - 1));
    const int b = act ? bin[d] : 0;
    __syncwarp();
    if (act) {
      pos[v] = (unsigned short)(b + rank);
      vert[b + rank] = (unsigned short)v;
      if (rank == 0) bin[d] = b + __popc(peers);
    }
    __syncwarp();
  }
  // bin[d] is now the END of bucket d: shift down to starts (descending chunks)
  for (int base = ((maxkey + 1) / 32) * 32; base >= 0; base -= 32) {
    const int d = base + lane;
    int prev = 0;
    if (d >= 1 && d <= maxkey + 1) prev = bin[d - 1];
    __syncwarp();
    if (d >= 1 && d <= maxkey + 1) bin[d] = prev;
    __syncwarp();
  }
  if (lane == 0) bin[0] = 0;
  __syncwarp();
}

constexpr int kRing = 16;  // rows in flight when the adjacency does not fit in shared memory (covers the DRAM latency at ~15 steps)

__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int kKcWarps = 4;  // warps of the k-core CTA (large graphs: one degree class per warp; small graphs: warp 0 alone)

// Bucket moves of one warp's neighbour list nbl[0..cnt), 32 neighbours at a time.  Moves into different buckets commute; the members
// u_0 < u_1 < ... of one bucket (same current degree, ranks from __match_any_sync) are applied in id order by pmc: "swap u_t with
// the vertex on slot bin + t".  That sequence has a closed form: u_t ends on slot bin + t, and the vertex y that is not a member
// but sat on one of the target slots ends on the old slot of the member found by walking  slot s -> member that sat there -> its
// target slot -> ... ; each member that sat OUTSIDE the target slots walks that chain backwards from its own rank and hands its
// old slot to the non-member it reaches (verified against the sequential mechanic, tests + DESIGN.md 5.3).
// above_own: the calling warp's bitset (neighbours leave it); add_next: bitset that receives neighbours whose new degree is still
// above the level (the same bitset in the single-warp path, the next lower degree class otherwise).
__device__ __forceinline__ void kcore_apply_moves(const unsigned short* __restrict__ nbl, int cnt, int dv, int* __restrict__ bin,
                                                  unsigned short* __restrict__ deg, unsigned short* __restrict__ pos,
                                                  unsigned short* __restrict__ vert, unsigned short* __restrict__ mrk,
                                                  uint32_t* __restrict__ above_own, uint32_t* __restrict__ add_next, bool classes) {
  const int lane = lane_id();
  const unsigned lt = (1u << lane) - 1u;
  for (int c0 = 0; c0 < cnt; c0 += 32) {
    const int e = c0 + lane;
    const bool act = e < cnt;
    const int u = act ? nbl[e] : 0;
    const int du = act ? deg[u] : -1 - lane;
    const unsigned grp = __match_any_sync(0xffffffffu, du);
    const int rank = __popc(grp & lt), m = __popc(grp);
    int b0 = 0, pu = 0;
    if (act) {
      b0 = bin[du];
      pu = pos[u];
      mrk[u] = (unsigned short)(rank + 1);
    }
    __syncwarp();
    int y = -1;  // the non-member that moves to this member's old slot
    if (act && pu >= b0 + m) {
      int curk = rank;
      for (;;) {
        y = vert[b0 + curk];
        const int r = mrk[y];
        if (r == 0) break;
        curk = r - 1;
      }
    }
    __syncwarp();
    if (act) {
      vert[b0 + rank] = (unsigned short)u; pos[u] = (unsigned short)(b0 + rank);
      if (y >= 0) { vert[pu] = (unsigned short)y; pos[y] = (unsigned short)pu; }
      mrk[u] = 0;
      deg[u] = (unsigned short)(du - 1);
      const uint32_t bit = 1u << (u & 31);
      if (classes) {
        atomicAnd(&above_own[u >> 5], ~bit);                       // u leaves this degree class ...
        if (du - 1 > dv) atomicOr(&add_next[u >> 5], bit);         // ... and joins the next lower one unless it reached the level
      } else if (du - 1 == dv) {
        atomicAnd(&above_own[u >> 5], ~bit);
      }
      if (rank == 0) bin[du] = b0 + m;
    }
    __syncwarp();
  }
}

// live words of this lane -> ascending list (word order = (lane, k)); returns the list length
template <int WPL>
__device__ __forceinline__ int kcore_expand(const uint32_t (&w)[WPL], int w0, unsigned short* __restrict__ nbl) {
  int c = 0;
#pragma unroll
  for (int k = 0; k < WPL; ++k) c += __popc(w[k]);
  int cnt;
  int off = warp_excl_scan(c, &cnt);
  if (cnt != 0) {
#pragma unroll
    for (int k = 0; k < WPL; ++k) {
      uint32_t x = w[k];
      const int basebit = (w0 + k) * 32;
      while (x) {
        const int b = __ffs(x) - 1;
        x &= x - 1;
        nbl[off++] = (unsigned short)(basebit + b);
      }
    }
  }
  return cnt;
}

// One CTA of kKcWarps warps per pair.  Lane l owns the nwl = ceil(nbw / 32) CONSECUTIVE adjacency words l * nwl .. l * nwl + nwl - 1 of the
// row being peeled (nwl <= WPL, W <= 32 * WPL), so the ascending neighbour list needs one warp scan per step whatever L is.
//   small graphs (the whole adjacency fits into the shared-memory row area): warp 0 alone, no block barrier at all;
//   large graphs: every warp owns the degree buckets of one residue class (bucket e belongs to warp e mod 4).  A step's events on
//     different buckets commute, so the four warps apply their classes' events concurrently from their own `above` bitsets; a
//     neighbour whose degree drops moves to the next lower class through a double-buffered `add` bitset that the receiving warp
//     merges at the start of the next step -- ONE block barrier per step.  Rows arrive through a cp.async ring of kRing rows (warp 0 prefetches kRing - 1 steps ahead).
// smem: bin (int x (Ls + 2)) | above [4][32 WPL] | add [2][4][32 WPL] | rows [row_words] | deg, pos, vert, mrk (u16 x Ls) | nbl [4][Ls] u16,
// Ls = min(Lc, kKcoreSmemVerts).  A pair with L > Ls keeps bin .. nbl in its slot of `ws` (kcore_ws_bytes(Lc) each, L2-resident) and
// uses the whole shared area behind the bitsets as its prefetch ring: the same code runs on either set of arrays.  The two cases are
// two instances (kWs = false: pairs with L <= Ls, true: the others), so every array access keeps its address space (LDS / LDG).
template <int WPL, bool kWs>
__global__ void __maxnreg__(168) kcore_kernel(const uint32_t* __restrict__ adj, const int* __restrict__ deg_in,
                                                              const int* __restrict__ n_corr, const PairSolve* __restrict__ solve, int Lc, int W,
                                                              int Ls, int row_words, unsigned char* __restrict__ ws, int* __restrict__ kcore,
                                                              int* __restrict__ korder, int* __restrict__ rank_of, int* __restrict__ by_rank,
                                                              int* __restrict__ kbin, int* __restrict__ max_core_out) {
  constexpr int NW = kKcWarps, AW = 32 * WPL;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int ring_tag[kRing];

  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (solve[pair].mode == QB200_INLIER_NONE) return;                 // no graph: iota_clique_kernel fills the pair
  const int L = n_corr[pair];
  if ((L > Ls) != kWs) return;                                       // the other instance runs this pair
  constexpr bool in_smem = !kWs;
  const int Lv = in_smem ? Ls : Lc;                                  // capacity of the per-vertex arrays
  int* bin = in_smem ? reinterpret_cast<int*>(smem_raw)              // [Lv + 2] start of every degree bucket
                     : reinterpret_cast<int*>(ws + (size_t)pair * kcore_ws_bytes(Lc));
  uint32_t* above = in_smem ? reinterpret_cast<uint32_t*>(bin + Ls + 2)  // [NW][AW] vertices with current degree > current level (per class)
                            : reinterpret_cast<uint32_t*>(smem_raw);
  uint32_t* add = above + NW * AW;                                   // [2][NW][AW] arrivals of the next step, by parity
  uint32_t* rows = add + 2 * NW * AW;                                // [row_words] adjacency cache or prefetch ring
  unsigned short* deg = in_smem ? reinterpret_cast<unsigned short*>(rows + row_words) : reinterpret_cast<unsigned short*>(bin + Lc + 2);
  unsigned short* pos = deg + Lv;
  unsigned short* vert = pos + Lv;
  unsigned short* mrk = vert + Lv;                                   // mrk[u] = 1 + rank of u inside its group during a pass, else 0
  unsigned short* nbl_all = mrk + Lv;                                // [NW][Lv] ascending list of a warp's live neighbours of the step
  int* __restrict__ kc = kcore + (size_t)pair * (Lc + 2);
  int* __restrict__ ko = korder + (size_t)pair * (Lc + 2);
  int* __restrict__ ro = rank_of + (size_t)pair * (Lc + 2);
  int* __restrict__ br = by_rank + (size_t)pair * (Lc + 2);
  int* __restrict__ kb = kbin + (size_t)pair * (Lc + 2);
  if (L <= 0) {
    if (tid == 0) max_core_out[pair] = 0;
    return;
  }
  const uint32_t* __restrict__ G = adj + (size_t)pair * Lc * W;
  const int nbw = (L + 31) >> 5;   // adjacency words per row in use
  const int nwl = (nbw + 31) >> 5; // words per lane in use (<= WPL)
  const bool cached = in_smem && (long long)L * nbw <= (long long)row_words;
  const int rs = in_smem ? Ls / 32 : W;  // row stride of the prefetch ring (>= nbw)
  const int w0 = lane * nwl;       // first adjacency word of this lane
  unsigned short* nbl = nbl_all + (size_t)warp * Lv;

  // ---- set-up: degrees, row cache, bucket sort by degree (warp 0 sorts; everybody helps loading) ----
  int md = 0;
  for (int v = tid; v < L; v += NW * 32) {
    const int d = deg_in[(size_t)pair * Lc + v];
    deg[v] = (unsigned short)d;
    mrk[v] = 0;
    md = max(md, d);
  }
  if (cached)  // the peel is a chain of dependent row reads: stage the whole graph once
    for (int idx = tid; idx < L * nbw; idx += NW * 32) rows[idx] = G[(size_t)(idx / nbw) * W + (idx % nbw)];
  for (int wd = tid; wd < 3 * NW * AW; wd += NW * 32) above[wd] = 0u;  // above + add
  __shared__ int s_md[NW];
  md = warp_max(md);
  if (lane == 0) s_md[warp] = md;
  __syncthreads();
  md = max(max(s_md[0], s_md[1]), max(s_md[2], s_md[3]));
  if (warp == 0) warp_bucket_sort(deg, L, md, bin, pos, vert);
  __syncthreads();
  // membership of `above`: everything (single-warp path) / by degree class
  for (int v = tid; v < L; v += NW * 32) {
    const int c = cached ? 0 : (int)deg[v] % NW;
    atomicOr(&above[c * AW + (v >> 5)], 1u << (v & 31));
  }
  __syncthreads();

  int cur = -1;  // current level: every vertex with degree <= cur has its bit in `above` cleared
  if (cached) {
    // ================= small graph: warp 0 alone, rows from the cache, no block barrier =================
    if (warp != 0) return;
    for (int i = 0; i < L; ++i) {
      const int v = vert[i];
      const int dv = deg[v];
      if (dv > cur) {  // level rise: bucket dv = positions [i, bin[dv+1]) leaves `above`
        const int end = bin[dv + 1];
        for (int p = i + lane; p < end; p += 32) {
          const int x = vert[p];
          atomicAnd(&above[x >> 5], ~(1u << (x & 31)));
        }
        cur = dv;
        __syncwarp();
      }
      uint32_t w[WPL];
#pragma unroll
      for (int k = 0; k < WPL; ++k) w[k] = (k < nwl && w0 + k < nbw) ? (rows[v * nbw + w0 + k] & above[w0 + k]) : 0u;
      const int cnt = kcore_expand<WPL>(w, w0, nbl);
      if (cnt == 0) continue;
      __syncwarp();
      kcore_apply_moves(nbl, cnt, dv, bin, deg, pos, vert, mrk, above, above, false);
    }
  } else {
    // ================= large graph: one degree class per warp, rows through the cp.async ring =================
    uint32_t* above_w = above + warp * AW;                                  // buckets e with e % NW == warp
    const int lower = (warp + NW - 1) % NW;                                 // class that receives my neighbours after a decrement
    auto fetch = [&](int p) {  // warp 0: prefetch the row of the vertex that sits at position p right now into its ring slot
      if (p < L) {
        const int x = vert[p], sl = p % kRing;
        if (lane == 0) ring_tag[sl] = x;
#pragma unroll
        for (int k = 0; k < WPL; ++k)
          if (k < nwl && w0 + k < nbw) cp_async4(rows + sl * rs + w0 + k, G + (size_t)x * W + w0 + k);
      }
      cp_async_commit();
    };
    if (warp == 0) {
      for (int p = 0; p < kRing - 1; ++p) fetch(p);
      cp_async_wait<kRing - 2>();  // position 0 has landed
    }
    __syncthreads();
    for (int i = 0; i < L; ++i) {
      const int v = vert[i];
      const int dv = deg[v];
      const int par = i & 1;
      if (warp == 0) fetch(i + kRing - 1);  // into the slot of step i - 1, which every warp left before the last barrier
      // arrivals of the previous step (written by the next higher class) join my bitset
      uint32_t* add_in = add + ((par ^ 1) * NW + warp) * AW;
      uint32_t w[WPL];
      const int sl = i % kRing;
      const bool hit = ring_tag[sl] == v;  // positions inside the current bucket are final: the prefetch usually holds the right row
#pragma unroll
      for (int k = 0; k < WPL; ++k) {
        w[k] = 0u;
        if (k < nwl && w0 + k < nbw) {
          const uint32_t a = add_in[w0 + k];
          if (a) { above_w[w0 + k] |= a; add_in[w0 + k] = 0u; }
          w[k] = hit ? rows[sl * rs + w0 + k] : G[(size_t)v * W + w0 + k];
        }
      }
      __syncwarp();
      if (dv > cur) {  // level rise: bucket dv leaves `above` -- it lives in class dv % NW only
        if (dv % NW == warp) {
          const int end = bin[dv + 1];
          for (int p = i + lane; p < end; p += 32) {
            const int x = vert[p];
            atomicAnd(&above_w[x >> 5], ~(1u << (x & 31)));
          }
          __syncwarp();
        }
        cur = dv;
      }
#pragma unroll
      for (int k = 0; k < WPL; ++k) w[k] = (k < nwl && w0 + k < nbw) ? (w[k] & above_w[w0 + k]) : 0u;
      const int cnt = kcore_expand<WPL>(w, w0, nbl);
      if (cnt != 0) {
        __syncwarp();
        kcore_apply_moves(nbl, cnt, dv, bin, deg, pos, vert, mrk, above_w, add + (par * NW + lower) * AW, true);
      }
      if (warp == 0) cp_async_wait<kRing - 2>();  // the row of position i + 1 has landed
      __syncthreads();  // every class is done with step i: vert / deg / add are consistent, the next row is visible
    }
    if (warp == 0) cp_async_wait<0>();
    if (warp != 0) return;
  }
  __syncwarp();
  // ---- outputs (warp 0): kcore = core + 1, peel order, max core ----
  const int max_core = deg[vert[L - 1]];
  for (int v = lane; v < L; v += 32) {
    kc[v] = (int)deg[v] + 1;
    ko[v] = vert[v];
  }
  if (lane == 0) max_core_out[pair] = max_core;
  __syncwarp();
  // ---- (kcore, id) ranks for the clique search: stable bucket sort by core number ----
  warp_bucket_sort(deg, L, max_core, bin, pos, vert);
  for (int v = lane; v < L; v += 32) {
    ro[v] = pos[v];
    br[v] = vert[v];
  }
  for (int d = lane; d <= max_core + 1; d += 32) kb[d] = bin[d];
}

// adjacency rows/columns renumbered by rank: adjp[rank(v)] bit rank(u) = adj[v] bit u.  One warp per row.
__global__ void __launch_bounds__(256) permute_adj_kernel(const uint32_t* __restrict__ adj, const int* __restrict__ n_corr, int Lc, int W,
                                                          const PairSolve* __restrict__ solve, const int* __restrict__ rank_of,
                                                          uint32_t* __restrict__ adjp) {
  extern __shared__ uint32_t rows[];  // [8][W]
  const int pair = blockIdx.y;
  if (solve[pair].mode == QB200_INLIER_NONE) return;
  const int L = n_corr[pair];
  const int wib = threadIdx.x >> 5, lane = lane_id();
  const int v = blockIdx.x * 8 + wib;
  if (v >= L) return;
  uint32_t* row = rows + wib * W;
  const int nb = (L + 31) >> 5;
  for (int w = lane; w < nb; w += 32) row[w] = 0;
  __syncwarp();
  const int* __restrict__ ro = rank_of + (size_t)pair * (Lc + 2);
  const uint32_t* __restrict__ src = adj + ((size_t)pair * Lc + v) * W;
  for (int w = lane; w < nb; w += 32) {
    uint32_t x = src[w];
    while (x) {
      const int b = __ffs(x) - 1;
      x &= x - 1;
      const int r = ro[w * 32 + b];
      atomicOr(&row[r >> 5], 1u << (r & 31));
    }
  }
  __syncwarp();
  uint32_t* __restrict__ dst = adjp + ((size_t)pair * Lc + ro[v]) * W;
  for (int w = lane; w < nb; w += 32) dst[w] = row[w];  // the descent never reads beyond ceil(L/32) words
}

// One greedy descent by one warp in rank space.  P = candidates of start vertex rv with rank >= thr; returns the chain
// length + 1 (the start vertex), or 0 when |P| <= mc.  WPL = adjacency words per lane.
template <int WPL>
__device__ __forceinline__ int clique_descent(const uint32_t* __restrict__ rows, int stride, int nbw, int rv, int thr, int mc,
                                              unsigned short* __restrict__ chain) {
  const int lane = lane_id();
  uint32_t P[WPL];
  int psize = 0;
#pragma unroll
  for (int k = 0; k < WPL; ++k) {
    const int wi = lane + 32 * k;
    uint32_t x = wi < nbw ? rows[(size_t)rv * stride + wi] : 0u;
    const int lo = wi * 32;
    if (thr >= lo + 32) x = 0;
    else if (thr > lo) x &= ~0u << (thr - lo);
    P[k] = x;
    psize += __popc(x);
  }
  psize = warp_sum(psize);
  if (psize <= mc) return 0;
  int sz = 1;
  for (;;) {
    int top = -1;  // highest set bit of P across the warp = largest (kcore, id)
#pragma unroll
    for (int k = 0; k < WPL; ++k)
      if (P[k]) top = max(top, (lane + 32 * k) * 32 + 31 - __clz(P[k]));
    top = warp_max(top);
    if (top < 0) break;
    if (lane == 0) chain[sz - 1] = (unsigned short)top;
    ++sz;
#pragma unroll
    for (int k = 0; k < WPL; ++k) {
      const int wi = lane + 32 * k;
      P[k] &= wi < nbw ? rows[(size_t)top * stride + wi] : 0u;
    }
  }
  return sz;
}

// One CTA (8 warps) per pair: PMC heuristic in rank space, start vertices tried speculatively by the warps and committed
// in sequential order.  smem: chains [8][Ls] u16 (Ls = min(Lc, kKcoreSmemVerts)), ids bitset [W], adjacency cache [cache_words].
// A pair with L > Ls keeps its chains in its slot of chain_ws ([8][Lc] u16 per pair).
__global__ void __launch_bounds__(kCliqueWarps * 32) clique_cta_kernel(const uint32_t* __restrict__ adjp, const int* __restrict__ n_corr, int Lc, int W,
                                                                       int Ls, unsigned short* __restrict__ chain_ws,
                                                                       const int* __restrict__ kcore, const int* __restrict__ korder,
                                                                       const int* __restrict__ rank_of, const int* __restrict__ by_rank,
                                                                       const int* __restrict__ kbin, const int* __restrict__ max_core_in,
                                                                       const PairSolve* __restrict__ solve, int cache_words, int* __restrict__ clique,
                                                                       int* __restrict__ n_clique) {
  constexpr int NT = kCliqueWarps * 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* idbits = reinterpret_cast<uint32_t*>(smem_raw + (size_t)kCliqueWarps * Ls * sizeof(unsigned short));  // [W]
  uint32_t* cache = idbits + W;                                                // [cache_words]
  __shared__ int s_sz[kCliqueWarps];
  __shared__ int s_scan[33];
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // PMC_EXACT starts from the heuristic clique (graph.cc:88-104: in.lb = pmc_heu.search, returned as is when lb == ub)
  const int mode = solve[pair].mode;
  if (mode == QB200_INLIER_NONE) return;
  const double kcore_thr = solve[pair].kcore_thr;
  const int L = n_corr[pair];
  const bool in_smem = L <= Ls;
  unsigned short* chains = in_smem ? reinterpret_cast<unsigned short*>(smem_raw) : chain_ws + (size_t)pair * kCliqueWarps * Lc;
  const int Lv = in_smem ? Ls : Lc;  // chain capacity
  int* __restrict__ out = clique + (size_t)pair * Lc;
  if (L <= 0) {
    if (tid == 0) n_clique[pair] = 0;
    return;
  }
  const int* __restrict__ kc = kcore + (size_t)pair * (Lc + 2);
  const int* __restrict__ ko = korder + (size_t)pair * (Lc + 2);
  const int* __restrict__ ro = rank_of + (size_t)pair * (Lc + 2);
  const int* __restrict__ br = by_rank + (size_t)pair * (Lc + 2);
  const int* __restrict__ kb = kbin + (size_t)pair * (Lc + 2);
  const uint32_t* __restrict__ G = adjp + (size_t)pair * Lc * W;
  const int max_core = max_core_in[pair];
  const int nbw = (L + 31) >> 5;
  const int nwl = (nbw + 31) >> 5;
  for (int w = tid; w < W; w += NT) idbits[w] = 0;

  if (mode == QB200_KCORE_HEU && qb_kcore_heu_shortcut(kcore_thr, L, max_core)) {
    // src/graph.cc:67-82: keep every vertex whose k_cores entry (core + 1) is >= max_core
    __syncthreads();
    for (int v = tid; v < L; v += NT)
      if (kc[v] >= max_core) atomicOr(&idbits[v >> 5], 1u << (v & 31));
  } else {
    // every descent step is a dependent row load: keep the rank-space adjacency in shared memory when it fits
    const bool cached = (long long)L * nbw <= (long long)cache_words;
    if (cached)
      for (int idx = tid; idx < L * nbw; idx += NT) cache[idx] = G[(size_t)(idx / nbw) * W + (idx % nbw)];
    const uint32_t* rows = cached ? cache : G;
    const int stride = cached ? nbw : W;
    unsigned short* chain = chains + (size_t)warp * Lv;
    const int ub = max_core + 1;  // src/graph.cc:84-86
    int mc = 0, i = L - 1;
    __syncthreads();
    while (i >= 0 && mc < ub) {
      // warp k tries the start vertex at peel position i - k against the current incumbent size mc
      const int my_i = i - warp;
      int sz = -1;  // -1: kcore[v] <= mc here, hence for every later start vertex too (kcore is non-increasing along the
                    //     reversed peel order and mc only grows)
      if (my_i >= 0) {
        const int v = ko[my_i];
        if (kc[v] > mc) {
          // candidates: neighbours of v with kcore > mc  <=>  rank >= kb[mc]  (first rank whose core >= mc)
          const int thr = kb[min(mc, max_core + 1)];
          const int rv = ro[v];
          if (nwl == 1) sz = clique_descent<1>(rows, stride, nbw, rv, thr, mc, chain);
          else if (nwl <= 4) sz = clique_descent<4>(rows, stride, nbw, rv, thr, mc, chain);
          else if (nwl <= 8) sz = clique_descent<8>(rows, stride, nbw, rv, thr, mc, chain);
          else if (nwl <= 16) sz = clique_descent<16>(rows, stride, nbw, rv, thr, mc, chain);
          else sz = clique_descent<32>(rows, stride, nbw, rv, thr, mc, chain);
        }
      }
      if (lane == 0) s_sz[warp] = sz;
      __syncthreads();
      int win = -1;
      bool stop = false;
#pragma unroll
      for (int k = 0; k < kCliqueWarps; ++k) {
        if (win < 0 && !stop) {
          const int s = s_sz[k];
          if (s < 0) stop = true;
          else if (s > mc) win = k;
        }
      }
      if (win >= 0) {  // commit the first improvement in sequential order; later warps saw a stale mc and are redone
        const int wsz = s_sz[win];
        for (int w = tid; w < W; w += NT) idbits[w] = 0;
        __syncthreads();
        if (warp == win) {
          for (int t = lane; t < wsz - 1; t += 32) {
            const int id = br[chain[t]];
            atomicOr(&idbits[id >> 5], 1u << (id & 31));
          }
          if (lane == 0) {
            const int v = ko[i - win];
            atomicOr(&idbits[v >> 5], 1u << (v & 31));
          }
        }
        mc = wsz;
        i = i - win - 1;
      } else if (stop) {
        i = -1;
      } else {
        i -= kCliqueWarps;
      }
      __syncthreads();
    }
  }
  __syncthreads();
  // ascending ids (std::sort(max_clique_), quatro.hpp:806)
  int csize = 0;
  for (int base = 0; base < W; base += NT) {
    const int w = base + tid;
    uint32_t x = w < W ? idbits[w] : 0;
    int tot;
    int off = csize + block_excl_scan(__popc(x), s_scan, &tot);
    while (x) {
      const int b = __ffs(x) - 1;
      x &= x - 1;
      out[off++] = w * 32 + b;
    }
    csize += tot;
  }
  if (tid == 0) n_clique[pair] = csize;
}


// ------------------------------------------------------------------------------------------------
// PMC_EXACT: bit-parallel branch and bound with greedy-colouring bounds, ONE WARP per pair, in rank space.
// Replaces the exact finder call of src/graph.cc:106-127 ([EXT] pmc::pmcx_maxclique::search_dense); the canonical search order
// (which of several maximum cliques is returned) is the canonical sequential one of DESIGN.md 5.3 -- the incumbent is the
// heuristic clique, root candidates = vertices of core number >= |incumbent|, colour classes take the lowest rank first, the
// branch runs from the end of the (colour, rank) list, a level dies when |C| + colour <= |incumbent|, the search ends after
// node_limit expanded nodes (QB200_FLAG_CLIQUE_TRUNCATED).  The warp keeps a candidate set as WPL words per lane (word index
// lane + 32 k, like clique_descent); the level stack -- one candidate bitset and one (rank | colour << 16) list segment per
// depth -- lives in global scratch (L1/L2-resident: the live part is a few KB), rows come from the shared-memory adjacency cache
// when the graph fits.  Stack or list-pool exhaustion ends the search like the node limit does.  Both limits exist on the device
// only (the CPU search grows its stack): a search that would go deeper than kExactDepth levels, or whose lists on the current path
// hold more than kExactPool entries, stops with QB200_FLAG_CLIQUE_TRUNCATED and the best clique found so far.  The root list (at
// most L entries) always fits.
// ------------------------------------------------------------------------------------------------
constexpr int kExactDepth = 1024;      // levels of the stack (a clique larger than this ends the search with the truncation flag)
constexpr int kExactPool = 1 << 17;    // list entries per pair
static_assert(kExactPool >= QB200_MAX_CORR, "the root colour list of a pair must fit into the list pool");
constexpr int kExactChunk = 64;        // pairs searched by one launch (the scratch is sized for these, not for max_batch_slots)

template <int WPL>
__device__ __forceinline__ int exact_colour_sort(const uint32_t* __restrict__ rows, int stride, int nbw, const uint32_t (&P)[WPL], int kmin,
                                                 uint32_t* __restrict__ list, int cap) {
  const int lane = lane_id();
  uint32_t Q[WPL], Qk[WPL];
#pragma unroll
  for (int k = 0; k < WPL; ++k) Q[k] = P[k];
  int col = 0, cnt = 0;
  for (;;) {
    uint32_t any = 0u;
#pragma unroll
    for (int k = 0; k < WPL; ++k) any |= Q[k];
    if (!__any_sync(0xffffffffu, any != 0u)) break;
    ++col;
#pragma unroll
    for (int k = 0; k < WPL; ++k) Qk[k] = Q[k];
    for (;;) {
      int cand = 0x7fffffff;  // lowest rank left in the class candidates (a lane's words ascend with k)
#pragma unroll
      for (int k = WPL - 1; k >= 0; --k)
        if (Qk[k]) cand = (lane + 32 * k) * 32 + __ffs(Qk[k]) - 1;
      const int v = __reduce_min_sync(0xffffffffu, cand);
      if (v == 0x7fffffff) break;
      const int vw = v >> 5;
      const uint32_t vbit = 1u << (v & 31);
#pragma unroll
      for (int k = 0; k < WPL; ++k) {
        const int wi = lane + 32 * k;
        if (wi < nbw) {
          uint32_t drop = rows[(size_t)v * stride + wi];
          if (wi == vw) { drop |= vbit; Q[k] &= ~vbit; }
          Qk[k] &= ~drop;
        }
      }
      if (col > kmin) {
        if (cnt >= cap) return -1;  // list pool exhausted (warp-uniform)
        if (lane == 0) list[cnt] = (uint32_t)v | ((uint32_t)col << 16);
        ++cnt;
      }
    }
  }
  return cnt;
}

template <int WPL>
__global__ void __launch_bounds__(32) clique_exact_kernel(const uint32_t* __restrict__ adjp, const int* __restrict__ n_corr, int Lc, int W,
                                                         const int* __restrict__ by_rank, const int* __restrict__ rank_of,
                                                         const int* __restrict__ kbin, const int* __restrict__ max_core_in,
                                                         const PairSolve* __restrict__ solve, int cache_words, int pair_base, uint32_t* __restrict__ stackP, uint32_t* __restrict__ pool,
                                                         int* __restrict__ lvl_begin, int* __restrict__ lvl_n, unsigned short* __restrict__ cur_c,
                                                         int* __restrict__ clique, int* __restrict__ n_clique, int* __restrict__ flags) {
  extern __shared__ uint32_t ex_cache[];  // [cache_words] rank-space adjacency when it fits
  const int pair = pair_base + blockIdx.x, slot = blockIdx.x, lane = lane_id();   // scratch is per launch slot, data per pair
  if (solve[pair].mode != QB200_PMC_EXACT) return;
  const long long node_limit = solve[pair].node_limit;
  const int L = n_corr[pair];
  if (L <= 0) return;
  int best = n_clique[pair];
  const int max_core = max_core_in[pair];
  const int ub = max_core + 1;
  if (best <= 0 || best >= ub) return;  // graph.cc:96-104: the heuristic clique already meets the k-core bound
  const int nbw = (L + 31) >> 5;
  const uint32_t* __restrict__ G = adjp + (size_t)pair * Lc * W;
  const bool cached = (long long)L * nbw <= (long long)cache_words;
  if (cached)
    for (int idx = lane; idx < L * nbw; idx += 32) ex_cache[idx] = G[(size_t)(idx / nbw) * W + (idx % nbw)];
  __syncwarp();
  const uint32_t* rows = cached ? ex_cache : G;
  const int stride = cached ? nbw : W;
  const int* __restrict__ br = by_rank + (size_t)pair * (Lc + 2);
  const int* __restrict__ kb = kbin + (size_t)pair * (Lc + 2);
  uint32_t* __restrict__ SP = stackP + (size_t)slot * kExactDepth * W;
  uint32_t* __restrict__ LP = pool + (size_t)slot * kExactPool;
  int* __restrict__ lb = lvl_begin + (size_t)slot * kExactDepth;
  int* __restrict__ ln = lvl_n + (size_t)slot * kExactDepth;
  unsigned short* __restrict__ C = cur_c + (size_t)slot * kExactDepth;
  int* __restrict__ out = clique + (size_t)pair * Lc;

  uint32_t P[WPL];
  {  // root: ranks >= kb[best] (core number >= |incumbent|)
    const int thr = kb[min(best, max_core + 1)];
#pragma unroll
    for (int k = 0; k < WPL; ++k) {
      const int wi = lane + 32 * k, lo = wi * 32;
      uint32_t x = 0u;
      const int a = max(thr, lo), b = min(L, lo + 32);  // ranks [a, b) of this word are candidates
      if (wi < nbw && a < b) x = (b - lo >= 32 ? ~0u : ((1u << (b - lo)) - 1u)) & (~0u << (a - lo));
      P[k] = x;
      if (wi < nbw) SP[wi] = x;
    }
  }
  int used = exact_colour_sort<WPL>(rows, stride, nbw, P, best, LP, kExactPool);
  bool truncated = used < 0;
  int depth = truncated ? -1 : 0;
  if (lane == 0 && !truncated) { lb[0] = 0; ln[0] = used; }
  __syncwarp();
  long long nodes = 0;
  bool improved = false;
  while (depth >= 0) {
    const int n_here = ln[depth];
    if (n_here == 0) { --depth; continue; }
    const int begin = lb[depth];
    const uint32_t e = LP[begin + n_here - 1];
    __syncwarp();
    if (lane == 0) ln[depth] = n_here - 1;
    const int v = (int)(e & 0xFFFFu), col = (int)(e >> 16);
    if (depth + col <= best) {  // nothing left on this level can beat the incumbent
      if (lane == 0) ln[depth] = 0;
      __syncwarp();
      continue;
    }
    if (lane == 0) C[depth] = (unsigned short)v;
    uint32_t* __restrict__ Pl = SP + (size_t)depth * W;
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < WPL; ++k) {
      const int wi = lane + 32 * k;
      uint32_t x = 0u;
      if (wi < nbw) {
        const uint32_t pw = Pl[wi];
        x = pw & rows[(size_t)v * stride + wi];
        if (wi == (v >> 5)) Pl[wi] = pw & ~(1u << (v & 31));  // v leaves this level's candidates
      }
      P[k] = x;
      cnt += __popc(x);
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    __syncwarp();
    if (cnt == 0) {
      if (depth + 1 > best) {  // a maximal clique larger than the incumbent: record it (ranks -> ids, sorted at the end)
        best = depth + 1;
        improved = true;
        for (int t = lane; t <= depth; t += 32) out[t] = br[C[t]];
        __syncwarp();
        if (best >= ub) break;
      }
      continue;
    }
    if (depth + 1 + cnt <= best) continue;
    if (++nodes > node_limit || depth + 1 >= kExactDepth) { truncated = true; break; }
    const int nbegin = begin + n_here - 1;  // the consumed entry's slot and everything behind it is free again
    uint32_t* __restrict__ Pn = SP + (size_t)(depth + 1) * W;
#pragma unroll
    for (int k = 0; k < WPL; ++k) {
      const int wi = lane + 32 * k;
      if (wi < nbw) Pn[wi] = P[k];
    }
    const int nl = exact_colour_sort<WPL>(rows, stride, nbw, P, best - (depth + 1), LP + nbegin, kExactPool - nbegin);
    if (nl < 0) { truncated = true; break; }
    if (lane == 0) { lb[depth + 1] = nbegin; ln[depth + 1] = nl; }
    __syncwarp();
    ++depth;
  }
  __syncwarp();
  if (improved) {
    // ascending ids (std::sort(max_clique_), quatro.hpp:806): rank = number of smaller ids (ids are distinct, cliques are small);
    // lvl_begin is free now and serves as the second buffer (best <= kExactDepth)
    for (int t = lane; t < best; t += 32) {
      const int x = out[t];
      int r = 0;
      for (int u = 0; u < best; ++u) r += out[u] < x ? 1 : 0;
      lb[r] = x;
    }
    __syncwarp();
    for (int t = lane; t < best; t += 32) out[t] = lb[t];
    if (lane == 0) n_clique[pair] = best;
  }
  if (lane == 0 && truncated) flags[pair] |= QB200_FLAG_CLIQUE_TRUNCATED;
}

// shared memory of the k-core peel: whole graphs up to L ~ 680 at max_corr 4096; the rest of the SM stays free for the dense
// kernels of the other lanes
constexpr size_t kKcoreSmemBudget = 144 * 1024;

template <int WPL>
static int launch_kcore(Lane* h, int n_pairs) {
  const int Lc = h->Lc, W = h->W;
  const int Ls = Lc < kKcoreSmemVerts ? Lc : kKcoreSmemVerts, Ws = Ls / 32;  // vertices / row words of the shared-memory layout
  const size_t bits = (size_t)3 * kKcWarps * 32 * WPL * sizeof(uint32_t);
  const size_t fixed = (size_t)(Ls + 2) * sizeof(int) + bits + (size_t)(4 + kKcWarps) * Ls * sizeof(unsigned short);
  // rows: what is left of the budget, at least the prefetch ring
  size_t row_words = fixed + 8 * 1024 < kKcoreSmemBudget ? (kKcoreSmemBudget - fixed) / 4 : 0;
  if (row_words < (size_t)kRing * Ws) row_words = (size_t)kRing * Ws;
  if (row_words > (size_t)Ls * Ws) row_words = (size_t)Ls * Ws;
  const size_t smem = fixed + row_words * 4;
  if (Ls < Lc && smem - bits < (size_t)kRing * W * 4) {  // a pair above Ls streams full-width rows through the area behind the bitsets
    h->fail(__FILE__, __LINE__, "k-core prefetch ring does not fit");
    return QB200_ERR_CUDA;
  }
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)kcore_kernel<WPL, false>, smem));
  kcore_kernel<WPL, false><<<n_pairs, kKcWarps * 32, smem, h->stream>>>(h->adj, h->deg, h->ctr.n_corr, h->d_solve, Lc, W, Ls, (int)row_words, h->kcore_ws,
                                                                        h->kcore, h->korder, h->rank_of, h->by_rank, h->kbin, h->ctr.max_core);
  if (Ls < Lc) {  // pairs above the shared-memory layout: same shared-memory size, per-vertex arrays in kcore_ws
    QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)kcore_kernel<WPL, true>, smem));
    kcore_kernel<WPL, true><<<n_pairs, kKcWarps * 32, smem, h->stream>>>(h->adj, h->deg, h->ctr.n_corr, h->d_solve, Lc, W, Ls, (int)row_words, h->kcore_ws,
                                                                         h->kcore, h->korder, h->rank_of, h->by_rank, h->kbin, h->ctr.max_core);
    h->launches++;
  }
  return QB200_OK;
}

// PMC_EXACT scratch (level stack, list pool), allocated on the first exact call of a handle: all of it or none
static int ensure_exact_scratch(Lane* h) {
  if (h->ex_stack) return QB200_OK;
  const size_t S = h->S < kExactChunk ? h->S : kExactChunk;
  DeviceMem<uint32_t> stack, pool;
  DeviceMem<int> lvl;
  DeviceMem<unsigned short> cur;
  QB_CUDA_TRY(h, stack.alloc(S * kExactDepth * (size_t)h->W));
  QB_CUDA_TRY(h, pool.alloc(S * (size_t)kExactPool));
  QB_CUDA_TRY(h, lvl.alloc(S * 2 * (size_t)kExactDepth));
  QB_CUDA_TRY(h, cur.alloc(S * (size_t)kExactDepth));
  h->ex_stack = std::move(stack);
  h->ex_pool = std::move(pool);
  h->ex_lvl = std::move(lvl);
  h->ex_cur = std::move(cur);
  return QB200_OK;
}

template <int WPL>
static int launch_exact(Lane* h, int n_pairs, int cache_words) {
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)clique_exact_kernel<WPL>, (size_t)cache_words * 4));
  const int chunk = h->S < kExactChunk ? h->S : kExactChunk;
  for (int base = 0; base < n_pairs; base += chunk) {   // chunks run one after the other on the stream and share the scratch
    const int np = n_pairs - base < chunk ? n_pairs - base : chunk;
    clique_exact_kernel<WPL><<<np, 32, (size_t)cache_words * 4, h->stream>>>(
        h->adjp, h->ctr.n_corr, h->Lc, h->W, h->by_rank, h->rank_of, h->kbin, h->ctr.max_core, h->d_solve, cache_words, base, h->ex_stack,
        h->ex_pool, h->ex_lvl, h->ex_lvl + (size_t)chunk * kExactDepth, h->ex_cur, h->clique, h->ctr.n_clique, h->ctr.flags);
    h->launches++;
  }
  return QB200_OK;
}

int launch_clique(Lane* h, int n_pairs, bool any_exact) {
  if (n_pairs <= 0) return QB200_OK;
  const int Lc = h->Lc, W = h->W;
  const int Ls = Lc < kKcoreSmemVerts ? Lc : kKcoreSmemVerts;
  // shared-memory adjacency cache of the descent: 14336 words (56 KB) hold graphs up to L ~ 660
  const int cache_words = 14336;
  const size_t sm_clique = (size_t)kCliqueWarps * Ls * sizeof(unsigned short) + (size_t)W * sizeof(uint32_t) + (size_t)cache_words * 4;
  int rc;
  QB_CUDA_TRY(h, ensure_dyn_smem(h->device, (const void*)clique_cta_kernel, sm_clique));
  if (any_exact && (rc = ensure_exact_scratch(h))) return rc;
  if (W <= 32) rc = launch_kcore<1>(h, n_pairs);
  else if (W <= 64) rc = launch_kcore<2>(h, n_pairs);
  else if (W <= 128) rc = launch_kcore<4>(h, n_pairs);
  else if (W <= 256) rc = launch_kcore<8>(h, n_pairs);
  else if (W <= 512) rc = launch_kcore<16>(h, n_pairs);
  else rc = launch_kcore<32>(h, n_pairs);
  if (rc) return rc;
  const dim3 gp((Lc + 7) / 8, n_pairs);
  permute_adj_kernel<<<gp, 256, 8 * W * sizeof(uint32_t), h->stream>>>(h->adj, h->ctr.n_corr, Lc, W, h->d_solve, h->rank_of, h->adjp);
  clique_cta_kernel<<<n_pairs, kCliqueWarps * 32, sm_clique, h->stream>>>(h->adjp, h->ctr.n_corr, Lc, W, Ls, h->chain_ws, h->kcore, h->korder,
                                                                          h->rank_of, h->by_rank, h->kbin, h->ctr.max_core, h->d_solve,
                                                                          cache_words, h->clique, h->ctr.n_clique);
  h->launches += 3;
  if (any_exact) {  // the PMC_EXACT pairs of the wave, each with its own node limit; the other pairs leave at once
    if (W <= 32) rc = launch_exact<1>(h, n_pairs, cache_words);
    else if (W <= 64) rc = launch_exact<2>(h, n_pairs, cache_words);
    else if (W <= 128) rc = launch_exact<4>(h, n_pairs, cache_words);
    else if (W <= 256) rc = launch_exact<8>(h, n_pairs, cache_words);
    else if (W <= 512) rc = launch_exact<16>(h, n_pairs, cache_words);
    else rc = launch_exact<32>(h, n_pairs, cache_words);
    if (rc) return rc;
  }
  QB_CUDA_TRY(h, cudaGetLastError());
  return QB200_OK;
}

}  // namespace qb
