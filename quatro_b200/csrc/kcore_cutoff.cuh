// kcore_cutoff.cuh -- the KCORE_HEU limit of src/graph.cc:67-70, shared by the CUDA library (clique.cu) and the CPU oracle.
//
// The reference takes the k-core shortcut when  max_core > static_cast<int>(kcore_heuristic_threshold * (double)n).  That cast is
// undefined in C++ for NaN and for products whose truncation lies outside int; the reference's only platform, x86-64, compiles it to
// cvttsd2si, which returns INT_MIN (0x80000000, the "integer indefinite" value) for all of them.  The device's cvt.rzi.s32.f64
// saturates instead (NaN -> 0, +inf -> INT_MAX), so neither side may write the cast itself: both call this function, which does the
// x86-64 conversion explicitly (deviation D18 of the oracle header, DESIGN.md section 2).
#pragma once
#include <limits.h>
#ifdef __CUDACC__
#define QB_KC_FN static __host__ __device__ __forceinline__
#else
#define QB_KC_FN static inline
#endif

// (int)(thr * L) as x86-64 computes it: the product truncated toward zero when that fits in int, INT_MIN otherwise (NaN included)
QB_KC_FN int qb_kcore_heu_limit(double thr, int L) {
  const double x = thr * (double)L;
  return (x > -2147483649.0 && x < 2147483648.0) ? (int)x : INT_MIN;
}

// src/graph.cc:67-70: KCORE_HEU keeps the vertices of the max core instead of searching (thr == 1 short-circuits the comparison)
QB_KC_FN bool qb_kcore_heu_shortcut(double thr, int L, int max_core) {
  return thr != 1.0 && max_core > qb_kcore_heu_limit(thr, L);
}

#undef QB_KC_FN
