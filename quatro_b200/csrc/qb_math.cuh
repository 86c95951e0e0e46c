// qb_math.cuh -- float32 transcendentals with a FIXED operation order (device copy).
//
// The FPFH / normal kernels need atan2f, acosf and sin/cos of the eigen-root angle.  CUDA's libm and
// the host's differ in the last ulp, which can move a Darboux angle across a histogram-bin edge, so
// both this library and the CPU oracle evaluate the same polynomial kernels with the same sequence of
// IEEE binary32 operations (coefficients: tools/fit_math.py; < 2 ulp of libm).  The library is built
// with -fmad=false, so no multiply-add below is contracted.  tests/test_math.py compiles this header
// for the host and checks it bit-for-bit against the oracle's copy.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>
#ifdef QB_HD            /* host test build defines QB_HD (empty) */
#define QB_HD_FN static inline
#else
#define QB_HD_FN static __host__ __device__ __forceinline__
#endif

#define QB_PI_F 3.14159274f
#define QB_PI_2_F 1.57079637f
#define QB_PI_4_F 0.785398185f

QB_HD_FN float qb_atan_core(float t) {  // |t| <= tan(pi/8)
  const float z = t * t;
  float p = -4.044491798e-02f;
  p = p * z + 7.135856152e-02f;
  p = p * z + -9.029050916e-02f;
  p = p * z + 1.110749617e-01f;
  p = p * z + -1.428561211e-01f;
  p = p * z + 1.999999881e-01f;
  p = p * z + -3.333333433e-01f;
  return t + t * (z * p);
}

QB_HD_FN int qb_signbitf(float v) {
#ifdef __CUDA_ARCH__
  return (int)(__float_as_uint(v) >> 31);
#else
  uint32_t u;
  memcpy(&u, &v, 4);
  return (int)(u >> 31);
#endif
}

QB_HD_FN float qb_atan2f(float y, float x) {
  if (x != x || y != y) return NAN;
  const float ax = fabsf(x), ay = fabsf(y);
  float r;
  if (ax == 0.0f && ay == 0.0f) {
    r = 0.0f;
  } else {
    const float hi = ax > ay ? ax : ay;
    const float lo = ax > ay ? ay : ax;
    float a = (hi == INFINITY) ? ((lo == INFINITY) ? 1.0f : 0.0f) : lo / hi;
    float base = 0.0f, t = a;
    if (a > 0.41421357f) {
      t = (a - 1.0f) / (a + 1.0f);
      base = QB_PI_4_F;
    }
    r = base + qb_atan_core(t);
    if (ay > ax) r = QB_PI_2_F - r;
  }
  if (qb_signbitf(x)) r = QB_PI_F - r;
  if (qb_signbitf(y)) r = -r;
  return r;
}

QB_HD_FN float qb_asin_poly(float z) {
  float q = 3.109041601e-02f;
  q = q * z + 1.048902422e-02f;
  q = q * z + 2.363533154e-02f;
  q = q * z + 3.026617132e-02f;
  q = q * z + 4.464783147e-02f;
  q = q * z + 7.499992102e-02f;
  q = q * z + 1.666666716e-01f;
  return q;
}

QB_HD_FN float qb_acosf(float x) {
  if (x != x) return NAN;
  const float ax = fabsf(x);
  if (ax > 1.0f) return NAN;
  float r;
  if (ax <= 0.5f) {
    const float z = ax * ax;
    r = QB_PI_2_F - (ax + ax * (z * qb_asin_poly(z)));
  } else {
    const float z = (1.0f - ax) * 0.5f;
    const float s = sqrtf(z);
    r = 2.0f * (s + s * (z * qb_asin_poly(z)));
  }
  if (x < 0.0f) r = QB_PI_F - r;
  return r;
}

// valid for x in [0, 1.1] (the eigen-root angle theta = atan2(sqrt(-q), half_b)/3 is in [0, pi/3])
QB_HD_FN void qb_sincosf(float x, float* s, float* c) {
  const float z = x * x;
  float ps = 1.469172284e-10f;
  ps = ps * z + -2.501203333e-08f;
  ps = ps * z + 2.755685500e-06f;
  ps = ps * z + -1.984126720e-04f;
  ps = ps * z + 8.333333768e-03f;
  ps = ps * z + -1.666666716e-01f;
  *s = x + x * (z * ps);
  float pc = 3.323700412e-06f;
  pc = pc * z + -1.105757929e-05f;
  pc = pc * z + 1.310664993e-05f;
  pc = pc * z + 1.771735151e-05f;
  pc = pc * z + -1.387358177e-03f;
  pc = pc * z + 4.166657478e-02f;
  *c = (1.0f - 0.5f * z) + (z * z) * pc;
}

// r % d for every 32-bit r and 1 <= d < 2^32 without a division: m = ceil(2^64 / d) (qb_fastmod_magic; d = 1 wraps to 0, which
// gives 0), then r % d = ((m * r mod 2^64) * d) >> 64 (Lemire, Kaser & Kurz, "Faster remainder by direct computation", 2019,
// Theorem 1: exact for N-bit r and d whenever the fraction has 2N bits).  tests/test_tuple_lazy.py checks it against % on the host.
QB_HD_FN uint64_t qb_fastmod_magic(uint32_t d) { return UINT64_MAX / d + 1u; }
QB_HD_FN uint32_t qb_fastmod(uint32_t r, uint64_t m, uint32_t d) {
  const uint64_t low = m * r;
#ifdef __CUDA_ARCH__
  return (uint32_t)__umul64hi(low, (uint64_t)d);
#else
  return (uint32_t)(((unsigned __int128)low * d) >> 64);
#endif
}
