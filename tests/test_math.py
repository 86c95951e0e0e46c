"""Portable transcendentals (oracle/qo_math.h, deviation D7) stay within a few ulp of libm, and the
CUDA copy (quatro_b200/csrc/qb_math.cuh) compiled for the host agrees with the oracle's bit for bit."""
import ctypes as C
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def ulps(a, truth):
    sp = np.spacing(np.abs(truth).astype(np.float32)).astype(np.float64)
    return np.abs(a.astype(np.float64) - truth) / sp


def test_atan2f_accuracy(oracle):
    rng = np.random.default_rng(0)
    y = rng.normal(size=20000).astype(np.float32)
    x = rng.normal(size=20000).astype(np.float32)
    got = oracle.atan2f(y, x)
    ref = np.arctan2(y.astype(np.float64), x.astype(np.float64))
    assert ulps(got, ref).max() < 4.0
    # quadrant / axis cases
    for yy, xx in [(0.0, 1.0), (1.0, 0.0), (0.0, -1.0), (-1.0, 0.0), (1.0, 1.0), (-1.0, -1.0), (1e-30, 1.0)]:
        assert abs(float(oracle.atan2f([yy], [xx])[0]) - np.arctan2(yy, xx)) < 1e-6
    assert float(oracle.atan2f([-0.0], [-1.0])[0]) == pytest.approx(-np.pi, abs=1e-6)  # sign of zero as libm
    assert np.isnan(oracle.atan2f([np.nan], [1.0])[0])


def test_acosf_accuracy(oracle):
    x = np.linspace(-1, 1, 20001).astype(np.float32)
    got = oracle.acosf(x)
    ref = np.arccos(x.astype(np.float64))
    err = np.abs(got.astype(np.float64) - ref)
    assert err.max() < 6e-7
    assert np.isnan(oracle.acosf([1.0000001])[0])  # like libm: acos(>1) = NaN (swap test then false)
    # monotone non-increasing on [0,1] (the only property the Darboux swap test uses)
    g = oracle.acosf(np.linspace(0, 1, 5001).astype(np.float32))
    assert np.all(np.diff(g) <= 0)


def test_sincosf_accuracy(oracle):
    x = np.linspace(0, 1.1, 5001).astype(np.float32)
    sc = oracle.sincosf(x)
    assert ulps(sc[:, 0], np.sin(x.astype(np.float64))).max() < 4
    assert ulps(sc[:, 1], np.cos(x.astype(np.float64))).max() < 4


def test_philox_known_answer(oracle):
    # Random123 known-answer vectors for philox4x32-10 use counter words 2,3 = 0 only when ctr < 2^64: check
    # self-consistency + the published KAT for an all-zero counter/key.
    o = oracle.philox(0, 0)
    assert [hex(v) for v in o] == ["0x6627e8d5", "0xe169c58d", "0xbc57ac4c", "0x9b00dbd8"]
    assert not np.array_equal(oracle.philox(0, 1), o)


def test_cuda_math_copy_matches_oracle_bitwise(tmp_path):
    """Compile quatro_b200/csrc/qb_math.cuh for the HOST and compare with oracle/qo_math.h on 1e6 inputs."""
    hdr = ROOT / "quatro_b200" / "csrc" / "qb_math.cuh"
    if not hdr.exists():
        pytest.skip("qb_math.cuh not written yet")
    src = tmp_path / "cmp.cpp"
    src.write_text(r'''
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <random>
#define QB_HD
#include "%s"
#include "%s"
static uint32_t bits(float f){ uint32_t u; memcpy(&u,&f,4); return u; }
int main(){
  std::mt19937 g(1); std::normal_distribution<float> nd(0.f,1.f); std::uniform_real_distribution<float> ud(-1.f,1.f);
  long bad=0;
  for(int i=0;i<1000000;++i){
    float y=nd(g), x=nd(g), u=ud(g), t=0.55f*(ud(g)+1.f);
    if(bits(qb_atan2f(y,x))!=bits(qo_atan2f(y,x))) ++bad;
    if(bits(qb_acosf(u))!=bits(qo_acosf(u))) ++bad;
    float s1,c1,s2,c2; qb_sincosf(t,&s1,&c1); qo_sincosf(t,&s2,&c2);
    if(bits(s1)!=bits(s2)||bits(c1)!=bits(c2)) ++bad;
  }
  printf("%%ld\n", bad); return bad!=0;
}''' % (hdr, ROOT / "oracle" / "qo_math.h"))
    exe = tmp_path / "cmp"
    subprocess.run(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-o", str(exe), str(src)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "0", r.stdout + r.stderr


def test_cuda_fpfh_math_matches_oracle_bitwise(tmp_path):
    """quatro_b200/csrc/fpfh_math.cuh (normal from covariance sums, Darboux features, bins) compiled for
    the HOST must agree bit-for-bit with the oracle's exported routines on random inputs."""
    hdr = ROOT / "quatro_b200" / "csrc" / "fpfh_math.cuh"
    from oracle import Oracle
    Oracle()  # builds oracle/build/libquatro_oracle.so if stale
    src = tmp_path / "cmp2.cpp"
    src.write_text(r'''
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <cmath>
#include <random>
#define QB_HD
#include "%s"
extern "C" void qo_test_normal_from_accu(const float*, int, const float*, float*);
extern "C" int qo_test_pair_features(const float*, const float*, const float*, const float*, float*);
extern "C" void qo_test_feature_bins(float, float, float, int*);
static bool same(float a, float b){ uint32_t x,y; memcpy(&x,&a,4); memcpy(&y,&b,4); return x==y || (a!=a && b!=b); }
int main(){
  std::mt19937 g(7); std::normal_distribution<float> nd(0.f,1.f); std::uniform_real_distribution<float> ud(-1.f,1.f);
  long bad=0;
  for(int it=0; it<200000; ++it){
    // a small neighbourhood around a far-away centre: accumulate like the kernels do
    float cx=60.f*ud(g), cy=60.f*ud(g), cz=2.f*ud(g); int cnt=3+(it%%20);
    float nx=nd(g), ny=nd(g), nz=nd(g);
    float accu[9]={0,0,0,0,0,0,0,0,0};
    for(int k=0;k<cnt;++k){ float a=0.5f*ud(g), b=0.5f*ud(g); float x=cx+a, y=cy+b, z=cz+0.02f*ud(g)+(it%%3==0? 0.3f*a*nx:0.f);
      accu[0]+=x*x; accu[1]+=x*y; accu[2]+=x*z; accu[3]+=y*y; accu[4]+=y*z; accu[5]+=z*z; accu[6]+=x; accu[7]+=y; accu[8]+=z; }
    (void)ny; (void)nz;
    float a1[9], o1[4], o2[4], p3[3]={cx,cy,cz}; memcpy(a1,accu,sizeof(a1));
    qb_normal_from_accu(a1, cnt, cx, cy, cz, o1);
    qo_test_normal_from_accu(accu, cnt, p3, o2);
    for(int k=0;k<4;++k) if(!same(o1[k],o2[k])) ++bad;
    // pair features on random unit-ish normals
    float p1[4]={ud(g),ud(g),ud(g),0}, p2[4]={ud(g),ud(g),ud(g),0}, n1[4]={nd(g),nd(g),nd(g),0}, n2[4]={nd(g),nd(g),nd(g),0};
    float l1=std::sqrt(n1[0]*n1[0]+n1[1]*n1[1]+n1[2]*n1[2]), l2=std::sqrt(n2[0]*n2[0]+n2[1]*n2[1]+n2[2]*n2[2]);
    for(int k=0;k<3;++k){ n1[k]/=l1; n2[k]/=l2; }
    if(it%%50==0){ n2[0]=n1[0]; n2[1]=n1[1]; n2[2]=n1[2]; }
    if(it%%77==0){ n1[0]=NAN; }
    float f[3]={0,0,0}, h1,h2,h3;
    bool okp = qb_pair_features(p1[0],p1[1],p1[2],n1[0],n1[1],n1[2],p2[0],p2[1],p2[2],n2[0],n2[1],n2[2],&h1,&h2,&h3);
    int oko = qo_test_pair_features(p1,n1,p2,n2,f);
    if((int)okp!=oko) ++bad;
    if(okp && oko){ if(!same(h1,f[0])||!same(h2,f[1])||!same(h3,f[2])) ++bad;
      int b[3], c1,c2,c3; qo_test_feature_bins(f[0],f[1],f[2],b); qb_feature_bins(h1,h2,h3,&c1,&c2,&c3);
      if(b[0]!=c1||b[1]!=c2||b[2]!=c3) ++bad; }
  }
  printf("%%ld\n", bad); return bad!=0;
}''' % hdr)
    exe = tmp_path / "cmp2"
    libdir = ROOT / "oracle" / "build"
    subprocess.run(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-o", str(exe), str(src), f"-L{libdir}", "-lquatro_oracle",
                    f"-Wl,-rpath,{libdir}"], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "0", r.stdout + r.stderr


# ---- the D7 kernels over every float near their branch points, on the host and as nvcc compiles them for the device ----------------
_EVAL_SRC = r'''
#include <cstdio>
#include <cstdint>
#include <cstring>
#define QB_HD
#include "%s"
int main(int argc, char** argv) {
  FILE* fi = fopen(argv[1], "rb"); FILE* fo = fopen(argv[2], "wb");
  float x;
  while (fread(&x, 4, 1, fi) == 1) {
    float o[5], s, c;
    qb_sincosf(x, &s, &c);
    o[0] = qb_acosf(x); o[1] = s; o[2] = c; o[3] = qb_atan2f(x, 1.0f); o[4] = qb_atan2f(1.0f, -x);
    fwrite(o, 4, 5, fo);
  }
  fclose(fi); fclose(fo); return 0;
}'''


def _floats(lo_bits, hi_bits, step=1):
    return np.arange(lo_bits, hi_bits, step, dtype=np.int64).astype(np.uint32).view(np.float32)


def _around(x, half=1 << 14):
    b = int(np.float32(x).view(np.uint32))
    return _floats(max(b - half, 0), b + half)


def test_d7_kernels_near_their_branch_points(tmp_path):
    """Host compile of qb_math.cuh on every float within 2^14 ulps of acos's 0.5 and 1, the atan reduction at 0.41421357, 1 (atan's
    octant switch), 0 and the smallest normal, all subnormals in stride, and a stride over the whole range: ulp bounds as measured by an
    exhaustive sweep (acos 1.24, sin 1.09, cos 1.39, atan2(y, 1) 2.62, atan2(1, -x) 1.51) plus a little headroom; acos monotone."""
    pos = np.concatenate([_around(0.5), _around(1.0), _around(0.41421357), _around(0.41421357 ** -1), _floats(0, 1 << 14),
                          _around(np.finfo(np.float32).tiny), _floats(1, 1 << 23, 997), _floats(1 << 23, 0x7F800000, 4099),
                          np.array([np.inf, 1.1, 1.0471976], np.float32)])
    x = np.unique(np.concatenate([pos, -pos]).astype(np.float32))
    src, exe = tmp_path / "ev.cpp", tmp_path / "ev"
    src.write_text(_EVAL_SRC % (ROOT / "quatro_b200" / "csrc" / "qb_math.cuh"))
    subprocess.run(["/usr/bin/g++", "-O2", "-ffp-contract=off", "-o", str(exe), str(src)], check=True)
    x.tofile(tmp_path / "in.bin")
    subprocess.run([str(exe), str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], check=True)
    o = np.fromfile(tmp_path / "out.bin", np.float32).reshape(-1, 5)
    x64 = x.astype(np.float64)
    dom = np.abs(x) <= 1
    assert np.isnan(o[~dom, 0]).all()
    assert ulps(o[dom, 0], np.arccos(x64[dom])).max() < 1.3
    xs = x[dom]
    a = o[dom, 0][np.argsort(xs, kind="stable")]
    assert np.all(np.diff(a) <= 0)                                      # non-increasing over [-1, 1]
    sc = (x >= 0) & (x <= np.float32(1.1))
    assert ulps(o[sc, 1], np.sin(x64[sc])).max() < 1.15
    assert ulps(o[sc, 2], np.cos(x64[sc])).max() < 1.45
    fin = np.isfinite(x) & (x > 0)
    assert ulps(o[fin, 3], np.arctan2(x64[fin], 1.0)).max() < 2.7
    assert ulps(o[fin, 4], np.arctan2(1.0, -x64[fin])).max() < 1.6
    assert o[x == np.inf, 3][0] == np.float32(np.pi / 2) and o[x == np.inf, 4][0] == np.float32(np.pi)
    sub = (x > 0) & (x < np.finfo(np.float32).tiny)
    assert (o[sub, 3] == x[sub]).all()                                  # atan2(y, 1) = y below FLT_MIN


_DEVICE_SRC = r'''
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "fpfh_math.cuh"

__global__ void eval_kernel(uint32_t b0, uint32_t n, int which, uint32_t* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = __uint_as_float(b0 + i);
  float s, c;
  if (which == 0) { out[i] = __float_as_uint(qb_acosf(x)); return; }
  qb_sincosf(x, &s, &c);
  out[2 * i] = __float_as_uint(s);
  out[2 * i + 1] = __float_as_uint(c);
}

__global__ void pair_kernel(const float* in, int n, float* out, int* bins) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* a = in + 12 * i;
  float f1 = 0.f, f2 = 0.f, f3 = 0.f;
  const bool ok = qb_pair_features(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8], a[9], a[10], a[11], &f1, &f2, &f3);
  out[3 * i] = f1; out[3 * i + 1] = f2; out[3 * i + 2] = f3;
  int b1, b2, b3;
  qb_feature_bins(f1, f2, f3, &b1, &b2, &b3);
  bins[4 * i] = ok; bins[4 * i + 1] = b1; bins[4 * i + 2] = b2; bins[4 * i + 3] = b3;
}

// every float of [lo, hi] (bit patterns, same sign) through acos (which = 0) or sincos (1) on the device, compared bit for bit with the
// host compile of the same header, in chunks of 2^22 floats; returns the mismatch count, or -1 on a CUDA error
extern "C" long long qbm_sweep(uint32_t lo, uint32_t hi, int which) {
  const uint32_t chunk = 1u << 22;
  const int w = which == 1 ? 2 : 1;
  uint32_t* d = nullptr;
  if (cudaMalloc(&d, (size_t)chunk * w * 4) != cudaSuccess) return -1;
  std::vector<uint32_t> h((size_t)chunk * w);
  long long bad = 0;
  for (uint64_t b0 = lo; b0 <= hi; b0 += chunk) {
    const uint32_t n = (uint32_t)((hi - b0 + 1) < chunk ? (hi - b0 + 1) : chunk);
    eval_kernel<<<(n + 255) / 256, 256>>>((uint32_t)b0, n, which, d);
    if (cudaMemcpy(h.data(), d, (size_t)n * w * 4, cudaMemcpyDeviceToHost) != cudaSuccess) { cudaFree(d); return -1; }
#pragma omp parallel for reduction(+ : bad) schedule(static)
    for (long long i = 0; i < (long long)n; ++i) {
      float x, s, c, r;
      const uint32_t xb = (uint32_t)(b0 + i);
      memcpy(&x, &xb, 4);
      uint32_t u[2];
      if (which == 0) { r = qb_acosf(x); memcpy(u, &r, 4); bad += u[0] != h[i]; }
      else { qb_sincosf(x, &s, &c); memcpy(u, &s, 4); memcpy(u + 1, &c, 4); bad += (u[0] != h[2 * i]) + (u[1] != h[2 * i + 1]); }
    }
  }
  cudaFree(d);
  return bad;
}

// qb_pair_features + qb_feature_bins of n pairs (p1, n1, p2, n2 as 12 floats each) on the device, written to f (n x 3) and
// bins (n x 4: ok, b1, b2, b3); returns the mismatch count against the host compile (the device returns the canonical NaN where x86
// propagates an operand's payload: NaN matches NaN), or -1 on a CUDA error
extern "C" long long qbm_pairs(const float* in, int n, float* f_out, int* bins_out) {
  float *d_in, *d_out; int* d_bins;
  cudaMalloc(&d_in, (size_t)n * 48); cudaMalloc(&d_out, (size_t)n * 12); cudaMalloc(&d_bins, (size_t)n * 16);
  cudaMemcpy(d_in, in, (size_t)n * 48, cudaMemcpyHostToDevice);
  pair_kernel<<<(n + 127) / 128, 128>>>(d_in, n, d_out, d_bins);
  std::vector<float> out((size_t)n * 3); std::vector<int> bins((size_t)n * 4);
  if (cudaMemcpy(out.data(), d_out, (size_t)n * 12, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  cudaMemcpy(bins.data(), d_bins, (size_t)n * 16, cudaMemcpyDeviceToHost);
  cudaFree(d_in); cudaFree(d_out); cudaFree(d_bins);
  memcpy(f_out, out.data(), (size_t)n * 12);
  memcpy(bins_out, bins.data(), (size_t)n * 16);
  long long bad = 0;
  auto same = [](float x, float y) { return memcmp(&x, &y, 4) == 0 || (x != x && y != y); };  // a NaN's payload is not part of the result
  for (int i = 0; i < n; ++i) {
    const float* a = in + 12 * i;
    float f[3] = {0.f, 0.f, 0.f};
    const bool ok = qb_pair_features(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8], a[9], a[10], a[11], &f[0], &f[1], &f[2]);
    int b[3];
    qb_feature_bins(f[0], f[1], f[2], &b[0], &b[1], &b[2]);
    bad += !same(f[0], out[3 * i]) || !same(f[1], out[3 * i + 1]) || !same(f[2], out[3 * i + 2]);
    bad += (int)ok != bins[4 * i] || b[0] != bins[4 * i + 1] || b[1] != bins[4 * i + 2] || b[2] != bins[4 * i + 3];
  }
  return bad;
}
'''


@pytest.mark.gpu
def test_device_compile_of_the_d7_kernels_matches_the_host(tmp_path):
    """qb_math.cuh / fpfh_math.cuh compiled by nvcc with the library's own flags: every float of acos's domain [-1, 1] and every float of
    [0, 1.1] through sincos on the device equal the host compile of the same header bit for bit.  The device's Darboux features and bins
    of the adversarial pairs of test_fpfh_adversarial.py and of random pairs equal the host compile and the float32 restatement of
    computePairFeatures (independent_ref.py), so a slip in fpfh_math.cuh cannot pass by changing both compiles alike."""
    from quatro_b200 import _build
    src, lib = tmp_path / "qbm.cu", tmp_path / "libqbm.so"
    src.write_text(_DEVICE_SRC)
    cmd = [_build.nvcc_path(), *_build.NVCC_FLAGS, "-ccbin", _build.HOST_CXX, "-Xcompiler", "-fopenmp,-ffp-contract=off", "-I",
           str(_build.CSRC), "-o", str(lib), str(src), "-lcudart", "-lgomp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    L = C.CDLL(str(lib))
    L.qbm_sweep.restype = C.c_longlong
    L.qbm_sweep.argtypes = [C.c_uint32, C.c_uint32, C.c_int]
    L.qbm_pairs.restype = C.c_longlong
    L.qbm_pairs.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    one = int(np.float32(1.0).view(np.uint32))
    assert L.qbm_sweep(0, one, 0) == 0                                   # [+0, 1]
    assert L.qbm_sweep(0x80000000, 0x80000000 | one, 0) == 0             # [-0, -1]
    assert L.qbm_sweep(0, int(np.float32(1.1).view(np.uint32)), 1) == 0
    import test_fpfh_adversarial as T
    cases = T.pair_cases()
    rng = np.random.default_rng(3)
    rand = rng.normal(size=(20000, 12)).astype(np.float32)
    arr = np.concatenate([np.array([np.concatenate(c[1:]) for c in cases], np.float32), rand])
    arr = np.ascontiguousarray(arr)
    f = np.zeros((len(arr), 3), np.float32)
    bins = np.zeros((len(arr), 4), np.int32)
    assert L.qbm_pairs(arr.ctypes.data, len(arr), f.ctypes.data, bins.ctypes.data) == 0
    import independent_ref as R
    pf = R.pair_features_pcl32(arr[:, 0:3], arr[:, 3:6], arr[:, 6:9], arr[:, 9:12], R.D7_MATH)
    ok = pf["ok"]
    assert np.array_equal(bins[:, 0].astype(bool), ok)
    want = np.stack([pf["f1"], pf["f2"], pf["f3"]], 1).astype(np.float32)
    same = (f[ok].view(np.uint32) == want[ok].view(np.uint32)) | (np.isnan(f[ok]) & np.isnan(want[ok]))
    assert same.all(), np.flatnonzero(~same.all(1))[:10]
    assert np.array_equal(bins[ok, 1:], pf["bins"][ok]), np.flatnonzero((bins[ok, 1:] != pf["bins"][ok]).any(1))[:10]
