// Host restatement of tim_graph_kernel's pair tests (quatro_b200/csrc/graph.cu), compiled by tests/test_graph_adversarial.py with
// g++ -O2 -ffp-contract=off: every fp32 operation below is the kernel's, in the kernel's order and nesting, with std::fmaf where the
// kernel writes fmaf / __fmaf_rn.  Line numbers refer to graph.cu.  For every pair test of a set it reports the fp32 decision,
// whether the kernel hands the test to the literal fp64 expression (and why), that expression, and t and s' in __float128: A and B
// are sums of squares of float differences, so the quad values are exact far below the 2^-24 scale of the error band q.
//
// usage: graph_band IN OUT [nofix]
//   IN:  int32 n_sets, then per set: int32 L, int32 0, double noise_bound, double cbar2, float a[L][4], float b[L][4]
//   OUT: per pair test (row i, column j; both orders inside a diagonal 32 x 32 block, as the kernel evaluates them) one Rec
//   nofix: leave out the guard !(Mj <= 2^62) of graph.cu:220 (the kernel before that guard)
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

namespace {

struct F4 { float x, y, z, w; };

struct Rec {
  int32_t set, i, j;
  uint8_t dec32;  // fp32 decision: sign(t) | sign(s') (graph.cu:191-192, 203)
  uint8_t to64;   // 1: |t_c| <= q (sign of w, graph.cu:193); 2: the smin net (graph.cu:208-220); 4: Mj beyond 2^62
  uint8_t lit;    // tim_consistent_fp64 (graph.cu:38-50)
  uint8_t exact;  // t <= 0 or s' <= 0 in __float128 (false for NaN)
  double ratio;   // |t_c - t| / q (NaN where t_c, t or q is not finite)
};
static_assert(sizeof(Rec) == 24, "record layout");

struct GraphConst { double beta; float b2, hb2q, twob2, b4, c1, c2, c3, two_b2_slack; };

// graph.cu:276-290
GraphConst graph_const(double noise_bound, double cbar2) {
  const double beta = 2 * noise_bound * std::sqrt(cbar2);
  const double u = 5.9604644775390625e-8;
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

// graph.cu:38-50
bool tim_consistent_fp64(const F4 ai, const F4 aj, const F4 bi, const F4 bj, double beta) {
  const double ax = (double)aj.x - (double)ai.x, ay = (double)aj.y - (double)ai.y, az = (double)aj.z - (double)ai.z;
  const double bx = (double)bj.x - (double)bi.x, by = (double)bj.y - (double)bi.y, bz = (double)bj.z - (double)bi.z;
  const double v1 = std::sqrt(ax * ax + ay * ay + az * az);
  const double v2 = std::sqrt(bx * bx + by * by + bz * bz);
  const double alpha_f = beta * (1.0 / v1);
  const double raw_f = v2 / v1;
  const bool in_f = std::fabs(raw_f - 1.0) <= alpha_f;
  const double alpha_r = beta * (1.0 / v2);
  const double raw_r = v1 / v2;
  const bool in_r = std::fabs(raw_r - 1.0) <= alpha_r;
  return in_f && in_r;
}

// the bit the kernel shifts in: every NaN an fp32 operation produces on the device is the canonical 0x7fffffff (sign bit clear)
inline bool sign_bit(float x) {
  if (std::isnan(x)) return false;
  uint32_t u;
  std::memcpy(&u, &x, 4);
  return u >> 31;
}

inline float norm2(const F4 p) { return std::fmaf(p.z, p.z, std::fmaf(p.y, p.y, p.x * p.x)); }  // graph.cu:135-136, 154-155

typedef __float128 Q;
inline Q qd(float a, float b) { return (Q)b - (Q)a; }

void run_set(int set, int L, const GraphConst& gc, const F4* A, const F4* B, bool fix, std::vector<Rec>& out) {
  const F4 zero4 = {0.f, 0.f, 0.f, 0.f};
  const int nb = (L + 31) >> 5;
  const float ntwob2 = -gc.twob2, nb4 = -gc.b4;                    // graph.cu:160
  const Q beta = (Q)gc.beta, beta2 = beta * beta;
  for (int bi = 0; bi < nb; ++bi) {
    // ---- the 32 staged rows of block bi (graph.cu:131-143); rows beyond L are zero points
    F4 r0[32], r1[32];
    float mm = 0.f;
    for (int lane = 0; lane < 32; ++lane) {
      const int i = bi * 32 + lane;
      const bool v = i < L;
      const F4 pa = v ? A[i] : zero4, pb = v ? B[i] : zero4;
      const float na = norm2(pa), nbn = norm2(pb);
      r0[lane] = {-2.0f * pa.x, -2.0f * pa.y, -2.0f * pa.z, na - gc.hb2q};
      r1[lane] = {-2.0f * pb.x, -2.0f * pb.y, -2.0f * pb.z, nbn - gc.hb2q};
      const float m = na + nbn;
      mm = lane == 0 ? m : std::fmax(mm, m);                      // the shuffle max: order-free, fmaxf drops NaN
    }
    for (int j = bi * 32; j < L; ++j) {                            // columns of blocks cbk >= bi (graph.cu:165, 202)
      const int cbk = j >> 5, lane = j & 31;
      // ---- the column (graph.cu:150-159)
      const F4 pa = A[j], pb = B[j];
      const float na = norm2(pa), nbn = norm2(pb);
      const F4 ca = {pa.x, pa.y, pa.z, na - gc.hb2q}, cb = {pb.x, pb.y, pb.z, nbn - gc.hb2q};
      const float cm = na + nbn;
      // ---- graph.cu:170-172
      const float Mj = (mm + cm + gc.two_b2_slack) * 1.00001f;
      const float qa = gc.c1 * Mj;
      const float qk = (gc.c2 * Mj + gc.c3) * Mj;
      // ---- the 32 row tests (graph.cu:180-196)
      float tv[32], Dv[32], qv[32];
      bool bt[32], bs[32], bw[32];
      float smin = 3.0e38f;
      for (int r = 0; r < 32; ++r) {
        const float Ap = std::fmaf(r0[r].x, ca.x, std::fmaf(r0[r].y, ca.y, std::fmaf(r0[r].z, ca.z, r0[r].w + ca.w)));
        const float Bp = std::fmaf(r1[r].x, cb.x, std::fmaf(r1[r].y, cb.y, std::fmaf(r1[r].z, cb.z, r1[r].w + cb.w)));
        const float D = Ap - Bp, sp = Ap + Bp;
        const float ng = std::fmaf(ntwob2, sp, nb4);
        const float t = std::fmaf(D, D, ng);
        const float q = std::fmaf(std::fabs(D), qa, qk);
        const float w = std::fabs(t) - q;
        tv[r] = t; Dv[r] = D; qv[r] = q;
        bt[r] = sign_bit(t); bs[r] = sign_bit(sp); bw[r] = sign_bit(w);
        smin = std::fmin(smin, sp);
      }
      // ---- the smin net (graph.cu:208-220): on the diagonal block the minimum is redone without row == lane
      float sm = smin;
      if (cbk == bi) {
        sm = 3.0e38f;
        for (int r = 0; r < 32; ++r) {
          const float Ap = std::fmaf(r0[r].x, ca.x, std::fmaf(r0[r].y, ca.y, std::fmaf(r0[r].z, ca.z, r0[r].w + ca.w)));
          const float Bp = std::fmaf(r1[r].x, cb.x, std::fmaf(r1[r].y, cb.y, std::fmaf(r1[r].z, cb.z, r1[r].w + cb.w)));
          if (r != lane) sm = std::fmin(sm, Ap + Bp);
        }
      }
      const bool net = sm <= std::fmaf(64.0f * 5.9604645e-8f, Mj, -gc.b2);
      const bool big = fix && !(Mj <= 0x1p62f);
      // ---- every live row (graph.cu:197-206, 221-233)
      for (int r = 0; r < 32; ++r) {
        const int i = bi * 32 + r;
        if (i >= L || i == j) continue;
        Rec rc;
        rc.set = set; rc.i = i; rc.j = j;
        rc.dec32 = bt[r] || bs[r];
        rc.to64 = (bw[r] ? 1 : 0) | (net ? 2 : 0) | (big ? 4 : 0);
        rc.lit = tim_consistent_fp64(A[i], A[j], B[i], B[j], gc.beta);
        const Q Aq = qd(A[i].x, A[j].x) * qd(A[i].x, A[j].x) + qd(A[i].y, A[j].y) * qd(A[i].y, A[j].y) + qd(A[i].z, A[j].z) * qd(A[i].z, A[j].z);
        const Q Bq = qd(B[i].x, B[j].x) * qd(B[i].x, B[j].x) + qd(B[i].y, B[j].y) * qd(B[i].y, B[j].y) + qd(B[i].z, B[j].z) * qd(B[i].z, B[j].z);
        const Q s = Aq + Bq - beta2;
        const Q t = s * s - 4 * Aq * Bq;
        rc.exact = t <= 0 || s <= 0;
        const Q e = (Q)tv[r] - t;
        const bool fin = std::isfinite(tv[r]) && std::isfinite(qv[r]) && std::isfinite(Dv[r]) && t == t && t - t == 0;
        rc.ratio = fin ? (double)((e < 0 ? -e : e) / (Q)qv[r]) : NAN;
        out.push_back(rc);
      }
    }
  }
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 3) { std::fprintf(stderr, "usage: %s IN OUT [nofix]\n", argv[0]); return 2; }
  const bool fix = !(argc > 3 && std::strcmp(argv[3], "nofix") == 0);
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  int32_t n_sets = 0;
  if (std::fread(&n_sets, 4, 1, f) != 1) return 4;
  std::vector<Rec> out;
  for (int s = 0; s < n_sets; ++s) {
    int32_t hdr[2];
    double prm[2];
    if (std::fread(hdr, 4, 2, f) != 2 || std::fread(prm, 8, 2, f) != 2) return 4;
    const int L = hdr[0];
    std::vector<F4> A(L), B(L);
    if (L > 0 && (std::fread(A.data(), 16, L, f) != (size_t)L || std::fread(B.data(), 16, L, f) != (size_t)L)) return 4;
    run_set(s, L, graph_const(prm[0], prm[1]), A.data(), B.data(), fix, out);
  }
  std::fclose(f);
  FILE* g = std::fopen(argv[2], "wb");
  if (!g) return 5;
  if (!out.empty() && std::fwrite(out.data(), sizeof(Rec), out.size(), g) != out.size()) return 6;
  std::fclose(g);
  return 0;
}
