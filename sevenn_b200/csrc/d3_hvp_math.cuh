// Per-pair and per-atom arithmetic of the D3 Hessian-vector product (d3.cu s7b_d3_hvp_strain): value, first and
// second derivative of the damping functions, of the coordination-number counting function and of the normalised
// C6 reference weights, and the tangent of a pair vector.  The arithmetic of the value and first derivative is the
// forward's (d3_kernels.cuh), so a jet's (g, g') is what the forward computes.  Host-compilable
// (tests/cpu_harness/d3_hvp_harness.cpp checks it against numpy on the CPU).
#pragma once
#include <cmath>

#include "hvp_math.cuh"

namespace s7b {

// the forward's fast intrinsics on the device, their libm counterparts on the host
S7B_HD float d3_expf(float x) {
#ifdef __CUDA_ARCH__
  return __expf(x);
#else
  return expf(x);
#endif
}
S7B_HD float d3_powf(float x, float y) {
#ifdef __CUDA_ARCH__
  return __powf(x, y);
#else
  return powf(x, y);
#endif
}
S7B_HD float d3_rsqrtf(float x) {
#ifdef __CUDA_ARCH__
  return rsqrtf(x);
#else
  return 1.0f / sqrtf(x);
#endif
}

// Becke-Johnson damping, E_pair = -C6 g(r): g = s6 / (r^6 + R0^6) + s8 r42x3 / (r^8 + R0^8), R0 = a1 sqrt(r42x3) + a2,
// r42x3 = 3 r2r4_i r2r4_j (bohr).  g1 = dg/dr, g2 = d2g/dr2.
S7B_HD void d3_damp_bj_jet(float r, float r42x3, float s6, float s8, float a1, float a2, float& g, float& g1, float& g2) {
  const float r2 = r * r;
  const float R0 = fmaf(a1, sqrtf(r42x3), a2);
  const float R0_2 = R0 * R0, R0_6 = R0_2 * R0_2 * R0_2, R0_8 = R0_6 * R0_2;
  const float r5 = r2 * r2 * r, r7 = r5 * r2;
  const float t6 = 1.0f / fmaf(r5, r, R0_6), t8 = 1.0f / fmaf(r7, r, R0_8);
  const float s8r = s8 * r42x3;
  g = fmaf(s8r, t8, s6 * t6);
  g1 = -fmaf(8.0f * s8r * r7, t8 * t8, 6.0f * s6 * r5 * t6 * t6);
  // d/dr (-6 r^5 t6^2) = -30 r^4 t6^2 + 72 r^10 t6^3 = t6 a6 (72 a6 - 30 / r), a6 = r^5 t6; likewise for t8
  const float a6 = r5 * t6, a8 = r7 * t8, ir = 1.0f / r;
  g2 = s6 * t6 * a6 * fmaf(72.0f, a6, -30.0f * ir) + s8r * t8 * a8 * fmaf(128.0f, a8, -56.0f * ir);
}

// Zero damping: g = s6 d6 / r^6 + 3 s8 r42 d8 / r^8, d_n = 1 / (1 + 6 (a r0 / r)^alp_n) (a = a1 for 6, a2 for 8).
// For h = c d r^-n, d = 1 / (1 + 6 t), t = (A / r)^alp, y = alp t d:
//   h' = c d r^-(n+1) (6 y - n),  h'' = c d r^-(n+2) [(6 y - n - 1)(6 y - n) - 6 alp y d].
S7B_HD void d3_damp_zero_jet(float r, float r0, float r42, float s6, float s8, float a1, float a2, float alp6, float alp8,
                             float& g, float& g1, float& g2) {
  const float rr = 1.0f / r;
  const float t6 = d3_powf(a1 * r0 * rr, alp6), t8 = d3_powf(a2 * r0 * rr, alp8);
  const float d6 = 1.0f / fmaf(6.0f, t6, 1.0f), d8 = 1.0f / fmaf(6.0f, t8, 1.0f);
  const float r2_rc = rr * rr, r6_rc = r2_rc * r2_rc * r2_rc, r8_rc = r6_rc * r2_rc;
  const float s8r = s8 * r42;
  g = r6_rc * fmaf(3.0f * r2_rc, s8r * d8, s6 * d6);
  g1 = 6.0f * r8_rc * r * (s6 * d6 * fmaf(alp6 * t6, d6, -1.0f) + r2_rc * s8r * d8 * fmaf(3.0f * alp8 * t8, d8, -4.0f));
  const float y6 = alp6 * t6 * d6, y8 = alp8 * t8 * d8;
  const float k6 = fmaf(6.0f, y6, -7.0f) * fmaf(6.0f, y6, -6.0f) - 6.0f * alp6 * y6 * d6;
  const float k8 = fmaf(6.0f, y8, -9.0f) * fmaf(6.0f, y8, -8.0f) - 6.0f * alp8 * y8 * d8;
  g2 = r8_rc * (s6 * d6 * k6 + 3.0f * r2_rc * s8r * d8 * k8);
}

// Counting function f = 1 / (1 + exp(-K1 (rc / r - 1))) of the coordination number at r^2 = r2 (bohr^2), with
// f1 = df/dr (the chain pass's dcnn) and f2 = d2f/dr2 = f1 (q (1 - e) / (1 + e) - 2 / r), q = K1 rc / r^2.
S7B_HD void d3_count_jet(float r2, float rc, float k1, float& f, float& f1, float& f2) {
  const float rr = d3_rsqrtf(r2);
  const float ex = d3_expf(-k1 * (rc * rr - 1.0f));
  f = 1.0f / (1.0f + ex);
  f1 = -k1 * rc * ex / (r2 * (ex + 1.0f) * (ex + 1.0f));
  const float q = k1 * rc * rr * rr;
  f2 = f1 * (q * (1.0f - ex) / (1.0f + ex) - 2.0f * rr);
}

// Normalised reference weights of one atom at coordination number cn and their first two CN-derivatives, in double
// as d3_weights_kernel: w_a = exp(k3 (CN - CN_a)^2) over the m references, W_a = w_a / D, D = sum_a w_a,
// w_a' = 2 k3 (CN - CN_a) w_a, w_a'' = ((2 k3 (CN - CN_a))^2 + 2 k3) w_a, W' = (w' - W D') / D,
// W'' = (w'' - 2 W' D' - W D'') / D.  D <= 1e-300: W is one-hot on the nearest reference and W' = W'' = 0.
S7B_HD void d3_weight_jet(float cn, const float* cnref, int m, double k3, double* W, double* W1, double* W2) {
  double w[5], w1[5], w2[5], D = 0.0, D1 = 0.0, D2 = 0.0;
  float best = 3.0e38f;
  int nb = 0;
  for (int a = 0; a < 5; ++a) {
    w[a] = w1[a] = w2[a] = 0.0;
    if (a >= m) continue;
    const float cr = cnref[a];
    const float d2 = (cr - cn) * (cr - cn);
    if (d2 < best) { best = d2; nb = a; }
    const double x = 2.0 * k3 * (double)(cn - cr);
    w[a] = exp(k3 * (double)d2);
    w1[a] = w[a] * x;
    w2[a] = w[a] * (x * x + 2.0 * k3);
    D += w[a];
    D1 += w1[a];
    D2 += w2[a];
  }
  for (int a = 0; a < 5; ++a) {
    if (D > 1e-300) {
      W[a] = w[a] / D;
      W1[a] = (w1[a] - W[a] * D1) / D;
      W2[a] = (w2[a] - 2.0 * W1[a] * D1 - W[a] * D2) / D;
    } else {
      W[a] = a == nb ? 1.0 : 0.0;
      W1[a] = W2[a] = 0.0;
    }
  }
}

// Tangent of the pair vector vec = x_j - x_i + tau along positions v (bohr, double) and a strain eps (row-major 3x3,
// applied as eps . vec; nullptr = none): dvec = v_j - v_i + eps . vec.
S7B_HD void d3_pair_dvec(const double* vi, const double* vj, const double* eps, const float vec[3], float dvec[3]) {
  for (int c = 0; c < 3; ++c) dvec[c] = (float)(vj[c] - vi[c]);
  if (eps) add_strain_tangent(eps, vec, dvec);
}

// r = |vec|, u = vec / r, dr = u . dvec, du = (I - u u^T) dvec / r
S7B_HD void d3_pair_tangent(const float vec[3], const float dvec[3], float& r, float u[3], float& dr, float du[3]) {
  r = sqrtf(vec[0] * vec[0] + vec[1] * vec[1] + vec[2] * vec[2]);
  const float ir = 1.0f / r;
  for (int c = 0; c < 3; ++c) u[c] = vec[c] * ir;
  dr = u[0] * dvec[0] + u[1] * dvec[1] + u[2] * dvec[2];
  for (int c = 0; c < 3; ++c) du[c] = (dvec[c] - dr * u[c]) * ir;
}

}  // namespace s7b
