// Per-edge and per-element arithmetic of the Hessian-vector product (engine.cu s7b_engine_hvp): the tangent of the
// edge geometry, the radial basis with its first and second r-derivatives, and the tangent of the edge backward.
// Host-compilable (tests/cpu_harness/hvp_harness.cpp checks it against numpy on the CPU).
#pragma once
#include <cmath>

#include "generated/sh.cuh"

namespace s7b {

// Envelope and its first two r-derivatives (edge_kernels.cuh envelope(); 0 from the cutoff on: both envelopes and
// their slopes vanish there, and the radial weights of an edge at or beyond it do not enter the energy).
// fn 0: XPLOR switching from r_on to rc; 1: polynomial of order p.
S7B_HD void envelope_jet(int fn, float rc, float r_on, int p, float r, float& env, float& d1, float& d2) {
  env = d1 = d2 = 0.0f;
  if (r >= rc) return;
  if (fn == 0) {
    if (r < r_on) { env = 1.0f; return; }
    const float r2 = r * r, on2 = r_on * r_on, c2 = rc * rc;
    const float den = (c2 - on2) * (c2 - on2) * (c2 - on2);
    const float a = c2 - r2, b = c2 + 2.0f * r2 - 3.0f * on2;
    env = a * a * b / den;
    d1 = (-4.0f * r * a * b + 4.0f * r * a * a) / den;
    d2 = (-4.0f * a * b + 8.0f * r2 * b - 32.0f * r2 * a + 4.0f * a * a) / den;
  } else {
    const float pf = (float)p, x = r / rc;
    float xm2 = 1.0f;                                    // x^(p-2)
    for (int i = 0; i < p - 2; ++i) xm2 *= x;
    const float xm1 = p >= 2 ? xm2 * x : 1.0f, xp = xm1 * x;
    const float c0 = (pf + 1.0f) * (pf + 2.0f) * 0.5f, c1 = pf * (pf + 2.0f), c2 = pf * (pf + 1.0f) * 0.5f;
    env = 1.0f - xp * (c0 - c1 * x + c2 * x * x);
    d1 = -xm1 * (c0 * pf - c1 * (pf + 1.0f) * x + c2 * (pf + 2.0f) * x * x) / rc;
    d2 = -(p >= 2 ? xm2 : 0.0f) * (c0 * pf * (pf - 1.0f) - c1 * (pf + 1.0f) * pf * x + c2 * (pf + 2.0f) * (pf + 1.0f) * x * x) / (rc * rc);
  }
}

// Bessel function 2/rc sin(c r)/r and its first two r-derivatives.  Below c r = 0.5, where the closed form of the
// second derivative cancels, the series of sin(x)/x = sum_k a_k x^2k to x^10 (truncation < 1e-10 relative).
S7B_HD void bessel_jet(float c, float rc, float r, float& b0, float& b1, float& b2) {
  const float pre = 2.0f / rc, cr = c * r;
  if (cr < 0.5f) {
    const float a[6] = {1.0f, -1.0f / 6.0f, 1.0f / 120.0f, -1.0f / 5040.0f, 1.0f / 362880.0f, -1.0f / 39916800.0f};
    const float x2 = cr * cr;
    float s0 = 0.0f, s1 = 0.0f, s2 = 0.0f;          // S(x), S'(x) / x, S''(x) by Horner in x^2
    for (int k = 5; k >= 0; --k) {
      s0 = s0 * x2 + a[k];
      if (k >= 1) s1 = s1 * x2 + 2.0f * k * a[k];
      if (k >= 1) s2 = s2 * x2 + 2.0f * k * (2.0f * k - 1.0f) * a[k];
    }
    b0 = pre * c * s0;
    b1 = pre * c * c * s1 * cr;
    b2 = pre * c * c * c * s2;
    return;
  }
  const float ir = 1.0f / r, sn = sinf(cr), cs = cosf(cr);
  b0 = pre * sn * ir;
  b1 = pre * (c * cs - sn * ir) * ir;
  b2 = pre * (-c * c * sn - 2.0f * c * cs * ir + 2.0f * sn * ir * ir) * ir;
}

// normalised silu s(z) = c z sigmoid(z) with s' and s''
S7B_HD void silu_n_jet(float z, float& s0, float& s1, float& s2) {
  const float sg = 1.0f / (1.0f + expf(-z));
  const float k = 1.6791767923989418f;                 // kSiluNorm (common.cuh)
  s0 = k * z * sg;
  s1 = k * sg * (1.0f + z * (1.0f - sg));
  s2 = k * sg * (1.0f - sg) * (2.0f + z * (1.0f - 2.0f * sg));
}

// Tangent of the edge geometry along d(edge_vec) = dv: dr = u . dv and dY = J_Y(u) du, du = (I - u u^T) dv / r
// (dY[0] = 0).  r = 0 (no direction) gives zeros.
template <int LMAX>
S7B_HD void edge_tangent(const float v[3], const float dv[3], float& dr, float* dY) {
  const float r = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const float ir = r > 0.0f ? 1.0f / r : 0.0f;
  const float u[3] = {v[0] * ir, v[1] * ir, v[2] * ir};
  dr = u[0] * dv[0] + u[1] * dv[1] + u[2] * dv[2];
  const float du[3] = {(dv[0] - dr * u[0]) * ir, (dv[1] - dr * u[1]) * ir, (dv[2] - dr * u[2]) * ir};
  SH2<LMAX>::jvp(u[0], u[1], u[2], du[0], du[1], du[2], dY);
}

// Structure of atom n in a batch whose structure b owns atoms [atom_ptr[b], atom_ptr[b+1]) (n < atom_ptr[n_sys]):
// the largest b with atom_ptr[b] <= n, so empty structures are skipped.
S7B_HD int structure_of(const int* atom_ptr, int n_sys, int n) {
  int lo = 0, hi = n_sys;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (atom_ptr[mid] <= n) lo = mid;
    else hi = mid;
  }
  return lo;
}

// dv += eps . v: the tangent of the edge vector under the homogeneous deformation r -> (I + s eps) r of atoms and
// cell (eps row-major 3x3, applied in fp64).
S7B_HD void add_strain_tangent(const double* eps, const float v[3], float dv[3]) {
  for (int a = 0; a < 3; ++a)
    dv[a] += (float)(eps[3 * a] * v[0] + eps[3 * a + 1] * v[1] + eps[3 * a + 2] * v[2]);
}

// Tangent of edge_bwd_kernel's f = ar u + (I - u u^T) J_Y^T gY / r along dv, given the tangents dgY of gY and dar
// of ar (gY[0], dgY[0] unused).  Writes df.
template <int LMAX>
S7B_HD void edge_bwd_tangent(const float v[3], const float dv[3], const float* gY, const float* dgY, float ar, float dar,
                             float df[3]) {
  const float r = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  const float ir = r > 0.0f ? 1.0f / r : 0.0f;
  const float u[3] = {v[0] * ir, v[1] * ir, v[2] * ir};
  const float dr = u[0] * dv[0] + u[1] * dv[1] + u[2] * dv[2];
  const float du[3] = {(dv[0] - dr * u[0]) * ir, (dv[1] - dr * u[1]) * ir, (dv[2] - dr * u[2]) * ir};
  float g[3], h[3], k[3];
  SH<LMAX>::vjp(u[0], u[1], u[2], gY, g[0], g[1], g[2]);
  SH2<LMAX>::hvp(u[0], u[1], u[2], gY, du[0], du[1], du[2], h[0], h[1], h[2]);
  SH<LMAX>::vjp(u[0], u[1], u[2], dgY, k[0], k[1], k[2]);
  const float dg[3] = {h[0] + k[0], h[1] + k[1], h[2] + k[2]};
  const float gu = g[0] * u[0] + g[1] * u[1] + g[2] * u[2];
  const float dgu = dg[0] * u[0] + dg[1] * u[1] + dg[2] * u[2] + g[0] * du[0] + g[1] * du[1] + g[2] * du[2];
  for (int c = 0; c < 3; ++c)
    df[c] = dar * u[c] + ar * du[c] + (dg[c] - dgu * u[c] - gu * du[c]) * ir - (g[c] - gu * u[c]) * ir * ir * dr;
}

}  // namespace s7b
