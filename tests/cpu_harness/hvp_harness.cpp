// Host-side harness: exposes the per-edge arithmetic of the Hessian-vector product (hvp_math.cuh, and the generated
// SH2<L> it calls) through a C interface so that tests/test_hvp_cpu.py can check it against numpy on the CPU.
// (Test infrastructure only; compiled with g++ by the test.)
#include "../../sevenn_b200/csrc/hvp_math.cuh"

using namespace s7b;

extern "C" {

int hv_sh_vjp(int L, const float* u, const float* gY, float* g) {
  if (L == 1) SH<1>::vjp(u[0], u[1], u[2], gY, g[0], g[1], g[2]);
  else if (L == 2) SH<2>::vjp(u[0], u[1], u[2], gY, g[0], g[1], g[2]);
  else if (L == 3) SH<3>::vjp(u[0], u[1], u[2], gY, g[0], g[1], g[2]);
  else return 1;
  return 0;
}

int hv_sh_hvp(int L, const float* u, const float* gY, const float* t, float* h) {
  if (L == 1) SH2<1>::hvp(u[0], u[1], u[2], gY, t[0], t[1], t[2], h[0], h[1], h[2]);
  else if (L == 2) SH2<2>::hvp(u[0], u[1], u[2], gY, t[0], t[1], t[2], h[0], h[1], h[2]);
  else if (L == 3) SH2<3>::hvp(u[0], u[1], u[2], gY, t[0], t[1], t[2], h[0], h[1], h[2]);
  else return 1;
  return 0;
}

int hv_edge_tangent(int L, const float* v, const float* dv, float* dr, float* dY) {
  if (L == 1) edge_tangent<1>(v, dv, *dr, dY);
  else if (L == 2) edge_tangent<2>(v, dv, *dr, dY);
  else if (L == 3) edge_tangent<3>(v, dv, *dr, dY);
  else return 1;
  return 0;
}

int hv_edge_bwd_tangent(int L, const float* v, const float* dv, const float* gY, const float* dgY, float ar, float dar,
                        float* df) {
  if (L == 1) edge_bwd_tangent<1>(v, dv, gY, dgY, ar, dar, df);
  else if (L == 2) edge_bwd_tangent<2>(v, dv, gY, dgY, ar, dar, df);
  else if (L == 3) edge_bwd_tangent<3>(v, dv, gY, dgY, ar, dar, df);
  else return 1;
  return 0;
}

// out[3 * i + k]: k-th r-derivative (k = 0, 1, 2) of envelope x Bessel function c at r[i]
void hv_radial_basis_jet(int fn, float rc, float r_on, int p, float c, const float* r, int n, float* out) {
  for (int i = 0; i < n; ++i) {
    float f0, f1, f2, b0, b1, b2;
    envelope_jet(fn, rc, r_on, p, r[i], f0, f1, f2);
    bessel_jet(c, rc, r[i], b0, b1, b2);
    out[3 * i] = b0 * f0;
    out[3 * i + 1] = b1 * f0 + b0 * f1;
    out[3 * i + 2] = b2 * f0 + 2.0f * b1 * f1 + b0 * f2;
  }
}

void hv_silu_n_jet(const float* z, int n, float* out) {
  for (int i = 0; i < n; ++i) silu_n_jet(z[i], out[3 * i], out[3 * i + 1], out[3 * i + 2]);
}

}  // extern "C"
