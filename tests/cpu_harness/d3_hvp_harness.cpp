// Host-side harness of the D3 Hessian-vector product's arithmetic (sevenn_b200/csrc/d3_hvp_math.cuh): the damping,
// counting-function and reference-weight jets and the pair tangent, through a C interface so that
// tests/test_d3_hvp_cpu.py checks them against numpy on the CPU.  (Test infrastructure only; compiled with g++ by
// the test.)
#include "../../sevenn_b200/csrc/d3_hvp_math.cuh"

using namespace s7b;

extern "C" {

// out[3 * k + (0, 1, 2)] = (g, g', g'') at r[k]; damping 1: Becke-Johnson (p = r42x3), 0: zero (p = r42, r0)
void d3h_damp_jet(int damping, const float* r, int n, float p, float r0, float s6, float s8, float a1, float a2,
                  float alp6, float alp8, float* out) {
  for (int k = 0; k < n; ++k) {
    if (damping == 1) d3_damp_bj_jet(r[k], p, s6, s8, a1, a2, out[3 * k], out[3 * k + 1], out[3 * k + 2]);
    else d3_damp_zero_jet(r[k], r0, p, s6, s8, a1, a2, alp6, alp8, out[3 * k], out[3 * k + 1], out[3 * k + 2]);
  }
}

// out[3 * k + (0, 1, 2)] = (f, f', f'') at r2[k] (bohr^2)
void d3h_count_jet(const float* r2, int n, float rc, float k1, float* out) {
  for (int k = 0; k < n; ++k) d3_count_jet(r2[k], rc, k1, out[3 * k], out[3 * k + 1], out[3 * k + 2]);
}

// out[15 * k + 5 * d + a]: d-th CN-derivative of W_a at cn[k]
void d3h_weight_jet(const float* cn, int n, const float* cnref, int m, double k3, double* out) {
  for (int k = 0; k < n; ++k) d3_weight_jet(cn[k], cnref, m, k3, out + 15 * k, out + 15 * k + 5, out + 15 * k + 10);
}

// dvec of d3_pair_dvec (eps may be null), then (r, u, dr, du) of d3_pair_tangent: out = [dvec(3), r, u(3), dr, du(3)]
void d3h_pair_tangent(const double* vi, const double* vj, const double* eps, const float* vec, float* out) {
  d3_pair_dvec(vi, vj, eps, vec, out);
  d3_pair_tangent(vec, out, out[3], out + 4, out[7], out + 8);
}

}  // extern "C"
