// Host-side harness of the strain tangent (hvp_math.cuh add_strain_tangent, structure_of) on top of the
// Hessian-vector product's harness, so that tests/test_elastic_cpu.py checks the per-edge arithmetic of
// hvp_edge_fwd_kernel with a strain against numpy.  (Test infrastructure only; compiled with g++ by the test.)
#include "hvp_harness.cpp"

extern "C" {

// hvp_edge_fwd_kernel's per-edge work: dv = (vs - vc, or 0 when vs is null) + eps . v, then (dr, dY) of edge_tangent
int hv_edge_strain_tangent(int L, const float* v, const float* vs, const float* vc, const double* eps, float* dv,
                           float* dr, float* dY) {
  for (int c = 0; c < 3; ++c) dv[c] = vs ? vs[c] - vc[c] : 0.0f;
  if (eps) add_strain_tangent(eps, v, dv);
  return hv_edge_tangent(L, v, dv, dr, dY);
}

int hv_structure_of(const int* atom_ptr, int n_sys, int n) { return structure_of(atom_ptr, n_sys, n); }

}  // extern "C"
