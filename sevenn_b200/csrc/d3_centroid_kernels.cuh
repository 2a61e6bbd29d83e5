// Kernels of the D3 per-atom centroid virial (d3.cu s7b_d3_centroid_virial, s7b_d3_centroid_pass; DESIGN.md §8.6),
// on the forward's cell list and sweep, with the forward's per-atom factors held.
//
// U_j = -1/2 sum_{k,tau} C6_jk(CN_j, CN_k) g(r_jk), self images included, as d3_pair_kernel's eatom, and
// Wc_i[a][b] = sum_j sum_i' (r_j - r_i')_a dU_j/dr_i',b over atom i and its images i'.  With vec = r_k + tau - r_i,
// u = vec / r, alpha_i = dE/dCN_i = -dc6i_i and f' = dCN/dr of the counting function (d3_chain_kernel's dcnn):
//   direct part               sum_k 1/2 C6 g'/r vec (x) vec: the forward pair pass's spair_i, read as it is
//   d3_centroid_moment_kernel beta_i = sum_{j, images} dU_j/dCN_i (r_j' - r_i) = -1/2 sum_k g dC6_ik/dCN_i vec
//                             (vdW radius; dC6 = 0 where the forward takes the "den <= 1e-99" branch)
//   d3_centroid_cn_kernel     Wc_i = spair_i - sum_m f'(r_im) (beta_m + beta_i + alpha_m vec_im) (x) u_im
//                             (CN radius, the chain pass's strict bound), in eV
// Self images contribute: their beta terms cancel between +-tau, their alpha term does not.  Summed over i the beta
// terms cancel pair by pair and the alpha term is schain's sum, so sum_i Wc_i is the virial.  Pair arithmetic in fp32,
// sums in fp64, one warp per atom, no atomics, fixed order: a batch member's rows are those of the structure alone.
#pragma once
#include "d3_hvp_math.cuh"
#include "d3_kernels.cuh"

namespace s7b {

// registers <= 64K / (128 x blocks), no spills (ptxas -v)
constexpr int kD3CentroidMomentBlocks = 7, kD3CentroidCnBlocks = 7;

struct D3Centroid {           // bin-sorted atom order
  double* beta;               // [n,3] beta_i (bohr x hartree / CN)
  float4* nb;                 // [n]   (beta_i, alpha_i) in float: what the CN pass reads of a neighbour, 16 bytes
  const double* spair;        // [n,6] the forward's pair rows (hartree; xx, yy, zz, xy, xz, yz)
  double* out;                // [n,9] Wc_i row-major (eV)
};

// ---- pass 1: beta_i, the moment of the CN adjoint ------------------------------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3CentroidMomentBlocks)
d3_centroid_moment_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, const float* __restrict__ dW, int3 R1,
                          int i_begin, int i_end, D3Centroid C) {
  __shared__ float sdV[kD3WarpsPerBlock][kD3MaxTypes][5];       // dV_i[t][b] over local types t, as d3_pair_kernel
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + wib;
  if (i >= i_end) return;
  const int ti = d3_row<kBatch>(A.type[i]), sb = kBatch ? A.sys[i] : 0;
  const int nloc = kBatch ? A.nloc[sb] : P.nrows;
  for (int q = lane; q < nloc * 5; q += 32) {
    const int t = q / 5, b = q % 5;
    const int tr = kBatch ? A.lrows[kD3MaxTypes * sb + t] : t;
    float dv = 0.0f;
#pragma unroll
    for (int a = 0; a < 5; ++a) dv = fmaf(__ldg(P.c6ref + ((ti * P.nrows + tr) * 5 + a) * 5 + b), dW[i * 5 + a], dv);
    sdV[wib][t][b] = dv;
  }
  __syncwarp();
  const float logDi = A.logD[i];
  const float r2r4i = P.r2r4[ti];
  double bx = 0.0, by = 0.0, bz = 0.0;
  d3_sweep_atom<kBatch>(g1, R1, A, i, 0, P.rthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool) {
    if (!(logDi + A.logD[j] > -227.95593f)) return;             // den <= 1e-99: dC6/dCN = 0
    const int twj = A.type[j], tj = d3_row<kBatch>(twj), lj = d3_local<kBatch>(twj);
    float dc6 = 0.0f;                                           // dC6_ij/dCN_i
#pragma unroll
    for (int b = 0; b < 5; ++b) dc6 = fmaf(sdV[wib][lj][b], A.W[j * 5 + b], dc6);
    float g, g1d, g2d;
    const float r = sqrtf(r2);
    if (P.damping == 1)
      d3_damp_bj_jet(r, r2r4i * P.r2r4[tj] * 3.0f, P.s6, P.s8, P.a1, P.a2, g, g1d, g2d);
    else
      d3_damp_zero_jet(r, __ldg(P.r0ab + ti * P.nrows + tj), r2r4i * P.r2r4[tj], P.s6, P.s8, P.a1, P.a2, P.alp6, P.alp8,
                       g, g1d, g2d);
    const float s = -0.5f * g * dc6;
    bx += (double)(s * dx); by += (double)(s * dy); bz += (double)(s * dz);
  });
  bx = warp_sum(bx); by = warp_sum(by); bz = warp_sum(bz);
  if (lane == 0) {
    C.beta[3 * (size_t)i] = bx; C.beta[3 * (size_t)i + 1] = by; C.beta[3 * (size_t)i + 2] = bz;
    C.nb[i] = make_float4((float)bx, (float)by, (float)bz, (float)(-A.dc6i[i]));
  }
}

// ---- pass 2: the CN part, plus spair, -> Wc_i in eV ----------------------------------------------------------------
// -sum_m f' (beta_m + alpha_m vec) (x) u per candidate; the beta_i term is beta_i (x) (-sum_m f' u), formed once at the
// end in fp64.
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3CentroidCnBlocks)
d3_centroid_cn_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, int3 R1, int i_begin, int i_end,
                      D3Centroid C) {
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= i_end) return;
  const float rci = P.rcov[d3_row<kBatch>(A.type[i])];
  const float cn2 = (float)P.cnthr;
  double w[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, su[3] = {0, 0, 0};
  d3_sweep_atom<kBatch>(g1, R1, A, i, 3, P.cnthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool) {
    if (r2 >= cn2) return;                                      // the chain pass's strict bound
    const float rc = rci + P.rcov[d3_row<kBatch>(A.type[j])];
    float f, f1, f2;
    d3_count_jet(r2, rc, kD3K1, f, f1, f2);
    const float c = -f1 * d3_rsqrtf(r2);                        // -f' / r
    const float4 bj = __ldg(C.nb + j);
    const float m[3] = {fmaf(bj.w, dx, bj.x), fmaf(bj.w, dy, bj.y), fmaf(bj.w, dz, bj.z)};
    const float cu[3] = {c * dx, c * dy, c * dz};
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) w[3 * a + b] += (double)(m[a] * cu[b]);
#pragma unroll
    for (int b = 0; b < 3; ++b) su[b] += (double)cu[b];
  });
#pragma unroll
  for (int q = 0; q < 9; ++q) w[q] = warp_sum(w[q]);
#pragma unroll
  for (int b = 0; b < 3; ++b) su[b] = warp_sum(su[b]);
  if (lane == 0) {
    const double* bi = C.beta + 3 * (size_t)i;
    const double* sp = C.spair + 6 * (size_t)i;
    const double s[9] = {sp[0], sp[3], sp[4], sp[3], sp[1], sp[5], sp[4], sp[5], sp[2]};
    double* o = C.out + 9 * (size_t)i;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) o[3 * a + b] = (s[3 * a + b] + w[3 * a + b] + bi[a] * su[b]) * kAuToEv;
  }
}

}  // namespace s7b
