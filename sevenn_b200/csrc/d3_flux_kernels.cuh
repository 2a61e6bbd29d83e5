// Kernels of the D3 heat flux (d3.cu s7b_d3_heat_flux, s7b_d3_heat_flux_pass): the potential part of the
// energy-barycentre flux of D3's atomic energies (DESIGN.md §8.4), on the forward's cell list and sweep, with the
// forward's per-atom factors held.
//
// U_j = -1/2 sum_{k,tau} C6_jk(CN_j, CN_k) g(r_jk), self images included, as d3_pair_kernel's eatom.  For velocities v
// and the moment M_j[X] = sum_i (r_j - r_i) (dX/dr_i . v_i) (i over every atom and image, an image moving with its
// atom), J_pot = sum_j M_j[U_j].  With vec = r_k + tau - r_j, u = vec / r, q_k = u . v_k:
//   d3_flux_cn_kernel    dCN_j = sum_k f' u . (v_k - v_j),  P_j = M_j[CN_j] = sum_k (-vec) f' q_k        (CN radius)
//   d3_flux_pair_kernel  R_j = M_j[U_j] = -1/2 [dc6i_j P_j + sum_k (D_jk g (P_k - vec dCN_k) - C6 g' vec q_k)]
//                        (vdW radius), D_jk = dC6_jk/dCN_k = sum_b V_j[t_k][b] W'_k[b]; P_k - vec dCN_k = M_j[CN_k]
// and the per-atom terms eatom_j v_j of the convective part.  Self images contribute (vec = tau, q = u . v_j): they
// carry no force, but their moment is not zero.  Where the forward takes the "den <= 1e-99" branch, D_jk = 0.  Pair
// arithmetic in fp32, sums in fp64, one warp per atom, no atomics, fixed order; d3_system_sums_kernel sums per
// structure.
#pragma once
#include "d3_hvp_math.cuh"
#include "d3_kernels.cuh"

namespace s7b {

// registers <= 64K / (128 x blocks), no spills (ptxas -v)
constexpr int kD3FluxCnBlocks = 7, kD3FluxPairBlocks = 6;

struct D3Flux {               // bin-sorted atom order
  const double* v;            // [n,3]  velocities (bohr x the caller's time unit)
  const double* eatom;        // [n]    the forward's atomic energies (hartree)
  double* cn4;                // [n,4]  dCN_j, P_j (x, y, z)
  float4* nb;                 // [n,2]  (P_j, dCN_j), (v_j, 0) in float: what the pair pass reads of a neighbour, one
                              //        32-byte sector (the pair arithmetic rounds them to float anyway)
  double* out;                // [n,6]  R_j (x, y, z), eatom_j v_j (x, y, z)
};

// ---- pass 1: dCN_j and the moment P_j of CN_j ---------------------------------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3FluxCnBlocks)
d3_flux_cn_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, int3 R1, int i_begin, int i_end, D3Flux X) {
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= i_end) return;
  const float rci = P.rcov[d3_row<kBatch>(A.type[i])];
  const float vi[3] = {(float)X.v[3 * i], (float)X.v[3 * i + 1], (float)X.v[3 * i + 2]};
  double dcn = 0.0, px = 0.0, py = 0.0, pz = 0.0;
  d3_sweep_atom<kBatch>(g1, R1, A, i, 3, P.cnthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool) {
    const float rc = rci + P.rcov[d3_row<kBatch>(A.type[j])];
    float f, f1, f2;
    d3_count_jet(r2, rc, kD3K1, f, f1, f2);
    const float ir = d3_rsqrtf(r2);
    const float vj[3] = {(float)X.v[3 * j], (float)X.v[3 * j + 1], (float)X.v[3 * j + 2]};
    const float q = (dx * vj[0] + dy * vj[1] + dz * vj[2]) * ir;
    const float qi = (dx * vi[0] + dy * vi[1] + dz * vi[2]) * ir;
    const float fq = f1 * q;
    dcn += (double)(f1 * (q - qi));
    px -= (double)(dx * fq); py -= (double)(dy * fq); pz -= (double)(dz * fq);
  });
  dcn = warp_sum(dcn); px = warp_sum(px); py = warp_sum(py); pz = warp_sum(pz);
  if (lane == 0) {
    X.cn4[4 * (size_t)i] = dcn;
    X.cn4[4 * (size_t)i + 1] = px; X.cn4[4 * (size_t)i + 2] = py; X.cn4[4 * (size_t)i + 3] = pz;
    X.nb[2 * (size_t)i] = make_float4((float)px, (float)py, (float)pz, (float)dcn);
    X.nb[2 * (size_t)i + 1] = make_float4(vi[0], vi[1], vi[2], 0.0f);
  }
}

// ---- pass 2: R_j = M_j[U_j] and eatom_j v_j -----------------------------------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3FluxPairBlocks)
d3_flux_pair_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, const float* __restrict__ dW, int3 R1,
                    int i_begin, int i_end, D3Flux X) {
  __shared__ float sV[kD3WarpsPerBlock][kD3MaxTypes][5];        // V_i[t][b] over local types t, as d3_pair_kernel
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + wib;
  if (i >= i_end) return;
  const int ti = d3_row<kBatch>(A.type[i]), sb = kBatch ? A.sys[i] : 0;
  const int nloc = kBatch ? A.nloc[sb] : P.nrows;
  for (int q = lane; q < nloc * 5; q += 32) {
    const int t = q / 5, b = q % 5;
    const int tr = kBatch ? A.lrows[kD3MaxTypes * sb + t] : t;
    float v = 0.0f;
#pragma unroll
    for (int a = 0; a < 5; ++a) v = fmaf(__ldg(P.c6ref + ((ti * P.nrows + tr) * 5 + a) * 5 + b), A.W[i * 5 + a], v);
    sV[wib][t][b] = v;
  }
  __syncwarp();
  const float logDi = A.logD[i];
  const int near_i = A.near[i];
  const float r2r4i = P.r2r4[ti];
  double rx = 0.0, ry = 0.0, rz = 0.0;
  d3_sweep_atom<kBatch>(g1, R1, A, i, 0, P.rthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool) {
    const int twj = A.type[j], tj = d3_row<kBatch>(twj), lj = d3_local<kBatch>(twj);
    float c6 = 0.0f, D = 0.0f;                                   // C6_ij and dC6_ij/dCN_j
    if (logDi + A.logD[j] > -227.95593f) {
#pragma unroll
      for (int b = 0; b < 5; ++b) {
        c6 = fmaf(sV[wib][lj][b], A.W[j * 5 + b], c6);
        D = fmaf(sV[wib][lj][b], dW[j * 5 + b], D);
      }
    } else {
      c6 = __ldg(P.c6ref + ((ti * P.nrows + tj) * 5 + near_i) * 5 + A.near[j]);
    }
    float g, g1d, g2d;
    const float r = sqrtf(r2);
    if (P.damping == 1)
      d3_damp_bj_jet(r, r2r4i * P.r2r4[tj] * 3.0f, P.s6, P.s8, P.a1, P.a2, g, g1d, g2d);
    else
      d3_damp_zero_jet(r, __ldg(P.r0ab + ti * P.nrows + tj), r2r4i * P.r2r4[tj], P.s6, P.s8, P.a1, P.a2, P.alp6, P.alp8,
                       g, g1d, g2d);
    const float4 pj = __ldg(X.nb + 2 * (size_t)j), vj = __ldg(X.nb + 2 * (size_t)j + 1);
    const float q = (dx * vj.x + dy * vj.y + dz * vj.z) / r;
    const float Dg = D * g, b = c6 * g1d * q;
    // D g (P_k - vec dCN_k) - C6 g' vec q_k = D g P_k - vec (D g dCN_k + C6 g' q_k)
    const float s = fmaf(Dg, pj.w, b);
    rx += (double)fmaf(Dg, pj.x, -s * dx);
    ry += (double)fmaf(Dg, pj.y, -s * dy);
    rz += (double)fmaf(Dg, pj.z, -s * dz);
  });
  rx = warp_sum(rx); ry = warp_sum(ry); rz = warp_sum(rz);
  if (lane == 0) {
    const double di = A.dc6i[i], e = X.eatom[i];
    const double* ci = X.cn4 + 4 * (size_t)i;
    double* o = X.out + 6 * (size_t)i;
    o[0] = -0.5 * (di * ci[1] + rx); o[1] = -0.5 * (di * ci[2] + ry); o[2] = -0.5 * (di * ci[3] + rz);
    o[3] = e * X.v[3 * i]; o[4] = e * X.v[3 * i + 1]; o[5] = e * X.v[3 * i + 2];
  }
}

// per-structure sums (d3_system_sums_kernel's sigma layout: R in 0..2, eatom v in 3..5) -> J_pot [B,3] and sum U v
// [B,3] in eV A x (the caller's velocity unit)
__global__ void d3_flux_results_kernel(int B, const double* __restrict__ sums, double* __restrict__ jpot,
                                       double* __restrict__ ju) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * B) return;
  const int b = t / 3, c = t - 3 * b;
  jpot[t] = sums[6 * (size_t)b + c] * (kAuToEv * kAuToAng);
  if (ju) ju[t] = sums[6 * (size_t)b + 3 + c] * (kAuToEv * kAuToAng);
}

}  // namespace s7b
