// Kernels of the D3 Hessian-vector product (d3.cu s7b_d3_hvp_strain): forward over reverse of the three D3 passes
// along a tangent of the positions v and a per-structure strain eps, on the forward's cell list and sweep.
//
// E = -1/2 sum_{i,j,tau} C6_ij(CN_i, CN_j) g(r_ij), CN_i = sum_j f(r_ij).  Along dvec_ij = v_j - v_i + eps_b . vec_ij:
//   d3_hvp_cn_kernel      dCN_i = sum_j f'(r) dr                                                  (CN radius)
//   d3_hvp_weights_kernel dW = W' dCN, dW' = W'' dCN                                               (per atom)
//   d3_hvp_pair_kernel    -dF_i = sum_j (dC6 g' + C6 g'' dr) u + C6 g' du, dC6 = d_i C6 dCN_i + d_j C6 dCN_j,
//                         d(dc6i_i) = sum_j g' dr d_i C6 + g (d2_ii C6 dCN_i + d2_ij C6 dCN_j)     (vdW radius)
//   d3_hvp_chain_kernel   -dF_i = sum_j [(ddc_i + ddc_j) f' + S f'' dr] u + S f' du, S = dc6i_i + dc6i_j  (CN radius)
// The force tangent is accumulated as -dF = H v + Lambda eps (hartree/bohr^2 x bohr), and the pair and chain passes
// write the per-atom terms of the virial's tangent dW = -sum (dvec (x) f + vec (x) df) in the forward's order
// (xx, yy, zz, xy, xz, yz); d3_system_sums_kernel and d3_system_results_kernel then sum, unsort and convert them as
// they do the forward's.  Pair arithmetic in fp32, sums in fp64, one warp per atom, no atomics, fixed order.  Where
// the forward is piecewise constant (the pair-level "den <= 1e-99" branch, the one-hot weights of D <= 1e-300, the
// strict r^2 < cnthr bound of the chain pass) the tangent is 0; self images carry no force, as in the forward.
#pragma once
#include "d3_hvp_math.cuh"
#include "d3_kernels.cuh"

namespace s7b {

// registers <= 64K / (128 x blocks), no spills (ptxas -v)
constexpr int kD3HvpCnBlocks = 8, kD3HvpPairBlocks = 4, kD3HvpChainBlocks = 5;

struct D3Hvp {                // bin-sorted atom order
  const double* v;            // [n,3]  position tangent (bohr)
  const double* strain;       // [B,9]  strain tangent per structure, or nullptr
  double* dcn;                // [n]    dCN
  float* dWt;                 // [n,5]  W' dCN (tangent of W)
  float* dW1t;                // [n,5]  W'' dCN (tangent of W')
  double* ddc;                // [n]    tangent of dc6i (after the pair pass)
  double* hforce;             // [n,3]  -dF
  double* spair;              // [n,6]  virial-tangent terms of the pair pass
  double* schain;             // [n,6]  virial-tangent terms of the chain pass
};

template <bool kBatch>
__device__ __forceinline__ const double* d3_hvp_eps(const D3Atoms& A, const D3Hvp& H, int i) {
  return H.strain ? H.strain + 9 * (kBatch ? A.sys[i] : 0) : nullptr;
}

// caller's atom order (Angstrom) -> sorted order (bohr); v == nullptr: zeros
__global__ void d3_hvp_gather_kernel(int n, const int* __restrict__ idx_sorted, const double* __restrict__ v,
                                     double* __restrict__ vs) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3 * n) return;
  const int s = t / 3, c = t - 3 * s;
  vs[t] = v ? v[3 * (size_t)idx_sorted[s] + c] / kAuToAng : 0.0;
}

// ---- pass 1: dCN_i = sum_j f'(r_ij) dr_ij -----------------------------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3HvpCnBlocks)
d3_hvp_cn_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, int3 R1, int n, D3Hvp H) {
  const int i = blockIdx.x * kD3WarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  const float rci = P.rcov[d3_row<kBatch>(A.type[i])];
  const double* eps = d3_hvp_eps<kBatch>(A, H, i);
  const double* vi = H.v + 3 * i;
  double dcn = 0.0;
  d3_sweep_atom<kBatch>(g1, R1, A, i, 3, P.cnthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool) {
    const float rc = rci + P.rcov[d3_row<kBatch>(A.type[j])];
    float f, f1, f2, r, dr, u[3], du[3], dvec[3];
    const float vec[3] = {dx, dy, dz};
    d3_count_jet(r2, rc, kD3K1, f, f1, f2);
    d3_pair_dvec(vi, H.v + 3 * j, eps, vec, dvec);
    d3_pair_tangent(vec, dvec, r, u, dr, du);
    dcn += (double)(f1 * dr);
  });
  dcn = warp_sum(dcn);
  if (lane == 0) H.dcn[i] = dcn;
}

// ---- per atom: tangents of the reference weights and of their CN derivative ------------------------------------
__global__ void d3_hvp_weights_kernel(int n, const int* __restrict__ type, const double* __restrict__ cn,
                                      const float* __restrict__ cnref /*[nrows,5]*/, const int* __restrict__ mxc,
                                      const double* __restrict__ dcn, float* __restrict__ dWt, float* __restrict__ dW1t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = type[i] & 0xff;
  double W[5], W1[5], W2[5];
  d3_weight_jet((float)cn[i], cnref + 5 * t, mxc[t], kD3K3, W, W1, W2);
  const double dc = dcn[i];
#pragma unroll
  for (int a = 0; a < 5; ++a) {
    dWt[i * 5 + a] = (float)(W1[a] * dc);
    dW1t[i * 5 + a] = (float)(W2[a] * dc);
  }
}

// ---- pass 2: tangent of the explicit force, of dc6i and the pair virial ------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3HvpPairBlocks)
d3_hvp_pair_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, const float* __restrict__ dW, int3 R1, int n,
                   D3Hvp H) {
  // V_i[t][b], dV_i[t][b] (from W'), ddV_i[t][b] (from W'' dCN_i) over local types t
  __shared__ float sV[kD3WarpsPerBlock][kD3MaxTypes][15];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kD3WarpsPerBlock + wib;
  if (i >= n) return;
  const int ti = d3_row<kBatch>(A.type[i]), sb = kBatch ? A.sys[i] : 0;
  const int nloc = kBatch ? A.nloc[sb] : P.nrows;
  for (int q = lane; q < nloc * 5; q += 32) {
    const int t = q / 5, b = q % 5;
    const int tr = kBatch ? A.lrows[kD3MaxTypes * sb + t] : t;
    float v = 0.0f, dv = 0.0f, ddv = 0.0f;
#pragma unroll
    for (int a = 0; a < 5; ++a) {
      const float c = __ldg(P.c6ref + ((ti * P.nrows + tr) * 5 + a) * 5 + b);
      v = fmaf(c, A.W[i * 5 + a], v);
      dv = fmaf(c, dW[i * 5 + a], dv);
      ddv = fmaf(c, H.dW1t[i * 5 + a], ddv);
    }
    sV[wib][t][b] = v;
    sV[wib][t][5 + b] = dv;
    sV[wib][t][10 + b] = ddv;
  }
  __syncwarp();
  const float logDi = A.logD[i];
  const int near_i = A.near[i];
  const float r2r4i = P.r2r4[ti];
  const float dcni = (float)H.dcn[i];
  const double* eps = d3_hvp_eps<kBatch>(A, H, i);
  const double* vi = H.v + 3 * i;
  double hx = 0.0, hy = 0.0, hz = 0.0, ddc = 0.0;
  double sg[6] = {0, 0, 0, 0, 0, 0};
  d3_sweep_atom<kBatch>(g1, R1, A, i, 0, P.rthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool self) {
    const int twj = A.type[j], tj = d3_row<kBatch>(twj), lj = d3_local<kBatch>(twj);
    // c6 = C6, dc6 = d_i C6, dC6 = tangent of C6, ddc6 = tangent of d_i C6
    float c6 = 0.0f, dc6 = 0.0f, dC6 = 0.0f, ddc6 = 0.0f;
    if (logDi + A.logD[j] > -227.95593f) {
      float dcj = 0.0f;
#pragma unroll
      for (int b = 0; b < 5; ++b) {
        const float wj = A.W[j * 5 + b], twj5 = H.dWt[j * 5 + b];
        c6 = fmaf(sV[wib][lj][b], wj, c6);
        dc6 = fmaf(sV[wib][lj][5 + b], wj, dc6);
        dcj = fmaf(sV[wib][lj][b], twj5, dcj);
        ddc6 = fmaf(sV[wib][lj][10 + b], wj, fmaf(sV[wib][lj][5 + b], twj5, ddc6));
      }
      dC6 = fmaf(dc6, dcni, dcj);
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
    const float vec[3] = {dx, dy, dz};
    float rt, u[3], dr, du[3], dvec[3];
    d3_pair_dvec(vi, H.v + 3 * j, eps, vec, dvec);
    d3_pair_tangent(vec, dvec, rt, u, dr, du);
    // F_i = -b u with b = C6 g'; -dF_i = a u + b du, a = dC6 g' + C6 g'' dr
    const float a = fmaf(c6 * g2d, dr, dC6 * g1d), b = c6 * g1d;
    const float hf[3] = {fmaf(a, u[0], b * du[0]), fmaf(a, u[1], b * du[1]), fmaf(a, u[2], b * du[2])};
    if (!self) { hx += (double)hf[0]; hy += (double)hf[1]; hz += (double)hf[2]; }
    ddc += (double)fmaf(g1d * dr, dc6, g * ddc6);
    // the forward's sigma -= 1/2 f (x) vec with f = -b u: its tangent with df = -hf
    const float f[3] = {-b * u[0], -b * u[1], -b * u[2]};
    sg[0] += 0.5 * (double)(hf[0] * vec[0] - f[0] * dvec[0]);
    sg[1] += 0.5 * (double)(hf[1] * vec[1] - f[1] * dvec[1]);
    sg[2] += 0.5 * (double)(hf[2] * vec[2] - f[2] * dvec[2]);
    sg[3] += 0.5 * (double)(hf[0] * vec[1] - f[0] * dvec[1]);
    sg[4] += 0.5 * (double)(hf[0] * vec[2] - f[0] * dvec[2]);
    sg[5] += 0.5 * (double)(hf[1] * vec[2] - f[1] * dvec[2]);
  });
  hx = warp_sum(hx); hy = warp_sum(hy); hz = warp_sum(hz); ddc = warp_sum(ddc);
#pragma unroll
  for (int q = 0; q < 6; ++q) sg[q] = warp_sum(sg[q]);
  if (lane == 0) {
    H.hforce[3 * i] = hx; H.hforce[3 * i + 1] = hy; H.hforce[3 * i + 2] = hz;
    H.ddc[i] = ddc;
#pragma unroll
    for (int q = 0; q < 6; ++q) H.spair[6 * (size_t)i + q] = sg[q];
  }
}

// ---- pass 3: tangent of the chain-rule force and virial -----------------------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3HvpChainBlocks)
d3_hvp_chain_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, int3 R1, int n, D3Hvp H) {
  const int lane = threadIdx.x & 31;
  const int i = blockIdx.x * kD3WarpsPerBlock + (threadIdx.x >> 5);
  if (i >= n) return;
  const float rci = P.rcov[d3_row<kBatch>(A.type[i])];
  const double di = A.dc6i[i], ddi = H.ddc[i];
  const float cn2 = (float)P.cnthr;
  const double* eps = d3_hvp_eps<kBatch>(A, H, i);
  const double* vi = H.v + 3 * i;
  double hx = 0.0, hy = 0.0, hz = 0.0;
  double sg[6] = {0, 0, 0, 0, 0, 0};
  d3_sweep_atom<kBatch>(g1, R1, A, i, 3, P.cnthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool self) {
    if (r2 >= cn2) return;                                      // the forward's strict bound
    const float rc = rci + P.rcov[d3_row<kBatch>(A.type[j])];
    float f, f1, f2;
    d3_count_jet(r2, rc, kD3K1, f, f1, f2);
    const float S = (float)(di + A.dc6i[j]), dS = (float)(ddi + H.ddc[j]);
    const float vec[3] = {dx, dy, dz};
    float r, u[3], dr, du[3], dvec[3];
    d3_pair_dvec(vi, H.v + 3 * j, eps, vec, dvec);
    d3_pair_tangent(vec, dvec, r, u, dr, du);
    // F_i = -x u with x = S f'; -dF_i = dx u + x du, dx = dS f' + S f'' dr
    const float x = S * f1, dxs = fmaf(dS, f1, S * f2 * dr);
    const float hf[3] = {fmaf(dxs, u[0], x * du[0]), fmaf(dxs, u[1], x * du[1]), fmaf(dxs, u[2], x * du[2])};
    if (!self) { hx += (double)hf[0]; hy += (double)hf[1]; hz += (double)hf[2]; }
    // the forward's sigma += 1/2 (x u) (x) vec: its tangent
    const float w[3] = {x * u[0], x * u[1], x * u[2]};
    sg[0] += 0.5 * (double)(hf[0] * vec[0] + w[0] * dvec[0]);
    sg[1] += 0.5 * (double)(hf[1] * vec[1] + w[1] * dvec[1]);
    sg[2] += 0.5 * (double)(hf[2] * vec[2] + w[2] * dvec[2]);
    sg[3] += 0.5 * (double)(hf[0] * vec[1] + w[0] * dvec[1]);
    sg[4] += 0.5 * (double)(hf[0] * vec[2] + w[0] * dvec[2]);
    sg[5] += 0.5 * (double)(hf[1] * vec[2] + w[1] * dvec[2]);
  });
  hx = warp_sum(hx); hy = warp_sum(hy); hz = warp_sum(hz);
#pragma unroll
  for (int q = 0; q < 6; ++q) sg[q] = warp_sum(sg[q]);
  if (lane == 0) {
    H.hforce[3 * i] += hx; H.hforce[3 * i + 1] += hy; H.hforce[3 * i + 2] += hz;
#pragma unroll
    for (int q = 0; q < 6; ++q) H.schain[6 * (size_t)i + q] = sg[q];
  }
}

}  // namespace s7b
