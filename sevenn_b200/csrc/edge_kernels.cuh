// Edge-side kernels: geometry -> (radial table index, spherical harmonics, Bessel basis) and the
// end of the backward chain dE/dr, dE/dY -> dE/d(edge_vec) -> forces and virial.
//
// Reference counterparts:
//   EdgeEmbedding.forward (BesselBasis, XPLOR / polynomial cutoff, SphericalHarmonics)
//                                        sevenn/nn/edge_embedding.py:81-217
//   ForceStressOutputFromEdge.forward    sevenn/nn/force_output.py:171-230
#pragma once
#include "common.cuh"
#include "generated/sh.cuh"

namespace s7b {

struct RadialDesc {
  float cutoff;
  int cutoff_fn;       // 0: XPLOR, 1: polynomial
  float cutoff_on;     // XPLOR r_on
  int poly_p;
  int n_basis;         // <= 8
  float coeffs[8];     // trained Bessel frequencies
  float inv_h;         // table: 1 / interval
  int knots;           // table: number of intervals
};

// envelope and d(envelope)/dr
S7B_HD void envelope(const RadialDesc& d, float r, float& env, float& denv) {
  if (d.cutoff_fn == 0) {
    if (r < d.cutoff_on) { env = 1.0f; denv = 0.0f; return; }
    const float r2 = r * r, on2 = d.cutoff_on * d.cutoff_on, c2 = d.cutoff * d.cutoff;
    const float den = (c2 - on2) * (c2 - on2) * (c2 - on2);
    const float a = c2 - r2, b = c2 + 2.0f * r2 - 3.0f * on2;
    env = a * a * b / den;
    denv = (-4.0f * r * a * b + 4.0f * r * a * a) / den;
  } else {
    const float p = (float)d.poly_p;
    const float x = r / d.cutoff;
    float xp = 1.0f;
    for (int i = 0; i < d.poly_p - 1; ++i) xp *= x;       // x^(p-1)
    const float c0 = (p + 1.0f) * (p + 2.0f) * 0.5f, c1 = p * (p + 2.0f), c2 = p * (p + 1.0f) * 0.5f;
    env = 1.0f - xp * x * (c0 - c1 * x + c2 * x * x);
    denv = -xp * (c0 * p - c1 * (p + 1.0f) * x + c2 * (p + 2.0f) * x * x) / d.cutoff;
  }
}

// One thread per edge.  Writes rec = {src, interval, frac, r} (the cubic table's interval and fraction; the
// forward's value table has its own grid, which conv_fwd places r on), Y[e, 0..ny_stride) = Y_1.., r, and
// (exact-MLP mode) the radial embedding emb[e, 0..n_basis).
// The edge count is read from device memory and the grid is sized for the engine's edge capacity, so
// a captured CUDA graph of the step stays valid when the neighbour count changes between MD steps.
template <int LMAX>
__global__ void edge_fwd_kernel(const RadialDesc rd, const float* __restrict__ edge_vec,
                                const int* __restrict__ src, const int64_t* __restrict__ n_edges_p, int ny_stride,
                                int4* __restrict__ rec, float* __restrict__ Yout,
                                float* __restrict__ rlen, float* __restrict__ emb) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= *n_edges_p) return;
  const float vx = edge_vec[3 * e], vy = edge_vec[3 * e + 1], vz = edge_vec[3 * e + 2];
  const float r = sqrtf(vx * vx + vy * vy + vz * vz);
  // r == 0 (a caller's degenerate pair) has no direction: harmonics of the zero vector, no NaN downstream
  const float ir = r > 0.0f ? 1.0f / r : 0.0f;
  float Y[SH<LMAX>::NY];
  SH<LMAX>::eval(vx * ir, vy * ir, vz * ir, Y);
  float* yrow = Yout + e * ny_stride;
#pragma unroll
  for (int j = 1; j < SH<LMAX>::NY; ++j) yrow[j - 1] = Y[j];
  for (int j = SH<LMAX>::NY - 1; j < ny_stride; ++j) yrow[j] = 0.0f;
  const float s = r * rd.inv_h;
  int tk = (int)s;
  tk = tk < 0 ? 0 : (tk > rd.knots - 1 ? rd.knots - 1 : tk);
  // edges at or beyond the cutoff sit at the end of the last interval, where the envelope has taken the
  // weights (and, for XPLOR / polynomial cutoffs, their slope) to zero: no extrapolation of the last cubic
  const float tt = fminf(fmaxf(s - (float)tk, 0.0f), 1.0f);
  rec[e] = make_int4(__ldg(src + e), tk, __float_as_int(tt), __float_as_int(r));
  rlen[e] = r;
  if (emb != nullptr) {
    float env, denv;
    envelope(rd, r, env, denv);
    const float pre = 2.0f / rd.cutoff;
    for (int b = 0; b < rd.n_basis; ++b) emb[e * rd.n_basis + b] = pre * sinf(rd.coeffs[b] * r) * ir * env;
  }
}

// One thread per edge: total dE/d(edge_vec) from the accumulated per-l1 partials.
//   f = (dE/dr) r^ + (1/r) (I - r^ r^T) J_Y^T (dE/dY)
// dY_acc: [n_part, part_stride, ny_stride], dEdr_acc: [n_part, part_stride] (part_stride = edge
// capacity >= E); demb (optional, exact-MLP mode): [E, n_basis]
template <int LMAX>
__global__ void edge_bwd_kernel(const RadialDesc rd, const float* __restrict__ edge_vec,
                                const int64_t* __restrict__ n_edges_p, int64_t part_stride, int ny_stride, int n_part,
                                const float* __restrict__ dY_acc, const float* __restrict__ dEdr_acc,
                                const float* __restrict__ demb, float* __restrict__ fedge) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= *n_edges_p) return;
  const float vx = edge_vec[3 * e], vy = edge_vec[3 * e + 1], vz = edge_vec[3 * e + 2];
  const float r = sqrtf(vx * vx + vy * vy + vz * vz);
  const float ir = r > 0.0f ? 1.0f / r : 0.0f;
  const float ux = vx * ir, uy = vy * ir, uz = vz * ir;
  float gY[SH<LMAX>::NY];
  gY[0] = 0.0f;
#pragma unroll
  for (int j = 1; j < SH<LMAX>::NY; ++j) gY[j] = 0.0f;
  float gr = 0.0f;
  for (int p = 0; p < n_part; ++p) {
    const float* row = dY_acc + ((size_t)p * part_stride + e) * ny_stride;
#pragma unroll
    for (int j = 1; j < SH<LMAX>::NY; ++j) gY[j] += row[j - 1];
    if (dEdr_acc != nullptr) gr += dEdr_acc[(size_t)p * part_stride + e];
  }
  if (demb != nullptr) {
    float env, denv;
    envelope(rd, r, env, denv);
    const float pre = 2.0f / rd.cutoff;
    for (int b = 0; b < rd.n_basis; ++b) {
      const float c = rd.coeffs[b];
      const float sn = sinf(c * r), cs = cosf(c * r);
      const float bes = pre * sn * ir;
      const float dbes = pre * (c * cs * ir - sn * ir * ir);
      gr = fmaf(demb[e * rd.n_basis + b], dbes * env + bes * denv, gr);
    }
  }
  float gx, gy, gz;
  SH<LMAX>::vjp(ux, uy, uz, gY, gx, gy, gz);
  const float dot = gx * ux + gy * uy + gz * uz;
  fedge[3 * e + 0] = gr * ux + (gx - dot * ux) * ir;
  fedge[3 * e + 1] = gr * uy + (gy - dot * uy) * ir;
  fedge[3 * e + 2] = gr * uz + (gz - dot * uz) * ir;
}

// forces[i] = sum_{e: dst = i} f_e - sum_{e: src = i} f_e   (force_output.py:189-195)
// virial6   = -sum_e (r_x f_x, r_y f_y, r_z f_z, r_x f_y, r_y f_z, r_z f_x)   (:198-228, before / V)
// atomic_virial (optional, [n_nodes, 6]) = -(per-edge 6-vector scattered onto the neighbour), :198-214.
// One warp per centre atom for the CSR part; the neighbour part uses RED.ADD.
__global__ void force_scatter_kernel(const int* __restrict__ rowptr, const int* __restrict__ src,
                                     const float* __restrict__ edge_vec,
                                     const float* __restrict__ fedge, int n_dst,
                                     float* __restrict__ forces, double* __restrict__ virial,
                                     float* __restrict__ atomic_virial) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  float fx = 0.f, fy = 0.f, fz = 0.f;
  float v[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (n < n_dst) {
    const int e0 = __ldg(rowptr + n), e1 = __ldg(rowptr + n + 1);
    for (int e = e0 + lane; e < e1; e += 32) {
      const float ax = fedge[3 * (size_t)e], ay = fedge[3 * (size_t)e + 1], az = fedge[3 * (size_t)e + 2];
      const float rx = edge_vec[3 * (size_t)e], ry = edge_vec[3 * (size_t)e + 1], rz = edge_vec[3 * (size_t)e + 2];
      fx += ax; fy += ay; fz += az;
      const int s = __ldg(src + e);
      atomicAdd(forces + 3 * (size_t)s + 0, -ax);
      atomicAdd(forces + 3 * (size_t)s + 1, -ay);
      atomicAdd(forces + 3 * (size_t)s + 2, -az);
      const float w6[6] = {rx * ax, ry * ay, rz * az, rx * ay, ry * az, rz * ax};
#pragma unroll
      for (int q = 0; q < 6; ++q) v[q] += w6[q];
      if (atomic_virial != nullptr) {      // per-atom virial lives on the neighbour atom, negated
#pragma unroll
        for (int q = 0; q < 6; ++q) atomicAdd(atomic_virial + 6 * (size_t)s + q, -w6[q]);
      }
    }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    fx += __shfl_xor_sync(0xffffffffu, fx, off);
    fy += __shfl_xor_sync(0xffffffffu, fy, off);
    fz += __shfl_xor_sync(0xffffffffu, fz, off);
#pragma unroll
    for (int q = 0; q < 6; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], off);
  }
  if (n < n_dst && lane == 0) {
    atomicAdd(forces + 3 * (size_t)n + 0, fx);
    atomicAdd(forces + 3 * (size_t)n + 1, fy);
    atomicAdd(forces + 3 * (size_t)n + 2, fz);
  }
  __shared__ double sm[32][6];
  const int wib = threadIdx.x >> 5;
  if (lane == 0)
    for (int q = 0; q < 6; ++q) sm[wib][q] = (double)v[q];
  __syncthreads();
  if (threadIdx.x < 6) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sm[i][threadIdx.x];
    atomicAdd(virial + threadIdx.x, -t);
  }
}

}  // namespace s7b
