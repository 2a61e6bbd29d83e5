// Kernels of the Hessian-vector product pass (engine.cu s7b_engine_hvp): forward-over-reverse through the edge
// geometry, the radial MLP, the gate and the edge backward.  The convolution's second order reuses the operator's
// conv_jvp_kernel / conv_bwd_tangent_kernel, the node linears and the force scatter are the step's own kernels.
#pragma once
#include "common.cuh"
#include "edge_kernels.cuh"
#include "hvp_math.cuh"
#include "node_kernels.cuh"

namespace s7b {

// One warp per centre atom, lanes over its CSR row: dvec[e] = v[src] - v[centre] + strain[b] . edge_vec[e], dr[e] =
// u . dvec and the tangent of the harmonics dY[e, 0..ny_stride) (Y_1.., the layout of the step's Y).  v null: no
// position tangent.  strain null: no strain tangent; else [n_sys][3][3] fp64, b the centre's structure in atom_ptr
// [n_sys + 1] (edges never join two structures).
template <int LMAX>
__global__ void hvp_edge_fwd_kernel(const int* __restrict__ rowptr, const int* __restrict__ src,
                                    const float* __restrict__ edge_vec, const float* __restrict__ v,
                                    const double* __restrict__ strain, const int* __restrict__ atom_ptr, int n_sys,
                                    int n_dst, int ny_stride, float* __restrict__ dvec, float* __restrict__ dr,
                                    float* __restrict__ dY) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= n_dst) return;
  const double* eps = strain ? strain + 9 * (size_t)structure_of(atom_ptr, n_sys, n) : nullptr;
  float vc[3] = {0.0f, 0.0f, 0.0f};
  if (v) for (int c = 0; c < 3; ++c) vc[c] = v[3 * (size_t)n + c];
  for (int e = rowptr[n] + lane; e < rowptr[n + 1]; e += 32) {
    const int s = src[e];
    const float ev[3] = {edge_vec[3 * (size_t)e], edge_vec[3 * (size_t)e + 1], edge_vec[3 * (size_t)e + 2]};
    float dv[3] = {0.0f, 0.0f, 0.0f};
    if (v) for (int c = 0; c < 3; ++c) dv[c] = v[3 * (size_t)s + c] - vc[c];
    if (eps) add_strain_tangent(eps, ev, dv);
    float t[SH<LMAX>::NY], d;
    edge_tangent<LMAX>(ev, dv, d, t);
    for (int c = 0; c < 3; ++c) dvec[3 * (size_t)e + c] = dv[c];
    dr[e] = d;
    float* row = dY + (size_t)e * ny_stride;
#pragma unroll
    for (int j = 1; j < SH<LMAX>::NY; ++j) row[j - 1] = t[j];
    for (int j = SH<LMAX>::NY - 1; j < ny_stride; ++j) row[j] = 0.0f;
  }
}

// The radial embedding and its first two r-derivatives, stacked [3][E][n_basis] (the rows of three GEMMs in one).
__global__ void hvp_radial_basis_kernel(const RadialDesc rd, const float* __restrict__ edge_vec, int64_t E,
                                        float* __restrict__ emb3) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float vx = edge_vec[3 * e], vy = edge_vec[3 * e + 1], vz = edge_vec[3 * e + 2];
  const float r = sqrtf(vx * vx + vy * vy + vz * vz);
  float f0, f1, f2;
  envelope_jet(rd.cutoff_fn, rd.cutoff, rd.cutoff_on, rd.poly_p, r, f0, f1, f2);
  const int nb = rd.n_basis;
  for (int b = 0; b < nb; ++b) {
    float b0, b1, b2;
    bessel_jet(rd.coeffs[b], rd.cutoff, r, b0, b1, b2);
    emb3[e * nb + b] = b0 * f0;
    emb3[(E + e) * nb + b] = b1 * f0 + b0 * f1;
    emb3[(2 * E + e) * nb + b] = b2 * f0 + 2.0f * b1 * f1 + b0 * f2;
  }
}

// In place over [3][rows]: (z, z', z'') -> (s(z), s'(z) z', s''(z) z'^2 + s'(z) z'') with s the normalised silu
__global__ void hvp_silu_jet_kernel(float* __restrict__ z3, int64_t rows) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (int64_t)gridDim.x * blockDim.x) {
    const float z = z3[i], z1 = z3[rows + i], z2 = z3[2 * rows + i];
    float s0, s1, s2;
    silu_n_jet(z, s0, s1, s2);
    z3[i] = s0;
    z3[rows + i] = s1 * z1;
    z3[2 * rows + i] = fmaf(s2 * z1, z1, s1 * z2);
  }
}

// dw[e, k] = w'[e, k] dr[e]
__global__ void hvp_scale_rows_kernel(const float* __restrict__ w1, const float* __restrict__ dr, int64_t E, int W,
                                      float* __restrict__ dw) {
  const int64_t total = E * W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    dw[i] = w1[i] * dr[i / W];
}

// One warp per edge: ar[e] += sum_k aw w',  dar[e] += sum_k (daw1 + daw2) w' + dr sum_k aw w''
__global__ void hvp_radial_reduce_kernel(const float* __restrict__ aw, const float* __restrict__ daw1,
                                         const float* __restrict__ daw2, const float* __restrict__ w1,
                                         const float* __restrict__ w2, const float* __restrict__ dr, int64_t E, int W,
                                         float* __restrict__ ar, float* __restrict__ dar) {
  const int64_t e = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (e >= E) return;
  float a = 0.0f, b = 0.0f, c = 0.0f;
  for (int k = lane; k < W; k += 32) {
    const size_t i = (size_t)e * W + k;
    a = fmaf(aw[i], w1[i], a);
    b = fmaf(daw1[i] + daw2[i], w1[i], b);
    c = fmaf(aw[i], w2[i], c);
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, off);
    b += __shfl_xor_sync(0xffffffffu, b, off);
    c += __shfl_xor_sync(0xffffffffu, c, off);
  }
  if (lane == 0) {
    ar[e] += a;
    dar[e] += fmaf(dr[e], c, b);
  }
}

// Tangent of gate_fwd_kernel: dh = gate'(g) dg                                    one thread per output element
__global__ void gate_jvp_kernel(const GateDesc d, const float* __restrict__ g, const float* __restrict__ dg,
                                float* __restrict__ dh, int n_nodes) {
  const size_t total = (size_t)n_nodes * d.dim_h;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / d.dim_h), c = (int)(idx - (size_t)n * d.dim_h);
    const float* grow = g + (size_t)n * d.dim_g;
    const float* trow = dg + (size_t)n * d.dim_g;
    float s0, s1, s2, v;
    if (c < d.n_scalars) {
      silu_n_jet(grow[c], s0, s1, s2);
      v = s1 * trow[c];
    } else {
      int l = 1;
      while (l < d.lmax && c >= d.h_off[l + 1]) ++l;
      const int rel = c - d.h_off[l];
      const int gi = d.gate_off[l] + rel % d.mul[l];
      silu_n_jet(grow[gi], s0, s1, s2);
      v = fmaf(trow[d.g_off[l] + rel], s0, grow[d.g_off[l] + rel] * s1 * trow[gi]);
    }
    dh[idx] = v;
  }
}

// Tangent of gate_bwd_kernel's dg = gate'(g)^T ah along (dg_t, dah): gate''(g)[dg_t, ah] + gate'(g)^T dah
// one thread per element of the output
__global__ void gate_bwd_tangent_kernel(const GateDesc d, const float* __restrict__ g, const float* __restrict__ tg,
                                        const float* __restrict__ ah, const float* __restrict__ dah,
                                        float* __restrict__ out, int n_nodes) {
  const size_t total = (size_t)n_nodes * d.dim_g;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / d.dim_g), c = (int)(idx - (size_t)n * d.dim_g);
    const float* grow = g + (size_t)n * d.dim_g;
    const float* trow = tg + (size_t)n * d.dim_g;
    const float* hrow = ah + (size_t)n * d.dim_h;
    const float* drow = dah + (size_t)n * d.dim_h;
    float s0, s1, s2, v;
    silu_n_jet(grow[c], s0, s1, s2);
    if (c < d.n_scalars) {
      v = fmaf(drow[c], s1, hrow[c] * s2 * trow[c]);
    } else if (c < d.g_off[1] || d.lmax == 0) {
      int l = 1;                                      // a gate scalar: find its l
      while (l < d.lmax && c >= d.gate_off[l + 1]) ++l;
      const int u = c - d.gate_off[l];
      float p = 0.0f, q = 0.0f;
      for (int i = 0; i < 2 * l + 1; ++i) {
        const int k = i * d.mul[l] + u;
        p = fmaf(hrow[d.h_off[l] + k], grow[d.g_off[l] + k], p);
        q = fmaf(drow[d.h_off[l] + k], grow[d.g_off[l] + k], q);
        q = fmaf(hrow[d.h_off[l] + k], trow[d.g_off[l] + k], q);
      }
      v = fmaf(q, s1, p * s2 * trow[c]);
    } else {
      int l = 1;
      while (l < d.lmax && c >= d.g_off[l + 1]) ++l;
      const int rel = c - d.g_off[l];
      const int gi = d.gate_off[l] + rel % d.mul[l];
      silu_n_jet(grow[gi], s0, s1, s2);
      v = fmaf(drow[d.h_off[l] + rel], s0, hrow[d.h_off[l] + rel] * s1 * trow[gi]);
    }
    out[idx] = v;
  }
}

// dE/dh of the last layer: scale[species] * wr (the seed readout_kernel leaves, without the energy sums)
__global__ void hvp_readout_seed_kernel(const float* __restrict__ wr, const float* __restrict__ scale,
                                        const int* __restrict__ species, int n_nodes, int width,
                                        float* __restrict__ dh) {
  const size_t total = (size_t)n_nodes * width;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / width), c = (int)(i - (size_t)n * width);
    dh[i] = __ldg(scale + species[n]) * __ldg(wr + c);
  }
}

// One thread per edge: -(tangent of edge_bwd_kernel's output), from the primal and tangent dE/dY rows (one part each)
// and dE/dr with its tangent.  The force scatter of it is H v.
template <int LMAX>
__global__ void hvp_edge_bwd_kernel(const float* __restrict__ edge_vec, const float* __restrict__ dvec, int64_t E,
                                    int ny_stride, const float* __restrict__ gY_acc, const float* __restrict__ dgY_acc,
                                    const float* __restrict__ ar, const float* __restrict__ dar,
                                    float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const float v[3] = {edge_vec[3 * e], edge_vec[3 * e + 1], edge_vec[3 * e + 2]};
  const float dv[3] = {dvec[3 * e], dvec[3 * e + 1], dvec[3 * e + 2]};
  float gY[SH<LMAX>::NY], dgY[SH<LMAX>::NY];
  gY[0] = dgY[0] = 0.0f;
#pragma unroll
  for (int j = 1; j < SH<LMAX>::NY; ++j) {
    gY[j] = gY_acc[e * ny_stride + j - 1];
    dgY[j] = dgY_acc[e * ny_stride + j - 1];
  }
  float df[3];
  edge_bwd_tangent<LMAX>(v, dv, gY, dgY, ar[e], dar[e], df);
  for (int c = 0; c < 3; ++c) out[3 * e + c] = -df[c];
}

// a[i] -= b[i]
__global__ void hvp_sub_kernel(double* __restrict__ a, const double* __restrict__ b, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] -= b[i];
}

}  // namespace s7b
