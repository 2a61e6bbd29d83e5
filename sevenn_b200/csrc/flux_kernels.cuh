// Kernels of the heat-flux pass (engine.cu s7b_engine_heat_flux, DESIGN.md §8.3): the edge tangents of the four
// channels, the first-order radial jet, and the readout of the tangents with the per-structure sums.  The
// convolution's four-channel JVP is conv_flux_jvp_kernel (conv_kernels.cuh); the node linears and gate_jvp_kernel
// are those of the Hessian-vector product.
//
// Channels (c = 0..3): T = sum_i dh_j/dr_i . v_i, and R_a = sum_i (r_j - r_i)_a (dh_j/dr_i . v_i) for a = x, y, z.
#pragma once
#include "common.cuh"
#include "hvp_math.cuh"
#include "neighbor.cuh"   // kSysBlock

namespace s7b {

constexpr int kFluxChannels = 4;

// One warp per centre j, lanes over its CSR row.  Edge e: centre j, neighbour k = src[e], vec = edge_vec[e] (the
// vector from j to k's image).  The channels' edge-vector tangents are
//   T:   dvec = v_k - v_j
//   R_a: dvec = -vec_a v_k         (the image of k sees j at -vec)
// and per channel c: dr[c][e] = u . dvec, dY[c][e, 0..ny_stride) the tangent of Y_1.. (the layout of the step's Y).
template <int LMAX>
__global__ void flux_edge_kernel(const int* __restrict__ rowptr, const int* __restrict__ src,
                                 const float* __restrict__ edge_vec, const float* __restrict__ v, int n_dst,
                                 int64_t E, int ny_stride, float* __restrict__ dr, float* __restrict__ dY) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= n_dst) return;
  const float vj[3] = {v[3 * (size_t)n], v[3 * (size_t)n + 1], v[3 * (size_t)n + 2]};
  for (int e = rowptr[n] + lane; e < rowptr[n + 1]; e += 32) {
    const int s = src[e];
    const float ev[3] = {edge_vec[3 * (size_t)e], edge_vec[3 * (size_t)e + 1], edge_vec[3 * (size_t)e + 2]};
    const float vk[3] = {v[3 * (size_t)s], v[3 * (size_t)s + 1], v[3 * (size_t)s + 2]};
#pragma unroll
    for (int c = 0; c < kFluxChannels; ++c) {
      float dv[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) dv[a] = c == 0 ? vk[a] - vj[a] : -ev[c - 1] * vk[a];
      float t[SH<LMAX>::NY], d;
      edge_tangent<LMAX>(ev, dv, d, t);
      dr[c * E + e] = d;
      float* row = dY + ((size_t)c * E + e) * ny_stride;
#pragma unroll
      for (int j = 1; j < SH<LMAX>::NY; ++j) row[j - 1] = t[j];
      for (int j = SH<LMAX>::NY - 1; j < ny_stride; ++j) row[j] = 0.0f;
    }
  }
}

// In place over [2][rows]: (z, z') -> (s(z), s'(z) z') with s the normalised silu (hvp_silu_jet_kernel's first two
// rows, the same arithmetic)
__global__ void flux_silu_jet_kernel(float* __restrict__ z2, int64_t rows) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += (int64_t)gridDim.x * blockDim.x) {
    const float z = z2[i], z1 = z2[rows + i];
    float s0, s1, s2;
    silu_n_jet(z, s0, s1, s2);
    z2[i] = s0;
    z2[rows + i] = s1 * z1;
  }
}

// Per structure b, one block over its atoms [atom_ptr[b], atom_ptr[b+1]) in a fixed order (deterministic, and a
// batch member's sums are the structure's alone), everything in fp64:
//   jpot[b, a] = sum_j scale[s_j] sum_c (wr + wr_lo)[c] R_a[j, c]      (the readout of the R channels' last tangent)
//   ju[b, a]   = sum_j U_j v_j,a                                          (U_j the step's atomic_energy64), if ju
// R_a = th + (1 + a) ch_stride, rows of `width` floats; th null: no J_pot (jpot is not written).
__global__ void __launch_bounds__(kSysBlock) flux_sums_kernel(
    const int* __restrict__ atom_ptr, const float* __restrict__ th, size_t ch_stride, int width,
    const float* __restrict__ wr, const float* __restrict__ wr_lo, const float* __restrict__ scale,
    const int* __restrict__ species, const double* __restrict__ atomic_energy, const float* __restrict__ v,
    double* __restrict__ jpot, double* __restrict__ ju) {
  const int b = blockIdx.x;
  const int a0 = atom_ptr[b], a1 = atom_ptr[b + 1];
  double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int j = a0 + threadIdx.x; j < a1; j += kSysBlock) {
    const double sc = scale[species[j]];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (th) {
        const float* row = th + (1 + a) * ch_stride + (size_t)j * width;
        double acc = 0.0;
        for (int c = 0; c < width; ++c)
          acc = fma((double)row[c], (double)wr[c] + (wr_lo != nullptr ? (double)wr_lo[c] : 0.0), acc);
        s[a] += sc * acc;
      }
      if (ju) s[3 + a] += atomic_energy[j] * (double)v[3 * (size_t)j + a];
    }
  }
  __shared__ double sm[6][kSysBlock];
#pragma unroll
  for (int q = 0; q < 6; ++q) sm[q][threadIdx.x] = s[q];
  __syncthreads();
  for (int k = kSysBlock >> 1; k > 0; k >>= 1) {
    if (threadIdx.x < k)
#pragma unroll
      for (int q = 0; q < 6; ++q) sm[q][threadIdx.x] += sm[q][threadIdx.x + k];
    __syncthreads();
  }
  if (th && threadIdx.x < 3) jpot[3 * (size_t)b + threadIdx.x] = sm[threadIdx.x][0];
  if (ju && threadIdx.x < 3) ju[3 * (size_t)b + threadIdx.x] = sm[3 + threadIdx.x][0];
}

}  // namespace s7b
