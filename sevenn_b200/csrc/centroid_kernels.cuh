// Edge end of the centroid-virial pass (engine.cu s7b_engine_centroid_virial, DESIGN.md §8.5).  The convolution's
// four-channel backward is conv_centroid_bwd_kernel (conv_kernels.cuh); the radial jet, the node linears and
// gate_bwd_kernel are those of the heat flux and the step.
//
// Channels (c = 0..3): A = dE/d(feature), and B_a = sum_m (r_m - r_j)_a dU_m/d(feature of j) for a = x, y, z.
#pragma once
#include "common.cuh"
#include "edge_kernels.cuh"

namespace s7b {

// d(.)/d(edge_vec) of one channel from its dE/dY_1.. row (gY[0] unused) and dE/dr: the arithmetic of edge_bwd_kernel
template <int LMAX>
__device__ __forceinline__ void centroid_edge_grad(float ux, float uy, float uz, float ir, float (&gY)[SH<LMAX>::NY],
                                                   float gr, float (&out)[3]) {
  float gx, gy, gz;
  SH<LMAX>::vjp(ux, uy, uz, gY, gx, gy, gz);
  const float dot = gx * ux + gy * uy + gz * uz;
  out[0] = gr * ux + (gx - dot * ux) * ir;
  out[1] = gr * uy + (gy - dot * uy) * ir;
  out[2] = gr * uz + (gz - dot * uz) * ir;
}

// One warp per centre j, lanes over its CSR row.  Edge e (neighbour k = src[e], vector vec) has from channel 0 the
// edge force f = dE/dvec and from channel 1 + a the row G'_a = d((B_a - vec_a A) . mid_j)/dvec = G_a - vec_a f, summed
// over the layers (dY [4][E, ny_stride], dr [4][E]).  Then
//   Wc_k[a][b] += G'_a,b                  (the neighbour end: RED.ADD.F64)
//   Wc_j[a][b] -= G'_a,b + vec_a f_b      (the centre end: a warp sum, one add per entry)
// which sum to -vec (x) f over both ends.  wc [n_nodes, 9] row-major in fp64, zeroed by the caller: G' and vec (x) f
// nearly cancel in the centre's sum.
template <int LMAX>
__global__ void centroid_scatter_kernel(const int* __restrict__ rowptr, const int* __restrict__ src,
                                        const float* __restrict__ edge_vec, const float* __restrict__ dY,
                                        const float* __restrict__ dr, int64_t E, int ny_stride, int n_dst,
                                        double* __restrict__ wc) {
  const int n = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= n_dst) return;                   // whole warps: n_dst is per warp
  double acc[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int e = __ldg(rowptr + n) + lane; e < __ldg(rowptr + n + 1); e += 32) {
    const float v[3] = {edge_vec[3 * (size_t)e], edge_vec[3 * (size_t)e + 1], edge_vec[3 * (size_t)e + 2]};
    const float r = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    const float ir = r > 0.0f ? 1.0f / r : 0.0f;
    const float ux = v[0] * ir, uy = v[1] * ir, uz = v[2] * ir;
    float G[4][3];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float gY[SH<LMAX>::NY];
      gY[0] = 0.0f;
      const float* row = dY + ((size_t)c * E + e) * ny_stride;
#pragma unroll
      for (int j = 1; j < SH<LMAX>::NY; ++j) gY[j] = row[j - 1];
      centroid_edge_grad<LMAX>(ux, uy, uz, ir, gY, dr[(size_t)c * E + e], G[c]);
    }
    const int k = __ldg(src + e);
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int b = 0; b < 3; ++b) {
        const double g = (double)G[1 + a][b];
        atomicAdd(wc + 9 * (size_t)k + 3 * a + b, g);
        acc[3 * a + b] -= g + (double)v[a] * (double)G[0][b];
      }
  }
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1)
#pragma unroll
    for (int q = 0; q < 9; ++q) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], off);
  if (lane < 9) {
    double s = acc[0];
#pragma unroll
    for (int q = 1; q < 9; ++q) if (lane == q) s = acc[q];
    atomicAdd(wc + 9 * (size_t)n + lane, s);
  }
}

}  // namespace s7b
