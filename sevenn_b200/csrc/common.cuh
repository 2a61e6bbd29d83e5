// Shared declarations for the sevenn_b200 CUDA library (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

#include "vec_ops.cuh"

namespace s7b {

constexpr float kSiluNorm = 1.6791767923989418f;   // e3nn normalize2mom(silu), see spec.py
constexpr int kMaxPaths = 12;                      // l1 = 2 with lmax 3 has 11 paths
constexpr int kMaxL = 4;                           // l = 0..3

// y = c * silu(z)
S7B_HD float silu_n(float z) {
  const float s = 1.0f / (1.0f + expf(-z));
  return kSiluNorm * z * s;
}
// d/dz [c * silu(z)]
S7B_HD float dsilu_n(float z) {
  const float s = 1.0f / (1.0f + expf(-z));
  return kSiluNorm * s * (1.0f + z * (1.0f - s));
}

// One (layer, l1) role of the fused convolution: which slice of x it reads, which weight
// columns and which mid-feature columns each of its paths owns.  Passed by value (constant bank).
struct ConvRole {
  int x_off;                  // offset of the l1 block inside a node row of x   (cm layout)
  int mul;                    // channels of l1 == component stride inside the block
  int tab_off;                // first channel pair of this role's radial table image (table mode, see ConvArgs::table)
  int w_off[kMaxPaths];       // per path: first column in weight[E, W]
  int out_off[kMaxPaths];     // per path: offset inside a mid row of element (k = 0, u = 0)
  int out_stride[kMaxPaths];  // per path: K_l3 (component stride in the fused mid block)
  int ftab_off;               // first channel pair of this role's value-table image (table mode, see ConvArgs::ftable)
};

// Floats per edge of the stored harmonics Y_1 .. Y_{NY-1} (Y_0 = 1 is implicit), padded to whole float4s.
__host__ __device__ constexpr int y_stride(int ny) { return (ny - 1 + 3) / 4 * 4; }

// Return code of the per-group convolution dispatch (conv_dispatch.cuh) for a role whose multiplicity no kernel
// runs (not a positive multiple of 32; the engine refuses such models when their layers are configured).
constexpr int kConvWrongMul = 3;
// ... and for an l1 role whose kind has no path (for example l1 > lmax_filter with lmax_out = 0): nothing launched.
constexpr int kConvNoPath = 4;

struct ConvArgs {
  const int* rowptr;          // [n_dst + 1] CSR over destination (centre) atoms
  const int4* rec;            // [E] {src, cubic-table interval, its frac bits, edge length r bits}
  const float* Y;             // [E, y_stride(NY)]  Y_1 .. Y_{NY-1} (Y_0 = 1 implicit), zero padded
  const float* x;             // [n_nodes, dim_x]
  // Radial tables: one image per l1 role at ConvRole::tab_off (cubic, backward) or ConvRole::ftab_off (values,
  // forward), laid out [knot][path of the role][channel pair] (engine.cu role_table_images), so that one edge
  // reaches all paths of its role from one address.
  const float4* table;        // {a0e,a0o,a1e,a1o}: value and slope*h of the cubic, per channel pair
  const uint2* table23;       // {half2(a2e,a2o), half2(a3e,a3o)}: the two small cubic terms in fp16
  const float* w;             // [E, W] stored weights (operator boundary / exact-MLP mode)
  int n_begin, n_dst;        // centre atoms [n_begin, n_dst) of this launch (multi-GPU: interior / boundary ranges)
  int dim_x, dim_mid, w_numel;
  float inv_h;                // 1 / table interval
  unsigned int* row_max;      // optional [n_dst, rows_per_node]: running max |out| bits of every (l3, k) row of the mid
  int rows_per_node;          // features (row l3^2 + k), for the tensor-core linear that consumes them (tc_gemm.cuh)
  const float2* ftable;       // w at knots 0..ftab_knots, per channel pair (forward: linear interpolation)
  float ftab_inv_h;           // ftab_knots / cutoff
  int ftab_knots;             // intervals of the value table over [0, cutoff]
};

// Tangents of the convolution backward's inputs x, Y and w (second order, conv_jvp_kernel / conv_bwd_tangent_kernel),
// in the layouts of ConvArgs::x, ::Y and ::w.  A null pointer is a zero tangent.
struct ConvTangents {
  const float* x;
  const float* Y;
  const float* w;
};

// Operands of the heat flux's four-channel convolution JVP (conv_flux_jvp_kernel): the channel c's array starts at
// c times its stride.  T [n_nodes, dim_x] and R [3][n_nodes, dim_x] are the tangents of x (null: zero, the first
// layer); w1 = dw/dr [E, W] (the layout of ConvArgs::w); dr [4][E]; dY [4][E, y_stride]; vec = edge_vec [E, 3].
struct FluxTangents {
  const float* T;
  const float* R;
  const float* w1;
  const float* dr;
  const float* dY;
  const float* vec;
  size_t x_stride, dr_stride, dY_stride, out_stride;
};

// Operands of the centroid virial's four-channel convolution backward (conv_centroid_bwd_kernel): the channel c's
// array starts at c times its stride.  g [4][n_nodes, dim_mid]: the adjoints (A, B_x, B_y, B_z) of mid; w1 = dw/dr
// [E, W]; vec = edge_vec [E, 3].  Accumulated: dx [4][n_nodes, dim_x] (null: not needed, the first layer),
// dY [4][E, y_stride] (dE/dY_1..), dr [4][E] (dE/dr through w).
struct CentroidAdjoints {
  const float* g;
  const float* w1;
  const float* vec;
  float* dx;
  float* dY;
  float* dr;
  size_t g_stride, x_stride, dY_stride, dr_stride;
};

// The kernel families of the fused convolution, one launcher type each (conv_dispatch.cuh): X(family, ...) for each
#define S7B_CONV_FAMILIES(X, ...) X(ConvFwd, __VA_ARGS__) X(ConvBwd, __VA_ARGS__) X(ConvJvp, __VA_ARGS__) \
  X(ConvBwdTangent, __VA_ARGS__) X(ConvFlux, __VA_ARGS__) X(ConvCentroid, __VA_ARGS__)

// Launch family F's kernel for the l1 role of the kinds (l1, lf, lo) over the centres [a.n_begin, a.n_dst)
// (conv_dispatch.cu): 0 when launched or when there is nothing to launch, 1 with the error set.
template <class F>
int launch_conv(int l1, int lf, int lo, const F& f, const ConvArgs& a, const ConvRole& role, cudaStream_t st);

}  // namespace s7b

#define S7B_CUDA_CHECK(expr)                                                            \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      s7b::set_error(__FILE__, __LINE__, cudaGetErrorString(_e));                       \
      return 1;                                                                         \
    }                                                                                   \
  } while (0)

namespace s7b {
void set_error(const char* file, int line, const char* msg);
}
