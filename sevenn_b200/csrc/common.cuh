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
  int w_off[kMaxPaths];       // per path: first column in weight[E, W] / table row
  int out_off[kMaxPaths];     // per path: offset inside a mid row of element (k = 0, u = 0)
  int out_stride[kMaxPaths];  // per path: K_l3 (component stride in the fused mid block)
};

struct ConvArgs {
  const int* rowptr;          // [n_dst + 1] CSR over destination (centre) atoms
  const int4* rec;            // [E] {src, table interval, frac bits, 0}
  const float* Y;             // [E, ny_stride]  Y_1 .. Y_{NY-1} (Y_0 = 1 implicit), zero padded
  const float* x;             // [n_nodes, dim_x]
  const float4* table;        // [knots, W/2] {a0e,a0o,a1e,a1o}: value and slope*h of the cubic, per channel pair
  const uint2* table23;       // [knots, W/2] {half2(a2e,a2o), half2(a3e,a3o)}: the two small cubic terms in fp16
  const float* w;             // [E, W] stored weights (operator boundary / exact-MLP mode)
  int n_begin, n_dst;        // centre atoms [n_begin, n_dst) of this launch (multi-GPU: interior / boundary ranges)
  int dim_x, dim_mid, w_numel, ny_stride;
  float inv_h;                // 1 / table interval
  unsigned int* row_max;      // optional [n_dst, rows_per_node]: running max |out| bits of every (l3, k) row of the mid
  int rows_per_node;          // features (row l3^2 + k), for the tensor-core linear that consumes them (tc_gemm.cuh)
};

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
