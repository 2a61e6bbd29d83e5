// Per-lane arithmetic of the convolution's second-order kernels (conv_jvp_kernel, conv_bwd_tangent_kernel): the
// generated first-order bodies TPKind::fwd / bwd (gen_kernels.py) run with substituted operands.
//
// TP(x, Y, w) is linear in each of x, Y and w.  Given tangents (tx, tY, tw) of the backward's inputs and
// ga = dE/d out of the forward:
//   jvp: acc += TP(tx, Y, w) + TP(x, tY, w) + TP(x, Y, tw)
//   bwd: dw   = d_w [TP(tx, Y, .) + TP(x, tY, .)]^T ga
//        dx   = d_x [TP(., tY, w) + TP(., Y, tw)]^T ga
//        dY  += d_Y [TP(tx, ., w) + TP(x, ., tw)]^T ga      (partial over channels, like TPKind::bwd; dY[0] untouched)
// A term whose tangent is absent (has_* false) is skipped.  Y_0 = 1 is a constant the generated code never reads
// (its l2 = 0 paths use the literal 1), so tY carries no Y_0 part: the tY terms run with the weights of the l2 = 0
// paths set to zero and drop the dw of those paths.
//
// Host-compilable (tests/cpu_harness) like the generated headers.
#pragma once
#include "generated/tp_kinds.cuh"

namespace s7b {

S7B_HD void set_zero(float& v) { v = 0.0f; }
S7B_HD void set_zero(V2& v) { v = splat2(0.0f); }

template <class Kind>
struct TPTangent {
  // w with the l2 = 0 paths zeroed: TP(x, tY, w0) is TP(x, tY, w) for a tY whose l = 0 component is 0
  template <class V>
  S7B_HD static void drop_l2_0(const V* __restrict__ w, V* __restrict__ w0) {
#pragma unroll
    for (int p = 0; p < Kind::NPATH; ++p) {
      if (Kind::path_l2(p) == 0) set_zero(w0[p]);
      else w0[p] = w[p];
    }
  }

  template <class V>
  S7B_HD static void jvp(const V* __restrict__ x, const float* __restrict__ Y, const V* __restrict__ w,
                         const V* __restrict__ tx, const float* __restrict__ tY, const V* __restrict__ tw,
                         bool has_x, bool has_Y, bool has_w, V* __restrict__ acc) {
    if (has_x) Kind::fwd(tx, Y, w, acc);
    if (has_w) Kind::fwd(x, Y, tw, acc);
    if (has_Y) {
      V w0[Kind::NPATH];
      drop_l2_0(w, w0);
      Kind::fwd(x, tY, w0, acc);
    }
  }

  // DW / DX / DY: which outputs to compute (the kernels may split them over passes to bound register use); only
  // the terms feeding those outputs run
  template <bool DW, bool DX, bool DY, class V>
  S7B_HD static void bwd(const V* __restrict__ x, const float* __restrict__ Y, const V* __restrict__ w,
                         const V* __restrict__ ga, const V* __restrict__ tx, const float* __restrict__ tY,
                         const V* __restrict__ tw, bool has_x, bool has_Y, bool has_w,
                         V* __restrict__ dw, V* __restrict__ dx, V* __restrict__ dY) {
    V sdw[Kind::NPATH], sdx[Kind::D1], sdY[Kind::NY];
#pragma unroll
    for (int p = 0; p < Kind::NPATH; ++p) set_zero(dw[p]);
#pragma unroll
    for (int i = 0; i < Kind::D1; ++i) set_zero(dx[i]);
#pragma unroll
    for (int j = 0; j < Kind::NY; ++j) set_zero(sdY[j]);
    if ((DW || DY) && has_x) {                     // tx: dw and dY (its dx is d_x of a term without x)
      Kind::bwd(tx, Y, w, ga, sdw, sdx, DY ? dY : sdY);
      if (DW) {
#pragma unroll
        for (int p = 0; p < Kind::NPATH; ++p) dw[p] = add_(dw[p], sdw[p]);
      }
    }
    if ((DW || DX) && has_Y) {                     // tY: dw (l2 > 0 paths) and dx
      V w0[Kind::NPATH];
      drop_l2_0(w, w0);
      Kind::bwd(x, tY, w0, ga, sdw, sdx, sdY);
      if (DW) {
#pragma unroll
        for (int p = 0; p < Kind::NPATH; ++p)
          if (Kind::path_l2(p) != 0) dw[p] = add_(dw[p], sdw[p]);
      }
      if (DX) {
#pragma unroll
        for (int i = 0; i < Kind::D1; ++i) dx[i] = add_(dx[i], sdx[i]);
      }
    }
    if ((DX || DY) && has_w) {                     // tw: dx and dY
      Kind::bwd(x, Y, tw, ga, sdw, sdx, DY ? dY : sdY);
      if (DX) {
#pragma unroll
        for (int i = 0; i < Kind::D1; ++i) dx[i] = add_(dx[i], sdx[i]);
      }
    }
  }
};

}  // namespace s7b
