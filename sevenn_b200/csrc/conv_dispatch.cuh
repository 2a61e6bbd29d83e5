// Launch dispatch for one (lmax_filter, lmax_out) group of tensor-product kinds.  Each group is
// its own translation unit (conv_group_*.cu) so that the kinds compile in parallel.
#pragma once
#include "conv_kernels.cuh"

#ifndef S7B_BWD_L0_NV
#define S7B_BWD_L0_NV 2   // channel pairs per lane in the l1 = 0 backward kernels (1 is 6% faster but splits a
                          // (node, l1) role over two CTAs, whose per-edge dY/dE/dr sums then need atomics)
#endif

#ifndef S7B_FWD_L0_NV
#define S7B_FWD_L0_NV 2   // channel pairs per lane in the l1 = 0 forward kernels (1 was measured 4 % slower)
#endif
#ifndef S7B_FWD_ODD_PAIRS
#define S7B_FWD_ODD_PAIRS 1   // mul = 32 forward kernels: 1 = channel pairs on half warps (two nodes per warp, float2 math),
                              // 0 = one channel per lane.  Pairs are 29 % faster since the edge records are fetched
                              // cooperatively (0.099 vs 0.139 ms, 7net-0 l1 = 2); before that the scalar form won.
#endif

namespace s7b {

template <int MUL, int NV, int LPN, int CH = 2>
static inline dim3 conv_grid(const ConvArgs& a) {
  const int nodes_per_block = kConvWarpsPerBlock * (32 / LPN);
  return dim3((a.n_dst - a.n_begin + nodes_per_block - 1) / nodes_per_block, MUL / (CH * LPN * NV));
}

template <class Kind, int MUL, int NV, int LPN>
static int launch_fwd_one(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  const dim3 grid = conv_grid<MUL, NV, LPN>(a);
  if (table) conv_fwd_kernel<Kind, MUL, NV, LPN, true, V2><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  else conv_fwd_kernel<Kind, MUL, NV, LPN, false, V2><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

// one channel per lane, a full warp per node (alternative forward mapping for mul = 32, see S7B_FWD_ODD_PAIRS)
template <class Kind, int MUL>
static int launch_fwd_scalar(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  const dim3 grid = conv_grid<MUL, 1, 32, 1>(a);
  if (table) conv_fwd_kernel<Kind, MUL, 1, 32, true, float><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  else conv_fwd_kernel<Kind, MUL, 1, 32, false, float><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <class Kind, int MUL, int NV, int LPN, bool ALLOW_NODX>
static int launch_bwd_one(bool table, bool need_dx, const ConvArgs& a, const ConvRole& role,
                          const float* gout, float* dx, float* dY, float* dEdr, float* dw, cudaStream_t st) {
  const dim3 grid = conv_grid<MUL, NV, LPN>(a);
  const int blk = 32 * kConvWarpsPerBlock;
  if (!need_dx && ALLOW_NODX) {
    if (table) conv_bwd_kernel<Kind, MUL, NV, LPN, true, !ALLOW_NODX><<<grid, blk, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
    else conv_bwd_kernel<Kind, MUL, NV, LPN, false, !ALLOW_NODX><<<grid, blk, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
  } else {
    if (table) conv_bwd_kernel<Kind, MUL, NV, LPN, true, true><<<grid, blk, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
    else conv_bwd_kernel<Kind, MUL, NV, LPN, false, true><<<grid, blk, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

// Lane mapping by multiplicity: 128 | MUL -> a warp per node, 2 channel pairs per lane (only
// where MAXNV == 2); 64 | MUL -> a warp per node, 1 pair; else half a warp per node.
template <class Kind, int MUL, int MAXNV>
static int fwd_kind(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  if (role.mul != MUL) return kConvWrongMul;
  if constexpr (MAXNV >= 2 && MUL % 128 == 0) return launch_fwd_one<Kind, MUL, MAXNV, 32>(table, a, role, out, st);
  else if constexpr (MUL % 64 == 0) return launch_fwd_one<Kind, MUL, 1, 32>(table, a, role, out, st);
#if S7B_FWD_ODD_PAIRS
  else return launch_fwd_one<Kind, MUL, 1, 16>(table, a, role, out, st);
#else
  else return launch_fwd_scalar<Kind, MUL>(table, a, role, out, st);
#endif
}

// ALLOW_NODX: only the l1 = 0 kinds are ever run without dx (first layer: x depends on species only)
template <class Kind, int MUL, int MAXNV, bool ALLOW_NODX>
static int bwd_kind(bool table, bool need_dx, const ConvArgs& a, const ConvRole& role,
                    const float* gout, float* dx, float* dY, float* dEdr, float* dw, cudaStream_t st) {
  if (role.mul != MUL) return kConvWrongMul;
  if constexpr (MAXNV >= 2 && MUL % 128 == 0)
    return launch_bwd_one<Kind, MUL, MAXNV, 32, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
  else if constexpr (MUL % 64 == 0)
    return launch_bwd_one<Kind, MUL, 1, 32, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
  else
    return launch_bwd_one<Kind, MUL, 1, 16, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
}

}  // namespace s7b

// Defines  launch_conv_fwd_LF_LO / launch_conv_bwd_LF_LO  for l1 = 0..LF.
#define S7B_DEFINE_CONV_GROUP(LF, LO)                                                              \
  namespace s7b {                                                                                  \
  int launch_conv_fwd_##LF##_##LO(int l1, bool table, const ConvArgs& a, const ConvRole& role,     \
                                  float* out, cudaStream_t st) {                                   \
    switch (l1) {                                                                                  \
      case 0: return fwd_kind<TPKind<0, LF, LO>, kConvMul[0], S7B_FWD_L0_NV>(table, a, role, out, st);  \
      case 1: return fwd_kind<TPKind<1, LF, LO>, kConvMul[1], 1>(table, a, role, out, st);              \
      case 2: return fwd_kind<TPKind<2, LF, LO>, kConvMul[2], 1>(table, a, role, out, st);              \
      case 3: return fwd_kind<TPKind<(LF >= 3 ? 3 : 2), LF, LO>, kConvMul[3], 1>(table, a, role, out, st); \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  int launch_conv_bwd_##LF##_##LO(int l1, bool table, bool need_dx, const ConvArgs& a,             \
                                  const ConvRole& role, const float* gout, float* dx, float* dY,   \
                                  float* dEdr, float* dw, cudaStream_t st) {                       \
    switch (l1) {                                                                                  \
      case 0: return bwd_kind<TPKind<0, LF, LO>, kConvMul[0], S7B_BWD_L0_NV, true>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);  \
      case 1: return bwd_kind<TPKind<1, LF, LO>, kConvMul[1], 1, false>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
      case 2: return bwd_kind<TPKind<2, LF, LO>, kConvMul[2], 1, false>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
      case 3: return bwd_kind<TPKind<(LF >= 3 ? 3 : 2), LF, LO>, kConvMul[3], 1, false>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  }
