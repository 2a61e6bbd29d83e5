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

// grid.y = role channels / channels per lane group; MUL = 0 takes the width from role.mul
template <int MUL, int NV, int LPN, int CH = 2>
static inline dim3 conv_grid(const ConvArgs& a, const ConvRole& role) {
  const int nodes_per_block = kConvWarpsPerBlock * (32 / LPN);
  const int mul = MUL > 0 ? MUL : role.mul;
  return dim3((a.n_dst - a.n_begin + nodes_per_block - 1) / nodes_per_block, mul / (CH * LPN * NV));
}

template <class Kind, int MUL, int NV, int LPN>
static int launch_fwd_one(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  const dim3 grid = conv_grid<MUL, NV, LPN>(a, role);
  if (table) conv_fwd_kernel<Kind, MUL, NV, LPN, true, V2><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  else conv_fwd_kernel<Kind, MUL, NV, LPN, false, V2><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

// one channel per lane, a full warp per node (alternative forward mapping for mul = 32, see S7B_FWD_ODD_PAIRS)
template <class Kind, int MUL>
static int launch_fwd_scalar(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  const dim3 grid = conv_grid<MUL, 1, 32, 1>(a, role);
  if (table) conv_fwd_kernel<Kind, MUL, 1, 32, true, float><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  else conv_fwd_kernel<Kind, MUL, 1, 32, false, float><<<grid, 32 * kConvWarpsPerBlock, 0, st>>>(a, role, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <class Kind, int MUL, int NV, int LPN, bool ALLOW_NODX>
static int launch_bwd_one(bool table, bool need_dx, const ConvArgs& a, const ConvRole& role,
                          const float* gout, float* dx, float* dY, float* dEdr, float* dw, cudaStream_t st) {
  const dim3 grid = conv_grid<MUL, NV, LPN>(a, role);
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

// The runtime-width kernels (MUL = 0): the same lane mapping, chosen from role.mul at launch.  A width that
// spans several CTAs (grid.y > 1, e.g. 96 or 256) makes the backward add its per-edge sums atomically.
template <class Kind, int MAXNV>
static int fwd_kind_rt(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if constexpr (MAXNV >= 2)
    if (role.mul % 128 == 0) return launch_fwd_one<Kind, 0, MAXNV, 32>(table, a, role, out, st);
  if (role.mul % 64 == 0) return launch_fwd_one<Kind, 0, 1, 32>(table, a, role, out, st);
#if S7B_FWD_ODD_PAIRS
  return launch_fwd_one<Kind, 0, 1, 16>(table, a, role, out, st);
#else
  return launch_fwd_scalar<Kind, 0>(table, a, role, out, st);
#endif
}

template <class Kind, int MAXNV, bool ALLOW_NODX>
static int bwd_kind_rt(bool table, bool need_dx, const ConvArgs& a, const ConvRole& role,
                       const float* gout, float* dx, float* dY, float* dEdr, float* dw, cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if constexpr (MAXNV >= 2)
    if (role.mul % 128 == 0)
      return launch_bwd_one<Kind, 0, MAXNV, 32, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
  if (role.mul % 64 == 0)
    return launch_bwd_one<Kind, 0, 1, 32, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
  return launch_bwd_one<Kind, 0, 1, 16, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
}

// Second order (operator boundary only): runtime-width kernels with the lane mappings of the forward (jvp) and
// the backward (bwd_tangent) above.
template <class Kind, int NV, int LPN>
static int launch_jvp_one(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan, float* out, cudaStream_t st) {
  conv_jvp_kernel<Kind, NV, LPN><<<conv_grid<0, NV, LPN>(a, role), 32 * kConvWarpsPerBlock, 0, st>>>(a, role, tan, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <class Kind, int NV, int LPN>
static int launch_bwdt_one(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan, const float* gout,
                           float* dx, float* dY, float* dw, cudaStream_t st) {
  conv_bwd_tangent_kernel<Kind, NV, LPN><<<conv_grid<0, NV, LPN>(a, role), 32 * kConvWarpsPerBlock, 0, st>>>(
      a, role, tan, gout, dx, dY, dw);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <class Kind, int MAXNV>
static int jvp_kind_rt(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan, float* out, cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if constexpr (MAXNV >= 2)
    if (role.mul % 128 == 0) return launch_jvp_one<Kind, MAXNV, 32>(a, role, tan, out, st);
  if (role.mul % 64 == 0) return launch_jvp_one<Kind, 1, 32>(a, role, tan, out, st);
  return launch_jvp_one<Kind, 1, 16>(a, role, tan, out, st);
}

template <class Kind, int MAXNV>
static int bwdt_kind_rt(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan, const float* gout,
                        float* dx, float* dY, float* dw, cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if constexpr (MAXNV >= 2)
    if (role.mul % 128 == 0) return launch_bwdt_one<Kind, MAXNV, 32>(a, role, tan, gout, dx, dY, dw, st);
  if (role.mul % 64 == 0) return launch_bwdt_one<Kind, 1, 32>(a, role, tan, gout, dx, dY, dw, st);
  return launch_bwdt_one<Kind, 1, 16>(a, role, tan, gout, dx, dY, dw, st);
}

// Heat flux (engine.cu s7b_engine_heat_flux): the runtime-width lane mapping of the JVP with one channel pair per
// lane (NV = 1), flux_channels<Kind>() of the four tangent channels per walk
template <class Kind, int LPN>
static int launch_flux_one(const ConvArgs& a, const ConvRole& role, const FluxTangents& f, int c0, int* nch,
                           float* out, cudaStream_t st) {
  constexpr int NCH = flux_channels<Kind>();
  *nch = NCH;
  conv_flux_jvp_kernel<Kind, 1, LPN, NCH><<<conv_grid<0, 1, LPN>(a, role), 32 * kConvWarpsPerBlock, 0, st>>>(
      a, role, f, c0, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <class Kind>
static int flux_kind_rt(const ConvArgs& a, const ConvRole& role, const FluxTangents& f, int c0, int* nch, float* out,
                        cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if (role.mul % 64 == 0) return launch_flux_one<Kind, 32>(a, role, f, c0, nch, out, st);
  return launch_flux_one<Kind, 16>(a, role, f, c0, nch, out, st);
}

// Centroid virial (engine.cu s7b_engine_centroid_virial): the lane mapping of the flux, centroid_channels<Kind>()
// of the four adjoint channels per walk
template <class Kind, int LPN>
static int launch_centroid_one(const ConvArgs& a, const ConvRole& role, const CentroidAdjoints& g, int c0, int* nch,
                               cudaStream_t st) {
  constexpr int NCH = centroid_channels<Kind>();
  *nch = NCH;
  conv_centroid_bwd_kernel<Kind, LPN, NCH><<<conv_grid<0, 1, LPN>(a, role), 32 * kConvWarpsPerBlock, 0, st>>>(
      a, role, g, c0);
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

template <class Kind>
static int centroid_kind_rt(const ConvArgs& a, const ConvRole& role, const CentroidAdjoints& g, int c0, int* nch,
                            cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if (role.mul % 64 == 0) return launch_centroid_one<Kind, 32>(a, role, g, c0, nch, st);
  return launch_centroid_one<Kind, 16>(a, role, g, c0, nch, st);
}

// Paths (l2, l3) of the kind (l1, lmax_filter, lmax_out): the triangle rule with l2 <= LF, l3 <= LO
constexpr int tp_npath(int l1, int lf, int lo) {
  int n = 0;
  for (int l2 = 0; l2 <= lf; ++l2)
    for (int l3 = (l1 > l2 ? l1 - l2 : l2 - l1); l3 <= l1 + l2; ++l3) n += l3 <= lo;
  return n;
}

// One l1 role of a group.  MUL: the width its kernels are specialised for (kConvMul), 0 for none.  The
// specialised kernel runs when role.mul == MUL, the runtime-width kernel otherwise; a role without paths
// launches nothing.
template <int L1, int LF, int LO, int MUL, int MAXNV>
static int fwd_role(bool table, const ConvArgs& a, const ConvRole& role, float* out, cudaStream_t st) {
  if constexpr (tp_npath(L1, LF, LO) == 0) {
    return kConvNoPath;
  } else {
    if constexpr (MUL > 0)
      if (role.mul == MUL) return fwd_kind<TPKind<L1, LF, LO>, MUL, MAXNV>(table, a, role, out, st);
    return fwd_kind_rt<TPKind<L1, LF, LO>, MAXNV>(table, a, role, out, st);
  }
}

template <int L1, int LF, int LO, int MUL, int MAXNV>
static int bwd_role(bool table, bool need_dx, const ConvArgs& a, const ConvRole& role,
                    const float* gout, float* dx, float* dY, float* dEdr, float* dw, cudaStream_t st) {
  constexpr bool ALLOW_NODX = L1 == 0;
  if constexpr (tp_npath(L1, LF, LO) == 0) {
    return kConvNoPath;
  } else {
    if constexpr (MUL > 0)
      if (role.mul == MUL)
        return bwd_kind<TPKind<L1, LF, LO>, MUL, MAXNV, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
    return bwd_kind_rt<TPKind<L1, LF, LO>, MAXNV, ALLOW_NODX>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st);
  }
}

template <int L1, int LF, int LO, int MAXNV>
static int jvp_role(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan, float* out, cudaStream_t st) {
  if constexpr (tp_npath(L1, LF, LO) == 0) return kConvNoPath;
  else return jvp_kind_rt<TPKind<L1, LF, LO>, MAXNV>(a, role, tan, out, st);
}

template <int L1, int LF, int LO, int MAXNV>
static int bwdt_role(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan, const float* gout, float* dx,
                     float* dY, float* dw, cudaStream_t st) {
  if constexpr (tp_npath(L1, LF, LO) == 0) return kConvNoPath;
  else return bwdt_kind_rt<TPKind<L1, LF, LO>, MAXNV>(a, role, tan, gout, dx, dY, dw, st);
}

template <int L1, int LF, int LO>
static int flux_role(const ConvArgs& a, const ConvRole& role, const FluxTangents& f, int c0, int* nch, float* out,
                     cudaStream_t st) {
  if constexpr (tp_npath(L1, LF, LO) == 0) return kConvNoPath;
  else return flux_kind_rt<TPKind<L1, LF, LO>>(a, role, f, c0, nch, out, st);
}

template <int L1, int LF, int LO>
static int centroid_role(const ConvArgs& a, const ConvRole& role, const CentroidAdjoints& g, int c0, int* nch,
                         cudaStream_t st) {
  if constexpr (tp_npath(L1, LF, LO) == 0) return kConvNoPath;
  else return centroid_kind_rt<TPKind<L1, LF, LO>>(a, role, g, c0, nch, st);
}

}  // namespace s7b

// Defines  launch_conv_fwd_LF_LO / launch_conv_bwd_LF_LO  for l1 = 0..3.  SPEC = 1 for the groups of SevenNet-0
// and SevenNet-l3i5, which also get the kernels specialised for the widths kConvMul (l1 = 3 only with LF = 3);
// the other groups have only the runtime-width kernels.  launch_conv_jvp_LF_LO / launch_conv_bwdt_LF_LO: the
// second-order kernels, runtime width in every group; launch_conv_flux_LF_LO / launch_conv_centroid_LF_LO: the heat
// flux's and the centroid virial's, likewise.
#define S7B_CONV_SPEC_MUL(SPEC, LF, L1) ((SPEC) && ((L1) < 3 || (LF) >= 3) ? s7b::kConvMul[L1] : 0)
#define S7B_DEFINE_CONV_GROUP(LF, LO, SPEC)                                                        \
  namespace s7b {                                                                                  \
  int launch_conv_fwd_##LF##_##LO(int l1, bool table, const ConvArgs& a, const ConvRole& role,     \
                                  float* out, cudaStream_t st) {                                   \
    switch (l1) {                                                                                  \
      case 0: return fwd_role<0, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 0), S7B_FWD_L0_NV>(table, a, role, out, st); \
      case 1: return fwd_role<1, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 1), 1>(table, a, role, out, st); \
      case 2: return fwd_role<2, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 2), 1>(table, a, role, out, st); \
      case 3: return fwd_role<3, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 3), 1>(table, a, role, out, st); \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  int launch_conv_bwd_##LF##_##LO(int l1, bool table, bool need_dx, const ConvArgs& a,             \
                                  const ConvRole& role, const float* gout, float* dx, float* dY,   \
                                  float* dEdr, float* dw, cudaStream_t st) {                       \
    switch (l1) {                                                                                  \
      case 0: return bwd_role<0, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 0), S7B_BWD_L0_NV>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
      case 1: return bwd_role<1, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 1), 1>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
      case 2: return bwd_role<2, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 2), 1>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
      case 3: return bwd_role<3, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 3), 1>(table, need_dx, a, role, gout, dx, dY, dEdr, dw, st); \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  int launch_conv_jvp_##LF##_##LO(int l1, const ConvArgs& a, const ConvRole& role,                 \
                                  const ConvTangents& tan, float* out, cudaStream_t st) {          \
    switch (l1) {                                                                                  \
      case 0: return jvp_role<0, LF, LO, S7B_FWD_L0_NV>(a, role, tan, out, st);                    \
      case 1: return jvp_role<1, LF, LO, 1>(a, role, tan, out, st);                                \
      case 2: return jvp_role<2, LF, LO, 1>(a, role, tan, out, st);                                \
      case 3: return jvp_role<3, LF, LO, 1>(a, role, tan, out, st);                                \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  int launch_conv_bwdt_##LF##_##LO(int l1, const ConvArgs& a, const ConvRole& role,                \
                                   const ConvTangents& tan, const float* gout, float* dx,          \
                                   float* dY, float* dw, cudaStream_t st) {                        \
    switch (l1) {                                                                                  \
      case 0: return bwdt_role<0, LF, LO, S7B_BWD_L0_NV>(a, role, tan, gout, dx, dY, dw, st);      \
      case 1: return bwdt_role<1, LF, LO, 1>(a, role, tan, gout, dx, dY, dw, st);                  \
      case 2: return bwdt_role<2, LF, LO, 1>(a, role, tan, gout, dx, dY, dw, st);                  \
      case 3: return bwdt_role<3, LF, LO, 1>(a, role, tan, gout, dx, dY, dw, st);                  \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  int launch_conv_flux_##LF##_##LO(int l1, const ConvArgs& a, const ConvRole& role,                \
                                   const FluxTangents& f, int c0, int* nch, float* out,            \
                                   cudaStream_t st) {                                              \
    switch (l1) {                                                                                  \
      case 0: return flux_role<0, LF, LO>(a, role, f, c0, nch, out, st);                           \
      case 1: return flux_role<1, LF, LO>(a, role, f, c0, nch, out, st);                           \
      case 2: return flux_role<2, LF, LO>(a, role, f, c0, nch, out, st);                           \
      case 3: return flux_role<3, LF, LO>(a, role, f, c0, nch, out, st);                           \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  int launch_conv_centroid_##LF##_##LO(int l1, const ConvArgs& a, const ConvRole& role,            \
                                       const CentroidAdjoints& g, int c0, int* nch, cudaStream_t st) { \
    switch (l1) {                                                                                  \
      case 0: return centroid_role<0, LF, LO>(a, role, g, c0, nch, st);                            \
      case 1: return centroid_role<1, LF, LO>(a, role, g, c0, nch, st);                            \
      case 2: return centroid_role<2, LF, LO>(a, role, g, c0, nch, st);                            \
      case 3: return centroid_role<3, LF, LO>(a, role, g, c0, nch, st);                            \
    }                                                                                              \
    return 1;                                                                                      \
  }                                                                                                \
  }
