// Launch dispatch of the fused convolution.  Each kernel family (forward, backward, JVP, backward tangent, heat flux,
// centroid virial) is a launcher type that holds its operands and launches its kernel for the <Kind, MUL, NV, LPN>
// chosen below.  launch_conv_group dispatches one (lmax_filter, lmax_out) group of tensor-product kinds; each group is
// its own translation unit (conv_group_*.cu) so that the kinds compile in parallel.  launch_conv (conv_dispatch.cu)
// picks the group.
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

constexpr int kConvBlock = 32 * kConvWarpsPerBlock;

// The families.  kSpecialised: the family also has the kernels specialised for the widths kConvMul (in the groups
// with SPEC = 1, see S7B_DEFINE_CONV_GROUP); the others run the runtime-width kernels (MUL = 0) only.  kL0NV: the
// most channel pairs per lane of its l1 = 0 kernels (1 for l1 > 0).
struct ConvFwd {
  static constexpr bool kSpecialised = true;
  static constexpr int kL0NV = S7B_FWD_L0_NV;
  bool table;
  float* out;
  template <class Kind, int MUL, int NV, int LPN>
  void run(const ConvArgs& a, const ConvRole& role, cudaStream_t st) const {
    if constexpr (LPN == 16 && !S7B_FWD_ODD_PAIRS) {   // one channel per lane instead, a full warp per node
      const dim3 grid = conv_grid<MUL, 1, 32, 1>(a, role);
      if (table) conv_fwd_kernel<Kind, MUL, 1, 32, true, float><<<grid, kConvBlock, 0, st>>>(a, role, out);
      else conv_fwd_kernel<Kind, MUL, 1, 32, false, float><<<grid, kConvBlock, 0, st>>>(a, role, out);
    } else {
      const dim3 grid = conv_grid<MUL, NV, LPN>(a, role);
      if (table) conv_fwd_kernel<Kind, MUL, NV, LPN, true, V2><<<grid, kConvBlock, 0, st>>>(a, role, out);
      else conv_fwd_kernel<Kind, MUL, NV, LPN, false, V2><<<grid, kConvBlock, 0, st>>>(a, role, out);
    }
  }
};

struct ConvBwd {
  static constexpr bool kSpecialised = true;
  static constexpr int kL0NV = S7B_BWD_L0_NV;
  bool table, need_dx;
  const float* gout;
  float *dx, *dY, *dEdr, *dw;
  template <class Kind, int MUL, int NV, int LPN>
  void run(const ConvArgs& a, const ConvRole& role, cudaStream_t st) const {
    // only the l1 = 0 kinds are ever run without dx (first layer: x depends on species only)
    constexpr bool ALLOW_NODX = Kind::L1 == 0;
    const dim3 grid = conv_grid<MUL, NV, LPN>(a, role);
    if (!need_dx && ALLOW_NODX) {
      if (table) conv_bwd_kernel<Kind, MUL, NV, LPN, true, !ALLOW_NODX><<<grid, kConvBlock, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
      else conv_bwd_kernel<Kind, MUL, NV, LPN, false, !ALLOW_NODX><<<grid, kConvBlock, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
    } else {
      if (table) conv_bwd_kernel<Kind, MUL, NV, LPN, true, true><<<grid, kConvBlock, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
      else conv_bwd_kernel<Kind, MUL, NV, LPN, false, true><<<grid, kConvBlock, 0, st>>>(a, role, gout, dx, dY, dEdr, dw);
    }
  }
};

// Second order (operator boundary only): the lane mappings of the forward (JVP) and the backward (backward tangent)
struct ConvJvp {
  static constexpr bool kSpecialised = false;
  static constexpr int kL0NV = S7B_FWD_L0_NV;
  ConvTangents tan;
  float* out;
  template <class Kind, int MUL, int NV, int LPN>
  void run(const ConvArgs& a, const ConvRole& role, cudaStream_t st) const {
    conv_jvp_kernel<Kind, NV, LPN><<<conv_grid<MUL, NV, LPN>(a, role), kConvBlock, 0, st>>>(a, role, tan, out);
  }
};

struct ConvBwdTangent {
  static constexpr bool kSpecialised = false;
  static constexpr int kL0NV = S7B_BWD_L0_NV;
  ConvTangents tan;
  const float* gout;
  float *dx, *dY, *dw;
  template <class Kind, int MUL, int NV, int LPN>
  void run(const ConvArgs& a, const ConvRole& role, cudaStream_t st) const {
    conv_bwd_tangent_kernel<Kind, NV, LPN><<<conv_grid<MUL, NV, LPN>(a, role), kConvBlock, 0, st>>>(
        a, role, tan, gout, dx, dY, dw);
  }
};

// Heat flux (engine.cu s7b_engine_heat_flux): one channel pair per lane, flux_channels<Kind>() of the four tangent
// channels per walk, from channel c0.  *nch is set to that count when the walk launches; a walk that launches nothing
// leaves it as the caller started it (kFluxChannels: the whole row).
struct ConvFlux {
  static constexpr bool kSpecialised = false;
  static constexpr int kL0NV = 1;
  FluxTangents f;
  int c0;
  int* nch;
  float* out;
  template <class Kind, int MUL, int NV, int LPN>
  void run(const ConvArgs& a, const ConvRole& role, cudaStream_t st) const {
    constexpr int NCH = flux_channels<Kind>();
    *nch = NCH;
    conv_flux_jvp_kernel<Kind, NV, LPN, NCH><<<conv_grid<MUL, NV, LPN>(a, role), kConvBlock, 0, st>>>(a, role, f, c0, out);
  }
};

// Centroid virial (engine.cu s7b_engine_centroid_virial): the lane mapping of the flux, centroid_channels<Kind>() of
// the four adjoint channels per walk; *nch as for the flux
struct ConvCentroid {
  static constexpr bool kSpecialised = false;
  static constexpr int kL0NV = 1;
  CentroidAdjoints g;
  int c0;
  int* nch;
  template <class Kind, int MUL, int NV, int LPN>
  void run(const ConvArgs& a, const ConvRole& role, cudaStream_t st) const {
    constexpr int NCH = centroid_channels<Kind>();
    *nch = NCH;
    conv_centroid_bwd_kernel<Kind, LPN, NCH><<<conv_grid<MUL, NV, LPN>(a, role), kConvBlock, 0, st>>>(a, role, g, c0);
  }
};

// Lane mapping by multiplicity: 128 | mul -> a warp per node, maxnv channel pairs per lane; 64 | mul -> a warp per
// node, one pair; else half a warp per node.
struct ConvLanes { int nv, lpn; };
constexpr ConvLanes conv_lanes(int mul, int maxnv) {
  return mul % 128 == 0 ? ConvLanes{maxnv, 32} : mul % 64 == 0 ? ConvLanes{1, 32} : ConvLanes{1, 16};
}

// Launch kind Kind of family F with the lane mapping of role.mul.  MUL > 0: the kernel specialised for the width MUL
// (role.mul == MUL), chosen at compile time; MUL = 0: the runtime-width kernels, chosen at launch.  A runtime width
// that spans several CTAs (grid.y > 1, e.g. 96 or 256) makes the backward add its per-edge sums atomically.
template <class Kind, int MUL, int MAXNV, class F>
static int launch_lanes(const F& f, const ConvArgs& a, const ConvRole& role, cudaStream_t st) {
  if (role.mul <= 0 || role.mul % 32 != 0) return kConvWrongMul;
  if constexpr (MUL > 0) {
    constexpr ConvLanes m = conv_lanes(MUL, MAXNV);
    f.template run<Kind, MUL, m.nv, m.lpn>(a, role, st);
  } else {
    const ConvLanes m = conv_lanes(role.mul, MAXNV);
    if (m.lpn == 16) f.template run<Kind, 0, 1, 16>(a, role, st);
    else if (m.nv == 1) f.template run<Kind, 0, 1, 32>(a, role, st);
    else f.template run<Kind, 0, MAXNV, 32>(a, role, st);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : 1;
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
template <int L1, int LF, int LO, int MUL, class F>
static int launch_role(const F& f, const ConvArgs& a, const ConvRole& role, cudaStream_t st) {
  constexpr int MAXNV = L1 == 0 ? F::kL0NV : 1;
  if constexpr (tp_npath(L1, LF, LO) == 0) {
    return kConvNoPath;
  } else {
    if constexpr (MUL > 0)
      if (role.mul == MUL) return launch_lanes<TPKind<L1, LF, LO>, MUL, MAXNV>(f, a, role, st);
    return launch_lanes<TPKind<L1, LF, LO>, 0, MAXNV>(f, a, role, st);
  }
}

// SPEC of the group (LF, LO), set by its translation unit (S7B_DEFINE_CONV_GROUP)
template <int LF, int LO> struct ConvGroupSpec;

// l1 = 0..3 of the group (LF, LO).  SPEC = 1 for the groups of SevenNet-0 and SevenNet-l3i5, which also get the
// kernels specialised for the widths kConvMul (l1 = 3 only with LF = 3); the other groups have only the
// runtime-width kernels.
#define S7B_CONV_SPEC_MUL(SPEC, LF, L1) ((SPEC) && ((L1) < 3 || (LF) >= 3) ? s7b::kConvMul[L1] : 0)
template <int LF, int LO, class F>
int launch_conv_group(int l1, const F& f, const ConvArgs& a, const ConvRole& role, cudaStream_t st) {
  constexpr bool SPEC = F::kSpecialised && ConvGroupSpec<LF, LO>::value;
  switch (l1) {
    case 0: return launch_role<0, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 0)>(f, a, role, st);
    case 1: return launch_role<1, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 1)>(f, a, role, st);
    case 2: return launch_role<2, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 2)>(f, a, role, st);
    case 3: return launch_role<3, LF, LO, S7B_CONV_SPEC_MUL(SPEC, LF, 3)>(f, a, role, st);
  }
  return 1;
}

}  // namespace s7b

// The translation unit of the group (LF, LO): its SPEC and launch_conv_group for every family
#define S7B_CONV_INSTANTIATE_GROUP(F, LF, LO) \
  template int launch_conv_group<LF, LO, F>(int, const F&, const ConvArgs&, const ConvRole&, cudaStream_t);
#define S7B_DEFINE_CONV_GROUP(LF, LO, SPEC)                                             \
  namespace s7b {                                                                       \
  template <> struct ConvGroupSpec<LF, LO> { static constexpr bool value = SPEC; };     \
  S7B_CONV_FAMILIES(S7B_CONV_INSTANTIATE_GROUP, LF, LO)                                 \
  }
