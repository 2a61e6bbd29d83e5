// Fused neighbour-gather -> Clebsch-Gordan tensor product -> scatter-to-centre kernels.
//
// Replaces, for one interaction layer, the reference's
//   x[edge_src] gather                     sevenn/nn/convolution.py:131
//   e3nn TensorProduct ('uvu', per-edge w) sevenn/nn/convolution.py:84-100,131
//   message_gather scatter_reduce_         sevenn/nn/convolution.py:17-26,133
// and their autograd backward (sevenn/nn/force_output.py:177-182) with one forward and one
// backward kernel per l1 "kind" (see csrc/gen_kernels.py).
//
// Mapping: a group of LPN lanes (32 = a warp, or 16 = half a warp for 32-channel irreps) owns one
// destination atom n and one l1 block.  Every lane carries NV channel PAIRS (channels 2*lane,
// 2*lane+1, then +2*LPN): all per-channel arithmetic is written on channel pairs
// (csrc/vec_ops.cuh), every global access of a group is one contiguous
// 8-byte-per-lane segment of the component-major ("cm") layout, and the node accumulators of all
// paths stay in registers over the whole CSR row -- no atomics in the forward.
// The radial weights w_p,u(r) come either from tables indexed by the edge length (TABLE, L2-resident) or from a
// stored [E, W] array (!TABLE: the reference's plug-in boundary, where the radial MLP stays outside).  The forward
// only needs w: it interpolates linearly in a value table on a grid three times finer (per (knot, channel pair)
// one float2, 16 B per pair read per edge; edges shorter than kValueTableMinR are added by a second pass over the
// row from the cubic table, in the warps that have such an edge).  The
// backward needs w and dw/dr: it evaluates a cubic-Hermite table (per (knot, channel pair) {a0e,a0o,a1e,a1o} fp32 +
// {a2e,a2o,a3e,a3o} fp16 = 24 B).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "generated/tp_kinds.cuh"
#include "tp_tangent.cuh"

namespace s7b {

constexpr int kConvWarpsPerBlock = 4;
// Channels of the l1 = 0..3 blocks of x that the kernels are specialised for (those of SevenNet-0 and
// SevenNet-l3i5), in the (lmax_filter, lmax_out) groups (2, 2), (2, 0), (3, 3) and (3, 0); l1 = 3 only with
// lmax_filter = 3.  The multiplicity is then a template parameter, so that the component stride of x and the
// table offsets are immediates.  Every other width (any positive multiple of 32) and every other group runs the
// runtime-width instantiation MUL = 0, which reads the width from ConvRole::mul (conv_dispatch.cuh).
constexpr int kConvMul[kMaxL] = {128, 64, 32, 32};
// Widest l1 block of x the engine accepts: keeps the kernels' 32-bit radial-table index (knot row * paths of the
// role * channel pairs) far from overflow for any practical knot count.
constexpr int kConvMaxMul = 1024;

// Channels of a role: the compile-time width, or role.mul in the runtime-width instantiation (MUL = 0)
template <int MUL>
__device__ __forceinline__ int conv_mul(const ConvRole& role) {
  if constexpr (MUL > 0) return MUL;
  else return role.mul;
}
// Register budget, as the min-resident-CTAs argument of __launch_bounds__ (128-thread CTAs: 4 -> 128
// registers, 3 -> 168, 1 -> 255).  Chosen by A/B timing on the previous GPU generation (7net-0, 12k atoms;
// not re-tuned on H100):
//  * forward: an explicit 1 lets ptxas keep more gathers in flight for the l1 = 0 kernels (96 -> 128
//    registers, -22 % time); the l1 >= 1 kernels do not change;
//  * backward: l1 = 0 is fastest at 3 (-6 %), l1 = 1 at 4 (128 registers; 168 or 220 are 3-4 % slower),
//    l1 >= 2 at 3 (what ptxas picks by itself).  The l1 = 0 kernel without dx (first layer) at 4: it fits
//    in 122 registers without spilling; at 3 it took 138 and 0.245 instead of 0.22 ms (H100, 700 W).  The
//    lmax = 3 kinds need > 168 registers (they spill otherwise) and are left at 2.
//  * runtime-width backward (MUL = 0), from -Xptxas -v: the l1 >= 1 kernels at 2 (at 3 or 4 the lmax_filter = 2
//    kinds spill 4-156 bytes: the runtime stride and split flag cost registers, and lmax_out = 3 adds paths);
//    l1 = 0 as above, which does not spill.
#ifndef S7B_FWD_MINBLOCKS
#define S7B_FWD_MINBLOCKS 1
#endif
#define S7B_FWD_BOUNDS __launch_bounds__(32 * kConvWarpsPerBlock, S7B_FWD_MINBLOCKS)
#ifdef S7B_BWD_MINBLOCKS
#define S7B_BWD_BOUNDS __launch_bounds__(32 * kConvWarpsPerBlock, S7B_BWD_MINBLOCKS)
#else
#define S7B_BWD_BOUNDS __launch_bounds__(32 * kConvWarpsPerBlock, \
    (Kind::NY != 9 || (MUL == 0 && Kind::D1 > 1)) ? 2 : ((Kind::D1 == 3 || !NEED_DX) ? 4 : 3))
#endif
#ifndef S7B_COOP_REC
#define S7B_COOP_REC 1   // lanes of a group fetch the records of LPN consecutive edges at once (see EdgeRecs)
#endif

// The 16-byte edge record {neighbour, table interval, frac} heads the per-edge dependency chain
// (record -> gather address / table address -> loads -> math).  Loading it per edge costs one
// dependent L2 round trip per edge; instead lane i of a group loads the record of edge e0 + i of the
// row (one coalesced 16*LPN-byte request per LPN edges, i.e. about once per row) and every iteration
// takes its record by shuffle.  Prefetching record + harmonics into registers was measured slower
// (register pressure); this costs three registers.
// Below this edge length the forward evaluates the cubic table instead of the value table.  Linear interpolation
// errs by h^2 w'' / 12, and w'' grows steeply at distances no MD run reaches (0.2 A: 2.7e-4 eV on a SevenNet-0
// H-H dimer, against 2.5e-6 eV with the cubic); the shortest bond, H2, is 0.74 A.
constexpr float kValueTableMinR = 0.6f;

// How the forward reads an edge record {src, cubic interval, its fraction, r} (edge_fwd_kernel):
//  * kRecRaw: as stored (the backward, and the forward with stored weights);
//  * kRecValue: r placed on the value grid (a.ftab_knots intervals over [0, cutoff]) with the clamps the edge kernel
//    applies for the cubic table: an edge at or beyond the cutoff reads the end of the last interval, knot Kf, whose
//    value is exactly 0 (s7b_engine_set_param checks it).  The fraction is one FMA from r, so it keeps the bits of
//    the fp32 position r / h.  An edge shorter than kValueTableMinR is also sent to knot Kf, so it adds exactly 0,
//    and raises `short_seen`: the cubic pass adds it afterwards;
//  * kRecCubicShort: the cubic interval of a short edge, ~interval (< 0) for every other edge, which adds 0.
enum { kRecRaw = 0, kRecValue = 1, kRecCubicShort = 2 };
template <int MODE>
__device__ __forceinline__ int4 fwd_rec(const ConvArgs& a, int4 r, bool valid, bool& short_seen) {
  const float rr = __int_as_float(r.w);
  const bool is_short = valid && rr < kValueTableMinR;
  if (MODE == kRecValue) {
    short_seen = short_seen || is_short;
    const int k = is_short ? a.ftab_knots - 1 : min(max((int)(rr * a.ftab_inv_h), 0), a.ftab_knots - 1);
    const float t = is_short ? 1.0f : fminf(fmaxf(fmaf(rr, a.ftab_inv_h, -(float)k), 0.0f), 1.0f);
    return make_int4(r.x, k, __float_as_int(t), 0);
  }
  if (MODE == kRecCubicShort) return make_int4(r.x, is_short ? r.y : ~r.y, r.z, 0);
  return r;
}

template <int LPN>
struct EdgeRecs {
  int cx, cy, cz;
  __device__ __forceinline__ void fill(const ConvArgs& a, int e0, int len, int it, int sl) {
    const int ei = it + sl;
    int4 r = make_int4(0, 0, 0, 0);
    if (ei < len) r = __ldg(a.rec + (unsigned)(e0 + ei));
    cx = r.x; cy = r.y; cz = r.z;
  }
  template <int MODE>
  __device__ __forceinline__ void fill(const ConvArgs& a, int e0, int len, int it, int sl, bool& short_seen) {
    const int ei = it + sl;
    int4 r = make_int4(0, 0, 0, 0);
    if (ei < len) r = __ldg(a.rec + (unsigned)(e0 + ei));
    r = fwd_rec<MODE>(a, r, ei < len, short_seen);
    cx = r.x; cy = r.y; cz = r.z;
  }
  __device__ __forceinline__ int4 get(int it) const {
    const int l = it % LPN;
    return make_int4(__shfl_sync(0xffffffffu, cx, l, LPN), __shfl_sync(0xffffffffu, cy, l, LPN),
                     __shfl_sync(0xffffffffu, cz, l, LPN), 0);
  }
};

// Sum M values (M = 8 or 16) over the LPN lanes of a group with ~M-1+log2(LPN/M) shuffles instead
// of M*log2(LPN).  On return v[0] of group-lane sl holds the total of value (sl / (LPN/M)) % M.
template <int M, int LPN>
__device__ __forceinline__ void group_reduce_multi(float (&v)[M], int sl) {
  static_assert((M == 8 || M == 16) && (LPN == 16 || LPN == 32) && M <= LPN, "unsupported reduction shape");
  int off = LPN / 2;
#pragma unroll
  for (int m = M / 2; m >= 1; m >>= 1, off >>= 1) {
    const bool up = (sl & off) != 0;
#pragma unroll
    for (int j = 0; j < m; ++j) {
      const float send = up ? v[j] : v[j + m];
      const float keep = up ? v[j + m] : v[j];
      v[j] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
#pragma unroll
  for (; off >= 1; off >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
}

template <int LPN>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int off = LPN / 2; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

template <class Kind>
__device__ __forceinline__ void load_Y(const float* __restrict__ Yrow, float (&Y)[Kind::NY]) {
  Y[0] = 1.0f;
  constexpr int NQ = (Kind::NY - 1 + 3) / 4;
  const float4* p = reinterpret_cast<const float4*>(Yrow);
#pragma unroll
  for (int q = 0; q < NQ; ++q) {
    const float4 v = __ldg(p + q);
    if (4 * q + 1 < Kind::NY) Y[4 * q + 1] = v.x;
    if (4 * q + 2 < Kind::NY) Y[4 * q + 2] = v.y;
    if (4 * q + 3 < Kind::NY) Y[4 * q + 3] = v.z;
    if (4 * q + 4 < Kind::NY) Y[4 * q + 4] = v.w;
  }
}

// i * stride for a non-negative row index and stride (node, edge): one 32 x 32 -> 64-bit multiply
__device__ __forceinline__ size_t row_offset(int i, int stride) { return (size_t)(unsigned)i * (unsigned)stride; }

__device__ __forceinline__ float2 ldg2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }

// Per-lane value type: V2 = two adjacent channels (float2 math), float = one channel.
template <class V> struct VT;
template <> struct VT<V2> {
  static constexpr int CH = 2;
  static __device__ __forceinline__ V2 zero() { return splat2(0.0f); }
  static __device__ __forceinline__ V2 load(const float* p) { return ldg2(p); }
  static __device__ __forceinline__ void store(float* p, V2 v) { *reinterpret_cast<float2*>(p) = v; }
  static __device__ __forceinline__ float hsum(V2 v) { return v.x + v.y; }
  static __device__ __forceinline__ float amax(V2 v) { return fmaxf(fabsf(v.x), fabsf(v.y)); }
  // value-table entry of the channel pair at p
  static __device__ __forceinline__ V2 val(const float2* p, bool) { return __ldg(p); }
  // cubic coefficients of the channel pair at t01 / t23
  static __device__ __forceinline__ void coef(const float4* t01, const uint2* t23, bool, V2& a0, V2& a1, V2& a2, V2& a3) {
    const float4 c01 = __ldg(t01);
    const uint2 c23 = __ldg(t23);
    a0 = make_float2(c01.x, c01.y);
    a1 = make_float2(c01.z, c01.w);
    a2 = __half22float2(*reinterpret_cast<const __half2*>(&c23.x));
    a3 = __half22float2(*reinterpret_cast<const __half2*>(&c23.y));
  }
};
template <> struct VT<float> {
  static constexpr int CH = 1;
  static __device__ __forceinline__ float zero() { return 0.0f; }
  static __device__ __forceinline__ float load(const float* p) { return __ldg(p); }
  static __device__ __forceinline__ void store(float* p, float v) { *p = v; }
  static __device__ __forceinline__ float hsum(float v) { return v; }
  static __device__ __forceinline__ float amax(float v) { return fabsf(v); }
  // the odd or even channel of the value-table entry of the pair at p
  static __device__ __forceinline__ float val(const float2* p, bool odd) { return __ldg(reinterpret_cast<const float*>(p) + odd); }
  // the odd or even channel of the pair at t01 / t23
  static __device__ __forceinline__ void coef(const float4* t01, const uint2* t23, bool odd, float& a0, float& a1, float& a2, float& a3) {
    const float4 c01 = __ldg(t01);
    const uint2 c23 = __ldg(t23);
    const float2 h2 = __half22float2(*reinterpret_cast<const __half2*>(&c23.x));
    const float2 h3 = __half22float2(*reinterpret_cast<const __half2*>(&c23.y));
    a0 = odd ? c01.y : c01.x;
    a1 = odd ? c01.w : c01.z;
    a2 = odd ? h2.y : h2.x;
    a3 = odd ? h3.y : h3.x;
  }
};

// Which node / channel pair this lane works on.
template <int NV, int LPN, int CH>
struct LaneMap {
  int n, sl, uc0, e0, len, nmax;
  bool node_ok;
  __device__ __forceinline__ LaneMap(const ConvArgs& a) {
    constexpr int GPW = 32 / LPN;
    const int lane = threadIdx.x & 31;
    sl = lane % LPN;
    n = a.n_begin + (blockIdx.x * kConvWarpsPerBlock + (threadIdx.x >> 5)) * GPW + lane / LPN;
    node_ok = n < a.n_dst;
    uc0 = blockIdx.y * (CH * LPN * NV) + CH * sl;
    e0 = 0;
    len = 0;
    if (node_ok) {
      e0 = __ldg(a.rowptr + n);
      len = __ldg(a.rowptr + n + 1) - e0;
    }
    nmax = len;
    if (GPW > 1) nmax = max(len, __shfl_xor_sync(0xffffffffu, len, 16));
  }
};

// ------------------------------------------------------------------------------------------
// forward:  out[n, path block] = sum_{e in row n} w_e * CG(x[src_e], Y_e)
// grid = (ceil(n_dst / (kConvWarpsPerBlock * 32/LPN)), MUL / (CH*LPN*NV)), block = 32*kConvWarpsPerBlock
// MUL (= role.mul) is a compile-time constant: the component stride of x and the table offsets of the paths
// become immediates, and each edge costs one x address and one table address per lane.  MUL = 0 reads the
// width from role.mul (runtime-width instantiation; role.mul must be a multiple of CH*LPN*NV).
// ------------------------------------------------------------------------------------------
// The edge loop of conv_fwd_kernel over the CSR row of this lane's node: acc += w_e * CG(x[src_e], Y_e).  MODE
// (see fwd_rec) picks the radial weights: kRecRaw the stored [E, W] array, kRecValue the value table (linear),
// kRecCubicShort the cubic table for the edges shorter than kValueTableMinR (0 for the others).
template <class Kind, int MUL, int NV, int LPN, bool TABLE, class V, int MODE>
__device__ __forceinline__ void conv_fwd_edges(const ConvArgs& a, const ConvRole& role,
                                               const LaneMap<NV, LPN, VT<V>::CH>& m,
                                               V (&acc)[NV][Kind::NACC], bool& short_seen) {
  constexpr int CH = VT<V>::CH;
  const int mul = conv_mul<MUL>(role);
  const unsigned xlane = role.x_off + m.uc0;               // this lane's first element in a row of x
  // ... and its first pair in a knot row of the role's image of the value table or the cubic table
  const unsigned tlane = (MODE == kRecCubicShort ? role.tab_off : role.ftab_off) + (m.uc0 >> 1);
  const bool odd = (m.uc0 & 1) != 0;
  EdgeRecs<LPN> recs;
  for (int it = 0; it < m.nmax; ++it) {
    const bool valid = (LPN == 32) || (it < m.len);
    const int e = valid ? m.e0 + it : 0;
#if S7B_COOP_REC
    if (it % LPN == 0) recs.template fill<MODE>(a, m.e0, m.len, it, m.sl, short_seen);
    const int4 rec = recs.get(it);
#else
    const int4 rec = fwd_rec<MODE>(a, __ldg(a.rec + e), valid, short_seen);
#endif
    float Y[Kind::NY];
    load_Y<Kind>(a.Y + row_offset(e, y_stride(Kind::NY)), Y);
    const float* __restrict__ xrow = a.x + (row_offset(rec.x, a.dim_x) + xlane);
    const bool take = MODE != kRecCubicShort || rec.y >= 0;
    const int k = take ? rec.y : ~rec.y;
    const unsigned ti = tlane + k * (Kind::NPATH * mul / 2);     // knot row of the role's table image
    const float2* __restrict__ v0 = a.ftable + ti;                 // value table: knot k ...
    const float2* __restrict__ v1 = v0 + Kind::NPATH * mul / 2;    // ... and k + 1, one row further
    const float tt = __int_as_float(rec.z);
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = CH * LPN * c;                        // channel offset from m.uc0
      V x[Kind::D1], w[Kind::NPATH];
#pragma unroll
      for (int i = 0; i < Kind::D1; ++i) x[i] = VT<V>::load(xrow + i * mul + u);
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) {
        if (MODE == kRecValue) {          // (1 - t) v_k + t v_k+1 (knot values: engine.py radial_value_table)
          const V w0 = VT<V>::val(v0 + (p * (mul / 2) + u / 2), odd);
          const V w1 = VT<V>::val(v1 + (p * (mul / 2) + u / 2), odd);
          w[p] = fma_(tt, w1, fma_(-tt, w0, w0));
        } else if (MODE == kRecCubicShort) {
          V a0, a1, a2, a3;
          VT<V>::coef(a.table + ti + (p * (mul / 2) + u / 2), a.table23 + ti + (p * (mul / 2) + u / 2), odd, a0, a1, a2, a3);
          w[p] = take ? fma_(tt, fma_(tt, fma_(tt, a3, a2), a1), a0) : VT<V>::zero();
        } else {
          w[p] = VT<V>::load(a.w + (size_t)e * a.w_numel + role.w_off[p] + m.uc0 + u);
        }
        if (LPN != 32 && !valid) w[p] = VT<V>::zero();
      }
      Kind::fwd(x, Y, w, acc[c]);
    }
  }
}

template <class Kind, int MUL, int NV, int LPN, bool TABLE, class V>
__global__ void S7B_FWD_BOUNDS
conv_fwd_kernel(const ConvArgs a, const ConvRole role, float* __restrict__ out) {
  constexpr int CH = VT<V>::CH;
  static_assert(MUL % (CH * LPN * NV) == 0, "channels must fill whole lane groups");
  const LaneMap<NV, LPN, CH> m(a);
  if (m.nmax == 0 && !m.node_ok) return;      // whole warp beyond the last node (uniform)

  V acc[NV][Kind::NACC];
#pragma unroll
  for (int c = 0; c < NV; ++c)
#pragma unroll
    for (int q = 0; q < Kind::NACC; ++q) acc[c][q] = VT<V>::zero();

  // value table (or stored weights) for every edge; then, only in a warp that met an edge shorter than
  // kValueTableMinR, the cubic table for those edges (the first pass added 0 for them)
  bool short_seen = false;
  conv_fwd_edges<Kind, MUL, NV, LPN, TABLE, V, TABLE ? kRecValue : kRecRaw>(a, role, m, acc, short_seen);
  if constexpr (TABLE)
    if (__any_sync(0xffffffffu, short_seen))
      conv_fwd_edges<Kind, MUL, NV, LPN, TABLE, V, kRecCubicShort>(a, role, m, acc, short_seen);

  // row maxima of the mid features for the tensor-core self_interaction_2 (fixed-point row scaling): one
  // group reduction and one atomicMax per (l3, k) row this role contributes to -- saves a pass over the mid tensor
  if (a.row_max != nullptr) {
#pragma unroll
    for (int l3 = 0; l3 < kMaxL; ++l3) {
      bool present = false;
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) present = present || (Kind::path_l3(p) == l3);
      if (!present) continue;
#pragma unroll
      for (int k = 0; k < 2 * l3 + 1; ++k) {
        float mx = 0.0f;
#pragma unroll
        for (int c = 0; c < NV; ++c)
#pragma unroll
          for (int p = 0; p < Kind::NPATH; ++p)
            if (Kind::path_l3(p) == l3) mx = fmaxf(mx, VT<V>::amax(acc[c][Kind::acc_off(p) + k]));
#pragma unroll
        for (int off = LPN / 2; off >= 1; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        if (m.node_ok && m.sl == 0) atomicMax(a.row_max + (size_t)m.n * a.rows_per_node + l3 * l3 + k, __float_as_uint(mx));
      }
    }
  }
  if (!m.node_ok) return;
  float* __restrict__ orow = out + (size_t)m.n * a.dim_mid;
#pragma unroll
  for (int c = 0; c < NV; ++c) {
    const int u = m.uc0 + CH * LPN * c;
#pragma unroll
    for (int p = 0; p < Kind::NPATH; ++p) {
#pragma unroll
      for (int k = 0; k < 2 * Kind::path_l3(p) + 1; ++k)
        VT<V>::store(orow + role.out_off[p] + k * role.out_stride[p] + u, acc[c][Kind::acc_off(p) + k]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// backward (centre-major): given ga = dE/d out[n, :], per edge of row n
//   TABLE : dEdr_acc[e] += sum_{p,u} (dE/dw_{p,u}) * w'_{p,u}(r_e)         (radial chain rule)
//   !TABLE: dw[e, :]     = dE/dw                                          (plug-in boundary)
//   dY_acc[e, 1..]      += sum_u dE/dY                                    (group reduction)
//   dx[src_e, :]        += dE/dx                                          (RED.ADD.F32x2, NEED_DX)
// dY_acc / dEdr_acc / dw rows are owned by exactly one group of one launch: plain read-modify-write,
// unless the role's channels are spread over several CTAs (SPLIT, gridDim.y > 1): then they are added atomically.
// MUL = 0 (runtime width, role.mul): SPLIT is read from the launch geometry.
// ------------------------------------------------------------------------------------------
template <class Kind, int MUL, int NV, int LPN, bool TABLE, bool NEED_DX>
__global__ void S7B_BWD_BOUNDS
conv_bwd_kernel(const ConvArgs a, const ConvRole role, const float* __restrict__ gout,
                float* __restrict__ dx, float* __restrict__ dY_acc, float* __restrict__ dEdr_acc,
                float* __restrict__ dw) {
  static_assert(MUL % (2 * LPN * NV) == 0, "channels must fill whole lane groups");
  const int mul = conv_mul<MUL>(role);
  const bool SPLIT = (MUL > 0) ? (MUL > 2 * LPN * NV) : (gridDim.y > 1);
  const LaneMap<NV, LPN, 2> m(a);
  if (m.nmax == 0) return;                    // uniform: no edges in any row of this warp

  V2 ga[NV][Kind::NACC];
  {
    const float* __restrict__ grow = gout + (size_t)(m.node_ok ? m.n : 0) * a.dim_mid;
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = m.uc0 + 2 * LPN * c;
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p)
#pragma unroll
        for (int k = 0; k < 2 * Kind::path_l3(p) + 1; ++k)
          ga[c][Kind::acc_off(p) + k] = ldg2(grow + role.out_off[p] + k * role.out_stride[p] + u);
    }
  }

  constexpr int NR = (Kind::NY <= 9) ? 8 : 16;   // values reduced with the transposing butterfly
  constexpr bool RIDE = TABLE && (Kind::NY - 1 < NR);     // a free slot of the butterfly carries dE/dr
  constexpr int PER = LPN / NR;
  const int idx = (m.sl / PER) % NR;                      // which reduced value ends up in this lane
  const bool is_dY = idx + 1 < Kind::NY;
  const bool writer = (m.sl % PER) == 0 && (is_dY || (RIDE && idx == NR - 1));
  const unsigned xlane = role.x_off + m.uc0;               // this lane's first element in a row of x / dx
  const unsigned tlane = role.tab_off + (m.uc0 >> 1);       // ... and its first pair in a knot row of the table
  EdgeRecs<LPN> recs;
  for (int it = 0; it < m.nmax; ++it) {
    const bool valid = (LPN == 32) || (it < m.len);
    const int e = valid ? m.e0 + it : 0;
#if S7B_COOP_REC
    if (it % LPN == 0) recs.fill(a, m.e0, m.len, it, m.sl);
    const int4 rec = recs.get(it);
#else
    const int4 rec = __ldg(a.rec + e);
#endif
    float Y[Kind::NY];
    load_Y<Kind>(a.Y + row_offset(e, y_stride(Kind::NY)), Y);
    const size_t xo = row_offset(rec.x, a.dim_x) + xlane;
    const unsigned ti = tlane + rec.y * (Kind::NPATH * mul / 2);   // knot row of the role's table image
    const float4* __restrict__ k01 = a.table + ti;
    const uint2* __restrict__ k23 = a.table23 + ti;
    const float tt = __int_as_float(rec.z);
    V2 dY[Kind::NY];
#pragma unroll
    for (int j = 0; j < Kind::NY; ++j) dY[j] = splat2(0.0f);
    V2 dEdr2 = splat2(0.0f);
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = 2 * LPN * c;                         // channel offset from m.uc0
      V2 x[Kind::D1], w[Kind::NPATH], wd[Kind::NPATH], dwv[Kind::NPATH], dxv[Kind::D1];
#pragma unroll
      for (int i = 0; i < Kind::D1; ++i) x[i] = ldg2(a.x + xo + (i * mul + u));
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) {
        if (TABLE) {
          const float4 c01 = __ldg(k01 + (p * (mul / 2) + u / 2));
          const uint2 c23 = __ldg(k23 + (p * (mul / 2) + u / 2));
          const V2 a0 = make_float2(c01.x, c01.y), a1 = make_float2(c01.z, c01.w);
          const V2 a2 = __half22float2(*reinterpret_cast<const __half2*>(&c23.x));
          const V2 a3 = __half22float2(*reinterpret_cast<const __half2*>(&c23.y));
          w[p] = fma_(tt, fma_(tt, fma_(tt, a3, a2), a1), a0);
          wd[p] = mul_(fma_(tt, fma_(3.0f * tt, a3, mul_(a2, 2.0f)), a1), a.inv_h);
        } else {
          w[p] = ldg2(a.w + (size_t)e * a.w_numel + role.w_off[p] + m.uc0 + u);
        }
      }
      Kind::bwd(x, Y, w, ga[c], dwv, dxv, dY);
      if (valid) {
#pragma unroll
        for (int p = 0; p < Kind::NPATH; ++p) {
          if (TABLE) dEdr2 = fma_(dwv[p], wd[p], dEdr2);
          else *reinterpret_cast<float2*>(dw + (size_t)e * a.w_numel + role.w_off[p] + m.uc0 + u) = dwv[p];
        }
        if (NEED_DX) {
#pragma unroll
          for (int i = 0; i < Kind::D1; ++i)
            atomicAdd(reinterpret_cast<float2*>(dx + xo + (i * mul + u)), dxv[i]);
        }
      }
    }
    // cross-channel reduction of dE/dY (NY-1 values) and dE/dr (1 value) over the group
    const float dEdr = dEdr2.x + dEdr2.y;
    float red[NR];
#pragma unroll
    for (int j = 0; j < NR; ++j) red[j] = (j + 1 < Kind::NY) ? dY[j + 1].x + dY[j + 1].y : 0.0f;
    if (RIDE) red[NR - 1] = dEdr;
    group_reduce_multi<NR, LPN>(red, m.sl);
    // a (node, l1) role normally belongs to one group -> plain read-modify-write (deterministic);
    // SPLIT (the role's channels are spread over several CTAs) adds atomically
    if (valid && writer) {
      float* dst = is_dY ? dY_acc + row_offset(e, y_stride(Kind::NY)) + idx : dEdr_acc + e;
      if (SPLIT) atomicAdd(dst, red[0]);
      else *dst += red[0];      // (requesting the old value at the top of the iteration was measured 1 % slower)
    }
    if (TABLE && !RIDE) {
      const float s = group_sum<LPN>(dEdr);
      if (valid && m.sl == 0) {
        if (SPLIT) atomicAdd(dEdr_acc + e, s);
        else dEdr_acc[e] += s;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// second order (operator boundary: stored weights, runtime width only).  Given tangents t = (tx, tY, tw) of the
// backward's inputs, any of them absent (null pointer: zero, its terms skipped), and g = dE/d out:
//   jvp:         out[n]      = sum_{e in row n} TP(tx[src],Y,w) + TP(x[src],tY,w) + TP(x[src],Y,tw)
//   bwd_tangent: dx[src_e]  += (d_x TP(.,tY,w) + d_x TP(.,Y,tw))^T g[n]                (RED.ADD.F32x2, as dx)
//                dY_acc[e]  += sum_u (d_Y TP(tx,.,w) + d_Y TP(x,.,tw))^T g[n]           (as dY_acc)
//                dw[e, :]    = (d_w TP(tx,Y,.) + d_w TP(x,tY,.))^T g[n]
// The per-lane arithmetic is TPTangent (tp_tangent.cuh); lane mapping, edge walk and reductions are those of
// conv_fwd_kernel / conv_bwd_kernel, the tangents are read at the same offsets as their primals.  The backward's
// per-edge sums go atomic when the role spans several CTAs (gridDim.y > 1), as in conv_bwd_kernel.
// ------------------------------------------------------------------------------------------
template <class Kind, int NV, int LPN>
__global__ void S7B_FWD_BOUNDS
conv_jvp_kernel(const ConvArgs a, const ConvRole role, const ConvTangents tan, float* __restrict__ out) {
  const LaneMap<NV, LPN, 2> m(a);
  if (m.nmax == 0 && !m.node_ok) return;      // whole warp beyond the last node (uniform)
  const int mul = role.mul;
  const bool hx = tan.x != nullptr, hY = tan.Y != nullptr, hw = tan.w != nullptr;

  V2 acc[NV][Kind::NACC];
#pragma unroll
  for (int c = 0; c < NV; ++c)
#pragma unroll
    for (int q = 0; q < Kind::NACC; ++q) acc[c][q] = splat2(0.0f);

  const unsigned xlane = role.x_off + m.uc0;
  EdgeRecs<LPN> recs;
  for (int it = 0; it < m.nmax; ++it) {
    const bool valid = (LPN == 32) || (it < m.len);
    const int e = valid ? m.e0 + it : 0;
    if (it % LPN == 0) recs.fill(a, m.e0, m.len, it, m.sl);
    const int4 rec = recs.get(it);
    float Y[Kind::NY], tY[Kind::NY];
    load_Y<Kind>(a.Y + row_offset(e, y_stride(Kind::NY)), Y);
    if (hY) load_Y<Kind>(tan.Y + row_offset(e, y_stride(Kind::NY)), tY);
    const size_t xo = row_offset(rec.x, a.dim_x) + xlane;
    const size_t wo = (size_t)e * a.w_numel + m.uc0;
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = 2 * LPN * c;                         // channel offset from m.uc0
      V2 x[Kind::D1], tx[Kind::D1], w[Kind::NPATH], tw[Kind::NPATH];
#pragma unroll
      for (int i = 0; i < Kind::D1; ++i) {
        x[i] = ldg2(a.x + xo + (i * mul + u));
        if (hx) tx[i] = ldg2(tan.x + xo + (i * mul + u));
      }
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) {
        w[p] = ldg2(a.w + wo + (role.w_off[p] + u));
        if (hw) tw[p] = ldg2(tan.w + wo + (role.w_off[p] + u));
        if (LPN != 32 && !valid) w[p] = tw[p] = splat2(0.0f);   // every term has w or tw as a factor
      }
      TPTangent<Kind>::jvp(x, Y, w, tx, tY, tw, hx, hY, hw, acc[c]);
    }
  }
  if (!m.node_ok) return;
  float* __restrict__ orow = out + (size_t)m.n * a.dim_mid;
#pragma unroll
  for (int c = 0; c < NV; ++c) {
    const int u = m.uc0 + 2 * LPN * c;
#pragma unroll
    for (int p = 0; p < Kind::NPATH; ++p) {
#pragma unroll
      for (int k = 0; k < 2 * Kind::path_l3(p) + 1; ++k)
        VT<V2>::store(orow + role.out_off[p] + k * role.out_stride[p] + u, acc[c][Kind::acc_off(p) + k]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// heat flux (engine.cu s7b_engine_heat_flux, DESIGN.md §8.3): the JVP of conv_jvp_kernel for the channels
// c = c0 .. c0 + NCH - 1 of the four (T, R_x, R_y, R_z), in one walk of the row.  x, Y, w and w' are read once per
// edge and shared by the channels; per channel the operand tangents are formed in registers:
//   dx_c = T[src]                                   (c = 0)
//          R_a[src] - vec_a T[src]                  (c = 1 + a; f.T null: dx = 0 for every channel)
//   dY_c = f.dY[c],  dw_c = w' f.dr[c][e]
// out + c * f.out_stride: the channel's mid rows.  NCH is the largest of 4, 2, 1 whose accumulators fit the
// register budget (flux_channels); the host walks each row 4 / NCH times.
// ------------------------------------------------------------------------------------------
template <class Kind>
constexpr int flux_channels() {
  return Kind::NACC * 4 <= 40 ? 4 : (Kind::NACC * 2 <= 50 ? 2 : 1);
}

template <class Kind, int NV, int LPN, int NCH>
__global__ void S7B_FWD_BOUNDS
conv_flux_jvp_kernel(const ConvArgs a, const ConvRole role, const FluxTangents f, int c0, float* __restrict__ out) {
  const LaneMap<NV, LPN, 2> m(a);
  if (m.nmax == 0 && !m.node_ok) return;      // whole warp beyond the last node (uniform)
  const int mul = role.mul;
  const bool hx = f.T != nullptr;

  V2 acc[NCH][NV][Kind::NACC];
#pragma unroll
  for (int k = 0; k < NCH; ++k)
#pragma unroll
    for (int c = 0; c < NV; ++c)
#pragma unroll
      for (int q = 0; q < Kind::NACC; ++q) acc[k][c][q] = splat2(0.0f);

  const unsigned xlane = role.x_off + m.uc0;
  EdgeRecs<LPN> recs;
  for (int it = 0; it < m.nmax; ++it) {
    const bool valid = (LPN == 32) || (it < m.len);
    const int e = valid ? m.e0 + it : 0;
    if (it % LPN == 0) recs.fill(a, m.e0, m.len, it, m.sl);
    const int4 rec = recs.get(it);
    float Y[Kind::NY];
    load_Y<Kind>(a.Y + row_offset(e, y_stride(Kind::NY)), Y);
    float ev[3], dr[NCH];
#pragma unroll
    for (int q = 0; q < 3; ++q) ev[q] = __ldg(f.vec + 3 * (size_t)e + q);
#pragma unroll
    for (int k = 0; k < NCH; ++k) dr[k] = __ldg(f.dr + (size_t)(c0 + k) * f.dr_stride + e);
    const size_t xo = row_offset(rec.x, a.dim_x) + xlane;
    const size_t wo = (size_t)e * a.w_numel + m.uc0;
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = 2 * LPN * c;                         // channel offset from m.uc0
      V2 x[Kind::D1], T[Kind::D1], w[Kind::NPATH], w1[Kind::NPATH];
#pragma unroll
      for (int i = 0; i < Kind::D1; ++i) {
        x[i] = ldg2(a.x + xo + (i * mul + u));
        if (hx) T[i] = ldg2(f.T + xo + (i * mul + u));
      }
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) {
        w[p] = ldg2(a.w + wo + (role.w_off[p] + u));
        w1[p] = ldg2(f.w1 + wo + (role.w_off[p] + u));
        if (LPN != 32 && !valid) w[p] = w1[p] = splat2(0.0f);   // every term has w or w' as a factor
      }
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const int ch = c0 + k;
        float tY[Kind::NY];
        load_Y<Kind>(f.dY + (size_t)ch * f.dY_stride + row_offset(e, y_stride(Kind::NY)), tY);
        if constexpr (NCH == 1) {      // the widest kinds: the tangents replace T and w' in their registers
          if (hx && ch > 0) {
#pragma unroll
            for (int i = 0; i < Kind::D1; ++i)
              T[i] = fma_(-ev[ch - 1], T[i], ldg2(f.R + (size_t)(ch - 1) * f.x_stride + xo + (i * mul + u)));
          }
#pragma unroll
          for (int p = 0; p < Kind::NPATH; ++p) w1[p] = mul_(w1[p], dr[k]);
          TPTangent<Kind>::jvp(x, Y, w, T, tY, w1, hx, true, true, acc[k][c]);
        } else {
          V2 tx[Kind::D1], tw[Kind::NPATH];
          if (hx) {
#pragma unroll
            for (int i = 0; i < Kind::D1; ++i) {
              if (ch == 0) tx[i] = T[i];
              else tx[i] = fma_(-ev[ch - 1], T[i], ldg2(f.R + (size_t)(ch - 1) * f.x_stride + xo + (i * mul + u)));
            }
          }
#pragma unroll
          for (int p = 0; p < Kind::NPATH; ++p) tw[p] = mul_(w1[p], dr[k]);
          TPTangent<Kind>::jvp(x, Y, w, tx, tY, tw, hx, true, true, acc[k][c]);
        }
      }
    }
  }
  if (!m.node_ok) return;
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    float* __restrict__ orow = out + (size_t)(c0 + k) * f.out_stride + (size_t)m.n * a.dim_mid;
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = m.uc0 + 2 * LPN * c;
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) {
#pragma unroll
        for (int q = 0; q < 2 * Kind::path_l3(p) + 1; ++q)
          VT<V2>::store(orow + role.out_off[p] + q * role.out_stride[p] + u, acc[k][c][Kind::acc_off(p) + q]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// centroid virial (engine.cu s7b_engine_centroid_virial, DESIGN.md §8.5): the backward of conv_bwd_kernel (stored
// weights) for the channels c = c0 .. c0 + NCH - 1 of the four adjoints (A, B_x, B_y, B_z) of mid, in one walk of
// the row.  The centre's A and B are held in registers; x, Y, w and w' are read once per edge and shared by the
// channels.  Edge e (centre n, neighbour k, vector vec) gives channel c the adjoint
//   g_c = A[n]                      (c = 0)
//         B_a[n] - vec_a A[n]       (c = 1 + a, formed in registers)
// and, with TP the edge's tensor product,
//   dx[c][k]  += TP_x^T(g_c)                                 (RED.ADD.F32x2, c.dx not null)
//   dY[c][e]  += sum_u dE/dY                                  (group reduction)
//   dr[c][e]  += sum_{p,u} (dE/dw_{p,u}) w'_{p,u}            (dE/dr through w, folded in registers)
// The per-edge sums go atomic when the role spans several CTAs (gridDim.y > 1), as in conv_bwd_kernel.  NCH is the
// largest of 4, 2, 1 whose adjoints fit the register budget (centroid_channels); the host walks each row 4 / NCH
// times.
// ------------------------------------------------------------------------------------------
template <class Kind>
constexpr int centroid_channels() {
  return Kind::NACC * 5 <= 50 ? 4 : (Kind::NACC * 3 <= 50 ? 2 : 1);
}

template <class Kind, int LPN, int NCH>
__global__ void S7B_FWD_BOUNDS
conv_centroid_bwd_kernel(const ConvArgs a, const ConvRole role, const CentroidAdjoints g, int c0) {
  const LaneMap<1, LPN, 2> m(a);
  if (m.nmax == 0) return;                    // uniform: no edges in any row of this warp
  const int mul = role.mul;
  const bool SPLIT = gridDim.y > 1;
  const bool need_dx = g.dx != nullptr;

  // A is held in registers where several channels share a walk; the widest kinds (one channel per walk) re-read it
  // per edge from L1 instead (holding it spilled 100-900 bytes for the lmax-3 kinds)
  constexpr bool A_REG = NCH > 1;
  V2 gA[A_REG ? Kind::NACC : 1], gB[NCH][Kind::NACC];
  const size_t ro = (size_t)(m.node_ok ? m.n : 0) * a.dim_mid + m.uc0;
#pragma unroll
  for (int p = 0; p < Kind::NPATH; ++p)
#pragma unroll
    for (int q = 0; q < 2 * Kind::path_l3(p) + 1; ++q) {
      const size_t o = ro + role.out_off[p] + q * role.out_stride[p];
      if constexpr (A_REG) gA[Kind::acc_off(p) + q] = ldg2(g.g + o);
#pragma unroll
      for (int k = 0; k < NCH; ++k) gB[k][Kind::acc_off(p) + q] = ldg2(g.g + (size_t)(c0 + k) * g.g_stride + o);
    }

  constexpr int NR = (Kind::NY <= 9) ? 8 : 16;   // values reduced with the transposing butterfly
  constexpr int PER = LPN / NR;
  const int idx = (m.sl / PER) % NR;                      // which reduced value ends up in this lane
  const bool writer = (m.sl % PER) == 0 && idx + 1 < Kind::NY;
  const unsigned xlane = role.x_off + m.uc0;
  EdgeRecs<LPN> recs;
  for (int it = 0; it < m.nmax; ++it) {
    const bool valid = (LPN == 32) || (it < m.len);
    const int e = valid ? m.e0 + it : 0;
    if (it % LPN == 0) recs.fill(a, m.e0, m.len, it, m.sl);
    const int4 rec = recs.get(it);
    float Y[Kind::NY];
    load_Y<Kind>(a.Y + row_offset(e, y_stride(Kind::NY)), Y);
    float ev[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) ev[q] = __ldg(g.vec + 3 * (size_t)e + q);
    const size_t xo = row_offset(rec.x, a.dim_x) + xlane;
    const size_t wo = (size_t)e * a.w_numel + m.uc0;
    V2 x[Kind::D1], w[Kind::NPATH], w1[Kind::NPATH];
#pragma unroll
    for (int i = 0; i < Kind::D1; ++i) x[i] = ldg2(a.x + xo + i * mul);
#pragma unroll
    for (int p = 0; p < Kind::NPATH; ++p) {
      w[p] = ldg2(a.w + wo + role.w_off[p]);
      w1[p] = ldg2(g.w1 + wo + role.w_off[p]);
      if (LPN != 32 && !valid) w[p] = w1[p] = splat2(0.0f);   // every output has w or w' as a factor
    }
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int ch = c0 + k;
      V2 gc[Kind::NACC], dY[Kind::NY], dwv[Kind::NPATH], dxv[Kind::D1];
      const float s = ch > 0 ? -ev[ch - 1] : 0.0f;
      if constexpr (A_REG) {
#pragma unroll
        for (int q = 0; q < Kind::NACC; ++q) gc[q] = ch > 0 ? fma_(s, gA[q], gB[k][q]) : gB[k][q];
      } else {
#pragma unroll
        for (int p = 0; p < Kind::NPATH; ++p)
#pragma unroll
          for (int q = 0; q < 2 * Kind::path_l3(p) + 1; ++q) {
            const int i = Kind::acc_off(p) + q;
            gc[i] = ch > 0 ? fma_(s, ldg2(g.g + ro + role.out_off[p] + q * role.out_stride[p]), gB[k][i]) : gB[k][i];
          }
      }
#pragma unroll
      for (int j = 0; j < Kind::NY; ++j) dY[j] = splat2(0.0f);
      Kind::bwd(x, Y, w, gc, dwv, dxv, dY);
      V2 dr2 = splat2(0.0f);
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) dr2 = fma_(dwv[p], w1[p], dr2);
      if (valid && need_dx) {
        float* dxc = g.dx + (size_t)ch * g.x_stride + xo;
#pragma unroll
        for (int i = 0; i < Kind::D1; ++i) atomicAdd(reinterpret_cast<float2*>(dxc + i * mul), dxv[i]);
      }
      float red[NR];
#pragma unroll
      for (int j = 0; j < NR; ++j) red[j] = (j + 1 < Kind::NY) ? dY[j + 1].x + dY[j + 1].y : 0.0f;
      group_reduce_multi<NR, LPN>(red, m.sl);
      const float dEdr = group_sum<LPN>(dr2.x + dr2.y);
      if (valid && writer) {
        float* dst = g.dY + (size_t)ch * g.dY_stride + row_offset(e, y_stride(Kind::NY)) + idx;
        if (SPLIT) atomicAdd(dst, red[0]);
        else *dst += red[0];
      }
      if (valid && m.sl == 0) {
        float* dst = g.dr + (size_t)ch * g.dr_stride + e;
        if (SPLIT) atomicAdd(dst, dEdr);
        else *dst += dEdr;
      }
    }
  }
}

// One walk of conv_bwd_tangent_kernel over the CSR row of this lane's node, computing the outputs in OUT
// (kTanDw | kTanDx | kTanDY)
enum { kTanDw = 1, kTanDx = 2, kTanDY = 4 };
template <class Kind, int NV, int LPN, int OUT>
__device__ __forceinline__ void conv_bwd_tangent_edges(const ConvArgs& a, const ConvRole& role, const ConvTangents& tan,
                                                       const LaneMap<NV, LPN, 2>& m, const V2 (&ga)[NV][Kind::NACC],
                                                       float* __restrict__ dx, float* __restrict__ dY_acc,
                                                       float* __restrict__ dw) {
  constexpr bool DW = (OUT & kTanDw) != 0, DX = (OUT & kTanDx) != 0, DY = (OUT & kTanDY) != 0;
  const int mul = role.mul;
  const bool SPLIT = gridDim.y > 1;
  const bool hx = tan.x != nullptr, hY = tan.Y != nullptr, hw = tan.w != nullptr;
  const bool need_dx = DX && (hY || hw);
  constexpr int NR = (Kind::NY <= 9) ? 8 : 16;   // values reduced with the transposing butterfly
  constexpr int PER = LPN / NR;
  const int idx = (m.sl / PER) % NR;                      // which reduced value ends up in this lane
  const bool writer = (m.sl % PER) == 0 && idx + 1 < Kind::NY;
  const unsigned xlane = role.x_off + m.uc0;
  EdgeRecs<LPN> recs;
  for (int it = 0; it < m.nmax; ++it) {
    const bool valid = (LPN == 32) || (it < m.len);
    const int e = valid ? m.e0 + it : 0;
    if (it % LPN == 0) recs.fill(a, m.e0, m.len, it, m.sl);
    const int4 rec = recs.get(it);
    float Y[Kind::NY], tY[Kind::NY];
    load_Y<Kind>(a.Y + row_offset(e, y_stride(Kind::NY)), Y);
    if (hY && (DW || DX)) load_Y<Kind>(tan.Y + row_offset(e, y_stride(Kind::NY)), tY);
    const size_t xo = row_offset(rec.x, a.dim_x) + xlane;
    const size_t wo = (size_t)e * a.w_numel + m.uc0;
    V2 dY[Kind::NY];
#pragma unroll
    for (int j = 0; j < Kind::NY; ++j) dY[j] = splat2(0.0f);
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = 2 * LPN * c;                         // channel offset from m.uc0
      V2 x[Kind::D1], tx[Kind::D1], w[Kind::NPATH], tw[Kind::NPATH], dwv[Kind::NPATH], dxv[Kind::D1];
#pragma unroll
      for (int i = 0; i < Kind::D1; ++i) {
        x[i] = ldg2(a.x + xo + (i * mul + u));
        if (hx && (DW || DY)) tx[i] = ldg2(tan.x + xo + (i * mul + u));
      }
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p) {
        w[p] = ldg2(a.w + wo + (role.w_off[p] + u));
        if (hw && (DX || DY)) tw[p] = ldg2(tan.w + wo + (role.w_off[p] + u));
      }
      TPTangent<Kind>::template bwd<DW, DX, DY>(x, Y, w, ga[c], tx, tY, tw, hx, hY, hw, dwv, dxv, dY);
      if (valid) {
        if (DW) {
#pragma unroll
          for (int p = 0; p < Kind::NPATH; ++p)
            *reinterpret_cast<float2*>(dw + wo + (role.w_off[p] + u)) = dwv[p];
        }
        if (need_dx) {
#pragma unroll
          for (int i = 0; i < Kind::D1; ++i)
            atomicAdd(reinterpret_cast<float2*>(dx + xo + (i * mul + u)), dxv[i]);
        }
      }
    }
    if (DY) {
      float red[NR];
#pragma unroll
      for (int j = 0; j < NR; ++j) red[j] = (j + 1 < Kind::NY) ? dY[j + 1].x + dY[j + 1].y : 0.0f;
      group_reduce_multi<NR, LPN>(red, m.sl);
      if (valid && writer) {
        float* dst = dY_acc + row_offset(e, y_stride(Kind::NY)) + idx;
        if (SPLIT) atomicAdd(dst, red[0]);
        else *dst += red[0];
      }
    }
  }
}

// Kinds whose one-walk form needs more than 255 registers (from -Xptxas -v: it spilled 70-1300 bytes for every kind
// above this bound and for none below) walk the row once per output instead: each walk runs only the terms of its
// output, at about the register need of conv_bwd_kernel, for a second read of the row's operands.
template <class Kind>
constexpr bool tangent_walk_per_output() { return Kind::NACC * (Kind::D1 + Kind::NY) > 400; }

template <class Kind, int NV, int LPN>
__global__ void S7B_FWD_BOUNDS
conv_bwd_tangent_kernel(const ConvArgs a, const ConvRole role, const ConvTangents tan, const float* __restrict__ gout,
                        float* __restrict__ dx, float* __restrict__ dY_acc, float* __restrict__ dw) {
  const LaneMap<NV, LPN, 2> m(a);
  if (m.nmax == 0) return;                    // uniform: no edges in any row of this warp

  V2 ga[NV][Kind::NACC];
  {
    const float* __restrict__ grow = gout + (size_t)(m.node_ok ? m.n : 0) * a.dim_mid;
#pragma unroll
    for (int c = 0; c < NV; ++c) {
      const int u = m.uc0 + 2 * LPN * c;
#pragma unroll
      for (int p = 0; p < Kind::NPATH; ++p)
#pragma unroll
        for (int k = 0; k < 2 * Kind::path_l3(p) + 1; ++k)
          ga[c][Kind::acc_off(p) + k] = ldg2(grow + role.out_off[p] + k * role.out_stride[p] + u);
    }
  }
  if constexpr (!tangent_walk_per_output<Kind>()) {
    conv_bwd_tangent_edges<Kind, NV, LPN, kTanDw | kTanDx | kTanDY>(a, role, tan, m, ga, dx, dY_acc, dw);
  } else {
    // dw is always written (zero without tx and tY); dx and dY_acc arrive zeroed
    conv_bwd_tangent_edges<Kind, NV, LPN, kTanDw>(a, role, tan, m, ga, dx, dY_acc, dw);
    if (tan.Y != nullptr || tan.w != nullptr) conv_bwd_tangent_edges<Kind, NV, LPN, kTanDx>(a, role, tan, m, ga, dx, dY_acc, dw);
    if (tan.x != nullptr || tan.w != nullptr) conv_bwd_tangent_edges<Kind, NV, LPN, kTanDY>(a, role, tan, m, ga, dx, dY_acc, dw);
  }
}

}  // namespace s7b
