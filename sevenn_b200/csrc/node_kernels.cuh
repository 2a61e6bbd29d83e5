// Node-side (per-atom) kernels: block-diagonal irreps linears as tiled FP32 GEMMs, the gate,
// species-row gathers, readout and reductions.
//
// Reference counterparts:
//   IrrepsLinear / e3nn o3.Linear         sevenn/nn/linear.py:94-100  (SI1, SI2, self-connection)
//   EquivariantGate / e3nn nn.Gate        sevenn/nn/equivariant_gate.py:57-59
//   SelfConnectionOutro (x + sc)          sevenn/nn/self_connection.py:131-138 (beta = 1 epilogue)
//   FullyConnectedNet (radial MLP)        sevenn/nn/convolution.py:93-95,121 (exact-MLP mode)
//   reduce_* + SpeciesWiseRescale + sum   sevenn/model_build.py:102-123, sevenn/nn/scale.py:155-162
#pragma once
#include "common.cuh"

namespace s7b {

// One irrep block of a block-diagonal linear:  C[(n,i), :N] (+)= A[(n,i), :K] * W[K, N]
// with A row = A + n*lda + a_off + i*a_cs, C row = C + n*ldc + c_off + i*c_cs  (cm layout).
struct LinBlock {
  const float* W;       // [K, N] row-major, normalisation folded in
  int d;                // 2l+1 rows per node
  int K, N;
  int a_off, a_cs;
  int c_off, c_cs;
};

enum LinEpilogue { kEpiNone = 0, kEpiSiluStoreZ = 1, kEpiMulDsilu = 2 };

struct LinArgs {
  const float* A;
  float* C;
  const float* aux_in;   // kEpiMulDsilu: z with C's addressing
  float* aux_out;        // kEpiSiluStoreZ: receives z with C's addressing
  int lda, ldc;
  int n_nodes;
  int accumulate;        // 1: C += result
  int epilogue;
  int nblocks;
  LinBlock blk[kMaxL];
};

constexpr int kGemmBM = 128, kGemmBN = 64, kGemmBK = 16, kGemmThreads = 256;
constexpr int kGemmPadM = kGemmBM + 4;

// FP32 SIMT GEMM tile: 128 x 64 per CTA, 8 x 4 per thread, inner product on float2 pairs
// (scalar-broadcast A element x a pair of B columns).  grid = (ceil(max rows / BM), ceil(max N / BN), nblocks)
__global__ void __launch_bounds__(kGemmThreads, 3) blocklin_gemm_kernel(const LinArgs a) {
  const LinBlock b = a.blk[blockIdx.z];
  const int rows = a.n_nodes * b.d;
  const int row0 = blockIdx.x * kGemmBM, col0 = blockIdx.y * kGemmBN;
  if (row0 >= rows || col0 >= b.N) return;

  __shared__ __align__(16) float As[kGemmBK][kGemmPadM];
  __shared__ __align__(16) float Bs[kGemmBK][kGemmBN];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  // A loader: thread -> rows (tid/4, tid/4 + 64), k-quad tid%4
  const int a_row = tid >> 2, a_kq = tid & 3;
  const float* a_ptr[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int gr = row0 + a_row + 64 * h;
    a_ptr[h] = nullptr;
    if (gr < rows) {
      const int n = gr / b.d, i = gr - n * b.d;
      a_ptr[h] = a.A + (size_t)n * a.lda + b.a_off + i * b.a_cs;
    }
  }
  // B loader: thread -> (k, col-quad)
  const int b_k = tid >> 4, b_cq = tid & 15;
  const int gc = col0 + b_cq * 4;

  V2 acc[8][2];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i][0] = acc[i][1] = splat2(0.0f);

  float4 ra[2], rb;
  auto load_tiles = [&](int k0) {
    const int ka = k0 + a_kq * 4;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      ra[h] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (a_ptr[h] != nullptr) {
        if (ka + 3 < b.K) ra[h] = __ldg(reinterpret_cast<const float4*>(a_ptr[h] + ka));
        else {
          if (ka + 0 < b.K) ra[h].x = __ldg(a_ptr[h] + ka + 0);
          if (ka + 1 < b.K) ra[h].y = __ldg(a_ptr[h] + ka + 1);
          if (ka + 2 < b.K) ra[h].z = __ldg(a_ptr[h] + ka + 2);
        }
      }
    }
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    const int kb = k0 + b_k;
    if (kb < b.K) {
      const float* wp = b.W + (size_t)kb * b.N + gc;
      if (gc + 3 < b.N) rb = __ldg(reinterpret_cast<const float4*>(wp));
      else {
        if (gc + 0 < b.N) rb.x = __ldg(wp + 0);
        if (gc + 1 < b.N) rb.y = __ldg(wp + 1);
        if (gc + 2 < b.N) rb.z = __ldg(wp + 2);
      }
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      As[a_kq * 4 + 0][a_row + 64 * h] = ra[h].x;
      As[a_kq * 4 + 1][a_row + 64 * h] = ra[h].y;
      As[a_kq * 4 + 2][a_row + 64 * h] = ra[h].z;
      As[a_kq * 4 + 3][a_row + 64 * h] = ra[h].w;
    }
    *reinterpret_cast<float4*>(&Bs[b_k][b_cq * 4]) = rb;
  };

  load_tiles(0);
  for (int k0 = 0; k0 < b.K; k0 += kGemmBK) {
    store_tiles();
    __syncthreads();
    if (k0 + kGemmBK < b.K) load_tiles(k0 + kGemmBK);
#pragma unroll
    for (int k = 0; k < kGemmBK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float aa[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const V2 b0 = make_float2(bv.x, bv.y), b1 = make_float2(bv.z, bv.w);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i][0] = fma_(aa[i], b0, acc[i][0]);
        acc[i][1] = fma_(aa[i], b1, acc[i][1]);
      }
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = row0 + ty * 8 + i;
    if (r >= rows) continue;
    const int n = r / b.d, ii = r - n * b.d;
    const size_t coff = (size_t)n * a.ldc + b.c_off + ii * b.c_cs;
    const float vals[4] = {acc[i][0].x, acc[i][0].y, acc[i][1].x, acc[i][1].y};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = col0 + tx * 4 + j;
      if (c >= b.N) continue;
      float v = vals[j];
      if (a.accumulate) v += a.C[coff + c];
      if (a.epilogue == kEpiSiluStoreZ) {
        a.aux_out[coff + c] = v;
        v = silu_n(v);
      } else if (a.epilogue == kEpiMulDsilu) {
        v *= dsilu_n(a.aux_in[coff + c]);
      }
      a.C[coff + c] = v;
    }
  }
}

// Gate description for one layer (cm layout).
struct GateDesc {
  int n_scalars;            // scalars kept as they are (after activation)
  int lmax;                 // highest gated l (0: no gates)
  int mul[kMaxL];           // output multiplicities per l (mul[0] = n_scalars)
  int dim_g, dim_h;         // row widths of gate input and output
  int g_off[kMaxL];         // offset of block l inside a g row; block 0 holds scalars | gates
  int h_off[kMaxL];
  int gate_off[kMaxL];      // column (inside block 0 of g) of the first gate scalar of l
};

// h = [silu_n(scalars), gated_l * silu_n(gate_l) ...]           one thread per output element
__global__ void gate_fwd_kernel(const GateDesc d, const float* __restrict__ g, float* __restrict__ h,
                                int n_nodes) {
  const size_t total = (size_t)n_nodes * d.dim_h;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / d.dim_h), c = (int)(idx - (size_t)n * d.dim_h);
    const float* grow = g + (size_t)n * d.dim_g;
    float v;
    if (c < d.n_scalars) {
      v = silu_n(grow[c]);
    } else {
      int l = 1;
      while (l < d.lmax && c >= d.h_off[l + 1]) ++l;
      const int rel = c - d.h_off[l];
      const int u = rel % d.mul[l];
      v = grow[d.g_off[l] + rel] * silu_n(grow[d.gate_off[l] + u]);
    }
    h[idx] = v;
  }
}

// dg from dh (one thread per element of dg)
__global__ void gate_bwd_kernel(const GateDesc d, const float* __restrict__ g,
                                const float* __restrict__ dh, float* __restrict__ dg, int n_nodes) {
  const size_t total = (size_t)n_nodes * d.dim_g;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / d.dim_g), c = (int)(idx - (size_t)n * d.dim_g);
    const float* grow = g + (size_t)n * d.dim_g;
    const float* hrow = dh + (size_t)n * d.dim_h;
    float v;
    if (c < d.n_scalars) {
      v = hrow[c] * dsilu_n(grow[c]);
    } else if (c < d.g_off[1] || d.lmax == 0) {
      // a gate scalar: find its l
      int l = 1;
      while (l < d.lmax && c >= d.gate_off[l + 1]) ++l;
      const int u = c - d.gate_off[l];
      float s = 0.0f;
      for (int i = 0; i < 2 * l + 1; ++i)
        s = fmaf(hrow[d.h_off[l] + i * d.mul[l] + u], grow[d.g_off[l] + i * d.mul[l] + u], s);
      v = s * dsilu_n(grow[c]);
    } else {
      int l = 1;
      while (l < d.lmax && c >= d.g_off[l + 1]) ++l;
      const int rel = c - d.g_off[l];
      const int u = rel % d.mul[l];
      v = hrow[d.h_off[l] + rel] * silu_n(grow[d.gate_off[l] + u]);
    }
    dg[idx] = v;
  }
}

// Warp-per-node variants of the two gate kernels that ALSO leave the row exponents of their output for the
// tensor-core linears that consume it (tc_gemm.cuh: fixed-point row scaling needs max |a| of every (l, component)
// row): E[n, l^2 + i] = exponent with max |row| < 2^E, or zero_row for an all-zero row.  Lanes walk the node's
// elements 32 at a time (coalesced); lanes holding elements of the same row combine with match.any + redux.sync.
__device__ __forceinline__ void row_max_update(unsigned int* smax, int r, float v, int lane) {
  const unsigned int m = __float_as_uint(v) & 0x7fffffffu;
  const unsigned int peers = __match_any_sync(0xffffffffu, r);
  const unsigned int mm = __reduce_max_sync(peers, m);
  if (r >= 0 && lane == __ffs(peers) - 1) smax[r] = max(smax[r], mm);
  __syncwarp();
}
// Row exponent of the tensor-core linear from max |a| over a row: E with max |a| < 2^E.  zero_row for an all-zero
// row, a row of subnormals (flushed: the row gives exactly 0) and a row holding Inf or NaN (the transform's a * 0
// turns it into a NaN row).  E >= -104 keeps the slice scale 2^(23 - E) a normal float; a row whose maximum lies
// below 2^-104 keeps 23 - (-104 - log2 max|a|) bits.  The same rule is restated in tc_gemm.cuh (row_exponent_kernel
// and blocklin_tc_kernel's row_exp), each function self-contained (tests/test_simt_emulation.py compiles them one by one).
__device__ __forceinline__ void row_exponents_store(const unsigned int* smax, int* E, int rows, int lane, int zero_row) {
  if (lane < rows) {
    const int ex = (int)(smax[lane] >> 23);
    E[lane] = (ex == 0 || ex == 255) ? zero_row : max(ex - 126, -104);     // |a| < 2^(ex-126)
  }
}

__global__ void gate_fwd_rows_kernel(const GateDesc d, const float* __restrict__ g, float* __restrict__ h, int n_nodes,
                                     int* __restrict__ E, int rows_per_node, int zero_row) {
  __shared__ unsigned int smax[8][16];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + wib;
  if (lane < 16) smax[wib][lane] = 0u;
  __syncwarp();
  if (n >= n_nodes) return;
  const float* grow = g + (size_t)n * d.dim_g;
  float* hrow = h + (size_t)n * d.dim_h;
  for (int c0 = 0; c0 < d.dim_h; c0 += 32) {
    const int c = c0 + lane;
    float v = 0.0f;
    int r = -1;
    if (c < d.dim_h) {
      if (c < d.n_scalars) {
        v = silu_n(grow[c]);
        r = 0;
      } else {
        int l = 1;
        while (l < d.lmax && c >= d.h_off[l + 1]) ++l;
        const int rel = c - d.h_off[l];
        const int u = rel % d.mul[l];
        v = grow[d.g_off[l] + rel] * silu_n(grow[d.gate_off[l] + u]);
        r = l * l + rel / d.mul[l];
      }
      hrow[c] = v;
    }
    row_max_update(smax[wib], r, v, lane);
  }
  row_exponents_store(smax[wib], E + (size_t)n * rows_per_node, rows_per_node, lane, zero_row);
}

// dg from dh, one thread per element like gate_bwd_kernel (the gate-scalar elements chain 2l+1 dependent
// loads: a warp-per-node walk serialises them, one thread per element hides them), plus the row maxima of dg:
// the 32 elements of a warp lie in one (node, row) -- every multiplicity is a multiple of 32 -- so one warp
// reduction and one atomicMax on the bit pattern of |v| per warp.  bits [n_nodes, rows_per_node] is zeroed by the caller.
__global__ void gate_bwd_rows_kernel(const GateDesc d, const float* __restrict__ g, const float* __restrict__ dh,
                                     float* __restrict__ dg, int n_nodes, unsigned int* __restrict__ bits, int rows_per_node) {
  const size_t total = (size_t)n_nodes * d.dim_g;
  const int lane = threadIdx.x & 31;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(idx / d.dim_g), c = (int)(idx - (size_t)n * d.dim_g);
    const float* grow = g + (size_t)n * d.dim_g;
    const float* hrow = dh + (size_t)n * d.dim_h;
    float v;
    int r = 0;
    if (c < d.n_scalars) {
      v = hrow[c] * dsilu_n(grow[c]);
    } else if (c < d.g_off[1] || d.lmax == 0) {
      int l = 1;                                        // a gate scalar: find its l
      while (l < d.lmax && c >= d.gate_off[l + 1]) ++l;
      const int u = c - d.gate_off[l];
      float s = 0.0f;
      for (int i = 0; i < 2 * l + 1; ++i)
        s = fmaf(hrow[d.h_off[l] + i * d.mul[l] + u], grow[d.g_off[l] + i * d.mul[l] + u], s);
      v = s * dsilu_n(grow[c]);
    } else {
      int l = 1;
      while (l < d.lmax && c >= d.g_off[l + 1]) ++l;
      const int rel = c - d.g_off[l];
      const int u = rel % d.mul[l];
      v = hrow[d.h_off[l] + rel] * silu_n(grow[d.gate_off[l] + u]);
      r = l * l + rel / d.mul[l];
    }
    dg[idx] = v;
    const unsigned int mm = __reduce_max_sync(0xffffffffu, __float_as_uint(v) & 0x7fffffffu);
    if (lane == 0) atomicMax(bits + (size_t)n * rows_per_node + r, mm);
  }
}

// out[n, :width] = table[idx[n], :width]
__global__ void gather_rows_kernel(const float* __restrict__ table, const int* __restrict__ idx,
                                   float* __restrict__ out, int n_rows, int width, int ld_out) {
  const size_t total = (size_t)n_rows * width;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total;
       t += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(t / width), c = (int)(t - (size_t)n * width);
    out[(size_t)n * ld_out + c] = __ldg(table + (size_t)__ldg(idx + n) * width + c);
  }
}

// Ghost-exchange pack / unpack (multi-GPU; replaces pair_e3gnn_parallel.cpp:698-799's pack/unpack of
// x_ghost / dE_dx rows): out[i, :] = src[idx[i], :]  and  dst[idx[i], :] += in[i, :].  One thread per
// float4 (VEC) or float of a row; indices of one scatter call are unique, so the add is a plain
// read-modify-write and the summation order over peers (one call per peer) is deterministic.
template <bool VEC>
__global__ void gather_rows_idx_kernel(const float* __restrict__ src, int ld_src, const int* __restrict__ idx,
                                       long long n, int width, float* __restrict__ out) {
  const int w = VEC ? width >> 2 : width;
  const long long total = n * w;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long i = t / w;
    const int c = (int)(t - i * w);
    const float* row = src + (size_t)__ldg(idx + i) * ld_src;
    if (VEC) reinterpret_cast<float4*>(out)[t] = __ldg(reinterpret_cast<const float4*>(row) + c);
    else out[t] = __ldg(row + c);
  }
}
template <bool VEC>
__global__ void scatter_add_rows_idx_kernel(float* __restrict__ dst, int ld_dst, const int* __restrict__ idx,
                                            long long n, int width, const float* __restrict__ in) {
  const int w = VEC ? width >> 2 : width;
  const long long total = n * w;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long i = t / w;
    const int c = (int)(t - i * w);
    float* row = dst + (size_t)__ldg(idx + i) * ld_dst;
    if (VEC) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(in) + t);
      float4* p = reinterpret_cast<float4*>(row) + c;
      float4 o = *p;
      o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w;
      *p = o;
    } else {
      row[c] += __ldg(in + t);
    }
  }
}

// Readout (two bias-free linears folded into one vector wr = wr_hi + wr_lo, the fp32 pair of the fp64
// fold), species-wise rescale, energy sum and the seed of the backward pass dE/dh = scale[s] * wr.
// One warp per atom; the 128-term dot product, the rescale and the energy sum run in double so that the
// per-atom energy carries no parameter-rounding offset (identical atoms would all share its sign).
__global__ void readout_kernel(const float* __restrict__ h, const float* __restrict__ wr,
                               const float* __restrict__ wr_lo,
                               const float* __restrict__ scale, const float* __restrict__ shift,
                               const int* __restrict__ species, int n_nodes, int width,
                               float* __restrict__ atomic_energy, double* __restrict__ atomic_energy64,
                               double* __restrict__ energy, float* __restrict__ dh) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  double e_atom = 0.0;
  if (warp < n_nodes) {
    const float* row = h + (size_t)warp * width;
    const int s = __ldg(species + warp);
    const float sc = __ldg(scale + s);
    double acc = 0.0;
    for (int c = lane; c < width; c += 32) {
      const float w = __ldg(wr + c);
      const double wd = (double)w + (wr_lo != nullptr ? (double)__ldg(wr_lo + c) : 0.0);
      acc = fma((double)row[c], wd, acc);
      dh[(size_t)warp * width + c] = sc * w;
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    const double ea = fma((double)sc, acc, (double)__ldg(shift + s));
    if (lane == 0) {
      atomic_energy[warp] = (float)ea;
      atomic_energy64[warp] = ea;
      e_atom = ea;
    }
  }
  // block reduction in double, one atomic per block
  __shared__ double sm[32];
  const int wib = threadIdx.x >> 5;
  if (lane == 0) sm[wib] = e_atom;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += sm[i];
    atomicAdd(energy, t);
  }
}

// ---- species-wise linear: the 'nequip' self-connection (sevenn/nn/self_connection.py:11-67) -------------------
// FullyConnectedTensorProduct(x, S x0e, gate_in) with the species one-hot as second operand is a block-diagonal
// linear whose weight depends on the atom's species:  C_l[n] (+)= A_l[n] * W_l[species(n)].

// Counting sort of rows [0, n) by species, one CTA (launched with 2 * S ints of dynamic shared memory):
// perm[seg[s] .. seg[s+1]) lists the rows of species s, seg[S + 1 + s] is the first 64-row tile of species s and
// seg[2S + 1] the tile count.  Rows whose species lies outside [0, S) are left out.  The order of the rows inside
// one species is not fixed, which does not matter: every row of the linear is computed on its own.
constexpr int kSpTileRows = 64;
constexpr int kMaxSpeciesSc = 4096;     // 2 * S ints of shared memory in species_segment_kernel
__global__ void __launch_bounds__(1024) species_segment_kernel(const int* __restrict__ species, int n, int S,
                                                               int* __restrict__ perm, int* __restrict__ seg) {
  extern __shared__ int sp_sm[];
  int* cnt = sp_sm;
  int* cur = sp_sm + S;
  const int lane = threadIdx.x & 31;
  for (int s = threadIdx.x; s < S; s += blockDim.x) cnt[s] = 0;
  __syncthreads();
  // lanes holding the same species add once per warp (a one-species cell would otherwise serialise on one counter)
  for (int i0 = 0; i0 < n; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const int s = i < n ? __ldg(species + i) : -1;
    const unsigned int peers = __match_any_sync(0xffffffffu, s);
    if (s >= 0 && s < S && lane == __ffs(peers) - 1) atomicAdd(&cnt[s], __popc(peers));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int off = 0, tile = 0;
    for (int s = 0; s < S; ++s) {
      cur[s] = off;
      seg[s] = off;
      seg[S + 1 + s] = tile;
      off += cnt[s];
      tile += (cnt[s] + kSpTileRows - 1) / kSpTileRows;
    }
    seg[S] = off;
    seg[2 * S + 1] = tile;
  }
  __syncthreads();
  for (int i0 = 0; i0 < n; i0 += blockDim.x) {
    const int i = i0 + threadIdx.x;
    const int s = i < n ? __ldg(species + i) : -1;
    const unsigned int peers = __match_any_sync(0xffffffffu, s);
    const int leader = __ffs(peers) - 1;
    int base = 0;
    if (s >= 0 && s < S && lane == leader) base = atomicAdd(&cur[s], __popc(peers));
    base = __shfl_sync(peers, base, leader);
    if (s >= 0 && s < S) perm[base + __popc(peers & ((1u << lane) - 1u))] = i;
  }
}

// One irrep block of the species-wise linear: W_l of species s at W + s * w_stride + w_off, [K, N] row-major.
struct SpLinBlock {
  int w_off;
  int d;                // 2l+1 rows per node
  int K, N;
  int a_off, a_cs;
  int c_off, c_cs;
};

struct SpLinArgs {
  const float* A;
  float* C;
  const float* W;
  long long w_stride;   // floats per species
  const int* perm;      // species_segment_kernel output
  const int* seg;
  int S;
  int lda, ldc;
  int accumulate;       // 1: C += result
  int nblocks;
  SpLinBlock blk[kMaxL];
};

constexpr int kSpBN = 64, kSpBK = 16, kSpThreads = 256;

// Tile: up to 64 rows of one species x 64 columns of one (block, component); 4 x 4 outputs per thread.
// grid = (ceil(n / 64) + S, ceil(max N / 64), sum of 2l+1 over the blocks); tiles past the last one exit.  A rows
// are read and C rows written through the permutation; every C element is written once, summed over K in a fixed
// order, so a row's result does not depend on which other rows share its tile.  K, N, the offsets and the leading
// dimensions are multiples of 4 (checked by the launcher).
__global__ void __launch_bounds__(kSpThreads) species_linear_kernel(const SpLinArgs a) {
  int z = blockIdx.z, bi = 0;
  while (bi + 1 < a.nblocks && z >= a.blk[bi].d) { z -= a.blk[bi].d; ++bi; }
  const SpLinBlock b = a.blk[bi];
  const int comp = z;
  const int col0 = blockIdx.y * kSpBN;
  if (col0 >= b.N) return;
  const int* tile0 = a.seg + a.S + 1;
  const int tile = blockIdx.x;
  if (tile >= __ldg(tile0 + a.S)) return;
  int lo = 0, hi = a.S - 1;          // the species of this tile: the last s with tile0[s] <= tile
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(tile0 + mid) <= tile) lo = mid;
    else hi = mid - 1;
  }
  const int s = lo;
  const int r0 = __ldg(a.seg + s) + (tile - __ldg(tile0 + s)) * kSpTileRows;
  const int nr = min(kSpTileRows, __ldg(a.seg + s + 1) - r0);
  const float* W = a.W + (size_t)s * a.w_stride + b.w_off;

  __shared__ __align__(16) float As[kSpBK][kSpTileRows + 4];
  __shared__ __align__(16) float Bs[kSpBK][kSpBN];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int a_row = tid >> 2, a_kq = tid & 3;          // A loader: row, k quad
  const float* a_ptr = a_row < nr ? a.A + (size_t)__ldg(a.perm + r0 + a_row) * a.lda + b.a_off + comp * b.a_cs : nullptr;
  const int b_k = tid >> 4, gc = col0 + (tid & 15) * 4;  // W loader: k, column quad

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;

  float4 ra, rb;
  auto load_tiles = [&](int k0) {
    const int ka = k0 + a_kq * 4;
    ra = make_float4(0.f, 0.f, 0.f, 0.f);
    if (a_ptr != nullptr && ka < b.K) ra = __ldg(reinterpret_cast<const float4*>(a_ptr + ka));
    rb = make_float4(0.f, 0.f, 0.f, 0.f);
    const int kb = k0 + b_k;
    if (kb < b.K && gc < b.N) rb = __ldg(reinterpret_cast<const float4*>(W + (size_t)kb * b.N + gc));
  };
  load_tiles(0);
  for (int k0 = 0; k0 < b.K; k0 += kSpBK) {
    As[a_kq * 4 + 0][a_row] = ra.x;
    As[a_kq * 4 + 1][a_row] = ra.y;
    As[a_kq * 4 + 2][a_row] = ra.z;
    As[a_kq * 4 + 3][a_row] = ra.w;
    *reinterpret_cast<float4*>(&Bs[b_k][(tid & 15) * 4]) = rb;
    __syncthreads();
    if (k0 + kSpBK < b.K) load_tiles(k0 + kSpBK);
#pragma unroll
    for (int k = 0; k < kSpBK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(aa[i], bb[j], acc[i][j]);
    }
    __syncthreads();
  }

  const int c = col0 + tx * 4;
  if (c >= b.N) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = ty * 4 + i;
    if (r >= nr) continue;
    float4* cp = reinterpret_cast<float4*>(a.C + (size_t)__ldg(a.perm + r0 + r) * a.ldc + b.c_off + comp * b.c_cs + c);
    float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    if (a.accumulate) {
      const float4 o = *cp;
      v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
    }
    *cp = v;
  }
}

}  // namespace s7b
