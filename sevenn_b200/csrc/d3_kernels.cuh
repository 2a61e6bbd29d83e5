// DFT-D3 dispersion correction (Grimme 2010; zero and Becke-Johnson damping) on a cell list.
//
// Replaces the reference's CUDA D3 (sevenn/pair_e3gnn/pair_d3_for_ase.cu = pair_d3.cu without LAMMPS):
//   kernel_get_coordination_number        :1004-1058
//   kernel_get_dC6_dCNij                  :765-845
//   kernel_get_forces_without_dC6_{zero,bj}  :1263-1496, 1534-1745
//   kernel_get_forces_with_dC6            :1797-1962
// The reference enumerates all N(N+1)/2 atom pairs x all lattice translations (O(N^2 tau) work, an
// N(N+1)/2-sized C6 table, int indexing that overflows at 46 340 atoms, one GPU).  Here:
//   * atoms are binned on the fractional cell (neighbor.cuh) and one WARP per atom sweeps the bin images
//     inside the cutoff, one lane per bin image -> O(N * neighbours) work, any cell size (also cells
//     much smaller than the 50 A cutoff), 64-bit-free indexing (no pair table at all);
//   * C6_ij(CN_i, CN_j) is not tabulated per pair: the Gaussian weight of reference (a, b) factorises,
//     L_ij(a,b) = w_i(a) w_j(b), because the reference coordination numbers depend only on (element,
//     index) (asserted by tools/convert_d3_params.py), so with per-atom normalised weights W_i
//         C6_ij = sum_b V_i[t_j][b] W_j[b],   V_i[t][b] = sum_a c6ref[t_i][t][a][b] W_i[a]
//     costs 5 FMAs per pair (and 5 more for dC6/dCN_i) instead of 25 exponentials;
//   * every ordered pair (i <- j) is evaluated by i's warp only: forces, dE/dCN, energy and virial are plain
//     per-warp sums, no atomics; pair math in fp32 as the reference,
//     accumulation in fp64 (the reference's float image sums lose ~4.5e-5 of the NaCl golden energy);
//   * an atom range [i_begin, i_end) per launch: multi-GPU = atom decomposition with replicated positions
//     (the 50 A range is of the order of the box), three small all-gathers per step (sevenn_b200/d3.py).
//   * a batch of B structures in one pass: each structure has its own grid (a [B] table) and its own range of
//     bins of one key space, as in the neighbour list (neighbor.cuh); a sweep visits only its own structure's
//     bins.  A single structure is a batch of one.  The pair and chain passes write per-atom energy and virial
//     terms and one block per structure sums them in a fixed order (d3_system_sums_kernel): per-structure
//     results without atomics, independent of the other members of the batch.
// Units inside: bohr and hartree, as in the reference.
#pragma once
#include "common.cuh"
#include "neighbor.cuh"

namespace s7b {

constexpr int kD3MaxTypes = 16;       // elements per structure (the per-warp C6 table sV)
constexpr int kD3Elements = 94;       // rows of the full element tables (Z = 1..94)
constexpr int kD3WarpsPerBlock = 4;
// resident blocks per SM the cell-list passes are compiled for (registers <= 64K / (128 x blocks), no spills): the
// occupancy they had with the grid in kernel parameters
constexpr int kD3CnBlocks = 10, kD3PairBlocks = 6, kD3ChainBlocks = 7;
constexpr float kD3K1 = 16.0f;
constexpr double kD3K3 = -4.0;
constexpr double kAuToAng = 0.52917726, kAuToEv = 27.21138505;   // pair_d3_for_ase.h:200-201

// The passes are compiled twice from one source: kBatch = true reads every structure's grid, radii and local types
// from the [B] tables; kBatch = false (one structure, s7b_d3_set_system) takes the grid and radii as kernel parameters
// and the type index as both table row and local type, the arithmetic of the single-structure kernels unchanged.
//
// An atom's type word: kBatch, its row of the element tables in the low byte and its local type (rank among the
// elements of its own structure: the index of sV) above; one structure, its type index.
template <bool kBatch> __device__ __forceinline__ int d3_row(int tw) { return kBatch ? (tw & 0xff) : tw; }
template <bool kBatch> __device__ __forceinline__ int d3_local(int tw) { return kBatch ? (tw >> 8) : tw; }

struct D3Atoms {              // arrays over atoms in bin-sorted order
  const double* x;            // [n,3] wrapped cartesian positions (bohr)
  const int* type;            // [n]   type word (d3_row / d3_local)
  const int* sys;             // [n]   structure of each atom
  const float* W;             // [n,5] normalised C6 reference weights
  const float* logD;          // [n]   log of the weight sum (den <= 1e-99 fallback, pair_d3_for_ase.cu:824-844)
  const int* near;            // [n]   nearest reference index
  const double* dc6i;         // [n]   -dE/dCN (after the pair pass)
  const int* bin_start;       // [nbins + 1]
  const int* bin_of;          // [n]   bin key of each (sorted) atom: bin_off[structure] + local bin
  // per structure (kBatch)
  const NLGrid* grids;        // [B]   cell (bohr), bins per direction, pbc
  const int* bin_off;         // [B+1]
  const int* R;               // [B,6] search radii in bins: R_vdw (x,y,z), R_cn (x,y,z)
  const int* lrows;           // [B,kD3MaxTypes] table row of every local type
  const int* nloc;            // [B]   local types
};

struct D3Params {
  int nrows, damping;         // rows of the element tables; damping: 0 = zero, 1 = Becke-Johnson
  float s6, s8, a1, a2, alp6, alp8;
  double rthr, cnthr;         // squared cutoffs (bohr^2)
  float rcov[kD3Elements], r2r4[kD3Elements];
  const float* r0ab;          // [nrows, nrows] (bohr)
  const float* c6ref;         // [nrows, nrows, 5, 5]
};

struct D3Out {
  double* cn;                 // [n]   (sorted order)
  double* dc6i;               // [n]
  double* force;              // [n,3]
  double* eatom;              // [n]   pair energy of each atom (pass 2)
  double* spair;              // [n,6] pair virial terms of each atom (pass 2; xx, yy, zz, xy, xz, yz)
  double* schain;             // [n,6] chain-rule virial terms of each atom (pass 3)
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off >= 1; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// Sweep of all (bin image, atom) candidates around atom i with one lane per bin image over the bins [boff, ...) of
// grid g.  f(j, dx, dy, dz, r2, self) is called for every candidate with r2 <= cut2 (self: j == i, other image).
// kBatch: g is in global memory, and its cell is re-read (L1-resident) at each bin image rather than held in 18
// registers for the whole sweep (a volatile load is not hoisted out of the loop).
__device__ __forceinline__ double d3_ld_cell(const double* p) {
  double v;
  asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

template <bool kBatch, class F>
__device__ __forceinline__ void d3_sweep(const NLGrid& g, const int (&R)[3], int boff, const D3Atoms& A, int i, double cut2,
                                         int lane, F&& f) {
  const double xi = A.x[3 * i], yi = A.x[3 * i + 1], zi = A.x[3 * i + 2];
  const int k = A.bin_of[i] - boff;
  const int b2 = k % g.nb[2], b1 = (k / g.nb[2]) % g.nb[1], b0 = k / (g.nb[2] * g.nb[1]);
  const int n1 = 2 * R[1] + 1, n2 = 2 * R[2] + 1;
  const int total = (2 * R[0] + 1) * n1 * n2;
  for (int m = lane; m < total; m += 32) {
    const int d2 = m % n2 - R[2], d1 = (m / n2) % n1 - R[1], d0 = m / (n2 * n1) - R[0];
    int q0 = b0 + d0, q1 = b1 + d1, q2 = b2 + d2, s0 = 0, s1 = 0, s2 = 0;
    if (g.pbc[0]) { s0 = (q0 >= 0) ? q0 / g.nb[0] : -((-q0 + g.nb[0] - 1) / g.nb[0]); q0 -= s0 * g.nb[0]; }
    else if (q0 < 0 || q0 >= g.nb[0]) continue;
    if (g.pbc[1]) { s1 = (q1 >= 0) ? q1 / g.nb[1] : -((-q1 + g.nb[1] - 1) / g.nb[1]); q1 -= s1 * g.nb[1]; }
    else if (q1 < 0 || q1 >= g.nb[1]) continue;
    if (g.pbc[2]) { s2 = (q2 >= 0) ? q2 / g.nb[2] : -((-q2 + g.nb[2] - 1) / g.nb[2]); q2 -= s2 * g.nb[2]; }
    else if (q2 < 0 || q2 >= g.nb[2]) continue;
    double c[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) c[q] = kBatch ? d3_ld_cell(g.cell + q) : g.cell[q];
    const double sx = s0 * c[0] + s1 * c[3] + s2 * c[6] - xi;
    const double sy = s0 * c[1] + s1 * c[4] + s2 * c[7] - yi;
    const double sz = s0 * c[2] + s1 * c[5] + s2 * c[8] - zi;
    const int nbin = boff + (q0 * g.nb[1] + q1) * g.nb[2] + q2;
    const bool same_image = (s0 == 0 && s1 == 0 && s2 == 0);
    const int e = A.bin_start[nbin + 1];
    for (int j = A.bin_start[nbin]; j < e; ++j) {
      if (same_image && j == i) continue;
      const double dx = A.x[3 * j] + sx, dy = A.x[3 * j + 1] + sy, dz = A.x[3 * j + 2] + sz;
      const double r2 = dx * dx + dy * dy + dz * dz;
      if (r2 <= cut2) f(j, (float)dx, (float)dy, (float)dz, (float)r2, j == i);
    }
  }
}

// The sweep of atom i over its own structure's bins: kBatch from the [B] tables (rsel = 0: R_vdw, 3: R_cn), else
// the grid g1 and radii R1 of the one structure.
template <bool kBatch, class F>
__device__ __forceinline__ void d3_sweep_atom(const NLGrid& g1, int3 R1, const D3Atoms& A, int i, int rsel, double cut2,
                                              int lane, F&& f) {
  if constexpr (kBatch) {
    const int sb = A.sys[i];
    const int R[3] = {A.R[6 * sb + rsel], A.R[6 * sb + rsel + 1], A.R[6 * sb + rsel + 2]};
    d3_sweep<true>(A.grids[sb], R, A.bin_off[sb], A, i, cut2, lane, f);
  } else {
    const int R[3] = {R1.x, R1.y, R1.z};
    d3_sweep<false>(g1, R, 0, A, i, cut2, lane, f);
  }
}

// ---- pass 1: coordination numbers (:1004-1058) -----------------------------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3CnBlocks)
d3_cn_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, int3 R1, int i_begin, int i_end, D3Out out) {
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= i_end) return;
  const float rci = P.rcov[d3_row<kBatch>(A.type[i])];
  double cn = 0.0;
  d3_sweep_atom<kBatch>(g1, R1, A, i, 3, P.cnthr, lane, [&](int j, float, float, float, float r2, bool) {
    const float rc = rci + P.rcov[d3_row<kBatch>(A.type[j])];
    const float rr = rsqrtf(r2);
    cn += (double)(1.0f / (1.0f + __expf(-kD3K1 * (rc * rr - 1.0f))));
  });
  cn = warp_sum(cn);
  if (lane == 0) out.cn[i] = cn;
}

// ---- per atom: normalised Gaussian weights of the C6 references and their CN derivative (:765-845) --
// W[a] = w_a / D, dW[a] = d W[a] / d CN, w_a = exp(K3 (CN_ref[a] - CN)^2), D = sum_a w_a (double: the
// exponents reach -400 for highly coordinated atoms)
__global__ void d3_weights_kernel(int n, const int* __restrict__ type, const double* __restrict__ cn,
                                  const float* __restrict__ cnref /*[nrows,5]*/, const int* __restrict__ mxc,
                                  float* __restrict__ W, float* __restrict__ dW, float* __restrict__ logD,
                                  int* __restrict__ near) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int t = type[i] & 0xff, m = mxc[t];                 // the table row of either type word
  const float cni = (float)cn[i];                           // the reference holds CN as a float here (:780)
  double w[5], dw[5], D = 0.0, dD = 0.0;
  float best = 3.0e38f;
  int nb = 0;
  for (int a = 0; a < 5; ++a) {
    w[a] = dw[a] = 0.0;
    if (a >= m) continue;
    const float cr = cnref[t * 5 + a];
    const float d2 = (cr - cni) * (cr - cni);
    if (d2 < best) { best = d2; nb = a; }
    w[a] = exp(kD3K3 * (double)d2);
    dw[a] = w[a] * 2.0 * kD3K3 * (double)(cni - cr);
    D += w[a];
    dD += dw[a];
  }
  // exponent bookkeeping for the reference's "denominator <= 1e-99" branch: log D without underflow
  double lD;
  if (D > 1e-300) lD = log(D);
  else lD = kD3K3 * (double)best;                            // dominated by the nearest reference
  for (int a = 0; a < 5; ++a) {
    const double Wn = D > 1e-300 ? w[a] / D : (a == nb ? 1.0 : 0.0);
    const double dWn = D > 1e-300 ? (dw[a] - Wn * dD) / D : 0.0;
    W[i * 5 + a] = (float)Wn;
    dW[i * 5 + a] = (float)dWn;
  }
  logD[i] = (float)lD;
  near[i] = nb;
}

// ---- pass 2: pair energy, explicit-r forces, dE/dCN (:1263-1745) -----------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3PairBlocks)
d3_pair_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, const float* __restrict__ dW, int3 R1, int i_begin,
               int i_end, D3Out out) {
  __shared__ float sV[kD3WarpsPerBlock][kD3MaxTypes][10];      // V_i[t][b], dV_i[t][b] over local types t
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + wib;
  if (i >= i_end) return;
  double e = 0.0, fx = 0.0, fy = 0.0, fz = 0.0, dc = 0.0;
  double sg[6] = {0, 0, 0, 0, 0, 0};                              // xx, yy, zz, xy, xz, yz
  const int ti = d3_row<kBatch>(A.type[i]), sb = kBatch ? A.sys[i] : 0;
  // V_i[t][b] = sum_a c6ref[ti][row(t)][a][b] W_i[a]  (lanes over (t, b))
  const int nloc = kBatch ? A.nloc[sb] : P.nrows;
  for (int q = lane; q < nloc * 5; q += 32) {
    const int t = q / 5, b = q % 5;
    const int tr = kBatch ? A.lrows[kD3MaxTypes * sb + t] : t;
    float v = 0.0f, dv = 0.0f;
#pragma unroll
    for (int a = 0; a < 5; ++a) {
      const float c = __ldg(P.c6ref + ((ti * P.nrows + tr) * 5 + a) * 5 + b);
      v = fmaf(c, A.W[i * 5 + a], v);
      dv = fmaf(c, dW[i * 5 + a], dv);
    }
    sV[wib][t][b] = v;
    sV[wib][t][5 + b] = dv;
  }
  __syncwarp();
  const float logDi = A.logD[i];
  const int near_i = A.near[i];
  const float r2r4i = P.r2r4[ti];
  d3_sweep_atom<kBatch>(g1, R1, A, i, 0, P.rthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool self) {
    const int twj = A.type[j], tj = d3_row<kBatch>(twj), lj = d3_local<kBatch>(twj);
    float c6 = 0.0f, dc6 = 0.0f;
    if (logDi + A.logD[j] > -227.95593f) {                      // den > 1e-99
#pragma unroll
      for (int b = 0; b < 5; ++b) {
        const float wj = A.W[j * 5 + b];
        c6 = fmaf(sV[wib][lj][b], wj, c6);
        dc6 = fmaf(sV[wib][lj][5 + b], wj, dc6);
      }
    } else {
      c6 = __ldg(P.c6ref + ((ti * P.nrows + tj) * 5 + near_i) * 5 + A.near[j]);
    }
    float gfun, dgdr;                                           // E_pair = -C6 g(r)
    const float r = sqrtf(r2);
    if (P.damping == 1) {
      const float r42x3 = r2r4i * P.r2r4[tj] * 3.0f;
      const float R0 = fmaf(P.a1, sqrtf(r42x3), P.a2);
      const float R0_2 = R0 * R0, R0_6 = R0_2 * R0_2 * R0_2, R0_8 = R0_6 * R0_2;
      const float r5 = r2 * r2 * r, r7 = r5 * r2;
      const float t6 = 1.0f / fmaf(r5, r, R0_6), t8 = 1.0f / fmaf(r7, r, R0_8);
      const float s8r = P.s8 * r42x3;
      gfun = fmaf(s8r, t8, P.s6 * t6);
      dgdr = -fmaf(8.0f * s8r * r7, t8 * t8, 6.0f * P.s6 * r5 * t6 * t6);
    } else {
      const float r0 = __ldg(P.r0ab + ti * P.nrows + tj);
      const float r42 = r2r4i * P.r2r4[tj];
      const float rr = 1.0f / r;
      const float t6 = __powf(P.a1 * r0 * rr, P.alp6), t8 = __powf(P.a2 * r0 * rr, P.alp8);
      const float d6 = 1.0f / fmaf(6.0f, t6, 1.0f), d8 = 1.0f / fmaf(6.0f, t8, 1.0f);
      const float r2_rc = rr * rr, r6_rc = r2_rc * r2_rc * r2_rc, r8_rc = r6_rc * r2_rc;
      const float s8r = P.s8 * r42;
      gfun = r6_rc * fmaf(3.0f * r2_rc, s8r * d8, P.s6 * d6);
      // d/dr [ s6 d6 r^-6 + 3 s8 r42 d8 r^-8 ]
      dgdr = 6.0f * r8_rc * r * (P.s6 * d6 * fmaf(P.alp6 * t6, d6, -1.0f) + r2_rc * s8r * d8 * fmaf(3.0f * P.alp8 * t8, d8, -4.0f));
    }
    e -= 0.5 * (double)(c6 * gfun);
    dc += (double)(gfun * dc6);                                 // dc6i_i = sum g dC6/dCN_i
    const float dEdr = -c6 * dgdr;                              // of the full pair
    const float s = dEdr / r;
    const float vx = s * dx, vy = s * dy, vz = s * dz;          // dE/d(r_ij) direction (r_ij = x_j - x_i + tau)
    if (!self) { fx += (double)vx; fy += (double)vy; fz += (double)vz; }
    sg[0] -= 0.5 * (double)(vx * dx); sg[1] -= 0.5 * (double)(vy * dy); sg[2] -= 0.5 * (double)(vz * dz);
    sg[3] -= 0.5 * (double)(vx * dy); sg[4] -= 0.5 * (double)(vx * dz); sg[5] -= 0.5 * (double)(vy * dz);
  });
  e = warp_sum(e); fx = warp_sum(fx); fy = warp_sum(fy); fz = warp_sum(fz); dc = warp_sum(dc);
#pragma unroll
  for (int q = 0; q < 6; ++q) sg[q] = warp_sum(sg[q]);
  if (lane == 0) {
    out.force[3 * i] = fx; out.force[3 * i + 1] = fy; out.force[3 * i + 2] = fz;
    out.dc6i[i] = dc;
    out.eatom[i] = e;
#pragma unroll
    for (int q = 0; q < 6; ++q) out.spair[6 * (size_t)i + q] = sg[q];
  }
}

// ---- pass 3: chain rule through the coordination numbers (:1797-1962) ------------------------------
template <bool kBatch>
__global__ void __launch_bounds__(32 * kD3WarpsPerBlock, kD3ChainBlocks)
d3_chain_kernel(const NLGrid g1, const D3Atoms A, const D3Params P, int3 R1, int i_begin, int i_end, D3Out out) {
  const int lane = threadIdx.x & 31;
  const int i = i_begin + blockIdx.x * kD3WarpsPerBlock + (threadIdx.x >> 5);
  if (i >= i_end) return;
  double fx = 0.0, fy = 0.0, fz = 0.0;
  double sg[6] = {0, 0, 0, 0, 0, 0};
  const float rci = P.rcov[d3_row<kBatch>(A.type[i])];
  const double di = A.dc6i[i];
  const float cn2 = (float)P.cnthr;
  d3_sweep_atom<kBatch>(g1, R1, A, i, 3, P.cnthr, lane, [&](int j, float dx, float dy, float dz, float r2, bool self) {
    if (r2 >= cn2) return;                                      // the reference uses a strict bound here (:1843)
    const float rc = rci + P.rcov[d3_row<kBatch>(A.type[j])];
    const float rr = rsqrtf(r2);
    const float ex = __expf(-kD3K1 * (rc * rr - 1.0f));
    const float dcnn = -kD3K1 * rc * ex / (r2 * (ex + 1.0f) * (ex + 1.0f));     // d cnf / dr
    const float x1 = dcnn * (float)(di + A.dc6i[j]);            // -dE/dr of the pair through CN_i and CN_j
    const float s = x1 * rr;
    const float vx = s * dx, vy = s * dy, vz = s * dz;
    if (!self) { fx -= (double)vx; fy -= (double)vy; fz -= (double)vz; }
    sg[0] += 0.5 * (double)(vx * dx); sg[1] += 0.5 * (double)(vy * dy); sg[2] += 0.5 * (double)(vz * dz);
    sg[3] += 0.5 * (double)(vx * dy); sg[4] += 0.5 * (double)(vx * dz); sg[5] += 0.5 * (double)(vy * dz);
  });
  fx = warp_sum(fx); fy = warp_sum(fy); fz = warp_sum(fz);
#pragma unroll
  for (int q = 0; q < 6; ++q) sg[q] = warp_sum(sg[q]);
  if (lane == 0) {
    out.force[3 * i] += fx; out.force[3 * i + 1] += fy; out.force[3 * i + 2] += fz;
#pragma unroll
    for (int q = 0; q < 6; ++q) out.schain[6 * (size_t)i + q] = sg[q];
  }
}

// ---- per-structure sums, one block per structure, in a fixed order ----------------------------------------
// Over the atoms of [i_begin, i_end) in structure b (sorted order; a structure's atoms are contiguous there):
// eatom != nullptr: energy[b] = sum eatom, sigma[b] = sum s;  eatom == nullptr: sigma[b] += sum s.
// Atom a0 + k is summed by thread k % kD3SumBlock, so a structure's sums do not depend on where it sits in a batch.
constexpr int kD3SumBlock = 512;
__global__ void __launch_bounds__(kD3SumBlock)
d3_system_sums_kernel(const int* __restrict__ atom_ptr, int i_begin, int i_end, const double* __restrict__ eatom,
                      const double* __restrict__ s, double* __restrict__ energy, double* __restrict__ sigma) {
  const int b = blockIdx.x;
  const int a0 = max(atom_ptr[b], i_begin), a1 = min(atom_ptr[b + 1], i_end);
  double v[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = a0 + threadIdx.x; i < a1; i += kD3SumBlock) {
    if (eatom) v[0] += eatom[i];
#pragma unroll
    for (int q = 0; q < 6; ++q) v[1 + q] += s[6 * (size_t)i + q];
  }
  __shared__ double sm[7][kD3SumBlock];
#pragma unroll
  for (int q = 0; q < 7; ++q) sm[q][threadIdx.x] = v[q];
  __syncthreads();
  for (int h = kD3SumBlock >> 1; h > 0; h >>= 1) {
    if (threadIdx.x < h)
#pragma unroll
      for (int q = 0; q < 7; ++q) sm[q][threadIdx.x] += sm[q][threadIdx.x + h];
    __syncthreads();
  }
  if (eatom) {
    if (threadIdx.x == 0) energy[b] = sm[0][0];
    if (threadIdx.x < 6) sigma[6 * (size_t)b + threadIdx.x] = sm[1 + threadIdx.x][0];
  } else if (threadIdx.x < 6) {
    sigma[6 * (size_t)b + threadIdx.x] += sm[1 + threadIdx.x][0];
  }
}

// ---- set-up on the device -------------------------------------------------------------------------------
// Positions (Angstrom) wrapped into the cell in ALL directions, as the reference does (pair_d3_for_ase.cu:1198-1212),
// in bohr: f = (p . inv_a) / au, f -= floor(f), x = f . cell, every operation rounded on its own (no FMA
// contraction), as the plain host expression, so that a structure's positions do not depend on where they were
// wrapped.  With numbers != nullptr also: table row = Z - 1, the structure's element presence [B,94], and the lowest
// structure with Z outside 1..94 in err[0].
__global__ void d3_prepare_kernel(int n, int B, const int* __restrict__ atom_ptr, const NLGrid* __restrict__ grids,
                                  const double* __restrict__ pos, const int* __restrict__ numbers, double* __restrict__ x,
                                  int* __restrict__ row, int* __restrict__ present, int* __restrict__ err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int sb = nl_system_of(atom_ptr, B, i);
  const double* inv = grids[sb].inv;
  const double* cell = grids[sb].cell;
  const double p0 = pos[3 * i], p1 = pos[3 * i + 1], p2 = pos[3 * i + 2];
  double f[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double d = __dadd_rn(__dadd_rn(__dmul_rn(p0, inv[0 * 3 + a]), __dmul_rn(p1, inv[1 * 3 + a])), __dmul_rn(p2, inv[2 * 3 + a]));
    f[a] = __ddiv_rn(d, kAuToAng);
    f[a] = __dsub_rn(f[a], floor(f[a]));
  }
#pragma unroll
  for (int c = 0; c < 3; ++c)
    x[3 * i + c] = __dadd_rn(__dadd_rn(__dmul_rn(f[0], cell[0 * 3 + c]), __dmul_rn(f[1], cell[1 * 3 + c])), __dmul_rn(f[2], cell[2 * 3 + c]));
  if (numbers) {
    const int z = numbers[i];
    if (z < 1 || z > kD3Elements) { atomicMin(err, sb); row[i] = 0; }
    else { row[i] = z - 1; present[kD3Elements * sb + z - 1] = 1; }
  }
}

// Local types of every structure: the rank of each present element (lrank [B,94]), the table row of every local type
// (lrows [B,kD3MaxTypes]) and their number (nloc [B]); the lowest structure with more than kD3MaxTypes elements
// in err[1].  One thread per structure.
__global__ void d3_local_types_kernel(int B, const int* __restrict__ present, int* __restrict__ lrank,
                                      int* __restrict__ lrows, int* __restrict__ nloc, int* __restrict__ err) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  int c = 0;
  for (int z = 0; z < kD3Elements; ++z) {
    if (!present[kD3Elements * b + z]) continue;
    if (c < kD3MaxTypes) lrows[kD3MaxTypes * b + c] = z;
    lrank[kD3Elements * b + z] = c++;
  }
  nloc[b] = c < kD3MaxTypes ? c : kD3MaxTypes;
  if (c > kD3MaxTypes) atomicMin(err + 1, b);
}

// gather / scatter between the caller's atom order and the bin-sorted order; the type word of every sorted atom
// (batch: row | lrank[structure][row] << 8; one structure, lrank == nullptr: the type index)
__global__ void d3_sort_gather_kernel(int n, const int* __restrict__ idx_sorted, const int* __restrict__ key_sorted,
                                      const double* __restrict__ wrapped, const int* __restrict__ row,
                                      const int* __restrict__ sys, const int* __restrict__ lrank,
                                      double* __restrict__ xs, int* __restrict__ ts, int* __restrict__ ss,
                                      int* __restrict__ bin_of) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int i = idx_sorted[s];
  xs[3 * s] = wrapped[3 * i]; xs[3 * s + 1] = wrapped[3 * i + 1]; xs[3 * s + 2] = wrapped[3 * i + 2];
  const int r = row[i], sb = sys[i];
  ts[s] = lrank ? (r | (lrank[kD3Elements * sb + r] << 8)) : r;
  ss[s] = sb;
  bin_of[s] = key_sorted[s];
}

// per-structure results in the caller's units and atom order: forces (eV/A), energy [B] (eV), virial [B,6] (eV;
// xx,yy,zz,xy,yz,zx of sum f (x) r, the order of the network's s7b_engine_system_results)
__global__ void d3_system_results_kernel(int n, int B, const int* __restrict__ idx_sorted, const double* __restrict__ force,
                                         const double* __restrict__ energy, const double* __restrict__ sigma,
                                         double* __restrict__ out_e, double* __restrict__ out_f, double* __restrict__ out_v) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < 3 * n) {
    const int s = t / 3, c = t - 3 * s;
    out_f[3 * (size_t)idx_sorted[s] + c] = force[t] * (kAuToEv / kAuToAng);
  }
  if (t < B) {
    const double* sg = sigma + 6 * (size_t)t;               // xx, yy, zz, xy, xz, yz
    out_e[t] = energy[t] * kAuToEv;
    out_v[6 * (size_t)t + 0] = sg[0] * kAuToEv; out_v[6 * (size_t)t + 1] = sg[1] * kAuToEv;
    out_v[6 * (size_t)t + 2] = sg[2] * kAuToEv; out_v[6 * (size_t)t + 3] = sg[3] * kAuToEv;
    out_v[6 * (size_t)t + 4] = sg[5] * kAuToEv; out_v[6 * (size_t)t + 5] = sg[4] * kAuToEv;
  }
}
__global__ void d3_unsort_kernel(int n, int width, const int* __restrict__ idx_sorted, const double* __restrict__ in,
                                 double scale, double* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * width) return;
  const int s = t / width, c = t - s * width;
  out[(size_t)idx_sorted[s] * width + c] = in[t] * scale;
}

}  // namespace s7b
