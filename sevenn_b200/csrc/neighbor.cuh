// Device neighbour list / graph build (SURVEY 8(f).1): positions + cell -> CSR over centre atoms.
//
// Replaces, for the calculator front-end, the CPU graph build the reference runs every step
//   sevenn/train/dataload.py:32-129  (matscipy / ASE neighbour_list 'ijDS' -> edge_index, edge_vec)
//   sevenn/pair_e3gnn/pair_e3gnn.cpp:118-170 (LAMMPS full neighbour list -> edge arrays)
// Semantics restated: a directed edge i <- j for every pair, every periodic image included (also
// self-images at non-zero shift), with |r_j - r_i + S.cell| < cutoff; edge_vec = r_j - r_i + S.cell
// evaluated in double and stored as float (the reference builds it in numpy float64, then casts).
//
// Method: atoms are binned on a grid of the fractional cell (bin width >= cutoff unless the cell is
// thinner than the cutoff), sorted by bin with a stable radix sort (deterministic neighbour order),
// then one thread per atom visits the (2R+1)^3 surrounding bins, R = ceil(cutoff / bin width), with
// the periodic image shift of every visited bin -- correct for any cell size, including cells much
// smaller than the cutoff.  Two passes (count, exclusive scan, fill) emit the CSR directly, so the
// engine needs no sort of the edge list.  Non-periodic directions use the bounding box and no images.
// D3's cell list (d3.cu) shares the lattice set-up (nl_lattice) and the binning (nl_bin_sort); only the bin
// policy, how many bins and how far to search, is each caller's own.
#pragma once
#include <cub/cub.cuh>
#include <string>

#include "common.cuh"

namespace s7b {

struct NLGrid {
  double cell[9];      // rows = lattice vectors a, b, c (for non-periodic systems: a bounding frame)
  double inv[9];       // inverse: frac = pos * inv  (row-vector convention)
  double fmin[3];      // offset of the binned fractional range (0 for periodic directions)
  double fspan[3];     // length of the binned fractional range (1 for periodic directions)
  int nb[3];           // bins per direction
  int R[3];            // search radius in bins
  int pbc[3];
  double cutoff2;
};

__device__ __forceinline__ void nl_frac(const NLGrid& g, const double* p, double* f) {
#pragma unroll
  for (int a = 0; a < 3; ++a) f[a] = p[0] * g.inv[0 * 3 + a] + p[1] * g.inv[1 * 3 + a] + p[2] * g.inv[2 * 3 + a];
}

// A batch is B independent structures; the atoms of structure b are [atom_ptr[b], atom_ptr[b+1]) and its bins
// are [bin_off[b], bin_off[b+1]) of one key space, so one stable sort and one bin_start cover the whole batch
// and no bin holds atoms of two structures.  A single structure is a batch of one.

// structure of atom i: the last b with atom_ptr[b] <= i (empty structures are skipped)
__device__ __forceinline__ int nl_system_of(const int* __restrict__ atom_ptr, int B, int i) {
  int lo = 0, hi = B;   // atom_ptr[lo] <= i < atom_ptr[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(atom_ptr + mid) <= i) lo = mid;
    else hi = mid;
  }
  return lo;
}

// Fractional bounding box [B, 6] = (lo_a, hi_a) per direction of every structure, one block per structure.
// Each fractional coordinate is rounded as the plain host expression p0*i0a + p1*i1a + p2*i2a (no FMA
// contraction), so a structure's grid does not depend on where or with what its bounding box was taken.
static __global__ void nl_bbox_kernel(const NLGrid* __restrict__ grids, const int* __restrict__ atom_ptr,
                                      const double* __restrict__ pos, double* __restrict__ lohi) {
  const int b = blockIdx.x;
  const int a0 = atom_ptr[b], a1 = atom_ptr[b + 1];
  const double* inv = grids[b].inv;
  double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
  for (int i = a0 + threadIdx.x; i < a1; i += blockDim.x) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double f = __dadd_rn(__dadd_rn(__dmul_rn(pos[3 * i], inv[0 * 3 + a]), __dmul_rn(pos[3 * i + 1], inv[1 * 3 + a])),
                                 __dmul_rn(pos[3 * i + 2], inv[2 * 3 + a]));
      lo[a] = f < lo[a] ? f : lo[a];
      hi[a] = f > hi[a] ? f : hi[a];
    }
  }
  __shared__ double sm[6][256];
#pragma unroll
  for (int a = 0; a < 3; ++a) { sm[2 * a][threadIdx.x] = lo[a]; sm[2 * a + 1][threadIdx.x] = hi[a]; }
  __syncthreads();
  for (int s = blockDim.x >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        const double l = sm[2 * a][threadIdx.x + s], h = sm[2 * a + 1][threadIdx.x + s];
        if (l < sm[2 * a][threadIdx.x]) sm[2 * a][threadIdx.x] = l;
        if (h > sm[2 * a + 1][threadIdx.x]) sm[2 * a + 1][threadIdx.x] = h;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x < 6) lohi[6 * (size_t)b + threadIdx.x] = sm[threadIdx.x][0];
}

// bin key per atom (bin_off[b] + local bin) + wrapped cartesian position + structure index
static __global__ void nl_bin_kernel(const NLGrid* __restrict__ grids, const int* __restrict__ atom_ptr,
                                     const int* __restrict__ bin_off, int B, const double* __restrict__ pos, int n,
                                     int* __restrict__ key, int* __restrict__ idx, double* __restrict__ wrapped,
                                     int* __restrict__ sys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int sb = nl_system_of(atom_ptr, B, i);
  const NLGrid g = grids[sb];
  const double p[3] = {pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]};
  double f[3];
  nl_frac(g, p, f);
  int b[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (g.pbc[a]) f[a] -= floor(f[a]);
    int q = (int)floor((f[a] - g.fmin[a]) / g.fspan[a] * g.nb[a]);
    b[a] = q < 0 ? 0 : (q >= g.nb[a] ? g.nb[a] - 1 : q);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) wrapped[3 * i + c] = f[0] * g.cell[0 * 3 + c] + f[1] * g.cell[1 * 3 + c] + f[2] * g.cell[2 * 3 + c];
  key[i] = bin_off[sb] + (b[0] * g.nb[1] + b[1]) * g.nb[2] + b[2];
  idx[i] = i;
  sys[i] = sb;
}

// first sorted position of every bin (bin_start[nbins] = n)
static __global__ void nl_bin_start_kernel(const int* __restrict__ key_sorted, int n, int nbins, int* __restrict__ bin_start) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n) return;
  const int prev = (s == 0) ? -1 : key_sorted[s - 1];
  const int cur = (s == n) ? nbins : key_sorted[s];
  for (int b = prev + 1; b <= cur; ++b) bin_start[b] = s;
}

// Lattice set-up from the rows in g.cell: g.inv and height[a], the spacing of the lattice planes of direction a.
// Non-zero when the cell is singular.
inline int nl_lattice(NLGrid& g, double height[3]) {
  const double* m = g.cell;
  const double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
  if (fabs(det) < 1e-12) return 1;
  const double id = 1.0 / det;
  g.inv[0] = (m[4] * m[8] - m[5] * m[7]) * id; g.inv[1] = (m[2] * m[7] - m[1] * m[8]) * id; g.inv[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  g.inv[3] = (m[5] * m[6] - m[3] * m[8]) * id; g.inv[4] = (m[0] * m[8] - m[2] * m[6]) * id; g.inv[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  g.inv[6] = (m[3] * m[7] - m[4] * m[6]) * id; g.inv[7] = (m[1] * m[6] - m[0] * m[7]) * id; g.inv[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  for (int a = 0; a < 3; ++a)        // |column a of inv| = 1 / height_a
    height[a] = 1.0 / sqrt(g.inv[a] * g.inv[a] + g.inv[3 + a] * g.inv[3 + a] + g.inv[6 + a] * g.inv[6 + a]);
  return 0;
}

// Device arrays of the binning of a batch's n > 0 atoms (in: grids, atom_ptr, bin_off, pos; out: the rest).
struct NLBinArgs {
  const NLGrid* grids;
  const int *atom_ptr, *bin_off;
  const double* pos;
  int B, n;
  long long nbins;
  int *key, *idx, *key_sorted, *idx_sorted, *sys, *bin_start;
  double* wrapped;
};

// Bin keys, one stable radix sort over the bits the keys use, and bin_start.  Sizes the cub workspace `tmp` (the
// caller's buffer type) to the larger of the sort's need and tmp_other, what the caller runs from it afterwards;
// reports a failed allocation through the caller's `fail` and adds its launches to *launches (nullptr: not counted).
template <class Buf>
int nl_bin_sort(const NLBinArgs& a, Buf& tmp, size_t tmp_other, int (*fail)(const std::string&), int64_t* launches, cudaStream_t st) {
  nl_bin_kernel<<<(a.n + 127) / 128, 128, 0, st>>>(a.grids, a.atom_ptr, a.bin_off, a.B, a.pos, a.n, a.key, a.idx, a.wrapped, a.sys);
  S7B_CUDA_CHECK(cudaGetLastError());
  int end_bit = 1;                   // keys are < nbins
  while ((1LL << end_bit) < a.nbins) ++end_bit;
  size_t tmp_sort = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, a.key, a.key_sorted, a.idx, a.idx_sorted, a.n, 0, end_bit, st);
  if (tmp.ensure((tmp_sort > tmp_other ? tmp_sort : tmp_other) + 256)) return fail("cudaMalloc failed for cub workspace");
  size_t bytes = tmp.bytes;
  S7B_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, a.key, a.key_sorted, a.idx, a.idx_sorted, a.n, 0, end_bit, st));
  nl_bin_start_kernel<<<(a.n + 1 + 255) / 256, 256, 0, st>>>(a.key_sorted, a.n, (int)a.nbins, a.bin_start);
  if (launches) *launches += 3;
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// One thread per centre atom (centre c = centres[tid], or tid itself when centres == nullptr; original
// numbering).  FILL = false: count[tid] = neighbours; FILL = true: write src / edge_vec at rowptr[tid] +
// running offset.  A centre subset is what a rank of the multi-GPU runner asks for: the rows of its own atoms.
// Only the centre's own structure's bins are visited, so a batch has no cross-structure edges.
template <bool FILL>
__global__ void nl_pairs_kernel(const NLGrid* __restrict__ grids, const int* __restrict__ bin_off,
                                const int* __restrict__ sys, const double* __restrict__ wrapped,
                                const int* __restrict__ key, const int* __restrict__ idx_sorted,
                                const int* __restrict__ bin_start, int n, int* __restrict__ count,
                                const int* __restrict__ rowptr, int* __restrict__ src, float* __restrict__ edge_vec,
                                const int* __restrict__ centres = nullptr) {
  const int tid = blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= n) return;
  const int i = centres != nullptr ? centres[tid] : tid;
  const int sb = sys[i];
  const NLGrid g = grids[sb];
  const int boff = bin_off[sb];
  const double xi = wrapped[3 * i], yi = wrapped[3 * i + 1], zi = wrapped[3 * i + 2];
  const int k = key[i] - boff;
  const int b2 = k % g.nb[2], b1 = (k / g.nb[2]) % g.nb[1], b0 = k / (g.nb[2] * g.nb[1]);
  int out = FILL ? rowptr[tid] : 0;
  for (int d0 = -g.R[0]; d0 <= g.R[0]; ++d0) {
    int q0 = b0 + d0, s0 = 0;
    if (g.pbc[0]) { s0 = (q0 >= 0) ? q0 / g.nb[0] : -((-q0 + g.nb[0] - 1) / g.nb[0]); q0 -= s0 * g.nb[0]; }
    else if (q0 < 0 || q0 >= g.nb[0]) continue;
    for (int d1 = -g.R[1]; d1 <= g.R[1]; ++d1) {
      int q1 = b1 + d1, s1 = 0;
      if (g.pbc[1]) { s1 = (q1 >= 0) ? q1 / g.nb[1] : -((-q1 + g.nb[1] - 1) / g.nb[1]); q1 -= s1 * g.nb[1]; }
      else if (q1 < 0 || q1 >= g.nb[1]) continue;
      for (int d2 = -g.R[2]; d2 <= g.R[2]; ++d2) {
        int q2 = b2 + d2, s2 = 0;
        if (g.pbc[2]) { s2 = (q2 >= 0) ? q2 / g.nb[2] : -((-q2 + g.nb[2] - 1) / g.nb[2]); q2 -= s2 * g.nb[2]; }
        else if (q2 < 0 || q2 >= g.nb[2]) continue;
        const double sx = s0 * g.cell[0] + s1 * g.cell[3] + s2 * g.cell[6];
        const double sy = s0 * g.cell[1] + s1 * g.cell[4] + s2 * g.cell[7];
        const double sz = s0 * g.cell[2] + s1 * g.cell[5] + s2 * g.cell[8];
        const int nbin = boff + (q0 * g.nb[1] + q1) * g.nb[2] + q2;
        const bool same_image = (s0 == 0 && s1 == 0 && s2 == 0);
        for (int s = bin_start[nbin]; s < bin_start[nbin + 1]; ++s) {
          const int j = idx_sorted[s];
          if (same_image && j == i) continue;
          const double dx = wrapped[3 * j] + sx - xi, dy = wrapped[3 * j + 1] + sy - yi, dz = wrapped[3 * j + 2] + sz - zi;
          if (dx * dx + dy * dy + dz * dz < g.cutoff2) {
            if (FILL) {
              src[out] = j;
              edge_vec[3 * (size_t)out] = (float)dx;
              edge_vec[3 * (size_t)out + 1] = (float)dy;
              edge_vec[3 * (size_t)out + 2] = (float)dz;
            }
            ++out;
          }
        }
      }
    }
  }
  if (!FILL) count[tid] = out;
}

// Per-structure results of a batch, one block per structure, in a fixed order (deterministic): energy[b] = sum
// of the fp64 per-atom energies of [atom_ptr[b], atom_ptr[b+1]); virial[b] = -sum over the structure's edges
// [rowptr[atom_ptr[b]], rowptr[atom_ptr[b+1]]) of (r_x f_x, r_y f_y, r_z f_z, r_x f_y, r_y f_z, r_z f_x), each
// product in double.  The edges of a structure are contiguous: the CSR is by centre and structures are
// contiguous atom ranges.
constexpr int kSysBlock = 256;
static __global__ void __launch_bounds__(kSysBlock) system_sums_kernel(
    const int* __restrict__ atom_ptr, const int* __restrict__ rowptr, const double* __restrict__ atomic_energy,
    const float* __restrict__ edge_vec, const float* __restrict__ fedge, double* __restrict__ energy,
    double* __restrict__ virial) {
  const int b = blockIdx.x;
  const int a0 = atom_ptr[b], a1 = atom_ptr[b + 1];
  const int e0 = rowptr[a0], e1 = rowptr[a1];
  double v[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int i = a0 + threadIdx.x; i < a1; i += kSysBlock) v[0] += atomic_energy[i];
  for (int k = e0 + threadIdx.x; k < e1; k += kSysBlock) {
    const double rx = edge_vec[3 * (size_t)k], ry = edge_vec[3 * (size_t)k + 1], rz = edge_vec[3 * (size_t)k + 2];
    const double fx = fedge[3 * (size_t)k], fy = fedge[3 * (size_t)k + 1], fz = fedge[3 * (size_t)k + 2];
    v[1] += rx * fx; v[2] += ry * fy; v[3] += rz * fz;
    v[4] += rx * fy; v[5] += ry * fz; v[6] += rz * fx;
  }
  __shared__ double sm[7][kSysBlock];
#pragma unroll
  for (int q = 0; q < 7; ++q) sm[q][threadIdx.x] = v[q];
  __syncthreads();
  for (int s = kSysBlock >> 1; s > 0; s >>= 1) {
    if (threadIdx.x < s)
#pragma unroll
      for (int q = 0; q < 7; ++q) sm[q][threadIdx.x] += sm[q][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) energy[b] = sm[0][0];
  if (threadIdx.x < 6) virial[6 * (size_t)b + threadIdx.x] = -sm[1 + threadIdx.x][0];
}

}  // namespace s7b
