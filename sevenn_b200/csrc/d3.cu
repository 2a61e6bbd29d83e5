// Host side of the D3 dispersion C ABI (include/sevenn_b200.h, "D3" section): parameters, cell list, the set-up of
// one structure (host arrays) or of a batch (device arrays, s7b_d3_set_system_batch), stage launches, per-structure
// results, the Hessian-vector product (s7b_d3_hvp_strain), the heat flux (s7b_d3_heat_flux, or by range passes), the
// per-atom centroid virial (s7b_d3_centroid_virial, or by range passes) and the reference-named entry points
// (pair_init ... pair_fin) that sevenn/calculator.py:430-483 binds with ctypes.  Kernels: d3_kernels.cuh,
// d3_hvp_kernels.cuh, d3_flux_kernels.cuh, d3_centroid_kernels.cuh.
#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/sevenn_b200.h"
#include "common.cuh"
#include "d3_centroid_kernels.cuh"
#include "d3_flux_kernels.cuh"
#include "d3_hvp_kernels.cuh"
#include "d3_kernels.cuh"

namespace s7b {
static int d3_fail(const std::string& m) {
  set_error(__FILE__, 0, m.c_str());
  return 1;
}

struct D3Buf {
  void* p = nullptr;
  size_t bytes = 0;
  int ensure(size_t need) {
    if (need <= bytes) return 0;
    if (p) cudaFree(p);
    p = nullptr;
    bytes = 0;
    if (cudaMalloc(&p, need + need / 8 + 256) != cudaSuccess) { cudaGetLastError(); return 1; }
    bytes = need + need / 8 + 256;
    return 0;
  }
  void release() { if (p) cudaFree(p); p = nullptr; bytes = 0; }
  template <class T> T* as() const { return reinterpret_cast<T*>(p); }
};
}  // namespace s7b

using namespace s7b;

struct S7bD3 {
  D3Params P;                  // tables of s7b_d3_set_params: rows = the system's types
  D3Params Pe;                 // tables of s7b_d3_set_element_tables: rows = Z - 1
  bool have_params = false, have_elements = false, have_damping = false, have_system = false;
  bool batched = false;        // the current system came from s7b_d3_set_system_batch (element tables)
  int n = 0, B = 0;
  NLGrid grid1{};              // one structure: its grid and radii, passed to the kernels as parameters
  int3 R1_vdw{}, R1_cn{};
  D3Buf r0ab, c6ref, cnref, mxc, el_r0ab, el_c6ref, el_cnref, el_mxc;
  // set-up scratch: written before a set-up's checks have passed, so a refused set-up leaves the current system intact
  D3Buf pin, pos, wrapped, type, key, key_sorted, idx, tmp, sys, present, lrank, err, st_grids, st_aptr, st_lrows, st_nloc;
  // the current system; grids / aptr / lrows / nloc are swapped in from their st_ scratch once the checks have passed
  D3Buf grids, aptr, lrows, nloc, bin_off, rtab, idx_sorted, bin_start;
  D3Buf xs, ts, ss, bin_of, W, dW, logD, near_, cn, dc6i, force, eatom, spair, schain, energy, sigma, out_force;
  // the forward: stages 1..fw_stage run in order over one atom range [fw_lo, fw_hi) since the current system, tables
  // and damping were set (fw_stage 0..3).  The Hessian-vector product and the one-shot flux and centroid virial read
  // cn, W, dW and dc6i of all atoms and need 3 over [0, n); the range passes need 3 over a range containing theirs
  int fw_stage = 0, fw_lo = 0, fw_hi = 0;
  // the range passes run since the last forward stage: 0 none, 1 pass 1 over [lo, hi), 2 then pass 2 inside it
  int fx_pass = 0, fx_lo = 0, fx_hi = 0, ct_pass = 0, ct_lo = 0, ct_hi = 0;
  // Hessian-vector product scratch, allocated on its first call
  D3Buf hv_v, hv_dcn, hv_dWt, hv_dW1t, hv_ddc, hv_force, hv_spair, hv_schain, hv_sigma, hv_energy, hv_oute, hv_dvir;
  // heat-flux scratch, allocated on its first call
  D3Buf fx_v, fx_cn4, fx_nb, fx_out, fx_energy, fx_sums;
  // centroid-virial scratch, allocated on its first call
  D3Buf ct_beta, ct_nb, ct_out;
  std::vector<double> host_force;      // reference ABI: pair_get_force returns a pointer
  double host_energy = 0.0, host_sigma[6] = {0, 0, 0, 0, 0, 0};
  // reference-ABI staging (pair_set_atom / pair_set_domain / pair_run_settings / pair_run_coeff)
  std::vector<int> ref_types;
  std::vector<double> ref_pos;
  double ref_cell[9] = {0}, ref_rthr = 9000.0, ref_cnthr = 1600.0;
  int ref_pbc[3] = {1, 1, 1}, ref_ntypes = 0;
  std::string ref_damp = "damp_bj", ref_func = "pbe";
};

static bool d3_full_forward(const S7bD3* d) { return d->fw_stage == 3 && d->fw_lo == 0 && d->fw_hi == d->n; }

static D3Atoms d3_atoms(const S7bD3* d) {
  D3Atoms A;
  A.x = d->xs.as<double>();
  A.type = d->ts.as<int>();
  A.sys = d->ss.as<int>();
  A.W = d->W.as<float>();
  A.logD = d->logD.as<float>();
  A.near = d->near_.as<int>();
  A.dc6i = d->dc6i.as<double>();
  A.bin_start = d->bin_start.as<int>();
  A.bin_of = d->bin_of.as<int>();
  A.grids = d->grids.as<NLGrid>();
  A.bin_off = d->bin_off.as<int>();
  A.R = d->rtab.as<int>();
  A.lrows = d->lrows.as<int>();
  A.nloc = d->nloc.as<int>();
  return A;
}
static D3Out d3_out(const S7bD3* d) {
  D3Out o;
  o.cn = d->cn.as<double>();
  o.dc6i = d->dc6i.as<double>();
  o.force = d->force.as<double>();
  o.eatom = d->eatom.as<double>();
  o.spair = d->spair.as<double>();
  o.schain = d->schain.as<double>();
  return o;
}

// float tables on the device, r0ab converted from Angstrom to bohr (:326-337); rcov / r2r4 by value in P
static int d3_upload_tables(D3Params& P, int nrows, const double* rcov, const double* r2r4, const double* r0ab,
                            const double* c6ref, const double* cnref, const int32_t* mxc, D3Buf& d_r0ab, D3Buf& d_c6ref,
                            D3Buf& d_cnref, D3Buf& d_mxc) {
  std::vector<float> f0((size_t)nrows * nrows), fc((size_t)nrows * nrows * 25), fr((size_t)nrows * 5);
  for (int t = 0; t < nrows; ++t) { P.rcov[t] = (float)rcov[t]; P.r2r4[t] = (float)r2r4[t]; }
  for (size_t k = 0; k < f0.size(); ++k) f0[k] = (float)(r0ab[k] / kAuToAng);
  for (size_t k = 0; k < fc.size(); ++k) fc[k] = (float)c6ref[k];
  for (size_t k = 0; k < fr.size(); ++k) fr[k] = (float)cnref[k];
  if (d_r0ab.ensure(f0.size() * 4) || d_c6ref.ensure(fc.size() * 4) || d_cnref.ensure(fr.size() * 4) || d_mxc.ensure(nrows * 4))
    return d3_fail("cudaMalloc failed for the D3 tables");
  S7B_CUDA_CHECK(cudaMemcpy(d_r0ab.p, f0.data(), f0.size() * 4, cudaMemcpyHostToDevice));
  S7B_CUDA_CHECK(cudaMemcpy(d_c6ref.p, fc.data(), fc.size() * 4, cudaMemcpyHostToDevice));
  S7B_CUDA_CHECK(cudaMemcpy(d_cnref.p, fr.data(), fr.size() * 4, cudaMemcpyHostToDevice));
  S7B_CUDA_CHECK(cudaMemcpy(d_mxc.p, mxc, nrows * 4, cudaMemcpyHostToDevice));
  P.nrows = nrows;
  P.r0ab = d_r0ab.as<float>();
  P.c6ref = d_c6ref.as<float>();
  return 0;
}

extern "C" {

int s7b_d3_create(S7bD3** out) {
  if (!out) return d3_fail("null argument");
  *out = new S7bD3();
  memset(&(*out)->P, 0, sizeof(D3Params));
  memset(&(*out)->Pe, 0, sizeof(D3Params));
  return 0;
}

void s7b_d3_destroy(S7bD3* d) {
  if (!d) return;
  D3Buf* bufs[] = {&d->r0ab, &d->c6ref, &d->cnref, &d->mxc, &d->el_r0ab, &d->el_c6ref, &d->el_cnref, &d->el_mxc,
                   &d->pin, &d->pos, &d->wrapped, &d->type, &d->key, &d->key_sorted, &d->idx, &d->tmp, &d->sys,
                   &d->present, &d->lrank, &d->err, &d->st_grids, &d->st_aptr, &d->st_lrows, &d->st_nloc,
                   &d->grids, &d->aptr, &d->lrows, &d->nloc, &d->bin_off, &d->rtab, &d->idx_sorted, &d->bin_start,
                   &d->xs, &d->ts, &d->ss, &d->bin_of, &d->W, &d->dW, &d->logD, &d->near_, &d->cn, &d->dc6i,
                   &d->force, &d->eatom, &d->spair, &d->schain, &d->energy, &d->sigma, &d->out_force,
                   &d->hv_v, &d->hv_dcn, &d->hv_dWt, &d->hv_dW1t, &d->hv_ddc, &d->hv_force, &d->hv_spair,
                   &d->hv_schain, &d->hv_sigma, &d->hv_energy, &d->hv_oute, &d->hv_dvir,
                   &d->fx_v, &d->fx_cn4, &d->fx_nb, &d->fx_out, &d->fx_energy, &d->fx_sums,
                   &d->ct_beta, &d->ct_nb, &d->ct_out};
  for (D3Buf* b : bufs) b->release();
  delete d;
}

int s7b_d3_set_params(S7bD3* d, int32_t ntypes, const double* rcov, const double* r2r4, const double* r0ab,
                      const double* c6ref, const double* cnref, const int32_t* mxc) {
  if (!d || !rcov || !r2r4 || !r0ab || !c6ref || !cnref || !mxc) return d3_fail("null argument");
  if (ntypes < 1 || ntypes > kD3MaxTypes) return d3_fail("D3: 1.." + std::to_string(kD3MaxTypes) + " atom types are supported");
  if (d3_upload_tables(d->P, ntypes, rcov, r2r4, r0ab, c6ref, cnref, mxc, d->r0ab, d->c6ref, d->cnref, d->mxc)) return 1;
  d->have_params = true;
  d->fw_stage = d->fx_pass = d->ct_pass = 0;
  return 0;
}

int s7b_d3_set_element_tables(S7bD3* d, const double* rcov, const double* r2r4, const double* r0ab, const double* c6ref,
                              const double* cnref, const int32_t* mxc) {
  if (!d || !rcov || !r2r4 || !r0ab || !c6ref || !cnref || !mxc) return d3_fail("null argument");
  if (d3_upload_tables(d->Pe, kD3Elements, rcov, r2r4, r0ab, c6ref, cnref, mxc, d->el_r0ab, d->el_c6ref, d->el_cnref, d->el_mxc))
    return 1;
  d->have_elements = true;
  d->fw_stage = d->fx_pass = d->ct_pass = 0;
  return 0;
}

int s7b_d3_set_damping(S7bD3* d, int32_t damping, double s6, double s8, double a1, double a2, double alp6, double alp8,
                       double vdw_cutoff_au2, double cn_cutoff_au2) {
  if (!d) return d3_fail("null argument");
  if (damping != 0 && damping != 1) return d3_fail("D3 damping must be 0 (zero) or 1 (Becke-Johnson)");
  if (!(vdw_cutoff_au2 > 0) || !(cn_cutoff_au2 > 0)) return d3_fail("D3 cutoffs must be positive");
  for (D3Params* P : {&d->P, &d->Pe}) {
    P->damping = damping;
    P->s6 = (float)s6; P->s8 = (float)s8; P->a1 = (float)a1; P->a2 = (float)a2;
    P->alp6 = (float)alp6; P->alp8 = (float)alp8;
    P->rthr = (double)(float)vdw_cutoff_au2;      // the reference compares float r^2 with float thresholds
    P->cnthr = (double)(float)cn_cutoff_au2;
  }
  d->have_damping = true;
  d->fw_stage = d->fx_pass = d->ct_pass = 0;
  return 0;
}

}  // extern "C"

// Cell-list grid of one structure (cell rows in Angstrom -> bohr, then nl_lattice) with D3's bin policy: bins of
// ~6 A (1..128 per direction) and the search radii in bins R[0..2] = R_vdw, R[3..5] = R_cn.  Non-zero when the
// cell is singular.
static int d3_grid(const double* cell9, const int32_t* pbc3, double rthr, double cnthr, NLGrid& g, int* R) {
  memset(&g, 0, sizeof(g));
  for (int k = 0; k < 9; ++k) g.cell[k] = cell9[k] / kAuToAng;
  double height[3];
  if (nl_lattice(g, height)) return 1;
  for (int a = 0; a < 3; ++a) { g.pbc[a] = pbc3[a] ? 1 : 0; g.fmin[a] = 0.0; g.fspan[a] = 1.0; }
  g.cutoff2 = rthr;
  const double w_target = 6.0 / kAuToAng;           // ~10 atoms per bin in a dense solid
  const double rc_v = sqrt(rthr), rc_c = sqrt(cnthr);
  for (int a = 0; a < 3; ++a) {
    int nb = (int)floor(height[a] / w_target);
    nb = std::max(1, std::min(nb, 128));
    g.nb[a] = nb;
    const double w = height[a] / nb;
    int Rv = (int)ceil(rc_v / w - 1e-12), Rc = (int)ceil(rc_c / w - 1e-12);
    if (!g.pbc[a]) { Rv = std::min(Rv, nb - 1); Rc = std::min(Rc, nb - 1); }
    g.R[a] = Rv;
    R[a] = Rv;
    R[3 + a] = Rc;
  }
  return 0;
}

// Set-up of B structures whose grids / radii the host has computed.  Single structure (h_types, h_pos: host types and
// positions): the types are the table rows and the local types.  Batch (d_numbers, d_pos: device atomic numbers and
// positions): rows and local types are derived on the device and checked, with one readback.  Positions in Angstrom.
static int d3_setup(S7bD3* d, int B, const int32_t* atom_ptr, const std::vector<NLGrid>& grids, const std::vector<int>& R,
                    const int32_t* h_types, const double* h_pos, const int32_t* d_numbers, const double* d_pos,
                    cudaStream_t st) {
  const int n = atom_ptr[B];
  const size_t N = (size_t)std::max(n, 1), Bs = (size_t)B;
  const bool batch = d_numbers != nullptr;
  int rc = 0;
  rc |= d->pin.ensure(N * 24); rc |= d->pos.ensure(N * 24); rc |= d->wrapped.ensure(N * 24); rc |= d->type.ensure(N * 4);
  rc |= d->key.ensure(N * 4); rc |= d->key_sorted.ensure(N * 4); rc |= d->idx.ensure(N * 4); rc |= d->sys.ensure(N * 4);
  rc |= d->present.ensure(Bs * kD3Elements * 4); rc |= d->lrank.ensure(Bs * kD3Elements * 4); rc |= d->err.ensure(8);
  rc |= d->st_grids.ensure(Bs * sizeof(NLGrid)); rc |= d->st_aptr.ensure((Bs + 1) * 4);
  rc |= d->st_lrows.ensure(Bs * kD3MaxTypes * 4); rc |= d->st_nloc.ensure(Bs * 4);
  if (rc) return d3_fail("cudaMalloc failed for the D3 system");
  S7B_CUDA_CHECK(cudaMemcpyAsync(d->st_grids.p, grids.data(), Bs * sizeof(NLGrid), cudaMemcpyHostToDevice, st));
  S7B_CUDA_CHECK(cudaMemcpyAsync(d->st_aptr.p, atom_ptr, (Bs + 1) * 4, cudaMemcpyHostToDevice, st));
  if (!batch) {
    if (n > 0) {
      S7B_CUDA_CHECK(cudaMemcpyAsync(d->pin.p, h_pos, (size_t)n * 24, cudaMemcpyHostToDevice, st));
      S7B_CUDA_CHECK(cudaMemcpyAsync(d->type.p, h_types, (size_t)n * 4, cudaMemcpyHostToDevice, st));
    }
    int lrows[kD3MaxTypes] = {0}, nloc = d->P.nrows;
    for (int t = 0; t < nloc; ++t) lrows[t] = t;
    S7B_CUDA_CHECK(cudaMemcpyAsync(d->st_lrows.p, lrows, sizeof(lrows), cudaMemcpyHostToDevice, st));
    S7B_CUDA_CHECK(cudaMemcpyAsync(d->st_nloc.p, &nloc, 4, cudaMemcpyHostToDevice, st));
    d_pos = d->pin.as<double>();
  } else {
    S7B_CUDA_CHECK(cudaMemsetAsync(d->present.p, 0, Bs * kD3Elements * 4, st));
    S7B_CUDA_CHECK(cudaMemsetAsync(d->err.p, 0x7f, 8, st));         // 0x7f7f7f7f: no structure
  }
  if (n > 0) {
    d3_prepare_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, B, d->st_aptr.as<int>(), d->st_grids.as<NLGrid>(), d_pos, d_numbers,
                                                       d->pos.as<double>(), d->type.as<int>(), d->present.as<int>(), d->err.as<int>());
    S7B_CUDA_CHECK(cudaGetLastError());
  }
  if (batch) {
    d3_local_types_kernel<<<(B + 127) / 128, 128, 0, st>>>(B, d->present.as<int>(), d->lrank.as<int>(), d->st_lrows.as<int>(),
                                                           d->st_nloc.as<int>(), d->err.as<int>());
    S7B_CUDA_CHECK(cudaGetLastError());
    int err[2];
    S7B_CUDA_CHECK(cudaMemcpyAsync(err, d->err.p, 8, cudaMemcpyDeviceToHost, st));
    S7B_CUDA_CHECK(cudaStreamSynchronize(st));
    if (err[0] < B) return d3_fail("D3: structure " + std::to_string(err[0]) + " has an atomic number outside 1..94");
    if (err[1] < B)
      return d3_fail("D3: structure " + std::to_string(err[1]) + " has more than " + std::to_string(kD3MaxTypes) +
                     " elements (at most " + std::to_string(kD3MaxTypes) + " per structure are supported)");
  }
  // the checks have passed: from here on the set-up replaces the current system
  std::vector<int> bin_off(Bs + 1, 0);
  long long nbins = 0;
  for (int b = 0; b < B; ++b) {
    nbins += (long long)grids[b].nb[0] * grids[b].nb[1] * grids[b].nb[2];
    if (nbins > (1LL << 30)) return d3_fail("D3: cell-list grids of the batch too large (more than 2^30 bins in all)");
    bin_off[b + 1] = (int)nbins;
  }
  std::swap(d->grids, d->st_grids);
  std::swap(d->aptr, d->st_aptr);
  std::swap(d->lrows, d->st_lrows);
  std::swap(d->nloc, d->st_nloc);
  d->have_system = false;
  d->fw_stage = d->fx_pass = d->ct_pass = 0;
  rc = 0;
  rc |= d->bin_off.ensure((Bs + 1) * 4); rc |= d->rtab.ensure(Bs * 24); rc |= d->idx_sorted.ensure(N * 4);
  rc |= d->bin_start.ensure(((size_t)nbins + 1) * 4);
  rc |= d->xs.ensure(N * 24); rc |= d->ts.ensure(N * 4); rc |= d->ss.ensure(N * 4); rc |= d->bin_of.ensure(N * 4);
  rc |= d->W.ensure(N * 20); rc |= d->dW.ensure(N * 20); rc |= d->logD.ensure(N * 4); rc |= d->near_.ensure(N * 4);
  rc |= d->cn.ensure(N * 8); rc |= d->dc6i.ensure(N * 8); rc |= d->force.ensure(N * 24); rc |= d->out_force.ensure(N * 24);
  rc |= d->eatom.ensure(N * 8); rc |= d->spair.ensure(N * 48); rc |= d->schain.ensure(N * 48);
  rc |= d->energy.ensure(Bs * 8); rc |= d->sigma.ensure(Bs * 48);
  if (rc) return d3_fail("cudaMalloc failed for the D3 system");
  S7B_CUDA_CHECK(cudaMemcpyAsync(d->bin_off.p, bin_off.data(), (Bs + 1) * 4, cudaMemcpyHostToDevice, st));
  S7B_CUDA_CHECK(cudaMemcpyAsync(d->rtab.p, R.data(), Bs * 24, cudaMemcpyHostToDevice, st));
  if (n > 0) {
    // the binning of the model's neighbour list, uncounted (the D3 entry points do not feed the engine's launch count)
    const NLBinArgs bins{d->grids.as<NLGrid>(), d->aptr.as<int>(), d->bin_off.as<int>(), d->pos.as<double>(), B, n, nbins, d->key.as<int>(),
                         d->idx.as<int>(), d->key_sorted.as<int>(), d->idx_sorted.as<int>(), d->sys.as<int>(), d->bin_start.as<int>(), d->wrapped.as<double>()};
    if (nl_bin_sort(bins, d->tmp, 0, d3_fail, nullptr, st)) return 1;
    d3_sort_gather_kernel<<<(n + 255) / 256, 256, 0, st>>>(n, d->idx_sorted.as<int>(), d->key_sorted.as<int>(), d->wrapped.as<double>(),
                                                          d->type.as<int>(), d->sys.as<int>(), batch ? d->lrank.as<int>() : nullptr,
                                                          d->xs.as<double>(), d->ts.as<int>(), d->ss.as<int>(), d->bin_of.as<int>());
    S7B_CUDA_CHECK(cudaGetLastError());
  }
  d->grid1 = grids[0];
  d->R1_vdw = make_int3(R[0], R[1], R[2]);
  d->R1_cn = make_int3(R[3], R[4], R[5]);
  d->n = n;
  d->B = B;
  d->batched = batch;
  d->have_system = true;
  return 0;
}

extern "C" {

// positions [n,3] and cell rows in Angstrom; types 0-based indices into the tables of set_params
int s7b_d3_set_system(S7bD3* d, int32_t n, const int32_t* types, const double* positions, const double* cell9,
                      const int32_t* pbc3, void* stream) {
  if (!d || !types || !positions || !cell9 || !pbc3) return d3_fail("null argument");
  if (!d->have_params || !d->have_damping) return d3_fail("D3: set_params and set_damping come first");
  if (n < 1) return d3_fail("D3 needs at least one atom");
  std::vector<NLGrid> g(1);
  std::vector<int> R(6);
  if (d3_grid(cell9, pbc3, d->P.rthr, d->P.cnthr, g[0], R.data())) return d3_fail("D3 requires a cell (non-singular lattice vectors)");
  for (int i = 0; i < n; ++i)
    if (types[i] < 0 || types[i] >= d->P.nrows) return d3_fail("D3: atom type out of range");
  const int32_t atom_ptr[2] = {0, n};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d3_setup(d, 1, atom_ptr, g, R, types, positions, nullptr, nullptr, st)) return 1;
  S7B_CUDA_CHECK(cudaStreamSynchronize(st));     // the caller may reuse `types` / `positions` on return
  return 0;
}

// B structures from device-resident atomic numbers / positions (Angstrom); atom_ptr [B+1], cells [B,9] (rows) and
// pbc [B,3] on the host.  Empty structures are allowed (their cell is not used).
int s7b_d3_set_system_batch(S7bD3* d, int32_t B, const int32_t* atom_ptr, const int32_t* d_numbers, const double* d_positions,
                            const double* cells9, const int32_t* pbc3, void* stream) {
  if (!d || !atom_ptr || !cells9 || !pbc3) return d3_fail("null argument");
  if (!d->have_elements || !d->have_damping) return d3_fail("D3: set_element_tables and set_damping come first");
  if (B < 1) return d3_fail("D3: a batch needs at least one structure");
  if (atom_ptr[0] != 0) return d3_fail("D3: atom_ptr[0] must be 0");
  for (int b = 0; b < B; ++b)
    if (atom_ptr[b + 1] < atom_ptr[b]) return d3_fail("D3: atom_ptr decreases at structure " + std::to_string(b));
  if (atom_ptr[B] > 0 && (!d_numbers || !d_positions)) return d3_fail("null argument");
  std::vector<NLGrid> g((size_t)B);
  std::vector<int> R(6 * (size_t)B);
  static const double kUnit[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};       // an empty structure's grid is never swept
  for (int b = 0; b < B; ++b) {
    const bool empty = atom_ptr[b + 1] == atom_ptr[b];
    if (d3_grid(empty ? kUnit : cells9 + 9 * (size_t)b, pbc3 + 3 * (size_t)b, d->Pe.rthr, d->Pe.cnthr, g[b], &R[6 * (size_t)b]))
      return d3_fail("D3: structure " + std::to_string(b) + " has a singular cell (D3 requires non-singular lattice vectors)");
  }
  return d3_setup(d, B, atom_ptr, g, R, nullptr, nullptr, d_numbers, d_positions, reinterpret_cast<cudaStream_t>(stream));
}

// stage 1: coordination numbers of atoms [i_begin, i_end) (bin-sorted order);
// stage 2: reference weights of ALL atoms from cn[], then pair energy / forces / dE/dCN of the range; energy and
//          sigma become the range's pair sums (per structure);  stage 3: CN chain-rule forces of the range (needs
//          dc6i[] of all atoms), its virial added to sigma
int s7b_d3_run_stage(S7bD3* d, int32_t stage, int32_t i_begin, int32_t i_end, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (i_begin < 0 || i_end > d->n || i_begin > i_end) return d3_fail("D3: bad atom range");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n = d->n, cnt = i_end - i_begin;
  const int grd = (cnt + kD3WarpsPerBlock - 1) / kD3WarpsPerBlock, blk = 32 * kD3WarpsPerBlock;
  const D3Params& P = d->batched ? d->Pe : d->P;
  const D3Atoms A = d3_atoms(d);
  const D3Out O = d3_out(d);
  const bool bt = d->batched;
  if (stage == 1) {
    if (cnt > 0) {
      if (bt) d3_cn_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, O);
      else d3_cn_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, O);
    }
  } else if (stage == 2) {
    if (n > 0)
      d3_weights_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, d->ts.as<int>(), d->cn.as<double>(),
                                                        (bt ? d->el_cnref : d->cnref).as<float>(),
                                                        (bt ? d->el_mxc : d->mxc).as<int>(), d->W.as<float>(),
                                                        d->dW.as<float>(), d->logD.as<float>(), d->near_.as<int>());
    S7B_CUDA_CHECK(cudaMemsetAsync(d->force.p, 0, (size_t)n * 24, st));
    if (cnt > 0) {
      if (bt) d3_pair_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, i_begin, i_end, O);
      else d3_pair_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, i_begin, i_end, O);
    }
    d3_system_sums_kernel<<<d->B, kD3SumBlock, 0, st>>>(d->aptr.as<int>(), i_begin, i_end, d->eatom.as<double>(), d->spair.as<double>(),
                                                        d->energy.as<double>(), d->sigma.as<double>());
  } else if (stage == 3) {
    if (cnt > 0) {
      if (bt) d3_chain_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, O);
      else d3_chain_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, O);
    }
    d3_system_sums_kernel<<<d->B, kD3SumBlock, 0, st>>>(d->aptr.as<int>(), i_begin, i_end, nullptr, d->schain.as<double>(),
                                                        d->energy.as<double>(), d->sigma.as<double>());
  } else {
    return d3_fail("D3: unknown stage");
  }
  S7B_CUDA_CHECK(cudaGetLastError());
  if (stage == 1) { d->fw_lo = i_begin; d->fw_hi = i_end; }
  d->fw_stage = (stage == 1 || (stage <= d->fw_stage + 1 && i_begin == d->fw_lo && i_end == d->fw_hi)) ? stage : 0;
  d->fx_pass = d->ct_pass = 0;
  return 0;
}

// device buffers, bin-sorted atom order: "cn" double[n], "dc6i" double[n], "force" double[n,3] (hartree/bohr),
// "energy" double[B] (hartree), "sigma" double[B,6] (hartree; xx,yy,zz,xy,xz,yz), "order" int[n] (sorted -> caller index),
// "type" int[n] (type word: after a batched set-up Z - 1 | local type << 8, else the type index), "eatom" double[n]
// (hartree, the atomic energies of the pair pass); the records the range passes exchange: "ct_nb" float[n,4],
// "fx_nb" float[n,8], "ct_out" double[n,9] (eV), "fx_out" double[n,6] (null before the first pass of their kind)
void* s7b_d3_buffer(S7bD3* d, const char* name, size_t* numel) {
  if (!d || !name) return nullptr;
  const std::string nm(name);
  void* p = nullptr;
  size_t n = 0;
  if (nm == "cn") { p = d->cn.p; n = d->n; }
  else if (nm == "dc6i") { p = d->dc6i.p; n = d->n; }
  else if (nm == "force") { p = d->force.p; n = (size_t)d->n * 3; }
  else if (nm == "energy") { p = d->energy.p; n = d->B; }
  else if (nm == "sigma") { p = d->sigma.p; n = (size_t)d->B * 6; }
  else if (nm == "order") { p = d->idx_sorted.p; n = d->n; }
  else if (nm == "type") { p = d->ts.p; n = d->n; }
  else if (nm == "eatom") { p = d->eatom.p; n = d->n; }
  else if (nm == "ct_nb") { p = d->ct_nb.p; n = (size_t)d->n * 4; }
  else if (nm == "fx_nb") { p = d->fx_nb.p; n = (size_t)d->n * 8; }
  else if (nm == "ct_out") { p = d->ct_out.p; n = (size_t)d->n * 9; }
  else if (nm == "fx_out") { p = d->fx_out.p; n = (size_t)d->n * 6; }
  if (numel) *numel = n;
  return p;
}

// energy (eV), forces [n,3] (eV/A, caller's atom order), sigma6 (eV; xx,yy,zz,xy,xz,yz of sum f (x) r) -> host
int s7b_d3_results_host(S7bD3* d, double* energy, double* forces, double* sigma6, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (d->B != 1) return d3_fail("D3: the system is a batch; read its results with s7b_d3_system_results");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int n = d->n;
  d3_unsort_kernel<<<(n * 3 + 255) / 256, 256, 0, st>>>(n, 3, d->idx_sorted.as<int>(), d->force.as<double>(), kAuToEv / kAuToAng, d->out_force.as<double>());
  S7B_CUDA_CHECK(cudaGetLastError());
  double e = 0.0, s[6];
  S7B_CUDA_CHECK(cudaMemcpyAsync(&e, d->energy.p, 8, cudaMemcpyDeviceToHost, st));
  S7B_CUDA_CHECK(cudaMemcpyAsync(s, d->sigma.p, 48, cudaMemcpyDeviceToHost, st));
  if (forces) S7B_CUDA_CHECK(cudaMemcpyAsync(forces, d->out_force.p, (size_t)n * 24, cudaMemcpyDeviceToHost, st));
  S7B_CUDA_CHECK(cudaStreamSynchronize(st));
  if (energy) *energy = e * kAuToEv;
  if (sigma6) for (int q = 0; q < 6; ++q) sigma6[q] = s[q] * kAuToEv;
  return 0;
}

int s7b_d3_compute_host(S7bD3* d, double* energy, double* forces, double* sigma6, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  for (int stage = 1; stage <= 3; ++stage)
    if (s7b_d3_run_stage(d, stage, 0, d->n, stream)) return 1;
  return s7b_d3_results_host(d, energy, forces, sigma6, stream);
}

// after the three stages over [0, n): energy [B] (eV), forces [n,3] (eV/A, caller's atom order), virial [B,6] (eV;
// xx,yy,zz,xy,yz,zx of sum f (x) r), device pointers, no synchronisation
int s7b_d3_system_results(S7bD3* d, double* d_energy, double* d_forces, double* d_virial, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (!d_energy || !d_virial || (d->n > 0 && !d_forces)) return d3_fail("null output");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int threads = std::max(3 * d->n, d->B);
  d3_system_results_kernel<<<(threads + 255) / 256, 256, 0, st>>>(d->n, d->B, d->idx_sorted.as<int>(), d->force.as<double>(),
                                                                  d->energy.as<double>(), d->sigma.as<double>(), d_energy, d_forces, d_virial);
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// Along r -> (I + s eps_b) r + s v for the atoms and cell of every structure b, on the current system with its
// forward (stages 1-3 over [0, n)) held: out = H v + Lambda eps (eV/A^2 x A resp. eV/A, caller's atom order) and the
// virial's tangent [B, 6] (eV; xx,yy,zz,xy,yz,zx, the order and sign of s7b_engine_hvp_strain's).  Launches the four
// tangent passes and the forward's own sums and results kernels on scratch; no forward buffer is written.
int s7b_d3_hvp_strain(S7bD3* d, const double* d_v, const double* d_strain, double* d_out, double* d_dvirial, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (!d3_full_forward(d))
    return d3_fail("D3: the Hessian-vector product needs stages 1, 2 and 3 run over all atoms [0, n) of the current "
                   "system first");
  const int n = d->n, B = d->B;
  if (n > 0 && !d_out) return d3_fail("null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d_dvirial) S7B_CUDA_CHECK(cudaMemsetAsync(d_dvirial, 0, (size_t)B * 48, st));
  if (n == 0) return 0;
  if (!d_v && !d_strain) {
    S7B_CUDA_CHECK(cudaMemsetAsync(d_out, 0, (size_t)n * 24, st));
    return 0;
  }
  const size_t N = (size_t)n, Bs = (size_t)B;
  int rc = 0;
  rc |= d->hv_v.ensure(N * 24); rc |= d->hv_dcn.ensure(N * 8); rc |= d->hv_dWt.ensure(N * 20); rc |= d->hv_dW1t.ensure(N * 20);
  rc |= d->hv_ddc.ensure(N * 8); rc |= d->hv_force.ensure(N * 24); rc |= d->hv_spair.ensure(N * 48);
  rc |= d->hv_schain.ensure(N * 48); rc |= d->hv_sigma.ensure(Bs * 48); rc |= d->hv_energy.ensure(Bs * 8);
  rc |= d->hv_oute.ensure(Bs * 8); rc |= d->hv_dvir.ensure(Bs * 48);
  if (rc) return d3_fail("cudaMalloc failed for the D3 Hessian-vector product");
  const bool bt = d->batched;
  const D3Params& P = bt ? d->Pe : d->P;
  const D3Atoms A = d3_atoms(d);
  D3Hvp H;
  H.v = d->hv_v.as<double>();
  H.strain = d_strain;
  H.dcn = d->hv_dcn.as<double>();
  H.dWt = d->hv_dWt.as<float>();
  H.dW1t = d->hv_dW1t.as<float>();
  H.ddc = d->hv_ddc.as<double>();
  H.hforce = d->hv_force.as<double>();
  H.spair = d->hv_spair.as<double>();
  H.schain = d->hv_schain.as<double>();
  const int grd = (n + kD3WarpsPerBlock - 1) / kD3WarpsPerBlock, blk = 32 * kD3WarpsPerBlock;
  d3_hvp_gather_kernel<<<(3 * n + 255) / 256, 256, 0, st>>>(n, d->idx_sorted.as<int>(), d_v, d->hv_v.as<double>());
  if (bt) d3_hvp_cn_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, n, H);
  else d3_hvp_cn_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, n, H);
  d3_hvp_weights_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, d->ts.as<int>(), d->cn.as<double>(),
                                                        (bt ? d->el_cnref : d->cnref).as<float>(),
                                                        (bt ? d->el_mxc : d->mxc).as<int>(), H.dcn, H.dWt, H.dW1t);
  if (bt) d3_hvp_pair_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, n, H);
  else d3_hvp_pair_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, n, H);
  if (bt) d3_hvp_chain_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, n, H);
  else d3_hvp_chain_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, n, H);
  // per-structure virial tangent (the pair sum sets it, the chain sum adds; dcn stands in for the energy terms)
  d3_system_sums_kernel<<<B, kD3SumBlock, 0, st>>>(d->aptr.as<int>(), 0, n, H.dcn, H.spair, d->hv_energy.as<double>(),
                                                   d->hv_sigma.as<double>());
  d3_system_sums_kernel<<<B, kD3SumBlock, 0, st>>>(d->aptr.as<int>(), 0, n, nullptr, H.schain, d->hv_energy.as<double>(),
                                                   d->hv_sigma.as<double>());
  const int threads = std::max(3 * n, B);
  d3_system_results_kernel<<<(threads + 255) / 256, 256, 0, st>>>(n, B, d->idx_sorted.as<int>(), H.hforce,
                                                                  d->hv_energy.as<double>(), d->hv_sigma.as<double>(),
                                                                  d->hv_oute.as<double>(), d_out,
                                                                  d_dvirial ? d_dvirial : d->hv_dvir.as<double>());
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

}  // extern "C"

// ---- heat flux and centroid virial: two passes each, over an atom range of the bin-sorted order ---------------------
// Each pass is one warp per atom with no atomics and a fixed order, and reads of its centre the per-atom values a range
// forward leaves valid for its range (eatom, spair, dc6i) and its own pass-1 row, and of a neighbour only the packed
// float record of pass 1 (fx_nb, ct_nb) and what stage 2 computed for all atoms.  So the passes of several ranges,
// with the records gathered between them, write each row bit for bit as one pass over [0, n) does.

// refusals shared by the range passes; pass 2 also needs pass 1 of its kind (state 1 or 2) over a range containing its
static int d3_pass_check(const S7bD3* d, int pass, int i_begin, int i_end, int state, int lo, int hi, const char* what) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (pass != 1 && pass != 2) return d3_fail(std::string("D3: the ") + what + " has passes 1 and 2");
  if (d->fw_stage < 3)
    return d3_fail(std::string("D3: the ") + what + " pass needs stages 1, 2 and 3 run in order over one atom range "
                   "since the last set-up, table or damping change");
  if (i_begin < d->fw_lo || i_end > d->fw_hi || i_begin > i_end)
    return d3_fail(std::string("D3: the ") + what + " pass range [" + std::to_string(i_begin) + ", " +
                   std::to_string(i_end) + ") is not inside the forward's range [" + std::to_string(d->fw_lo) + ", " +
                   std::to_string(d->fw_hi) + ")");
  if (pass == 2 && (state < 1 || i_begin < lo || i_end > hi))
    return d3_fail(std::string("D3: the ") + what + " pass 2 needs pass 1 over a range containing its own since the "
                   "last forward stage");
  return 0;
}

static int d3_flux_scratch(S7bD3* d) {
  const size_t N = (size_t)d->n, Bs = (size_t)d->B;
  int rc = 0;
  rc |= d->fx_v.ensure(N * 24); rc |= d->fx_cn4.ensure(N * 32); rc |= d->fx_nb.ensure(N * 32); rc |= d->fx_out.ensure(N * 48);
  rc |= d->fx_energy.ensure(Bs * 8); rc |= d->fx_sums.ensure(Bs * 48);
  return rc ? d3_fail("cudaMalloc failed for the D3 heat flux") : 0;
}

static int d3_centroid_scratch(S7bD3* d) {
  const size_t N = (size_t)d->n;
  int rc = 0;
  rc |= d->ct_beta.ensure(N * 24); rc |= d->ct_nb.ensure(N * 16); rc |= d->ct_out.ensure(N * 72);
  return rc ? d3_fail("cudaMalloc failed for the D3 centroid virial") : 0;
}

static D3Flux d3_flux_args(const S7bD3* d) {
  D3Flux X;
  X.v = d->fx_v.as<double>();
  X.eatom = d->eatom.as<double>();
  X.cn4 = d->fx_cn4.as<double>();
  X.nb = d->fx_nb.as<float4>();
  X.out = d->fx_out.as<double>();
  return X;
}

static D3Centroid d3_centroid_args(const S7bD3* d) {
  D3Centroid C;
  C.beta = d->ct_beta.as<double>();
  C.nb = d->ct_nb.as<float4>();
  C.spair = d->spair.as<double>();
  C.out = d->ct_out.as<double>();
  return C;
}

// flux pass 1: the velocities of all atoms to the sorted order in bohr, then d3_flux_cn_kernel over the range;
// pass 2: d3_flux_pair_kernel over the range.  Scratch allocated, no checks.
static int d3_flux_launch(S7bD3* d, int pass, const double* d_v, int i_begin, int i_end, cudaStream_t st) {
  const int n = d->n, cnt = i_end - i_begin;
  const int grd = (cnt + kD3WarpsPerBlock - 1) / kD3WarpsPerBlock, blk = 32 * kD3WarpsPerBlock;
  const bool bt = d->batched;
  const D3Params& P = bt ? d->Pe : d->P;
  const D3Atoms A = d3_atoms(d);
  const D3Flux X = d3_flux_args(d);
  if (pass == 1) {
    if (n > 0) d3_hvp_gather_kernel<<<(3 * n + 255) / 256, 256, 0, st>>>(n, d->idx_sorted.as<int>(), d_v, d->fx_v.as<double>());
    if (cnt > 0) {
      if (bt) d3_flux_cn_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, X);
      else d3_flux_cn_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, X);
    }
  } else if (cnt > 0) {
    if (bt) d3_flux_pair_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, i_begin, i_end, X);
    else d3_flux_pair_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, i_begin, i_end, X);
  }
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// per structure over all n rows of fx_out: R in the sums' first three slots, eatom v in the last three (the energy sum
// goes to scratch), then J_pot and sum U v in eV A x (the unit of v)
static int d3_flux_sums_launch(S7bD3* d, double* d_jpot, double* d_ju, cudaStream_t st) {
  const int B = d->B;
  d3_system_sums_kernel<<<B, kD3SumBlock, 0, st>>>(d->aptr.as<int>(), 0, d->n, d->eatom.as<double>(), d->fx_out.as<double>(),
                                                   d->fx_energy.as<double>(), d->fx_sums.as<double>());
  d3_flux_results_kernel<<<(3 * B + 255) / 256, 256, 0, st>>>(B, d->fx_sums.as<double>(), d_jpot, d_ju);
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// centroid pass 1: d3_centroid_moment_kernel over the range; pass 2: d3_centroid_cn_kernel over the range (ct_out rows
// in eV, sorted order).  Scratch allocated, no checks.
static int d3_centroid_launch(S7bD3* d, int pass, int i_begin, int i_end, cudaStream_t st) {
  const int cnt = i_end - i_begin;
  if (cnt == 0) return 0;
  const int grd = (cnt + kD3WarpsPerBlock - 1) / kD3WarpsPerBlock, blk = 32 * kD3WarpsPerBlock;
  const bool bt = d->batched;
  const D3Params& P = bt ? d->Pe : d->P;
  const D3Atoms A = d3_atoms(d);
  const D3Centroid C = d3_centroid_args(d);
  if (pass == 1) {
    if (bt) d3_centroid_moment_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, i_begin, i_end, C);
    else d3_centroid_moment_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->dW.as<float>(), d->R1_vdw, i_begin, i_end, C);
  } else {
    if (bt) d3_centroid_cn_kernel<true><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, C);
    else d3_centroid_cn_kernel<false><<<grd, blk, 0, st>>>(d->grid1, A, P, d->R1_cn, i_begin, i_end, C);
  }
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

extern "C" {

// Potential part of the heat flux of D3's atomic energies, J_pot = sum_j sum_i (r_j - r_i) (dU_j/dr_i . v_i) per
// structure, and sum_j U_j v_j, on the current system with its forward (stages 1-3 over [0, n)) held: the two passes
// over [0, n) on scratch (d3_flux_kernels.cuh), then the sums; no forward buffer is written.
int s7b_d3_heat_flux(S7bD3* d, const double* d_v, double* d_jpot, double* d_ju, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (!d3_full_forward(d))
    return d3_fail("D3: the heat flux needs stages 1, 2 and 3 run over all atoms [0, n) of the current system first");
  const int n = d->n, B = d->B;
  if (!d_jpot || (n > 0 && !d_v)) return d3_fail("null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (n == 0) {
    S7B_CUDA_CHECK(cudaMemsetAsync(d_jpot, 0, (size_t)B * 24, st));
    if (d_ju) S7B_CUDA_CHECK(cudaMemsetAsync(d_ju, 0, (size_t)B * 24, st));
    return 0;
  }
  if (d3_flux_scratch(d) || d3_flux_launch(d, 1, d_v, 0, n, st) || d3_flux_launch(d, 2, nullptr, 0, n, st)) return 1;
  d->fx_pass = 2; d->fx_lo = 0; d->fx_hi = n;
  return d3_flux_sums_launch(d, d_jpot, d_ju, st);
}

// One pass of the heat flux over [i_begin, i_end) of a range forward: see the header
int s7b_d3_heat_flux_pass(S7bD3* d, int32_t pass, const double* d_v, int32_t i_begin, int32_t i_end, void* stream) {
  if (d3_pass_check(d, pass, i_begin, i_end, d ? d->fx_pass : 0, d ? d->fx_lo : 0, d ? d->fx_hi : 0, "heat flux")) return 1;
  if (pass == 1 && d->n > 0 && !d_v) return d3_fail("null argument");
  if (d3_flux_scratch(d) || d3_flux_launch(d, pass, d_v, i_begin, i_end, reinterpret_cast<cudaStream_t>(stream))) return 1;
  if (pass == 1) { d->fx_pass = 1; d->fx_lo = i_begin; d->fx_hi = i_end; }
  else d->fx_pass = 2;
  return 0;
}

int s7b_d3_heat_flux_sums(S7bD3* d, double* d_jpot, double* d_ju, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (d->fx_pass < 2) return d3_fail("D3: the heat flux sums need flux pass 2 since the last forward stage");
  if (!d_jpot) return d3_fail("null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d->n == 0) {
    S7B_CUDA_CHECK(cudaMemsetAsync(d_jpot, 0, (size_t)d->B * 24, st));
    if (d_ju) S7B_CUDA_CHECK(cudaMemsetAsync(d_ju, 0, (size_t)d->B * 24, st));
    return 0;
  }
  return d3_flux_sums_launch(d, d_jpot, d_ju, st);
}

// Per-atom centroid virial of D3's atomic energies, Wc_i = sum_j sum_i' (r_j - r_i') (x) dU_j/dr_i' [n,9] (eV,
// caller's atom order), on the current system with its forward (stages 1-3 over [0, n)) held: the two passes over
// [0, n) on scratch (d3_centroid_kernels.cuh) that read the forward's spair rows, then the forward's unsort; no forward
// buffer is written.
int s7b_d3_centroid_virial(S7bD3* d, double* d_out, void* stream) {
  if (!d || !d->have_system) return d3_fail("D3: no system set");
  if (!d3_full_forward(d))
    return d3_fail("D3: the centroid virial needs stages 1, 2 and 3 run over all atoms [0, n) of the current system "
                   "first");
  const int n = d->n;
  if (n == 0) return 0;
  if (!d_out) return d3_fail("null argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (d3_centroid_scratch(d) || d3_centroid_launch(d, 1, 0, n, st) || d3_centroid_launch(d, 2, 0, n, st)) return 1;
  d->ct_pass = 2; d->ct_lo = 0; d->ct_hi = n;
  d3_unsort_kernel<<<(n * 9 + 255) / 256, 256, 0, st>>>(n, 9, d->idx_sorted.as<int>(), d->ct_out.as<double>(), 1.0, d_out);
  S7B_CUDA_CHECK(cudaGetLastError());
  return 0;
}

// One pass of the centroid virial over [i_begin, i_end) of a range forward: see the header
int s7b_d3_centroid_pass(S7bD3* d, int32_t pass, int32_t i_begin, int32_t i_end, void* stream) {
  if (d3_pass_check(d, pass, i_begin, i_end, d ? d->ct_pass : 0, d ? d->ct_lo : 0, d ? d->ct_hi : 0, "centroid virial"))
    return 1;
  if (d3_centroid_scratch(d) || d3_centroid_launch(d, pass, i_begin, i_end, reinterpret_cast<cudaStream_t>(stream))) return 1;
  if (pass == 1) { d->ct_pass = 1; d->ct_lo = i_begin; d->ct_hi = i_end; }
  else d->ct_pass = 2;
  return 0;
}

}  // extern "C"

// ---- the reference's own entry points (sevenn/pair_e3gnn/pair_d3_for_ase.cu:2034-2082) ------------------
// Same names, argument meaning and call order as the ctypes binding in sevenn/calculator.py:430-483, so the
// reference's D3Calculator can load this library in place of its pair_d3.so.  The parameter tables come from
// weights/d3_params.bin (tools/convert_d3_params.py), found through $S7B_D3_PARAMS or relative to this library.
namespace s7b {
struct D3Tables {
  std::vector<double> r0ab, c6ref, cnref, r2r4, rcov;
  std::vector<int> mxc;
  std::map<std::string, std::vector<double>> func;     // "damp_bj/pbe" -> {s6, rs6, s18, rs18, alp}
  bool ok = false;
  std::string error;
};
static D3Tables& d3_tables() {
  static D3Tables T;
  if (T.ok || !T.error.empty()) return T;
  std::string path;
  if (const char* env = getenv("S7B_D3_PARAMS")) path = env;
  else {
    Dl_info info;
    if (dladdr((void*)&d3_tables, &info) && info.dli_fname) {
      std::string lib(info.dli_fname);
      const size_t k = lib.rfind('/');
      path = (k == std::string::npos ? std::string(".") : lib.substr(0, k)) + "/../../weights/d3_params.bin";
    }
  }
  FILE* f = fopen(path.c_str(), "rb");
  if (!f) { T.error = "cannot open " + path; return T; }
  auto rd = [&](std::vector<double>& v, size_t n) { v.resize(n); return fread(v.data(), 8, n, f) == n; };
  std::vector<double> m;
  bool good = rd(T.r0ab, 94 * 94) && rd(T.c6ref, 94 * 94 * 25) && rd(T.cnref, 94 * 5) && rd(m, 94) && rd(T.r2r4, 94) && rd(T.rcov, 94);
  if (good) {
    T.mxc.assign(94, 0);
    for (int i = 0; i < 94; ++i) T.mxc[i] = (int)m[i];
    char line[256];
    while (fgets(line, sizeof(line), f)) {
      char damp[64], name[64];
      double v[5];
      if (sscanf(line, "%63s %63s %lf %lf %lf %lf %lf", damp, name, &v[0], &v[1], &v[2], &v[3], &v[4]) == 7)
        T.func[std::string(damp) + "/" + name] = std::vector<double>(v, v + 5);
    }
  }
  fclose(f);
  if (!good || T.func.empty()) T.error = "malformed " + path;
  else T.ok = true;
  return T;
}
}  // namespace s7b

extern "C" {

S7bD3* pair_init(void) {
  S7bD3* d = nullptr;
  return s7b_d3_create(&d) ? nullptr : d;
}

void pair_set_atom(S7bD3* d, int natoms, int ntypes, int* type, double* x_flat) {
  if (!d) return;
  d->ref_types.assign(type, type + natoms);                  // 1-based, as LAMMPS / the reference
  d->ref_pos.assign(x_flat, x_flat + (size_t)natoms * 3);
  d->ref_ntypes = ntypes;
}

void pair_set_domain(S7bD3* d, int xperiodic, int yperiodic, int zperiodic, double* boxlo, double* boxhi, double xy,
                     double xz, double yz) {
  if (!d) return;
  const double c[9] = {boxhi[0] - boxlo[0], 0, 0, xy, boxhi[1] - boxlo[1], 0, xz, yz, boxhi[2] - boxlo[2]};   // :889-897
  memcpy(d->ref_cell, c, sizeof(c));
  d->ref_pbc[0] = xperiodic; d->ref_pbc[1] = yperiodic; d->ref_pbc[2] = zperiodic;
}

void pair_run_settings(S7bD3* d, double rthr, double cnthr, const char* damp_name, const char* func_name) {
  if (!d) return;
  d->ref_rthr = rthr;
  d->ref_cnthr = cnthr;
  d->ref_damp = damp_name ? damp_name : "";
  d->ref_func = func_name ? func_name : "";
}

void pair_run_coeff(S7bD3* d, int* atomic_numbers) {
  if (!d) return;
  D3Tables& T = d3_tables();
  if (!T.ok) { d3_fail("D3 tables: " + T.error); fprintf(stderr, "Error: %s\n", s7b_last_error()); return; }
  const int nt = d->ref_ntypes;
  std::vector<double> rcov(nt), r2r4(nt), r0((size_t)nt * nt), c6((size_t)nt * nt * 25), cr((size_t)nt * 5);
  std::vector<int> mxc(nt);
  for (int a = 0; a < nt; ++a) {
    const int za = atomic_numbers[a] - 1;
    if (za < 0 || za >= 94) { d3_fail("D3: atomic number out of range"); return; }
    rcov[a] = T.rcov[za]; r2r4[a] = T.r2r4[za]; mxc[a] = T.mxc[za];
    for (int q = 0; q < 5; ++q) cr[a * 5 + q] = T.cnref[za * 5 + q];
    for (int b = 0; b < nt; ++b) {
      const int zb = atomic_numbers[b] - 1;
      r0[a * nt + b] = T.r0ab[za * 94 + zb];
      for (int q = 0; q < 25; ++q) c6[((size_t)a * nt + b) * 25 + q] = T.c6ref[((size_t)za * 94 + zb) * 25 + q];
    }
  }
  if (s7b_d3_set_params(d, nt, rcov.data(), r2r4.data(), r0.data(), c6.data(), cr.data(), mxc.data())) { fprintf(stderr, "Error: %s\n", s7b_last_error()); return; }
  auto it = T.func.find(d->ref_damp + "/" + d->ref_func);
  if (it == T.func.end()) { d3_fail("Functional name unknown"); fprintf(stderr, "Error: Functional name unknown\n"); return; }
  const std::vector<double>& p = it->second;    // s6, rs6, s18, rs18, alp  ->  setfuncpar (:608-631)
  if (s7b_d3_set_damping(d, d->ref_damp == "damp_bj" ? 1 : 0, p[0], p[2], p[1], p[3], p[4], p[4] + 2.0, d->ref_rthr, d->ref_cnthr))
    fprintf(stderr, "Error: %s\n", s7b_last_error());
}

void pair_run_compute(S7bD3* d) {
  if (!d) return;
  const int n = (int)d->ref_types.size();
  std::vector<int> t0(n);
  for (int i = 0; i < n; ++i) t0[i] = d->ref_types[i] - 1;
  d->host_force.assign((size_t)n * 3, 0.0);
  if (s7b_d3_set_system(d, n, t0.data(), d->ref_pos.data(), d->ref_cell, d->ref_pbc, nullptr) ||
      s7b_d3_compute_host(d, &d->host_energy, d->host_force.data(), d->host_sigma, nullptr))
    fprintf(stderr, "Error: %s\n", s7b_last_error());
}

double pair_get_energy(S7bD3* d) { return d ? d->host_energy : 0.0; }
double* pair_get_force(S7bD3* d) { return d ? d->host_force.data() : nullptr; }
double* pair_get_stress(S7bD3* d) { return d ? d->host_sigma : nullptr; }
void pair_fin(S7bD3* d) { s7b_d3_destroy(d); }

}  // extern "C"
