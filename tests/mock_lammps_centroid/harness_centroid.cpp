// Mock-LAMMPS harness for the per-atom centroid virial of examples/lammps/pair_e3gnn_b200.cpp (CPU, test
// infrastructure): a cluster of atoms with a full neighbour list (with skin), the pair style's compute with the
// centroid flag set (LAMMPS's VIRIAL_CENTROID bit, as compute centroid/stress/atom requests it), against the Pair
// declarations of ./pair.h (those of tests/mock_lammps plus the centroid members).  Checks:
//   * the style advertises CENTROID_AVAIL;
//   * cvatom holds the library's rows in LAMMPS order (xx yy zz xy xz yz yx zx zy), xy = Wc[x][y];
//   * REAL_ENGINE (the library on the GPU): cvatom summed over the atoms is the virial (xx yy zz xy xz yz), and compute
//     heat/flux's contraction J_a = sum_i (cvatom_i v_i)_a equals s7b_engine_heat_flux's J_pot on the same atoms and
//     velocities.
// Without REAL_ENGINE the library is tests/mock_lammps/stub_s7b.cpp, and s7b_engine_centroid_virial_host is the toy
// below, whose rows are Wc_r[a][b] = 100 r + 10 a + b: every entry distinct, so any misplaced component shows.
#include <cmath>
#include <cstdio>
#include <random>
#include <stdexcept>
#include <vector>

#include "pair_e3gnn_b200.h"

#include "../../include/sevenn_b200.h"
#ifdef REAL_ENGINE
#include <cuda_runtime.h>
#endif

namespace LAMMPS_NS {
void Error::all(const char *f, int l, const char *m) { throw std::runtime_error(std::string(f) + ":" + std::to_string(l) + " " + m); }
void Error::one(const char *f, int l, const char *m) { throw std::runtime_error(std::string(f) + ":" + std::to_string(l) + " " + m); }
int Atom::map(tagint t) { return t - 1; }
int Atom::tag_consecutive() { return 1; }
void *Neighbor::add_request(Pair *, int) { return nullptr; }
void Pair::ev_init(int eflag, int vflag, int) {
  eflag_global = eflag & 1; eflag_atom = eflag & 2; vflag_global = vflag & 1; vflag_atom = vflag & 2;
  cvflag_atom = vflag & 8;         // VIRIAL_CENTROID
  eng_vdwl = 0.0;
  for (double &v : virial) v = 0.0;
}
}  // namespace LAMMPS_NS

using namespace LAMMPS_NS;

#ifndef REAL_ENGINE
static int g_rows = 0;       // rows of the toy centroid virial (the harness's atom count)
extern "C" int s7b_engine_centroid_virial_host(S7bEngine *, double *host_out, void *) {
  for (int r = 0; r < g_rows; ++r)
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) host_out[9 * (size_t)r + 3 * a + b] = 100.0 * r + 10.0 * a + b;
  return 0;
}
#endif

struct TestSerialPair : PairE3GNNB200 {
  Error err; Memory mem; Force frc; Neighbor nb;
  explicit TestSerialPair(Atom *a, const char *model) : PairE3GNNB200(nullptr) {
    error = &err; memory = &mem; atom = a; force = &frc; neighbor = &nb;
    frc.newton_pair = 1;
    if (model) {
      settings(0, nullptr);
      char a0[] = "*", a1[] = "*", sym[] = "Si";
      std::string mp(model);
      char *args[4] = {a0, a1, mp.data(), sym};
      coeff(4, args);
      init_style();
    } else {
      S7bModelDesc d{};
      d.n_layers = 3;
      d.cutoff = 3.0f;
      for (int t = 0; t <= 3; ++t) { d.n_l[t] = 1; d.muls[t][0] = 4; }
      if (s7b_engine_create(&d, &engine)) throw std::runtime_error("create");
      allocate();
      cutoff = d.cutoff;
      for (int t = 1; t <= a->ntypes; ++t) species_of_type[t] = t - 1;
    }
  }
  void set_list(NeighList *l) { list = l; }
  S7bEngine *eng() { return engine; }
  const std::vector<double> &rows() const { return cvatom_buf; }     // what the library returned to the style
};

int main(int argc, char **argv) {
  const char *model = argc > 1 ? argv[1] : nullptr;
#ifdef REAL_ENGINE
  if (!model) { std::printf("usage: harness_centroid <model.s7b>\n"); return 2; }
  const double a0 = 5.431, rc = 5.0, skin = 0.5;
  const int ntypes = 1;
#else
  const double a0 = 2.4, rc = 3.0, skin = 0.5;
  const int ntypes = 2;
#endif
  // a 2x2x1 block of diamond conventional cells, no periodicity, positions jittered by up to +-0.05 A
  const double basis[8][3] = {{0, 0, 0}, {0, .5, .5}, {.5, 0, .5}, {.5, .5, 0}, {.25, .25, .25}, {.25, .75, .75}, {.75, .25, .75}, {.75, .75, .25}};
  std::mt19937 rng(7);
  std::uniform_real_distribution<double> jit(-0.05, 0.05), vel(-1.0, 1.0);
  std::vector<double> xflat, vflat;
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j)
      for (int b = 0; b < 8; ++b) {
        xflat.push_back((i + basis[b][0]) * a0 + jit(rng));
        xflat.push_back((j + basis[b][1]) * a0 + jit(rng));
        xflat.push_back(basis[b][2] * a0 + jit(rng));
      }
  const int n = (int)xflat.size() / 3;
#ifndef REAL_ENGINE
  g_rows = n;
#endif
  for (int q = 0; q < 3 * n; ++q) vflat.push_back(vel(rng));
  std::vector<double> fflat((size_t)n * 3, 0.0), eatom(n, 0.0), cvflat((size_t)n * 9, 0.0);
  std::vector<double *> x(n), f(n), cv(n);
  std::vector<int> type(n), tag(n), ilist(n), numneigh(n);
  for (int i = 0; i < n; ++i) {
    x[i] = &xflat[3 * (size_t)i]; f[i] = &fflat[3 * (size_t)i]; cv[i] = &cvflat[9 * (size_t)i];
    type[i] = 1 + i % ntypes; tag[i] = i + 1; ilist[i] = i;
  }
  std::vector<std::vector<int>> nbrs(n);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) {
      if (i == j) continue;
      double r2 = 0;
      for (int a = 0; a < 3; ++a) r2 += (x[j][a] - x[i][a]) * (x[j][a] - x[i][a]);
      if (r2 < (rc + skin) * (rc + skin)) nbrs[i].push_back(j);
    }
  std::vector<int *> first(n);
  for (int i = 0; i < n; ++i) { numneigh[i] = (int)nbrs[i].size(); first[i] = nbrs[i].data(); }
  Atom atom{};
  atom.ntypes = ntypes; atom.nlocal = n; atom.nghost = 0; atom.map_style = Atom::MAP_ARRAY;
  atom.x = x.data(); atom.f = f.data(); atom.type = type.data(); atom.tag = tag.data();
  NeighList list{};
  list.inum = n; list.ilist = ilist.data(); list.numneigh = numneigh.data(); list.firstneigh = first.data();

  double virial[6];
  std::vector<double> rows((size_t)n * 9);
  double jpot_engine[3] = {0, 0, 0};
  bool avail = false;
  try {
    TestSerialPair sp(&atom, model);
    sp.set_list(&list);
    sp.eatom = eatom.data();
    sp.cvatom = cv.data();
    avail = sp.centroidstressflag == CENTROID_AVAIL;
    sp.compute(3, 1 | 8);
    for (int q = 0; q < 6; ++q) virial[q] = sp.virial[q];
    rows = sp.rows();
#ifdef REAL_ENGINE
    std::vector<float> v32(vflat.begin(), vflat.end());
    float *dv = nullptr;
    double *dj = nullptr;
    if (cudaMalloc(&dv, sizeof(float) * 3 * n) || cudaMalloc(&dj, sizeof(double) * 3)) throw std::runtime_error("cudaMalloc");
    cudaMemcpy(dv, v32.data(), sizeof(float) * 3 * n, cudaMemcpyHostToDevice);
    if (s7b_engine_heat_flux(sp.eng(), dv, dj, nullptr, nullptr)) throw std::runtime_error(s7b_last_error());
    cudaMemcpy(jpot_engine, dj, sizeof(jpot_engine), cudaMemcpyDeviceToHost);
    cudaFree(dv);
    cudaFree(dj);
#endif
  } catch (const std::exception &ex) {
    std::printf("FAIL serial pair style raised: %s\n", ex.what());
    return 1;
  }
  // cvatom in LAMMPS order against the library rows; sums against the virial; compute heat/flux's contraction
  const int lm[9] = {0, 4, 8, 1, 2, 5, 3, 6, 7};
  double drow = 0, dsum = 0, scale = 0, total = 0, J[3] = {0, 0, 0};
  for (int i = 0; i < n; ++i)
    for (int q = 0; q < 9; ++q) {
      drow = std::fmax(drow, std::fabs(cv[i][q] - rows[9 * (size_t)i + lm[q]]));
      scale = std::fmax(scale, std::fabs(cv[i][q]));
      total += std::fabs(cv[i][q]);
    }
  for (int q = 0; q < 6; ++q) {
    double t = 0;
    for (int i = 0; i < n; ++i) t += cv[i][q];
    dsum = std::fmax(dsum, std::fabs(t - virial[q]));
  }
  double jscale = 0;
  for (int i = 0; i < n; ++i) {      // compute_heat_flux.cpp: J_x = sum_i (s0 v0 + s3 v1 + s4 v2), cvatom order
    const double *s = cv[i], *v = &vflat[3 * (size_t)i];
    J[0] += s[0] * v[0] + s[3] * v[1] + s[4] * v[2];
    J[1] += s[6] * v[0] + s[1] * v[1] + s[5] * v[2];
    J[2] += s[7] * v[0] + s[8] * v[1] + s[2] * v[2];
    for (int q = 0; q < 9; ++q) jscale += std::fabs(s[q]);
  }
  double dj = 0;
#ifdef REAL_ENGINE
  for (int a = 0; a < 3; ++a) dj = std::fmax(dj, std::fabs(J[a] - jpot_engine[a]));
  dj /= jscale;
  const bool physics = dsum < 1e-5 * total && dj < 1e-5;    // the sum rule to the pass's fp32 rounding
#else
  const bool physics = true;      // the toy rows are no virial
#endif
  std::printf("atoms %d: CENTROID_AVAIL %d, max|cvatom - library rows| %.2e (max|cvatom| %.2e), max|sum cvatom - virial| %.2e, "
              "heat/flux J %.6e %.6e %.6e vs engine J_pot %.6e %.6e %.6e, err / sum|terms| %.2e\n",
              n, avail ? 1 : 0, drow, scale, dsum, J[0], J[1], J[2], jpot_engine[0], jpot_engine[1], jpot_engine[2], dj);
  // the rows are copied, so exactly
  const bool ok = avail && scale > 1e-6 && drow == 0.0 && physics;
  std::printf(ok ? "OK\n" : "FAIL\n");
  return ok ? 0 : 1;
}
