/* See pair_e3gnn_b200.h.  Per step: LAMMPS full neighbour list -> centre-major edge arrays on the
 * host -> one call of s7b_engine_compute_host (H2D, CSR build, model, forces, virial, D2H) ->
 * accumulate into f / eng_vdwl / virial / eatom. */
#include "pair_e3gnn_b200.h"

#include <string>
#include <type_traits>
#include <utility>

#include "atom.h"
#include "error.h"
#include "force.h"
#include "memory.h"
#include "neigh_list.h"
#include "neighbor.h"

#include "../s7b_model_file.h"

using namespace LAMMPS_NS;

namespace {
// Whether the LAMMPS Pair class carries the per-atom centroid virial (cvatom / centroidstressflag, LAMMPS since
// stable_29Oct2020).  Against older Pair declarations the style builds without centroid support and LAMMPS keeps
// its default for it.
template <class P, class = void>
struct HasCentroid : std::false_type {};
template <class P>
struct HasCentroid<P, std::void_t<decltype(std::declval<P &>().cvatom), decltype(std::declval<P &>().centroidstressflag)>>
    : std::true_type {};
}  // namespace

PairE3GNNB200::PairE3GNNB200(LAMMPS *lmp) : Pair(lmp) {
  single_enable = 0;
  restartinfo = 0;
  one_coeff = 1;
  manybody_flag = 1;
  no_virial_fdotr_compute = 1;     // the virial comes from the edge forces, not from f . r
  centroid_setup(this);
}

PairE3GNNB200::~PairE3GNNB200() {
  if (engine) s7b_engine_destroy(engine);
  if (allocated) {
    memory->destroy(setflag);
    memory->destroy(cutsq);
    memory->destroy(species_of_type);
  }
}

void PairE3GNNB200::allocate() {
  allocated = 1;
  const int n = atom->ntypes;
  memory->create(setflag, n + 1, n + 1, "pair:setflag");
  memory->create(cutsq, n + 1, n + 1, "pair:cutsq");
  memory->create(species_of_type, n + 1, "pair:species_of_type");
}

void PairE3GNNB200::settings(int narg, char ** /*arg*/) {
  if (narg != 0) error->all(FLERR, "Illegal pair_style command: e3gnn/b200 takes no arguments");
}

// pair_coeff * * <model.s7b> <symbol of type 1> <symbol of type 2> ...
void PairE3GNNB200::coeff(int narg, char **arg) {
  if (!allocated) allocate();
  const int ntypes = atom->ntypes;
  if (narg != 3 + ntypes) error->all(FLERR, "Incorrect args for pair coefficients: * * model.s7b + one element per atom type");
  if (std::string(arg[0]) != "*" || std::string(arg[1]) != "*") error->all(FLERR, "e3gnn/b200: pair_coeff must start with * *");

  s7b_file::Model model;
  const std::string err = s7b_file::load(arg[2], model);
  if (!err.empty()) error->all(FLERR, ("e3gnn/b200: " + err).c_str());
  if (engine) s7b_engine_destroy(engine);
  engine = model.engine;
  cutoff = model.desc.cutoff;

  for (int t = 1; t <= ntypes; ++t) {
    const int z = s7b_file::atomic_number(arg[2 + t]);
    const auto it = model.species_of_z.find(z);
    if (z == 0 || it == model.species_of_z.end())
      error->all(FLERR, (std::string("e3gnn/b200: element ") + arg[2 + t] + " is not known to the model").c_str());
    species_of_type[t] = it->second;
  }
  for (int i = 1; i <= ntypes; ++i)
    for (int j = 1; j <= ntypes; ++j) {
      setflag[i][j] = 1;
      cutsq[i][j] = cutoff * cutoff;
    }
}

void PairE3GNNB200::init_style() {
  if (force->newton_pair == 0) error->all(FLERR, "Pair style e3gnn/b200 requires newton pair on");
  if (atom->map_style == Atom::MAP_NONE) error->all(FLERR, "Pair style e3gnn/b200 requires an atom map (atom_modify map yes)");
  neighbor->add_request(this, NeighConst::REQ_FULL);
}

double PairE3GNNB200::init_one(int /*i*/, int /*j*/) { return cutoff; }

void PairE3GNNB200::compute(int eflag, int vflag) {
  ev_init(eflag, vflag);
  if (atom->tag_consecutive() == 0) error->all(FLERR, "Pair style e3gnn/b200 requires consecutive atom IDs");

  double **x = atom->x;
  double **f = atom->f;
  const int *type = atom->type;
  const tagint *tag = atom->tag;
  const int nlocal = list->inum;
  const int *ilist = list->ilist;
  const int *numneigh = list->numneigh;
  int **firstneigh = list->firstneigh;
  const double cut2 = cutoff * cutoff;

  // graph row r <-> local atom ilist[r]; neighbours that are periodic images or ghosts map back to
  // their owning local atom through the atom map (single process), the image shift stays in edge_vec
  species.resize(nlocal);
  row_of_atom.assign(atom->nlocal, -1);
  for (int r = 0; r < nlocal; ++r) {
    species[r] = species_of_type[type[ilist[r]]];
    row_of_atom[ilist[r]] = r;
  }
  edge_centre.clear();
  edge_neighbour.clear();
  edge_vec.clear();
  for (int r = 0; r < nlocal; ++r) {
    const int i = ilist[r];
    const int *jlist = firstneigh[i];
    for (int jj = 0; jj < numneigh[i]; ++jj) {
      const int j = jlist[jj] & NEIGHMASK;
      const double dx = x[j][0] - x[i][0], dy = x[j][1] - x[i][1], dz = x[j][2] - x[i][2];
      if (dx * dx + dy * dy + dz * dz >= cut2) continue;      // the list carries the skin
      const int owner = atom->map(tag[j]);
      if (owner < 0 || owner >= atom->nlocal || row_of_atom[owner] < 0) error->one(FLERR, "e3gnn/b200: neighbour without a local owner");
      edge_centre.push_back(r);                               // rows are visited in order: sorted by centre
      edge_neighbour.push_back(row_of_atom[owner]);
      edge_vec.push_back((float)dx);
      edge_vec.push_back((float)dy);
      edge_vec.push_back((float)dz);
    }
  }

  if (vflag_atom && !atomic_virial_on) {       // per-atom virial on demand (pair_e3gnn.cpp:263-275)
    if (s7b_engine_set_atomic_virial(engine, 1)) error->one(FLERR, s7b_last_error());
    atomic_virial_on = true;
  }
  forces.resize((size_t)nlocal * 3);
  eatom_buf.resize(nlocal);
  double energy = 0.0, v6[6] = {0, 0, 0, 0, 0, 0};
  if (s7b_engine_compute_host(engine, nlocal, (int64_t)edge_centre.size(), species.data(), edge_centre.data(),
                              edge_neighbour.data(), edge_vec.data(), &energy, eatom_buf.data(), forces.data(), v6,
                              /*stream=*/nullptr) != 0)
    error->one(FLERR, s7b_last_error());

  for (int r = 0; r < nlocal; ++r) {
    const int i = ilist[r];
    f[i][0] += forces[3 * r];
    f[i][1] += forces[3 * r + 1];
    f[i][2] += forces[3 * r + 2];
  }
  if (eflag_global) eng_vdwl += energy;
  if (eflag_atom)
    for (int r = 0; r < nlocal; ++r) eatom[ilist[r]] += eatom_buf[r];
  if (vflag_global) {
    // library order (xx, yy, zz, xy, yz, zx), value -sum r (x) dE/dr  ->  LAMMPS (xx, yy, zz, xy, xz, yz)
    virial[0] += v6[0];
    virial[1] += v6[1];
    virial[2] += v6[2];
    virial[3] += v6[3];
    virial[4] += v6[5];
    virial[5] += v6[4];
  }
  if (vflag_atom) {
    // the library's per-atom virial: -(v (x) f_e) of every edge on its NEIGHBOUR atom, order xx yy zz xy yz zx -- the
    // quantity the reference scatters onto edge_idx_dst and negates (pair_e3gnn.cpp:231-275)
    vatom_buf.resize((size_t)nlocal * 6);
    if (s7b_engine_read_rows_host(engine, "atomic_virial", 0, 0, nlocal, 6, vatom_buf.data(), nullptr)) error->one(FLERR, s7b_last_error());
    const int lm[6] = {0, 1, 2, 3, 5, 4};      // LAMMPS (xx, yy, zz, xy, xz, yz)
    for (int r = 0; r < nlocal; ++r)
      for (int q = 0; q < 6; ++q) vatom[ilist[r]][q] += vatom_buf[(size_t)r * 6 + lm[q]];
  }
  centroid_rows(this, nlocal, ilist);
}

// cvatom is the library's exact per-atom centroid virial (CENTROID_AVAIL, value 1 in LAMMPS's enum; the literal keeps
// this branch free of names an older Pair does not declare)
template <class P>
void PairE3GNNB200::centroid_setup(P *self) {
  if constexpr (HasCentroid<P>::value) self->centroidstressflag = 1;
}

// compute centroid/stress/atom (cvflag_atom): the library's centroid virial Wc_i[a][b] = sum_j (r_j - r_i)_a
// dU_j/dr_i,b (row-major, DESIGN.md §8.5), exact for the message-passing model, so that compute heat/flux's
// J_a = sum_b Wc_i[a][b] v_i,b is the model's potential flux.  The graph has no ghost rows (images map to their
// owners), so every row is an owned atom's.  LAMMPS order: xx yy zz xy xz yz yx zx zy.
template <class P>
void PairE3GNNB200::centroid_rows(P *self, int nlocal, const int *ilist) {
  if constexpr (HasCentroid<P>::value) {
    if (!self->cvflag_atom) return;
    cvatom_buf.resize((size_t)nlocal * 9);
    if (s7b_engine_centroid_virial_host(engine, cvatom_buf.data(), nullptr))
      error->one(FLERR, (std::string("e3gnn/b200: compute centroid/stress/atom needs the radial MLP in the model file "
                                     "(export_flat(..., radial_mlp=True)): ") + s7b_last_error()).c_str());
    const int lm[9] = {0, 4, 8, 1, 2, 5, 3, 6, 7};
    for (int r = 0; r < nlocal; ++r)
      for (int q = 0; q < 9; ++q) self->cvatom[ilist[r]][q] += cvatom_buf[(size_t)r * 9 + lm[q]];
  } else {
    (void)self;
    (void)nlocal;
    (void)ilist;
  }
}
