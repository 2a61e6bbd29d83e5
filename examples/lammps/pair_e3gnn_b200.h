/* LAMMPS pair style backed by libsevenn_b200.so (SURVEY section 8 f.3).
 *
 *   pair_style e3gnn/b200
 *   pair_coeff * * model.s7b Hf O        # one chemical symbol per LAMMPS atom type
 *
 * Same user contract as the reference's serial `pair_style e3gnn` (sevenn/pair_e3gnn/pair_e3gnn.cpp:
 * 302-411): metal units, `newton_pair on`, a full neighbour list, an atom map (`atom_modify map yes`),
 * one process.  Per-atom virial: `compute stress/atom` gets the pairwise split of the reference; `compute
 * centroid/stress/atom` gets the exact per-atom centroid virial, the one `compute heat/flux` needs for Green-Kubo
 * (DESIGN.md §8.5; a Pair class without the centroid members builds the style without it).  The model file comes from sevenn_b200/export.py:export_flat instead of `sevenn
 * get_model` (TorchScript); there is no libtorch in this pair style.
 * Written against LAMMPS stable_2Aug2023.  LAMMPS is not in the image: this repository compiles it against the
 * minimal declarations in tests/mock_lammps/ and runs it there on the CPU against a toy double of the library
 * (tests/mock_lammps/harness_parallel.cpp, tests/test_host_logic.py). */
#ifdef PAIR_CLASS
// clang-format off
PairStyle(e3gnn/b200, PairE3GNNB200)
// clang-format on
#else
#ifndef LMP_PAIR_E3GNN_B200_H
#define LMP_PAIR_E3GNN_B200_H

#include <vector>

#include "pair.h"

struct S7bEngine;

namespace LAMMPS_NS {

class PairE3GNNB200 : public Pair {
 public:
  PairE3GNNB200(class LAMMPS *);
  ~PairE3GNNB200() override;
  void compute(int, int) override;
  void settings(int, char **) override;
  void coeff(int, char **) override;
  void init_style() override;
  double init_one(int, int) override;

 protected:
  void allocate();
  template <class P> void centroid_setup(P *self);
  template <class P> void centroid_rows(P *self, int nlocal, const int *ilist);

  S7bEngine *engine = nullptr;
  double cutoff = 0.0;
  int *species_of_type = nullptr;     // LAMMPS type -> species index of the model
  // host staging, reused between steps
  std::vector<int> species, edge_centre, edge_neighbour, row_of_atom;
  std::vector<float> edge_vec, forces, eatom_buf, vatom_buf;
  std::vector<double> cvatom_buf;
  bool atomic_virial_on = false;
};

}  // namespace LAMMPS_NS
#endif
#endif
