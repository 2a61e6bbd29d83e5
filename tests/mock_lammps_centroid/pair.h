// Minimal stand-ins for the LAMMPS declarations examples/lammps/pair_e3gnn_b200.cpp uses, with the per-atom centroid
// virial of LAMMPS's Pair (cvatom, cvflag_atom, centroidstressflag and its CENTROID_* values), so that the serial pair
// style's centroid branch can be compiled and run in the CPU harness (harness_centroid.cpp) without LAMMPS.  The same
// declarations as tests/mock_lammps/pair.h otherwise, which stands in for a Pair without the centroid members.  Not
// LAMMPS code: member names and signatures follow the public LAMMPS developer documentation (stable_2Aug2023).
#pragma once
#include <cstdint>
#define FLERR __FILE__, __LINE__
#define NEIGHMASK 0x1FFFFFFF
namespace LAMMPS_NS {
typedef int tagint;
class LAMMPS;
struct Error {
  [[noreturn]] void all(const char *, int, const char *);
  [[noreturn]] void one(const char *, int, const char *);
};
struct Memory {       // leaks on purpose (test scaffolding): one flat block per array, row pointers for the 2-D form
  template <class T> T **create(T **&a, int n1, int n2, const char *) {
    T *flat = new T[(size_t)n1 * n2]();
    a = new T *[n1];
    for (int i = 0; i < n1; ++i) a[i] = flat + (size_t)i * n2;
    return a;
  }
  template <class T> T *create(T *&a, int n, const char *) { a = new T[n](); return a; }
  template <class T> void destroy(T &a) { a = nullptr; }
};
struct Atom {
  enum { MAP_NONE = 0, MAP_ARRAY = 1, MAP_HASH = 2, MAP_YES = 3 };
  int ntypes, nlocal, nghost, map_style;
  double **x, **f;
  int *type;
  tagint *tag;
  int map(tagint);
  int tag_consecutive();
};
struct Force { int newton_pair; };
struct NeighList {
  int inum;
  int *ilist, *numneigh, **firstneigh;
};
namespace NeighConst { enum { REQ_DEFAULT = 0, REQ_FULL = 1 }; }
enum { CENTROID_SAME = 0, CENTROID_AVAIL = 1, CENTROID_NOTAVAIL = 2 };
struct Neighbor { void *add_request(class Pair *, int); };
struct Comm {
  int me, nprocs;
  void forward_comm(class Pair *, int size = 0);
  void reverse_comm(class Pair *, int size = 0);
};
class Pointers {
 public:
  explicit Pointers(LAMMPS *) {}
  virtual ~Pointers() = default;
 protected:
  Error *error;
  Memory *memory;
  Atom *atom;
  Force *force;
  Neighbor *neighbor;
  Comm *comm;
};
class Pair : protected Pointers {
 public:
  explicit Pair(LAMMPS *lmp) : Pointers(lmp) {}
  virtual void compute(int, int) = 0;
  virtual void settings(int, char **) = 0;
  virtual void coeff(int, char **) = 0;
  virtual void init_style() {}
  virtual double init_one(int, int) { return 0.0; }
  virtual int pack_forward_comm(int, int *, double *, int, int *) { return 0; }
  virtual void unpack_forward_comm(int, int, double *) {}
  virtual int pack_reverse_comm(int, int, double *) { return 0; }
  virtual void unpack_reverse_comm(int, int *, double *) {}
  int comm_forward = 0, comm_reverse = 0;
  double eng_vdwl, virial[6];
  double *eatom, **vatom;
  double **cvatom = nullptr;               // per-atom centroid virial, 9 components (compute centroid/stress/atom)
  int centroidstressflag = CENTROID_SAME;
 protected:
  int allocated = 0, single_enable, restartinfo, one_coeff, manybody_flag, no_virial_fdotr_compute;
  int eflag_global, eflag_atom, vflag_global, vflag_atom;
  int cvflag_atom = 0;
  int **setflag;
  double **cutsq;
  NeighList *list;
  void ev_init(int, int, int = 1);
};
}  // namespace LAMMPS_NS
