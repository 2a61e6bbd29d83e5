// Stand-in for the LAMMPS header of the same name: every declaration the pair style uses is in pair.h.
#include "pair.h"
