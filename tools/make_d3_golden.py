"""Runs the reference's own CUDA D3 (oracle/_ref/libpaird3.so, built by oracle/Makefile from the unmodified
reference sources) on the rocksalt NaCl cells of tests/test_d3_gpu.py::test_matches_compiled_reference and on
the LAMMPS-frame systems of tests/d3_cells.py (sheared, slab, compressed_cs, species16; each with one functional
per damping that holds an extreme of the functional table), and stores its energies, forces and stresses in
tests/golden/d3_compiled_reference.npz, so that the tests compare the repository's D3 kernels and the fp64
oracle with the reference without needing the reference.  Needs a GPU.  When the output file exists, values it
already holds are kept and the tool reports how far the rerun is from each.

    python tools/make_d3_golden.py [output.npz]
"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import d3_cells  # noqa: E402
from sevenn_b200.neighbors import rocksalt_nacl  # noqa: E402

# (cells, damping) of the test; rocksalt_nacl(*cells, sigma=0.05, seed=11)
CASES = [((2, 2, 2), 'damp_bj'), ((6, 6, 4), 'damp_bj'), ((5, 5, 5), 'damp_zero')]
def case_key(cells, damping):
    return '{}x{}x{}_{}'.format(*cells, damping)




def reference_lib(path):
    lib = ctypes.CDLL(path)
    lib.pair_init.restype = ctypes.c_void_p
    lib.pair_get_energy.restype = ctypes.c_double
    lib.pair_get_force.restype = ctypes.POINTER(ctypes.c_double)
    lib.pair_get_stress.restype = ctypes.POINTER(ctypes.c_double * 6)
    for fn in ('pair_set_atom', 'pair_set_domain', 'pair_run_settings', 'pair_run_coeff', 'pair_run_compute', 'pair_fin'):
        getattr(lib, fn).restype = None
    lib.pair_get_energy.argtypes = lib.pair_get_force.argtypes = lib.pair_get_stress.argtypes = [ctypes.c_void_p]
    lib.pair_set_atom.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    lib.pair_set_domain.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_double] * 3
    lib.pair_run_settings.argtypes = [ctypes.c_void_p, ctypes.c_double, ctypes.c_double, ctypes.c_char_p, ctypes.c_char_p]
    lib.pair_run_coeff.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    lib.pair_run_compute.argtypes = lib.pair_fin.argtypes = [ctypes.c_void_p]
    return lib


def run_reference_d3(lib, z, pos, cell, damping, functional='pbe', pbc=(True, True, True)):
    """the compiled, unmodified reference, default cutoffs (orthogonal / lower-triangular cells only: no frame rotation)"""
    assert np.allclose(np.triu(np.asarray(cell), 1), 0.0), 'cell rows must be lower-triangular (LAMMPS frame)'
    uniq = list(dict.fromkeys(np.asarray(z).tolist()))
    types = np.ascontiguousarray([uniq.index(a) + 1 for a in z], dtype=np.int32)
    x = np.ascontiguousarray(pos, dtype=np.float64)
    nums = np.ascontiguousarray(uniq, dtype=np.int32)
    lo, hi = np.zeros(3), np.ascontiguousarray([cell[0, 0], cell[1, 1], cell[2, 2]], dtype=np.float64)
    p = lib.pair_init()
    lib.pair_set_atom(p, len(z), len(uniq), types.ctypes.data, x.ctypes.data)
    lib.pair_set_domain(p, *[int(bool(b)) for b in pbc], lo.ctypes.data, hi.ctypes.data, float(cell[1, 0]), float(cell[2, 0]), float(cell[2, 1]))
    lib.pair_run_settings(p, 9000.0, 1600.0, damping.encode(), functional.encode())
    lib.pair_run_coeff(p, nums.ctypes.data)
    lib.pair_run_compute(p)
    e = lib.pair_get_energy(p)
    f = np.ctypeslib.as_array(lib.pair_get_force(p), shape=(len(z) * 3,)).reshape(-1, 3).copy()
    s = np.array(lib.pair_get_stress(p).contents)
    lib.pair_fin(p)
    return e, f, s


def main(out):
    lib = reference_lib(os.path.join(ROOT, 'oracle', '_ref', 'libpaird3.so'))
    data = {}
    for cells, damping in CASES:
        pos, cell, z = rocksalt_nacl(*cells, sigma=0.05, seed=11)
        e, f, s = run_reference_d3(lib, z, pos, cell, damping)
        k = case_key(cells, damping)
        data[k + '_positions'] = pos
        data[k + '_energy'] = np.float64(e)
        data[k + '_forces'] = f
        data[k + '_stress'] = s
        print(k, len(z), 'atoms, E =', e)
    for fixture, damping, functional in d3_cells.GOLDEN_CASES:
        z, pos, cell, pbc = d3_cells.FIXTURES[fixture]()
        e, f, s = run_reference_d3(lib, z, pos, cell, damping, functional, pbc)
        k = d3_cells.golden_key(fixture, damping, functional)
        data[k + '_positions'] = pos
        data[k + '_energy'] = np.float64(e)
        data[k + '_forces'] = f
        data[k + '_stress'] = s
        print(k, len(z), 'atoms, E =', e)
    if os.path.exists(out):
        # the reference adds its fp64 forces with atomics, so a rerun can differ in the last bit: values already
        # stored are kept, and the rerun's difference from them is reported
        old = np.load(out)
        for k in old.files:
            if k in data:
                d = np.abs(np.asarray(data[k], dtype=np.float64) - old[k]).max()
                print(k, 'bit-identical' if np.array_equal(old[k], data[k]) else f'rerun differs by {d:.1e} (kept)')
            data[k] = old[k]
    np.savez_compressed(out, **data)


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden', 'd3_compiled_reference.npz'))
