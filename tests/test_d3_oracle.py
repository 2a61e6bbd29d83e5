"""The D3 CPU oracle (oracle/d3_oracle.py, fp64 numpy restatement of sevenn/pair_e3gnn/pair_d3_for_ase.cu)
against the reference's own golden values, tests/unit_tests/test_calculator.py:192-238 (PBE, Becke-Johnson).

Tolerances: forces agree to 3e-8 eV/A and the H2O energy to 5e-7 relative.  The NaCl energy / stress of the
reference are 4.5e-5 / 1.8e-5 (relative) smaller in magnitude than the fp64 sums: the reference accumulates the
~130 000 lattice images of every atom pair in a float (``disp_local``, pair_d3_for_ase.cu:1560,1700), and the
far images (each ~6e-8 of the running sum, i.e. at the fp32 rounding threshold) are partly absorbed.  The
oracle keeps the exact sum; the test bounds the difference and checks its sign."""
import os

import numpy as np
import pytest

import d3_cells as C
from oracle.d3_oracle import ase_results, d3_reference

NACL = dict(numbers=[11, 17], positions=[[0.0, 0.0, 0.0], [2.815, 0.0, 0.0]],
            cell=[[1.0, 2.815, 2.815], [2.815, 0.0, 2.815], [2.815, 2.815, 0.0]])
NACL_REF = dict(energy=-0.531393751583389,
                forces=[[-0.00570205, 0.00107457, 0.00107459], [0.00570205, -0.00107457, -0.00107459]],
                stress=[1.52403705e-02, 1.50417333e-02, 1.50417321e-02, -3.22684163e-05, -5.05532863e-05, -5.05586994e-05])
H2O_POS = np.array([[0.0, 0.2, 0.12], [0.0, 0.76, -0.48], [0.0, -0.76, -0.48]])
H2O_REF = dict(energy=-0.009889134535170716,
               forces=[[0.0, 2.04263840e-03, 1.27477674e-03], [0.0, -9.90038901e-05, 1.18046682e-06],
                       [0.0, -1.94363451e-03, -1.27595721e-03]])


def h2o_cell():
    # D3Calculator.calculate builds this cell for a molecule without one (sevenn/calculator.py:534-547)
    cut = np.sqrt(9000.0) * 0.52917726
    return np.diag(H2O_POS.max(0) - H2O_POS.min(0) + cut + 1.0)


def test_nacl_golden():
    r = ase_results(**NACL)
    assert np.allclose(r['forces'], NACL_REF['forces'], atol=5e-8, rtol=0)
    rel = r['energy'] / NACL_REF['energy'] - 1.0
    assert 0.0 < rel < 1e-4                      # exact sum is slightly MORE negative than the float-accumulated one
    assert np.allclose(r['stress'], NACL_REF['stress'], rtol=5e-5, atol=2e-8)


def test_h2o_golden():
    r = ase_results([8, 1, 1], H2O_POS, h2o_cell())
    assert abs(r['energy'] / H2O_REF['energy'] - 1.0) < 2e-6
    assert np.allclose(r['forces'], H2O_REF['forces'], atol=1e-7, rtol=0)


def test_forces_are_the_energy_gradient():
    rng = np.random.RandomState(0)
    cell = np.array([[7.0, 0.3, 0.0], [0.0, 6.5, 0.4], [0.2, 0.0, 7.5]])
    z = np.array([11, 17, 8, 1, 14, 14])
    pos = rng.uniform(0, 6, size=(6, 3))
    for damping in ('damp_bj', 'damp_zero'):
        kw = dict(damping=damping, vdw_cutoff=900.0, cn_cutoff=400.0)
        base = d3_reference(z, pos, cell, **kw)
        for (a, k) in ((0, 0), (3, 2), (5, 1)):
            h = 1e-4
            p1, p2 = pos.copy(), pos.copy()
            p1[a, k] += h
            p2[a, k] -= h
            fd = -(d3_reference(z, p1, cell, **kw)['energy'] - d3_reference(z, p2, cell, **kw)['energy']) / (2 * h)
            # the cutoffs are sharp: pairs crossing them make the energy non-smooth at the 1e-7 level
            assert abs(fd - base['forces'][a, k]) < 2e-6, (damping, a, k, fd, base['forces'][a, k])
        assert np.abs(base['forces'].sum(0)).max() < 1e-12
        assert np.allclose(base['sigma'], base['sigma'].T, atol=1e-12)


@pytest.mark.parametrize('fixture,damping,functional', C.GOLDEN_CASES)
def test_matches_compiled_reference_edge_cells(fixture, damping, functional):
    """The oracle against stored outputs of the reference's compiled D3 (tools/make_d3_golden.py) on a sheared
    cell, a slab, a compressed Cs cell (weight sums below 1e-300) and 16 species, each with a functional at an
    extreme of the table.  Measured: energy within 1.8e-6 (relative), forces within 2.7e-6 and stress within
    2.0e-6 of their largest component; the reference's fp32 image sums (see the module docstring) account for
    that, most on the 5.75 A Cs cell with its ~12 000 lattice images.  Bounds 1e-5."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'd3_compiled_reference.npz'))
    k = C.golden_key(fixture, damping, functional)
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    assert np.array_equal(pos, g[k + '_positions'])
    r = d3_reference(z, pos, cell, pbc, damping=damping, functional=functional)
    s = r['sigma']
    s6 = np.array([s[0, 0], s[1, 1], s[2, 2], s[0, 1], s[0, 2], s[1, 2]])
    f_ref, s_ref = g[k + '_forces'], g[k + '_stress']
    assert abs(r['energy'] / float(g[k + '_energy']) - 1.0) < 1e-5
    assert np.abs(r['forces'] - f_ref).max() < 1e-5 * np.abs(f_ref).max()
    assert np.abs(s6 - s_ref).max() < 1e-5 * np.abs(s_ref).max()
