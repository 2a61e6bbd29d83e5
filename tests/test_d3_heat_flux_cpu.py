"""The fp64 references of the D3 heat flux (tests/d3_flux_reference.py) on the CPU:

* the atomic energies sum to the oracle's energy;
* the recursion the kernels run equals Richardson differences of the atomic energies, J_pot = sum_j [r_j dU_j(v) -
  dU_j(w^a)], on a molecule and on periodic cells through their unfolded cluster (whose U_j equal the periodic ones);
* uniform velocity c: J_pot = W c with the oracle's virial W.

Also: the C signature of s7b_d3_heat_flux and its ctypes binding."""
import os
import re

import numpy as np
import pytest

import d3_cells
from d3_flux_reference import AU, atomic_energies, difference_flux, recursion_flux, unfold
from helpers import ROOT

SMALL = dict(vdw_cutoff=400.0, cn_cutoff=225.0)         # bohr^2: unfolded clusters of ~1 500 atoms
KW = dict(vdw_cutoff=2500.0, cn_cutoff=900.0)


def _generated(pos, kw):
    return np.eye(3) * (pos.max(0) - pos.min(0) + np.sqrt(max(kw['vdw_cutoff'], kw['cn_cutoff'])) * AU + 1.0)


def _nacl_primitive():
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(1, 1, 1, sigma=0.0)
    prim = 0.5 * np.array([[0, 1, 1], [1, 0, 1], [1, 1, 0]]) * cell[0, 0]
    p = np.array([[0.0, 0.0, 0.0], [0.5 * cell[0, 0], 0.0, 0.0]]) + np.array([[0.05, -0.08, 0.03], [-0.04, 0.02, 0.09]])
    return np.array([11, 17]), p, prim @ (np.eye(3) + 0.03 * np.array([[0, 1, 0], [0, 0, -1], [1, 0, 0]])).T


def _system(name, kw):
    if name == 'nacl2':
        z, pos, cell = _nacl_primitive()
        return z, pos, cell, (True, True, True)
    z, pos, cell, pbc = d3_cells.FIXTURES[name]()
    if np.asarray(cell).sum() == 0:
        return z, pos, _generated(pos, kw), (True, True, True)
    return z, pos, cell, pbc


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('name', ['molecule', 'nacl2', 'sheared'])
def test_atomic_energies_sum_to_the_energy(name, damping):
    from oracle.d3_oracle import d3_reference
    z, pos, cell, pbc = _system(name, KW)
    E = d3_reference(z, pos, cell, pbc, damping=damping, functional='pbe', **KW)['energy']
    U = atomic_energies(z, pos, cell, pbc, damping, **KW)
    _, _, U_rec = recursion_flux(z, pos, cell, pbc, np.zeros(pos.shape), damping, **KW)
    print(f'{name} {damping}: E = {E:.12e} eV, sum U - E = {U.sum() - E:.1e}, recursion {U_rec.sum() - E:.1e}')
    assert abs(U.sum() - E) < 1e-12 * np.abs(U).sum()
    assert np.abs(U_rec - U).max() < 1e-12 * np.abs(U).sum()


def test_unfolded_cluster_has_the_periodic_atomic_energies():
    z, pos, cell, pbc = _system('nacl2', SMALL)
    U_p = atomic_energies(z, pos, cell, pbc, 'damp_bj', **SMALL)
    radius = (np.sqrt(SMALL['vdw_cutoff']) + np.sqrt(SMALL['cn_cutoff'])) * AU + 1.0
    cpos, parent = unfold(pos, cell, pbc, radius)
    c = cpos - cpos.min(0) + 5.0
    box = np.diag(cpos.max(0) - cpos.min(0) + 10.0)
    U_c = atomic_energies(z[parent], c, box, (False,) * 3, 'damp_bj', **SMALL)[:len(z)]
    print(f'cluster of {len(cpos)} atoms: max|U_cluster - U_periodic| = {np.abs(U_c - U_p).max():.1e} eV')
    assert np.abs(U_c - U_p).max() < 1e-12 * np.abs(U_p).sum()


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('name', ['molecule', 'nacl2'])
def test_recursion_equals_differences(name, damping):
    z, pos, cell, pbc = _system(name, SMALL)
    rng = np.random.RandomState(7 + 2 * (name == 'nacl2') + (damping == 'damp_zero'))
    v = rng.normal(size=pos.shape)
    J, R, _ = recursion_flux(z, pos, cell, pbc, v, damping, **SMALL)
    # the molecule's generated cell has no image in range: its cluster is the molecule itself
    ref, per = difference_flux(z, pos, cell, pbc if name != 'molecule' else (False,) * 3, v, damping, **SMALL)
    err = np.abs(J - ref).max() / np.abs(per).sum()
    err_atoms = np.abs(R - per).max() / np.abs(per).sum()
    print(f'{name} {damping}: J_pot = {J}, differences {ref}, err / sum|J_j| = {err:.1e}, per atom {err_atoms:.1e}')
    assert err < 1e-7 and err_atoms < 1e-7


def test_self_images_contribute():
    """a one-atom cell: every pair is a self image, no force, yet J_pot = W v is not zero"""
    from oracle.d3_oracle import d3_reference
    z, pos = np.array([18]), np.zeros((1, 3))
    cell = np.array([[3.6, 0.2, 0.0], [0.1, 3.9, 0.3], [0.0, -0.2, 4.2]])
    c = np.array([0.4, -0.9, 1.3])
    J, _, _ = recursion_flux(z, pos, cell, (True,) * 3, c[None], 'damp_bj', **KW)
    W = d3_reference(z, pos, cell, (True,) * 3, damping='damp_bj', functional='pbe', **KW)['sigma']
    print(f'one atom: J_pot = {J}, W c = {W.T @ c}')
    assert np.abs(W.T @ c).max() > 1e-3
    assert np.abs(J - W.T @ c).max() < 1e-10 * np.abs(W.T @ c).max()


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('name', ['sheared', 'slab', 'compressed_cs', 'nacl2'])
def test_uniform_velocity_is_virial_times_c(name, damping):
    """sum_i dU_j/dr_i = 0 leaves J_pot = W c, W = -sum vec (x) dE/dvec: the oracle's sigma, transposed"""
    from oracle.d3_oracle import d3_reference
    z, pos, cell, pbc = _system(name, KW)
    c = np.array([0.3, -1.1, 0.7])
    J, _, _ = recursion_flux(z, pos, cell, pbc, np.tile(c, (len(z), 1)), damping, **KW)
    W = d3_reference(z, pos, cell, pbc, damping=damping, functional='pbe', **KW)['sigma']
    err = np.abs(J - W.T @ c).max() / np.abs(W.T @ c).max()
    print(f'{name} {damping}: J_pot = {J}, W c = {W.T @ c}, rel err {err:.1e}')
    assert err < 1e-10


def test_signature():
    hdr = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API int s7b_d3_heat_flux\(([^)]*)\)', hdr)
    assert m, 's7b_d3_heat_flux is not declared'
    args = [a.strip() for a in m.group(1).split(',')]
    assert args == ['S7bD3* d3', 'const double* d_v', 'double* d_jpot', 'double* d_ju', 'void* stream']
    src = open(os.path.join(ROOT, 'sevenn_b200', 'engine.py')).read()
    assert "lib.s7b_d3_heat_flux.argtypes = [vp, vp, vp, vp, vp]" in src
    assert "'s7b_d3_heat_flux'" in src
