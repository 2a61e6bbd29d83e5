"""The fp64 reference of D3's per-atom centroid virial (tests/d3_centroid_reference.py) on the CPU:

* J_pot is linear in the velocities, so J_pot(e_(i,b)) of ``recursion_flux`` (pinned to Richardson differences of
  the atomic energies in tests/test_d3_heat_flux_cpu.py) is column b of Wc_i: the reference equals those 3n columns;
* sum_i Wc_i is the oracle's virial, a one-atom cell of self images only included;
* with the CN cutoff below every interatomic distance the CN part vanishes and Wc_i is the symmetric pair row.

Also: the C signature of s7b_d3_centroid_virial and its ctypes binding."""
import os
import re

import numpy as np
import pytest

from d3_centroid_reference import centroid_virials, pairwise_split
from d3_flux_reference import recursion_flux
from helpers import ROOT
from test_d3_heat_flux_cpu import _system

SMALL = dict(vdw_cutoff=400.0, cn_cutoff=225.0)         # bohr^2
KW = dict(vdw_cutoff=2500.0, cn_cutoff=900.0)


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('name', ['molecule', 'nacl2'])
def test_reference_equals_one_hot_flux_columns(name, damping):
    z, pos, cell, pbc = _system(name, SMALL)
    n = len(z)
    W = centroid_virials(z, pos, cell, pbc, damping, **SMALL)
    cols = np.zeros((n, 3, 3))
    for i in range(n):
        for b in range(3):
            v = np.zeros((n, 3))
            v[i, b] = 1.0
            cols[i, :, b] = recursion_flux(z, pos, cell, pbc, v, damping, **SMALL)[0]
    err = np.abs(W - cols).max() / np.abs(W).sum()
    print(f'{name} {damping}: max|Wc - flux columns| / sum|Wc| = {err:.1e}')
    assert err < 1e-12


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('name', ['molecule', 'nacl2', 'sheared', 'slab', 'compressed_cs'])
def test_sum_is_the_virial(name, damping):
    from oracle.d3_oracle import d3_reference
    z, pos, cell, pbc = _system(name, KW)
    W = centroid_virials(z, pos, cell, pbc, damping, **KW)
    sigma = d3_reference(z, pos, cell, pbc, damping=damping, functional='pbe', **KW)['sigma']
    err = np.abs(W.sum(0) - sigma).max() / np.abs(sigma).max()
    print(f'{name} {damping}: max|sum_i Wc_i - W| / max|W| = {err:.1e}')
    assert err < 1e-10


def test_one_atom_cell():
    """every pair is a self image: no force, yet the atom's Wc is the whole virial, CN part included"""
    from oracle.d3_oracle import d3_reference
    z, pos = np.array([14]), np.zeros((1, 3))
    cell = np.array([[3.6, 0.2, 0.0], [0.1, 3.9, 0.3], [0.0, -0.2, 4.2]])
    W, _, cnp = centroid_virials(z, pos, cell, (True,) * 3, 'damp_bj', **KW, parts=True)
    sigma = d3_reference(z, pos, cell, (True,) * 3, damping='damp_bj', functional='pbe', **KW)['sigma']
    print(f'one atom: Wc = {W[0].ravel()}, CN part {cnp[0].ravel()}')
    assert np.abs(cnp).max() > 1e-2 * np.abs(W).max()
    assert np.abs(W[0] - sigma).max() < 1e-12 * np.abs(sigma).max()


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
def test_no_cn_pairs_leaves_the_pair_row(damping):
    """cn_cutoff below every distance: CN is 0 and constant, the CN part is zero and Wc_i is spair_i, symmetric"""
    z, pos, cell, pbc = _system('sheared', KW)
    kw = dict(vdw_cutoff=KW['vdw_cutoff'], cn_cutoff=0.25)
    W, direct, cnp = centroid_virials(z, pos, cell, pbc, damping, **kw, parts=True)
    split = pairwise_split(z, pos, cell, pbc, damping, **kw)
    assert not cnp.any()
    assert np.array_equal(W, direct) and np.array_equal(W, split)
    assert np.abs(W - W.transpose(0, 2, 1)).max() < 1e-14 * np.abs(W).max()


@pytest.mark.parametrize('name', ['sheared', 'nacl2'])
def test_pairwise_split(name):
    """the forward's per-atom rows spair + schain sum to the same virial.  Per atom they differ from Wc for a many-body
    energy (the sheared mixed cell), but not in rock salt: there CN (~5-9) lies far above the references of Na and Cl
    (0 and ~1), the weights are one-hot and dC6/dCN = 0, so D3 is a pair potential and the split is exact."""
    z, pos, cell, pbc = _system(name, KW)
    W = centroid_virials(z, pos, cell, pbc, 'damp_bj', **KW)
    split = pairwise_split(z, pos, cell, pbc, 'damp_bj', **KW)
    sum_err = np.abs(split.sum(0) - W.sum(0)).max() / np.abs(W.sum(0)).max()
    per = np.abs(split - W).max() / np.abs(W).max()
    print(f'{name}: sums agree to {sum_err:.1e}, per atom max|split - Wc| / max|Wc| = {per:.2e}')
    assert sum_err < 1e-10
    assert per > 1e-2 if name == 'sheared' else per < 1e-12


def test_signature():
    hdr = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API int s7b_d3_centroid_virial\(([^)]*)\)', hdr)
    assert m, 's7b_d3_centroid_virial is not declared'
    assert [a.strip() for a in m.group(1).split(',')] == ['S7bD3* d3', 'double* d_out', 'void* stream']
    src = open(os.path.join(ROOT, 'sevenn_b200', 'engine.py')).read()
    assert "lib.s7b_d3_centroid_virial.argtypes = [vp, vp, vp]" in src
    assert "'s7b_d3_centroid_virial'" in src
