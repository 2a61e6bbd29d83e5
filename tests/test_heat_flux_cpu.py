"""The fp64 reference heat flux (tests/flux_reference.py) on the CPU, against two closed forms:

* uniform velocity c: sum_i dU_j/dr_i = 0 (translation invariance) leaves J_pot = sum_i r_i (F_i . c) = W c, with
  W = sum_i r_i (x) F_i = -sum_e vec_e (x) f_e the 3x3 virial (f_e = dE/dvec_e);
* a one-layer model, where U_j depends on its own edges only: J_pot = -sum_e vec_e (f_e . v_src(e)), the pairwise
  (atomic-virial) form, exact here and only here.

Periodic cells are evaluated on their unfolded cluster, whose U_j must first equal the periodic U_j.  Also: the C
signature of s7b_engine_heat_flux and its ctypes binding."""
import os
import re

import numpy as np
import pytest

from flux_reference import atomic_energies, cluster_graph, make_oracle, reference_flux, unfold
from helpers import ROOT, model_weights


def _species(meta, z):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z], dtype=np.int64)


def _one_layer(tmp):
    from synthetic_models import convert, layered, write_checkpoint
    arch = layered('flux_one_layer', 2, 2, ['32x0e', '32x0e'])
    return convert(write_checkpoint(os.path.join(tmp, 'flux1.pth'), arch, seed=11), arch)


def _edge_forces(o, species, ei, ev):
    out = o.forward(species, ei, ev)
    return out['edge_force'].detach().cpu().numpy().astype(np.float64)


def test_uniform_velocity_is_virial_times_c():
    from sevenn_b200.neighbors import diamond_si
    from sevenn_b200.spec import build_spec
    meta, arrays = model_weights('sevennet_0')
    spec = build_spec(meta)
    o = make_oracle(meta, arrays, 'cpu')
    pos, _, z = diamond_si(1, 1, 1, sigma=0.08, seed=3)
    species = _species(meta, z)
    c = np.array([0.3, -1.1, 0.7])
    J, _ = reference_flux(o, spec, species, pos, np.tile(c, (len(pos), 1)))
    ei, ev = cluster_graph(pos - pos.mean(0), spec.cutoff)
    W = -ev.T @ _edge_forces(o, species, ei, ev)
    err = np.abs(J - W @ c).max() / np.abs(W @ c).max()
    print(f'uniform c: J_pot = {J}, W c = {W @ c}, rel err {err:.1e}')
    assert err < 1e-7


def test_one_layer_is_the_atomic_virial_form(tmp_path):
    from sevenn_b200.neighbors import build_graph, diamond_si
    from sevenn_b200.spec import build_spec
    meta, arrays = _one_layer(str(tmp_path))
    spec = build_spec(meta)
    assert len(spec.layers) == 1
    o = make_oracle(meta, arrays, 'cpu')
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.08, seed=5)
    species = _species(meta, z)
    v = np.random.RandomState(2).normal(size=pos.shape)
    # the periodic cell through its unfolded cluster: the cluster's U_j equal the periodic ones
    ei_p, ev_p = build_graph(pos, cell, True, spec.cutoff)
    U_p = atomic_energies(o, species, ei_p, ev_p)
    cpos, parent = unfold(pos, cell, spec.cutoff + 1.0)
    ei_c, ev_c = cluster_graph(cpos, spec.cutoff)
    U_c = atomic_energies(o, species[parent], ei_c, ev_c)[:len(pos)]
    print(f'cluster of {len(cpos)} atoms: max|U_cluster - U_periodic| = {np.abs(U_c - U_p).max():.1e}')
    assert np.abs(U_c - U_p).max() < 1e-10
    J, per = reference_flux(o, spec, species[parent], cpos, v[parent], n_cell=len(pos))
    f = _edge_forces(o, species, ei_p, ev_p)
    J_pair = -(ev_p * (f * v[ei_p[1]]).sum(1, keepdims=True)).sum(0)
    err = np.abs(J - J_pair).max() / np.abs(per).sum()
    print(f'one layer: J_pot = {J}, pairwise form {J_pair}, err / sum|J_j| = {err:.1e}')
    assert err < 1e-8


def test_signature():
    hdr = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API int s7b_engine_heat_flux\(([^)]*)\)', hdr)
    assert m, 's7b_engine_heat_flux is not declared'
    args = [a.strip() for a in m.group(1).split(',')]
    assert args == ['S7bEngine* eng', 'const float* d_v', 'double* d_jpot', 'double* d_ju', 'void* stream']
    src = open(os.path.join(ROOT, 'sevenn_b200', 'engine.py')).read()
    assert "lib.s7b_engine_heat_flux.argtypes = [vp, vp, vp, vp, vp]" in src
    assert "'s7b_engine_heat_flux'" in src
