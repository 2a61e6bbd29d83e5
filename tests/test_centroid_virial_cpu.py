"""The fp64 reference centroid virial (tests/centroid_reference.py) on the CPU, against the identities of DESIGN.md
§8.5 on molecules and periodic cells, for linear and species-wise ('nequip') self-connection models:

1. sum_i Wc_i = W, the oracle's virial -sum_e vec_e (x) f_e (f_e = dE/dvec_e);
2. sum_i Wc_i v_i = J_pot of the reference heat flux (tests/flux_reference.py, central differences) for random v;
3. a one-layer model: Wc_k = -sum_{e: neighbour k} vec_e (x) f_e, whose (xx, yy, zz, xy, yz, zx) entries are the
   oracle's atomic_virial row of k.

Periodic cells are evaluated on their unfolded cluster.  Also: the C signatures and their ctypes bindings."""
import os
import re

import numpy as np
import pytest

from centroid_reference import reference_centroid_cell
from flux_reference import make_oracle, reference_flux, unfold
from helpers import ROOT, model_weights


def _species(meta, z):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z], dtype=np.int64)


def _layered(tmp, name, irreps, seed=11):
    from synthetic_models import convert, layered, write_checkpoint
    arch = layered(name, 2, 2, irreps)
    return convert(write_checkpoint(os.path.join(tmp, f'{name}.pth'), arch, seed=seed), arch)


def _nequip(tmp, arch='B', seed=5):
    """synthetic model B (4 layers, lmax 1) with the species-wise self-connection"""
    from synthetic_nequip import convert, write_nequip_checkpoint
    return convert(write_nequip_checkpoint(os.path.join(tmp, f'wc_nequip_{arch}.pth'), arch, seed=seed), arch)


def _virial3(o, species, ei, ev):
    w = o.forward(species, ei, ev)['virial'].detach().cpu().numpy().astype(np.float64)
    return np.array([[w[0], w[3], w[5]], [w[3], w[1], w[4]], [w[5], w[4], w[2]]])


def _check_identities(meta, arrays, pos, cell, z, seed):
    from sevenn_b200.neighbors import build_graph
    from sevenn_b200.spec import build_spec
    from flux_reference import cluster_graph
    spec = build_spec(meta)
    o = make_oracle(meta, arrays, 'cpu')
    species = _species(meta, z)
    Wc = reference_centroid_cell(o, spec, species, pos, cell)
    scale = np.abs(Wc).sum()
    # 1: the virial
    if cell is None:
        ei, ev = cluster_graph(pos - pos.mean(0), spec.cutoff)
    else:
        ei, ev = build_graph(pos, cell, True, spec.cutoff)
    W = _virial3(o, species, ei, ev)
    err1 = np.abs(Wc.sum(0) - W).max() / scale
    asym = np.abs(Wc - Wc.transpose(0, 2, 1)).max() / np.abs(Wc).max()
    # 2: the heat flux for a random v
    v = np.random.RandomState(seed).normal(size=pos.shape)
    if cell is None:
        J, per = reference_flux(o, spec, species, pos, v)
    else:
        cpos, parent = unfold(pos, cell, len(spec.layers) * spec.cutoff + 1.0)
        J, per = reference_flux(o, spec, species[parent], cpos, v[parent], n_cell=len(pos))
    Jc = np.einsum('iab,ib->a', Wc, v)
    err2 = np.abs(Jc - J).max() / np.abs(per).sum()
    print(f'{meta.get("self_connection", "linear")} {"cluster" if cell is None else "periodic"}: '
          f'|sum Wc - W| / sum|Wc| = {err1:.1e}, |sum Wc v - J_pot| / sum|J_j| = {err2:.1e}, '
          f'max |Wc - Wc^T| / max |Wc| = {asym:.1e}')
    assert err1 < 1e-10         # W is symmetric, so the sum is, although no single Wc_i is (asym)
    assert err2 < 1e-7


@pytest.mark.parametrize('sc', ['linear', 'nequip'])
def test_identities_cluster(sc, tmp_path):
    from sevenn_b200.neighbors import diamond_si
    if sc == 'linear':
        meta, arrays = model_weights('sevennet_0')
    else:
        meta, arrays = _nequip(str(tmp_path))
    pos, _, z = diamond_si(1, 1, 1, sigma=0.08, seed=3)
    if sc == 'nequip':
        from synthetic_models import NUMBERS
        z = np.array([NUMBERS[i % 3] for i in range(len(pos))])
    _check_identities(meta, arrays, pos, None, z, seed=1)


@pytest.mark.parametrize('sc', ['linear', 'nequip'])
def test_identities_periodic(sc, tmp_path):
    from sevenn_b200.neighbors import diamond_si
    from synthetic_models import NUMBERS
    if sc == 'linear':
        meta, arrays = _layered(str(tmp_path), 'wc_two_layers', ['32x0e', '32x0e+32x1e+32x2e', '32x0e'])
    else:
        meta, arrays = _nequip(str(tmp_path))
    pos, cell, _ = diamond_si(1, 1, 1, sigma=0.08, seed=5)
    z = np.array([NUMBERS[i % 3] for i in range(len(pos))])
    _check_identities(meta, arrays, pos, cell, z, seed=2)


def test_one_layer_is_the_atomic_virial(tmp_path):
    from sevenn_b200.neighbors import build_graph, diamond_si
    from sevenn_b200.spec import build_spec
    meta, arrays = _layered(str(tmp_path), 'wc_one_layer', ['32x0e', '32x0e'])
    spec = build_spec(meta)
    assert len(spec.layers) == 1
    o = make_oracle(meta, arrays, 'cpu')
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.08, seed=5)
    species = _species(meta, z)
    Wc = reference_centroid_cell(o, spec, species, pos, cell)
    ei, ev = build_graph(pos, cell, True, spec.cutoff)
    out = o.forward(species, ei, ev)
    f = out['edge_force'].detach().cpu().numpy().astype(np.float64)
    pair = np.zeros((len(pos), 3, 3))
    np.add.at(pair, ei[1], -ev[:, :, None] * f[:, None, :])
    av = out['atomic_virial'].detach().cpu().numpy().astype(np.float64)
    rows = np.stack([Wc[:, 0, 0], Wc[:, 1, 1], Wc[:, 2, 2], Wc[:, 0, 1], Wc[:, 1, 2], Wc[:, 2, 0]], 1)
    scale = np.abs(Wc).sum()
    err = np.abs(Wc - pair).max() / scale
    err_av = np.abs(rows - av).max() / scale
    print(f'one layer: |Wc - pairwise| / sum|Wc| = {err:.1e}, |rows - atomic_virial| / sum|Wc| = {err_av:.1e}')
    assert err < 1e-10 and err_av < 1e-10


def test_signature():
    hdr = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    src = open(os.path.join(ROOT, 'sevenn_b200', 'engine.py')).read()
    for name, last in (('s7b_engine_centroid_virial', 'double* d_out'),
                       ('s7b_engine_centroid_virial_host', 'double* host_out')):
        m = re.search(rf'S7B_API int {name}\(([^)]*)\)', hdr)
        assert m, f'{name} is not declared'
        assert [a.strip() for a in m.group(1).split(',')] == ['S7bEngine* eng', last, 'void* stream']
        assert f'lib.{name}.argtypes = [vp, vp, vp]' in src
        assert f"'{name}'" in src
