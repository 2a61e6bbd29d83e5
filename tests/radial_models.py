"""Seeded synthetic checkpoints in the reference's layout whose radial part differs from the shipped models'
(cutoff 5.0, XPLOR 4.5 or poly_cut p = 6, 8 Bessel functions at n pi / rc, radial MLP [64, 64]).

  id  cutoff  envelope          n_basis  radial hidden  arch  why
  R1  6.0     XPLOR r_on 5.5    8        [64, 64]       B     the multi_modal / mf_ompa presets: r_on falls between
                                                              knots of a 2000-interval table
  R2  5.0     XPLOR r_on 4.5    8        [64, 64]       B     r_on on a knot of the 2000-interval table (control)
  R3  4.0     poly_cut p = 3    8        [64, 64]       A     short cutoff, low-order polynomial envelope
  R4  5.3     poly_cut p = 9    6        [48, 96]       A     cutoff not exact in fp32, n_basis and widths that are
                                                              not multiples of 4 / 8
  R5  5.3     XPLOR r_on 4.8    5        [50, 70]       B     r_on off the 2000-interval grid, odd radial GEMM shapes

The Bessel frequencies are n pi / rc perturbed by up to +-5 %, as training leaves them; the radial MLP weights are
N(0, 1) like e3nn's initialisation.  Everything else comes from synthetic_models.reference_checkpoint (archs A, B:
small widths keep the fp64 oracle cheap).
"""
from __future__ import annotations

import numpy as np

from synthetic_models import reference_checkpoint

CONFIGS = {
    'R1': dict(arch='B', cutoff=6.0, cutoff_fn='XPLOR', cutoff_on=5.5, n_basis=8, hidden=[64, 64]),
    'R2': dict(arch='B', cutoff=5.0, cutoff_fn='XPLOR', cutoff_on=4.5, n_basis=8, hidden=[64, 64]),
    'R3': dict(arch='A', cutoff=4.0, cutoff_fn='poly_cut', poly_p=3, n_basis=8, hidden=[64, 64]),
    'R4': dict(arch='A', cutoff=5.3, cutoff_fn='poly_cut', poly_p=9, n_basis=6, hidden=[48, 96]),
    'R5': dict(arch='B', cutoff=5.3, cutoff_fn='XPLOR', cutoff_on=4.8, n_basis=5, hidden=[50, 70]),
}


def radial_checkpoint(cid: str, hidden=None) -> dict:
    """{'config', 'model_state_dict'} of config ``cid``; ``hidden`` overrides the radial MLP's hidden widths"""
    import torch
    c = CONFIGS[cid]
    seed = 10 + sorted(CONFIGS).index(cid)
    ck = reference_checkpoint(c['arch'], seed=seed)
    cfg, sd = ck['config'], ck['model_state_dict']
    hidden = list(c['hidden'] if hidden is None else hidden)
    rc, nb = c['cutoff'], c['n_basis']
    cfg['cutoff'] = rc
    if c['cutoff_fn'] == 'XPLOR':
        cfg['cutoff_function'] = {'cutoff_function_name': 'XPLOR', 'cutoff_on': c['cutoff_on']}
    else:
        cfg['cutoff_function'] = {'cutoff_function_name': 'poly_cut', 'poly_cut_p_value': c['poly_p']}
    cfg['radial_basis'] = {'radial_basis_name': 'bessel', 'bessel_basis_num': nb}
    cfg['weight_nn_hidden_neurons'] = hidden
    rng = np.random.RandomState(500 + seed)
    t = lambda v: torch.tensor(np.asarray(v, dtype=np.float32))
    sd['edge_embedding.basis_function.coeffs'] = t(np.arange(1, nb + 1) * np.pi / rc * (1 + rng.uniform(-0.05, 0.05, nb)))
    for k in range(cfg['num_convolution_layer']):
        n_out = sd[f'{k}_convolution.weight_nn.layer2.weight'].shape[1]
        for j in range(3):
            sd.pop(f'{k}_convolution.weight_nn.layer{j}.weight')
        dims = [nb] + hidden + [n_out]
        for j in range(len(dims) - 1):
            sd[f'{k}_convolution.weight_nn.layer{j}.weight'] = t(rng.standard_normal((dims[j], dims[j + 1])))
    return ck


def write_radial_checkpoint(path, cid: str, hidden=None) -> str:
    import torch
    torch.save(radial_checkpoint(cid, hidden), str(path))
    return str(path)


def convert_radial(path, cid: str):
    """(meta, arrays) through the reference-checkpoint converter"""
    from sevenn_b200.checkpoint import convert_reference_checkpoint
    return convert_reference_checkpoint(str(path), f'radial_{cid}')
