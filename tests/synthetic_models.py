"""Seeded synthetic SevenNet checkpoints of architectures other than SevenNet-0 / SevenNet-l3i5, written in the
reference's checkpoint layout (config + model_state_dict with the reference's key names and Wigner-3j buffers), so
that the converter, the calculator and export_flat all see them as a user's trained model.

The stored linear and radial-MLP weights are N(0, 1) like e3nn's initialisation; e3nn (and the oracle) divide
by sqrt(fan_in) in the forward, so each layer acts with the ~1/sqrt(fan_in) scale of a trained model.  The shift
(-3 .. -6 eV per species), scale (~1.5) and convolution denominators (~ neighbour count of the test systems) are
realistic, so that energies are O(eV/atom) and absolute tolerances mean what they mean for the shipped models.

  id  irreps of the mid layers          lmax_edge / lmax_node  layers  what it runs
  A   32x0e+32x1e+32x2e                  2 / 2                  3       base-preset widths, runtime-width kernels
  B   64x0e+32x1e                        1 / 1                  4       groups (1, 1), (1, 0)
  C   128x0e+64x1e+32x2e                 3 / 2                  3       group (3, 2) at SevenNet-0 widths
  D   256x0e+96x1e+64x2e+32x3e           3 / 3                  2       split backward: 256 (NV = 2) and 96 (16 lanes)

``layered`` describes any other architecture by the irreps of every layer (tests/test_conv_table_gpu.py).
"""
from __future__ import annotations

import numpy as np

ELEMENTS = ['H', 'C', 'O', 'Na', 'Si', 'Cl', 'Hf']
NUMBERS = [1, 6, 8, 11, 14, 17, 72]

ARCHS = {
    'A': dict(mid='32x0e+32x1e+32x2e', lmax_edge=2, lmax_node=2, layers=3),
    'B': dict(mid='64x0e+32x1e', lmax_edge=1, lmax_node=1, layers=4),
    'C': dict(mid='128x0e+64x1e+32x2e', lmax_edge=3, lmax_node=2, layers=3),
    'D': dict(mid='256x0e+96x1e+64x2e+32x3e', lmax_edge=3, lmax_node=3, layers=2),
}


def layered(name: str, lmax_edge: int, lmax_node: int, irreps) -> dict:
    """An architecture of any lmax_edge / lmax_node with the irreps of every layer given (``irreps[t]``: the input
    of layer t, the last entry the output of the last layer), for ``reference_checkpoint`` in place of an ARCHS id"""
    return dict(name=name, lmax_edge=lmax_edge, lmax_node=lmax_node, layers=len(irreps) - 1, irreps=list(irreps))


def _arch(arch):
    return ARCHS[arch] if isinstance(arch, str) else arch


def _name(arch):
    return arch if isinstance(arch, str) else arch['name']


def irreps_per_layer(arch):
    a = _arch(arch)
    if 'irreps' in a:
        return list(a['irreps'])
    s0 = a['mid'].split('+')[0]
    return [s0] + [a['mid']] * (a['layers'] - 1) + [s0]


def reference_checkpoint(arch, seed: int = 0, parity: bool = False) -> dict:
    """{'config', 'model_state_dict'} of a reference checkpoint (torch tensors) for architecture ``arch``: an ARCHS
    id or a ``layered`` description"""
    import torch
    from sevenn_b200.cg import wigner_3j
    from sevenn_b200.checkpoint import random_weights
    from sevenn_b200.spec import build_spec, parse_even_irreps

    a = _arch(arch)
    irreps = irreps_per_layer(arch)
    cutoff = 5.0
    meta = dict(name=f'synthetic_{_name(arch)}', cutoff=cutoff, cutoff_fn='poly_cut', cutoff_on=0.0, poly_p=6, n_basis=8,
                lmax_filter=a['lmax_edge'], num_species=len(NUMBERS),
                type_map={str(z): i for i, z in enumerate(NUMBERS)}, chemical_species=ELEMENTS,
                radial_hidden=[64, 64], irreps_per_layer=irreps,
                readout_hidden=parse_even_irreps(irreps[-1])[0] // 2)
    spec = build_spec(meta)
    w = random_weights(meta, seed=seed)
    rng = np.random.RandomState(1000 + seed)
    t = lambda v: torch.tensor(np.asarray(v, dtype=np.float32))
    sd = {
        'edge_embedding.basis_function.coeffs': t(w['bessel_coeffs']),
        'onehot_to_feature_x.linear.weight': t(w['embed']),
        'reduce_input_to_hidden.linear.weight': t(w['readout1']),
        'reduce_hidden_to_energy.linear.weight': t(w['readout2']),
        'rescale_atomic_energy.shift': t(rng.uniform(-6.0, -3.0, size=len(NUMBERS))),
        'rescale_atomic_energy.scale': t(rng.uniform(1.2, 1.8, size=len(NUMBERS))),
    }
    for L in spec.layers:
        k = L.t
        sd[f'{k}_self_connection_intro.linear.weight'] = t(w[f'{k}.sc'])
        sd[f'{k}_self_interaction_1.linear.weight'] = t(w[f'{k}.si1'])
        sd[f'{k}_self_interaction_2.linear.weight'] = t(w[f'{k}.si2'])
        sd[f'{k}_convolution.denominator'] = t([rng.uniform(20.0, 40.0)])
        for j in range(3):
            sd[f'{k}_convolution.weight_nn.layer{j}.weight'] = t(w[f'{k}.mlp{j}'])
        for p in L.paths:
            sd[f'{k}_convolution.convolution._compiled_main_left_right._w3j_{p.l1}_{p.l2}_{p.l3}'] = \
                torch.tensor(wigner_3j(p.l1, p.l2, p.l3), dtype=torch.float32)
    config = {
        'version': '0.11.2', 'is_parity': parity, 'self_connection_type': 'linear', 'use_bias_in_linear': False,
        'act_gate': {'e': 'silu', 'o': 'tanh'}, 'act_scalar': {'e': 'silu', 'o': 'tanh'}, 'act_radial': 'silu',
        '_normalize_sph': True, 'num_convolution_layer': a['layers'], 'lmax': max(a['lmax_edge'], a['lmax_node']),
        'lmax_edge': a['lmax_edge'], 'lmax_node': a['lmax_node'], 'irreps_manual': irreps,
        'channel': parse_even_irreps(irreps[0])[0], 'cutoff': cutoff,
        'cutoff_function': {'cutoff_function_name': 'poly_cut', 'poly_cut_p_value': 6},
        'radial_basis': {'radial_basis_name': 'bessel', 'bessel_basis_num': 8},
        '_number_of_species': len(NUMBERS), '_type_map': {z: i for i, z in enumerate(NUMBERS)},
        'chemical_species': ELEMENTS, 'weight_nn_hidden_neurons': [64, 64],
    }
    return {'config': config, 'model_state_dict': sd}


def write_checkpoint(path, arch, seed: int = 0, parity: bool = False) -> str:
    import torch
    torch.save(reference_checkpoint(arch, seed, parity), str(path))
    return str(path)


def convert(path, arch):
    """(meta, arrays) of a checkpoint written by write_checkpoint, through the reference-checkpoint converter"""
    from sevenn_b200.checkpoint import convert_reference_checkpoint
    return convert_reference_checkpoint(str(path), f'synthetic_{_name(arch)}')
