"""Checkpoint reading: reference ``.pth`` -> a plain dict of numpy weights + JSON meta
(``.npz``), the only model format the engine, the oracle and the GPU box ever see.

Restates the parts of the reference loader that matter for inference
(``sevenn/checkpoint.py:286-370``, ``sevenn/scripts/backward_compatibility.py:79-184``):

* state-dict key names of >= 0.10 checkpoints (older "space" names are mapped),
* for checkpoints older than 0.11.0 the last radial-MLP layer's columns are stored in
  instruction-creation order and are permuted block-by-block into i_out-sorted order
  (``backward_compatibility.py:99-141``),
* where a checkpoint's stored Wigner-3j buffer is the negative of the current convention
  (``sevenn_b200.cg.wigner_3j``) the matching weight block is negated -- the same fix the
  reference applies (``backward_compatibility.py:127-134``) so that every consumer can use one
  set of coupling tensors.

The weights stay in e3nn's flat layout here (canonical form).  ``sevenn_b200.engine`` repacks
them for the GPU; ``oracle/oracle.py`` consumes them as they are.
"""
from __future__ import annotations

import io
import json
import os
from typing import Dict, Tuple

import numpy as np

from .cg import wigner_3j
from .spec import ModelSpec, build_spec, check_sc_weight, parse_even_irreps, sc_numel


def _version_tuple(v: str) -> Tuple[int, ...]:
    return tuple(int(x) for x in v.split('.')[:3])


_OLD_NAMES = {
    'EdgeEmbedding': 'edge_embedding',
    'reducing nn input to hidden': 'reduce_input_to_hidden',
    'reducing nn hidden to energy': 'reduce_hidden_to_energy',
    'rescale atomic energy': 'rescale_atomic_energy',
}


def convert_reference_checkpoint(path: str, name: str) -> Tuple[dict, Dict[str, np.ndarray]]:
    """Read a reference checkpoint with plain ``torch.load`` (no sevenn/e3nn import needed:
    the files pickle only tensors and builtins) and return ``(meta, arrays)``."""
    import torch

    try:       # the files hold tensors, builtins and a few numpy scalars/arrays: the restricted unpickler
        # with numpy's array reconstruction allow-listed is enough (no arbitrary code execution)
        import numpy._core.multiarray as ma
        allow = [(ma._reconstruct, 'numpy.core.multiarray._reconstruct'), (ma.scalar, 'numpy.core.multiarray.scalar'),
                 ma._reconstruct, ma.scalar, np.ndarray, np.dtype]
        allow += [type(np.dtype(t)) for t in ('f4', 'f8', 'i4', 'i8', 'b1', 'U1', 'S1')]
        with torch.serialization.safe_globals(allow):
            ck = torch.load(path, map_location='cpu', weights_only=True)
    except Exception as ex:   # noqa: BLE001
        if os.environ.get('S7B_UNSAFE_LOAD') != '1':
            raise RuntimeError(
                f'{path}: torch.load(weights_only=True) failed ({type(ex).__name__}: {ex}); if you trust the file, '
                f'set S7B_UNSAFE_LOAD=1 to allow full unpickling') from ex
        ck = torch.load(path, map_location='cpu', weights_only=False)
    cfg, sd = ck['config'], ck['model_state_dict']
    version = str(cfg['version'])
    vt = _version_tuple(version)

    if vt < (0, 10, 0):  # backward_compatibility.map_old_model
        fixed = {}
        for k, v in sd.items():
            head, _, tail = k.partition('.')
            tail = tail.replace('denumerator', 'denominator')
            for i in range(10):
                _OLD_NAMES.setdefault(f'{i} self connection intro', f'{i}_self_connection_intro')
                _OLD_NAMES.setdefault(f'{i} convolution', f'{i}_convolution')
                _OLD_NAMES.setdefault(f'{i} self interaction 2', f'{i}_self_interaction_2')
                _OLD_NAMES.setdefault(f'{i} equivariant gate', f'{i}_equivariant_gate')
            fixed[_OLD_NAMES.get(head, head) + '.' + tail] = v
        sd = fixed

    if cfg.get('is_parity', False):
        raise NotImplementedError('is_parity: True checkpoints are out of scope (SURVEY 0.9)')
    sc_type = cfg.get('self_connection_type', 'nequip')     # _const.py default
    if isinstance(sc_type, (list, tuple)):                   # one entry per layer is allowed by the reference
        if len(set(sc_type)) != 1:
            raise NotImplementedError(f'self_connection_type must be the same in every layer, got {list(sc_type)}')
        sc_type = sc_type[0]
    if sc_type not in ('linear', 'nequip'):
        raise NotImplementedError(f"self_connection_type {sc_type!r} is not supported (only 'linear' and 'nequip')")
    if cfg.get('use_bias_in_linear', False):
        raise NotImplementedError('use_bias_in_linear is not supported')
    if cfg.get('use_modality', False):
        raise NotImplementedError('multi-fidelity (modal) checkpoints are out of scope')
    if cfg.get('readout_as_fcn', False):
        raise NotImplementedError('readout_as_fcn is not supported')
    for key in ('act_gate', 'act_scalar'):
        if cfg[key].get('e', 'silu') != 'silu':
            raise NotImplementedError(f'{key} must be silu for even irreps')
    if cfg.get('act_radial', 'silu') != 'silu':
        raise NotImplementedError('act_radial must be silu')
    # patch_old_config (backward_compatibility.py:36-37): <= 0.9 checkpoints without the key
    # were trained with un-normalised spherical harmonics
    if not cfg.get('_normalize_sph', not (vt[0] == 0 and vt[1] <= 9)):
        raise NotImplementedError('_normalize_sph False (pre-July-2024 7net-0) is not supported')

    n_layers = int(cfg['num_convolution_layer'])
    lmax = int(cfg['lmax'])
    if cfg.get('irreps_manual', False):
        irreps = [str(s) for s in cfg['irreps_manual']]
    else:
        ch = int(cfg['channel'])
        lmax_node = int(cfg['lmax_node']) if int(cfg.get('lmax_node', -1)) > 0 else lmax
        full = '+'.join(f'{ch}x{l}e' for l in range(lmax_node + 1))
        irreps = [f'{ch}x0e'] + [full] * (n_layers - 1) + [f'{ch}x0e']
    lmax_filter = int(cfg['lmax_edge']) if int(cfg.get('lmax_edge', -1)) > 0 else lmax

    cf = cfg['cutoff_function']
    cf_name = cf['cutoff_function_name']
    meta = dict(
        name=name, source_version=version, cutoff=float(cfg['cutoff']),
        cutoff_fn='XPLOR' if cf_name == 'XPLOR' else 'poly_cut',
        cutoff_on=float(cf.get('cutoff_on', 0.0)), poly_p=int(cf.get('poly_cut_p_value', 6)),
        n_basis=int(cfg['radial_basis']['bessel_basis_num']), lmax_filter=lmax_filter,
        num_species=int(cfg['_number_of_species']),
        type_map={str(int(k)): int(v) for k, v in cfg['_type_map'].items()},
        chemical_species=list(cfg['chemical_species']),
        radial_hidden=[int(h) for h in cfg['weight_nn_hidden_neurons']],
        irreps_per_layer=irreps, readout_hidden=parse_even_irreps(irreps[-1])[0] // 2,
        self_connection=sc_type,
    )
    spec = build_spec(meta)

    def get(k):
        return sd[k].detach().cpu().numpy().astype(np.float32)

    arrays: Dict[str, np.ndarray] = {
        'bessel_coeffs': get('edge_embedding.basis_function.coeffs'),
        'embed': get('onehot_to_feature_x.linear.weight'),
        'readout1': get('reduce_input_to_hidden.linear.weight'),
        'readout2': get('reduce_hidden_to_energy.linear.weight'),
        'shift': get('rescale_atomic_energy.shift').reshape(-1),
        'scale': get('rescale_atomic_energy.scale').reshape(-1),
    }
    if arrays['shift'].size == 1:
        arrays['shift'] = np.full(spec.num_species, arrays['shift'][0], np.float32)
    if arrays['scale'].size == 1:
        arrays['scale'] = np.full(spec.num_species, arrays['scale'][0], np.float32)

    old_order = vt < (0, 11, 0)
    n_mlp = len(spec.radial_hidden) + 1
    for L in spec.layers:
        t = L.t
        # 'nequip': FullyConnectedTensorProduct(x, S x0e, gate_in) weight, blocks [mul_in, S, mul_out] per l
        sc_key = 'fc_tensor_product.weight' if sc_type == 'nequip' else 'linear.weight'
        arrays[f'{t}.sc'] = get(f'{t}_self_connection_intro.{sc_key}').reshape(-1)
        check_sc_weight(L, sc_type, spec.num_species, arrays[f'{t}.sc'].size)
        arrays[f'{t}.si1'] = get(f'{t}_self_interaction_1.linear.weight')
        arrays[f'{t}.si2'] = get(f'{t}_self_interaction_2.linear.weight')
        arrays[f'{t}.den'] = get(f'{t}_convolution.denominator').reshape(1)
        for j in range(n_mlp):
            arrays[f'{t}.mlp{j}'] = get(f'{t}_convolution.weight_nn.layer{j}.weight')
        w_last = arrays[f'{t}.mlp{n_mlp - 1}']
        assert w_last.shape[1] == L.weight_numel, (w_last.shape, L.weight_numel)
        if old_order:
            # columns arrive in creation order: block c holds path with created == c
            created_off, off = {}, 0
            for p in sorted(L.paths, key=lambda p: p.created):
                created_off[p.created] = off
                off += p.mul
            w_sorted = np.empty_like(w_last)
            for p in L.paths:
                w_sorted[:, p.w_off:p.w_off + p.mul] = \
                    w_last[:, created_off[p.created]:created_off[p.created] + p.mul]
            w_last = w_sorted
        # sign convention of the coupling tensors
        for p in L.paths:
            key = (f'{t}_convolution.convolution._compiled_main_left_right.'
                   f'_w3j_{p.l1}_{p.l2}_{p.l3}')
            if key in sd:
                stored = sd[key].numpy().astype(np.float64)
                mine = wigner_3j(p.l1, p.l2, p.l3)
                if np.allclose(stored, mine, atol=1e-6):
                    pass
                elif np.allclose(stored, -mine, atol=1e-6):
                    w_last[:, p.w_off:p.w_off + p.mul] *= -1.0
                else:
                    raise ValueError(f'w3j buffer {key} matches neither +/- convention')
        arrays[f'{t}.mlp{n_mlp - 1}'] = np.ascontiguousarray(w_last)
    return meta, arrays


def save_weights(path: str, meta: dict, arrays: Dict[str, np.ndarray]) -> None:
    np.savez_compressed(path, __meta__=np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8),
                        **arrays)


def load_weights(path: str) -> Tuple[dict, Dict[str, np.ndarray]]:
    with np.load(path) as z:
        meta = json.loads(bytes(z['__meta__']).decode())
        arrays = {k: z[k] for k in z.files if k != '__meta__'}
    return meta, arrays


def random_weights(meta: dict, seed: int = 0) -> Dict[str, np.ndarray]:
    """Random-init weights of a given architecture (for synthetic benchmarks when no
    converted checkpoint is available).  N(0,1) like e3nn's default initialisation."""
    spec = build_spec(meta)
    rng = np.random.RandomState(seed)
    S = spec.num_species

    def lin(in_muls, out_muls):
        return rng.standard_normal(sum(a * b for a, b in zip(in_muls, out_muls))).astype(np.float32)

    arrays = {
        'bessel_coeffs': (np.arange(1, spec.n_basis + 1) * np.pi / spec.cutoff).astype(np.float32),
        'embed': rng.standard_normal(S * spec.layers[0].x_muls[0]).astype(np.float32),
        'readout1': rng.standard_normal(spec.layers[-1].out_muls[0] * spec.readout_hidden).astype(np.float32),
        'readout2': rng.standard_normal(spec.readout_hidden).astype(np.float32),
        'shift': rng.standard_normal(S).astype(np.float32),
        'scale': np.full(S, 1.5, np.float32),
    }
    hs = [spec.n_basis] + list(spec.radial_hidden)
    for L in spec.layers:
        t = L.t
        if spec.self_connection == 'nequip':
            arrays[f'{t}.sc'] = rng.standard_normal(sc_numel(L, 'nequip', S)).astype(np.float32)
        else:
            arrays[f'{t}.sc'] = lin(L.x_muls, L.gate_muls)
        arrays[f'{t}.si1'] = lin(L.x_muls, L.x_muls)
        si2 = []
        for l3, K in enumerate(L.mid_K):
            si2.append(rng.standard_normal(K * L.gate_muls[l3]).astype(np.float32))
        arrays[f'{t}.si2'] = np.concatenate(si2)
        arrays[f'{t}.den'] = np.array([28.0], np.float32)
        dims = hs + [L.weight_numel]
        for j in range(len(dims) - 1):
            arrays[f'{t}.mlp{j}'] = rng.standard_normal((dims[j], dims[j + 1])).astype(np.float32)
    return arrays


def spec_from_meta(meta: dict) -> ModelSpec:
    return build_spec(meta)
