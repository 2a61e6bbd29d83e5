"""The synthetic checkpoints of synthetic_models.py with the 'nequip' self-connection, the default of the
reference's training presets (``sevenn/presets/base.yaml:32``, ``sevenn/_const.py``), in the reference layout:
``self_connection_type: 'nequip'`` and, per layer, ``{t}_self_connection_intro.fc_tensor_product.weight`` -- the
weight of ``FullyConnectedTensorProduct(x, S x0e, gate_in)``, one block [mul_in(l), S, mul_out(l)] per l.

``sc``:
  * 'random'       N(0, 1) blocks, like e3nn's initialisation (seeded);
  * 'from_linear'  W_l[:, s, :] = sqrt(S) * M_l for every species s, M_l the linear self-connection of the
                   same seed: the model then computes exactly what the linear-SC checkpoint computes;
  * 'one_species'  random blocks with every species slice but ``only`` zeroed.

SevenNet-0 widths (128x0e+64x1e+32x2e) are architecture C of synthetic_models.py."""
from __future__ import annotations

import numpy as np

from synthetic_models import ARCHS, NUMBERS, irreps_per_layer, reference_checkpoint

S = len(NUMBERS)


def layers(arch: str):
    from sevenn_b200.spec import build_layer, parse_even_irreps
    irreps = [parse_even_irreps(s) for s in irreps_per_layer(arch)]
    return [build_layer(t, irreps[t], irreps[t + 1], ARCHS[arch]['lmax_edge']) for t in range(len(irreps) - 1)]


def nequip_checkpoint(arch: str, seed: int = 0, sc: str = 'random', only: int = 0, parity: bool = False) -> dict:
    import torch
    from sevenn_b200.spec import sc_blocks
    ck = reference_checkpoint(arch, seed, parity)
    ck['config']['self_connection_type'] = 'nequip'
    sd = ck['model_state_dict']
    rng = np.random.RandomState(2000 + seed)
    for L in layers(arch):
        lin = sd.pop(f'{L.t}_self_connection_intro.linear.weight').numpy().astype(np.float64)
        parts, off = [], 0
        for k, n in sc_blocks(L):
            if sc == 'from_linear':
                M = lin[off:off + k * n].reshape(k, 1, n)
                parts.append(np.broadcast_to(np.sqrt(S) * M, (k, S, n)).ravel())
            else:
                W = rng.standard_normal((k, S, n))
                if sc == 'one_species':
                    W[:, np.arange(S) != only, :] = 0.0
                parts.append(W.ravel())
            off += k * n
        sd[f'{L.t}_self_connection_intro.fc_tensor_product.weight'] = torch.tensor(np.concatenate(parts), dtype=torch.float32)
    return ck


def write_nequip_checkpoint(path, arch: str, seed: int = 0, **kw) -> str:
    import torch
    torch.save(nequip_checkpoint(arch, seed, **kw), str(path))
    return str(path)


def convert(path, arch: str):
    from sevenn_b200.checkpoint import convert_reference_checkpoint
    return convert_reference_checkpoint(str(path), f'synthetic_{arch}_nequip')
