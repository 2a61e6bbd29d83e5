"""fp64 / fp32 oracle of models with the 'nequip' self-connection: ``oracle.oracle.Oracle`` with its
self_connection_intro replaced by the species-wise operator.  Test infrastructure; nothing under sevenn_b200/
imports it.

``SelfConnectionIntro`` (``sevenn/nn/self_connection.py:11-67``) is e3nn's
``FullyConnectedTensorProduct(x, S x0e, gate_in)`` with the species one-hot (``NODE_ATTR``,
``sevenn/nn/node_embedding.py:46``) as its second operand.  The operand is scalars only, so the instructions
are (l, 0e -> l), mode 'uvw', one weight block [mul_in(l), S, mul_out(l)] per l in instruction order.  With
e3nn's defaults (irrep_normalization 'component', path_normalization 'element') each path is scaled by
1/sqrt(mul_in(l) * S), and the coupling w3j(l, 0, l) = delta / sqrt(2l+1) times the component normalisation
sqrt(2l+1) is the identity, so

    sc_l[n, w, m] = 1/sqrt(mul_in(l) * S) * sum_u W_l[u, species(n), w] * x_l[n, u, m]

(restated from e3nn's published definition, as the oracle does for ``o3.Linear``; pinned to the linear path by
tests/test_nequip_sc_cpu.py: W_l[:, s, :] = sqrt(S) M_l is the linear self-connection with weights M_l)."""
from __future__ import annotations

import math

import numpy as np
import torch

from oracle.oracle import Oracle


def species_linear(x: torch.Tensor, flat_w: torch.Tensor, in_blocks, out_muls, species: torch.Tensor,
                   num_species: int) -> torch.Tensor:
    """the operator above on x [n, dim] (e3nn mul_ir layout); in_blocks: (l, mul, offset) of x"""
    n, S = x.shape[0], num_species
    outs = [torch.zeros(n, out_muls[l], 2 * l + 1, dtype=x.dtype, device=x.device) for l in range(len(out_muls))]
    present = [int(v) for v in torch.unique(species).tolist()]
    woff = 0
    for (l, mul, off) in in_blocks:
        if l >= len(out_muls) or out_muls[l] == 0:
            continue
        d = 2 * l + 1
        W = flat_w[woff:woff + mul * S * out_muls[l]].reshape(mul, S, out_muls[l])
        woff += mul * S * out_muls[l]
        xb = x[:, off:off + mul * d].reshape(n, mul, d)
        acc = outs[l]
        for s in present:
            rows = torch.nonzero(species == s).flatten()
            acc = acc.index_add(0, rows, torch.einsum('uw,nui->nwi', W[:, s, :], xb[rows]) / math.sqrt(mul * S))
        outs[l] = acc
    assert woff == flat_w.numel(), (woff, flat_w.numel())
    return torch.cat([o.reshape(n, o.shape[1] * o.shape[2]) for o in outs], dim=1)


class NequipOracle(Oracle):
    """Oracle whose self_connection_intro is the species-wise operator when the model's meta says 'nequip'
    (any other model: exactly Oracle)."""

    def forward(self, species, *args, **kw):
        self._species = torch.as_tensor(np.asarray(species), dtype=torch.long, device=self.device)
        return super().forward(species, *args, **kw)

    def linear(self, x, flat_w, in_blocks, out_muls):
        if self.spec.self_connection == 'nequip' and any(flat_w is self.w[f'{L.t}.sc'] for L in self.spec.layers):
            return species_linear(x, flat_w, in_blocks, out_muls, self._species, self.spec.num_species)
        return super().linear(x, flat_w, in_blocks, out_muls)


def nequip_oracle(meta, arrays, dtype=torch.float64, device='cpu') -> NequipOracle:
    return NequipOracle(meta, arrays, dtype=dtype, device=device)
