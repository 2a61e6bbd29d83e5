"""Static description of a SevenNet (NequIP-type, even-parity) model: layer irreps,
tensor-product paths, weight blocks and the two feature layouts used in this repo.

What the reference derives at model-build time
(``sevenn/model_build.py:448-636``, ``sevenn/nn/interaction_blocks.py:14-78``,
``sevenn/nn/convolution.py:61-91``) is restated here as plain data so that the CPU oracle,
the CUDA engine and the code generator all agree on one source of truth.

Two layouts of a node feature vector with irreps ``mul_0 x 0e + mul_1 x 1e + ...``:

* ``mul_ir`` (e3nn / reference boundary layout): block l is ``[mul_l, 2l+1]`` row-major,
  i.e. element (u, m) sits at ``off_l + u*(2l+1) + m``.
* ``cm`` (component-major, the engine's internal HBM layout): block l is ``[2l+1, mul_l]``
  row-major, element (m, u) at ``off_l + m*mul_l + u`` -- a warp whose lanes are channels
  reads and writes 128-byte contiguous segments.

The convolution output ("mid" features) in e3nn is one ``[mul_p, 2l3+1]`` block per path
slot p, slots sorted by l3.  Internally all slots with the same l3 are fused into one
``[2l3+1, K_l3]`` block (K_l3 = sum of their multiplicities) so that the following
``self_interaction_2`` linear sees a contiguous K axis.
"""
from __future__ import annotations

import dataclasses
import re
from typing import Dict, List, Tuple

import numpy as np

# e3nn ``normalize2mom(silu)``: (E_{z~N(0,1)} silu(z)^2)^-1/2 estimated by e3nn with
# ``torch.randn(1_000_000, generator=manual_seed(0), dtype=float64)``.  The value below is
# what this torch build produces (SURVEY Appendix A.7; recomputed in tools/make_golden.py).
SILU_NORM = 1.6791767923989418


def parse_even_irreps(s: str) -> List[int]:
    """'128x0e+64x1e+32x2e' -> [128, 64, 32].  Only sorted, simplified, even-parity irreps
    (``is_parity: False`` models: SevenNet-0, SevenNet-l3i5) are supported."""
    muls: List[int] = []
    for tok in str(s).replace(' ', '').split('+'):
        m = re.fullmatch(r'(\d+)x(\d+)([eo])', tok)
        if m is None:
            raise ValueError(f'cannot parse irreps token {tok!r}')
        mul, l, p = int(m.group(1)), int(m.group(2)), m.group(3)
        if p != 'e':
            raise NotImplementedError('odd-parity irreps (is_parity: True) are out of scope')
        if l != len(muls):
            raise NotImplementedError(f'irreps must list l = 0..lmax once each, got {s!r}')
        muls.append(mul)
    return muls


def irreps_dim(muls: List[int]) -> int:
    return sum((2 * l + 1) * m for l, m in enumerate(muls))


def irreps_offsets(muls: List[int]) -> List[int]:
    off, out = 0, []
    for l, m in enumerate(muls):
        out.append(off)
        off += (2 * l + 1) * m
    return out


def perm_cm_from_mulir(muls: List[int]) -> np.ndarray:
    """Index array P with  x_cm = x_mulir[..., P]."""
    p = np.empty(irreps_dim(muls), dtype=np.int64)
    for l, (m, off) in enumerate(zip(muls, irreps_offsets(muls))):
        d = 2 * l + 1
        for i in range(d):
            for u in range(m):
                p[off + i * m + u] = off + u * d + i
    return p


@dataclasses.dataclass(frozen=True)
class TPPath:
    """One 'uvu' instruction of the convolution (``sevenn/nn/convolution.py:61-82``)."""
    slot: int        # position in the i_out-sorted instruction list (= weight block order)
    l1: int          # node-feature irrep
    l2: int          # spherical-harmonic (edge filter) irrep
    l3: int          # output irrep
    mul: int         # channels (= mul of l1 in x)
    w_off: int       # column offset of this path's block in weight[E, W]
    out_off: int     # offset of the [mul, 2l3+1] block in the e3nn mid vector
    k_off: int       # column offset inside the fused [2l3+1, K_l3] internal mid block
    created: int     # position in instruction-creation order (old checkpoints, A.8)


@dataclasses.dataclass(frozen=True)
class LayerSpec:
    t: int
    x_muls: Tuple[int, ...]       # irreps of the layer input (and of x after self_interaction_1)
    gate_muls: Tuple[int, ...]    # irreps fed to the gate: (n_scalars + n_gates) x0e + gated
    out_muls: Tuple[int, ...]     # irreps after the gate (= next layer's x_muls)
    lmax_filter: int
    paths: Tuple[TPPath, ...]
    mid_K: Tuple[int, ...]        # K_l3 for l3 = 0..lmax_mid

    @property
    def dim_x(self) -> int:
        return irreps_dim(list(self.x_muls))

    @property
    def dim_gate(self) -> int:
        return irreps_dim(list(self.gate_muls))

    @property
    def dim_out(self) -> int:
        return irreps_dim(list(self.out_muls))

    @property
    def dim_mid(self) -> int:
        return irreps_dim(list(self.mid_K))

    @property
    def weight_numel(self) -> int:
        return sum(p.mul for p in self.paths)

    @property
    def n_scalars(self) -> int:
        return self.out_muls[0]

    def mid_perm_cm_from_mulir(self) -> np.ndarray:
        """P with  mid_internal = mid_e3nn[..., P]."""
        offs = irreps_offsets(list(self.mid_K))
        p = np.empty(self.dim_mid, dtype=np.int64)
        for pa in self.paths:
            d = 2 * pa.l3 + 1
            K = self.mid_K[pa.l3]
            for k in range(d):
                for u in range(pa.mul):
                    p[offs[pa.l3] + k * K + pa.k_off + u] = pa.out_off + u * d + k
        return p


def build_layer(t: int, x_muls: List[int], out_muls: List[int], lmax_filter: int) -> LayerSpec:
    """Restates ``NequIP_interaction_block`` + ``IrrepsConvolution.__init__`` for even-parity
    irreps: every triangle-allowed (l1, l2, l3) with l3 <= lmax(out) is a path."""
    lmax_out = len(out_muls) - 1
    created = []
    for l1, mul in enumerate(x_muls):
        for l2 in range(lmax_filter + 1):
            for l3 in range(abs(l1 - l2), l1 + l2 + 1):
                if l3 <= lmax_out:
                    created.append((l1, l2, l3, mul))
    order = sorted(range(len(created)), key=lambda c: (created[c][2], c))  # Irreps.sort(): by l, stable
    paths, w_off, out_off = [], 0, 0
    k_run: Dict[int, int] = {}
    for slot, c in enumerate(order):
        l1, l2, l3, mul = created[c]
        k_off = k_run.get(l3, 0)
        paths.append(TPPath(slot, l1, l2, l3, mul, w_off, out_off, k_off, c))
        k_run[l3] = k_off + mul
        w_off += mul
        out_off += mul * (2 * l3 + 1)
    mid_K = tuple(k_run.get(l, 0) for l in range(lmax_out + 1))
    # e3nn Gate input: scalars + one gate scalar per gated irrep channel, then the gated irreps
    n_gates = sum(out_muls[1:])
    gate_muls = (out_muls[0] + n_gates,) + tuple(out_muls[1:])
    return LayerSpec(t, tuple(x_muls), gate_muls, tuple(out_muls), lmax_filter, tuple(paths), mid_K)


@dataclasses.dataclass
class ModelSpec:
    name: str
    cutoff: float
    cutoff_fn: str                 # 'XPLOR' | 'poly_cut'
    cutoff_on: float               # XPLOR r_on
    poly_p: int                    # poly_cut p
    n_basis: int
    lmax_filter: int
    num_species: int
    type_map: Dict[int, int]       # atomic number -> species index
    radial_hidden: Tuple[int, ...]
    layers: List[LayerSpec]
    readout_hidden: int
    self_connection: str = 'linear'   # 'linear' (o3.Linear) | 'nequip' (species-wise FullyConnectedTensorProduct)

    @property
    def n_layers(self) -> int:
        return len(self.layers)

    @property
    def n_sh(self) -> int:
        return (self.lmax_filter + 1) ** 2


def build_spec(meta: dict) -> ModelSpec:
    irreps = [parse_even_irreps(s) for s in meta['irreps_per_layer']]
    layers = [build_layer(t, irreps[t], irreps[t + 1], int(meta['lmax_filter']))
              for t in range(len(irreps) - 1)]
    return ModelSpec(
        name=meta['name'], cutoff=float(meta['cutoff']), cutoff_fn=meta['cutoff_fn'],
        cutoff_on=float(meta.get('cutoff_on', 0.0)), poly_p=int(meta.get('poly_p', 6)),
        n_basis=int(meta['n_basis']), lmax_filter=int(meta['lmax_filter']),
        num_species=int(meta['num_species']),
        type_map={int(k): int(v) for k, v in meta['type_map'].items()},
        radial_hidden=tuple(int(h) for h in meta['radial_hidden']), layers=layers,
        readout_hidden=int(meta['readout_hidden']), self_connection=self_connection_of(meta))


SELF_CONNECTIONS = ('linear', 'nequip')


def self_connection_of(meta: dict) -> str:
    """The self-connection type a meta records; files written before the key existed are 'linear'."""
    sc = str(meta.get('self_connection', 'linear'))
    if sc not in SELF_CONNECTIONS:
        raise NotImplementedError(f'self_connection {sc!r} is not supported (one of {SELF_CONNECTIONS})')
    return sc


def sc_blocks(L: LayerSpec) -> List[Tuple[int, int]]:
    """(K, N) = (mul_in, mul_out) of the self-connection's weight blocks, l = 0 .. min(n_lx, n_lg) - 1, in weight
    order: one block per l for both types (an e3nn o3.Linear, or the uvw instructions (l, 0e -> l) of
    ``FullyConnectedTensorProduct(x, S x0e, gate_in)``, ``sevenn/nn/self_connection.py:11-67``)."""
    n = min(len(L.x_muls), len(L.gate_muls))
    return [(L.x_muls[l], L.gate_muls[l]) for l in range(n)]


def sc_numel(L: LayerSpec, kind: str, num_species: int) -> int:
    """Values of layer L's self-connection weight: sum K*N ('linear'), sum K*S*N ('nequip': blocks [K, S, N])."""
    per = sum(k * n for k, n in sc_blocks(L))
    return per * num_species if kind == 'nequip' else per


def check_sc_weight(L: LayerSpec, kind: str, num_species: int, size: int) -> None:
    want = sc_numel(L, kind, num_species)
    if int(size) != want:
        shape = ' + '.join(f'{k}x{num_species}x{n}' if kind == 'nequip' else f'{k}x{n}' for k, n in sc_blocks(L))
        raise ValueError(f'layer {L.t}: the {kind} self-connection weight has {int(size)} values, expected {want} ({shape})')
