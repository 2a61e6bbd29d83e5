"""Python host side of the engine: parameter repacking and a thin ctypes binding to the
C-ABI library ``sevenn_b200/lib/libsevenn_b200.so`` (``include/sevenn_b200.h``).

PyTorch is used only for device memory, streams and (in ``parallel.py``) NCCL; every kernel on
the energy/force path is in the shared library.  There is no CPU fallback: if the library is
missing, importing the binding raises.

Weight preparation restates the normalisations the reference applies at run time inside e3nn
modules (SURVEY Appendix A.5-A.7) and folds them into the arrays once, in float64:
  * ``o3.Linear``: 1/sqrt(fan_in) per output irrep (``sevenn/nn/linear.py:94-100``)
  * convolution ``x.div(denominator)`` (``sevenn/nn/convolution.py:135``) folded into self_interaction_2
  * the 'nequip' self-connection (``sevenn/nn/self_connection.py:11-67``, a linear whose weight depends on the
    atom's species): 1/sqrt(fan_in * num_species) per block; folded into ``embed_g0`` in layer 0
  * the two bias-free readout linears (``sevenn/model_build.py:102-123``) folded into one vector
  * the radial MLP ``FullyConnectedNet`` (``convolution.py:93-95,121``) either kept exact
    (``radial='mlp'``) or tabulated as cubic Hermite splines of the edge length (``radial='table'``)
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Dict, Optional

import numpy as np

from .spec import SILU_NORM, ModelSpec, build_spec, check_sc_weight, sc_blocks

_LIB_PATH = os.environ.get('S7B_LIB') or os.path.join(os.path.dirname(os.path.abspath(__file__)), 'lib', 'libsevenn_b200.so')
_lib = None

S7B_MAX_LAYERS, S7B_MAX_L = 8, 4
(STAGE_FWD_BEGIN, STAGE_FWD_LAYER, STAGE_FWD_END, STAGE_BWD_LAYER_A, STAGE_BWD_LAYER_B,
 STAGE_BWD_END, STAGE_FWD_LAYER_A, STAGE_FWD_LAYER_SC, STAGE_BWD_LAYER_B1, STAGE_BWD_LAYER_B2,
 STAGE_FWD_CONV_INTERIOR, STAGE_FWD_LAYER_A2, STAGE_BWD_LAYER_A1, STAGE_BWD_LAYER_A2) = range(14)


class S7bModelDesc(ctypes.Structure):
    _fields_ = [
        ('n_layers', ctypes.c_int32), ('lmax_filter', ctypes.c_int32),
        ('num_species', ctypes.c_int32), ('n_basis', ctypes.c_int32),
        ('cutoff', ctypes.c_float), ('cutoff_fn', ctypes.c_int32),
        ('cutoff_on', ctypes.c_float), ('poly_p', ctypes.c_int32),
        ('radial_hidden', ctypes.c_int32 * 2),
        ('n_l', ctypes.c_int32 * (S7B_MAX_LAYERS + 1)),
        ('muls', (ctypes.c_int32 * S7B_MAX_L) * (S7B_MAX_LAYERS + 1)),
        ('table_knots', ctypes.c_int32),
    ]


EXPORTS = [
    's7b_last_error', 's7b_version', 's7b_set_option', 's7b_dense_linear', 's7b_engine_create', 's7b_engine_destroy',
    's7b_engine_set_atomic_virial', 's7b_tc_pack_weights', 's7b_gather_rows', 's7b_scatter_add_rows',
    's7b_engine_set_interior', 's7b_block_linear', 's7b_tc_trace_enable', 's7b_engine_neighbor_rows_host',
    's7b_d3_create', 's7b_d3_destroy', 's7b_d3_set_params', 's7b_d3_set_damping', 's7b_d3_set_system', 's7b_d3_run_stage',
    's7b_d3_buffer', 's7b_d3_results_host', 's7b_d3_compute_host', 'pair_init', 'pair_set_atom', 'pair_set_domain',
    'pair_run_settings', 'pair_run_coeff', 'pair_run_compute', 'pair_get_energy', 'pair_get_force', 'pair_get_stress', 'pair_fin',
    's7b_engine_set_param', 's7b_engine_set_graph', 's7b_engine_run_stage', 's7b_engine_compute',
    's7b_engine_buffer', 's7b_engine_compute_host', 's7b_engine_set_positions_host',
    's7b_engine_compute_positions_host', 's7b_launch_count', 's7b_engine_graph_stats', 's7b_engine_stage_graph_stats', 's7b_engine_set_graph_host',
    's7b_engine_read_rows_host', 's7b_engine_write_rows_host', 's7b_engine_read_scalars_host', 's7b_engine_set_profiling',
    's7b_engine_profile_count', 's7b_engine_profile_entry', 's7b_conv_plan_create',
    's7b_conv_plan_destroy', 's7b_conv_plan_dims', 's7b_conv_forward', 's7b_conv_backward',
    's7b_engine_set_positions_batch', 's7b_engine_system_results',
    's7b_d3_set_element_tables', 's7b_d3_set_system_batch', 's7b_d3_system_results', 's7b_species_linear',
]


def load_library() -> ctypes.CDLL:
    """Load the CUDA library; fails loudly when it has not been built (no fallback path)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise ImportError(
            f'{_LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            f'or `make -C sevenn_b200/csrc`. sevenn_b200 has no CPU or PyTorch fallback.')
    lib = ctypes.CDLL(_LIB_PATH)
    vp, i32, i64, sz = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t
    lib.s7b_last_error.restype = ctypes.c_char_p
    lib.s7b_set_option.argtypes = [ctypes.c_char_p, ctypes.c_int]
    lib.s7b_dense_linear.argtypes = [vp, vp, vp, i64, i32, i32, i32, vp]
    lib.s7b_engine_create.argtypes = [ctypes.POINTER(S7bModelDesc), ctypes.POINTER(vp)]
    lib.s7b_engine_destroy.argtypes = [vp]
    lib.s7b_engine_destroy.restype = None
    lib.s7b_engine_set_atomic_virial.argtypes = [vp, ctypes.c_int]
    lib.s7b_tc_pack_weights.argtypes = [vp, i32, i32, vp, vp, ctypes.POINTER(i32)]
    lib.s7b_gather_rows.argtypes = [vp, i32, vp, i64, i32, vp, vp]
    lib.s7b_scatter_add_rows.argtypes = [vp, i32, vp, i64, i32, vp, vp]
    lib.s7b_engine_set_interior.argtypes = [vp, i32]
    lib.s7b_engine_neighbor_rows_host.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, ctypes.POINTER(i64), vp]
    lib.s7b_tc_trace_enable.argtypes = [i32, ctypes.POINTER(vp)]
    lib.s7b_block_linear.argtypes = [vp, i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, i32, i32, vp]
    lib.s7b_species_linear.argtypes = [vp, i32, i32, vp, i32, i32, vp, vp, vp, vp, i32, vp, vp, i32, vp]
    f64 = ctypes.c_double
    lib.s7b_d3_create.argtypes = [ctypes.POINTER(vp)]
    lib.s7b_d3_destroy.argtypes = [vp]
    lib.s7b_d3_destroy.restype = None
    lib.s7b_d3_set_params.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp]
    lib.s7b_d3_set_damping.argtypes = [vp, i32, f64, f64, f64, f64, f64, f64, f64, f64]
    lib.s7b_d3_set_system.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    lib.s7b_d3_run_stage.argtypes = [vp, i32, i32, i32, vp]
    lib.s7b_d3_buffer.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(sz)]
    lib.s7b_d3_buffer.restype = vp
    lib.s7b_d3_results_host.argtypes = [vp, vp, vp, vp, vp]
    lib.s7b_d3_compute_host.argtypes = [vp, vp, vp, vp, vp]
    lib.s7b_d3_set_element_tables.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    lib.s7b_d3_set_system_batch.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp]
    lib.s7b_d3_system_results.argtypes = [vp, vp, vp, vp, vp]
    lib.s7b_engine_set_param.argtypes = [vp, ctypes.c_char_p, ctypes.c_int, vp, sz]
    lib.s7b_engine_set_graph.argtypes = [vp, i32, i32, i64, vp, vp, vp, vp, vp]
    lib.s7b_engine_run_stage.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp]
    lib.s7b_engine_compute.argtypes = [vp, vp]
    lib.s7b_engine_buffer.argtypes = [vp, ctypes.c_char_p, ctypes.c_int, ctypes.POINTER(sz)]
    lib.s7b_engine_buffer.restype = vp
    lib.s7b_engine_compute_host.argtypes = [vp, i32, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.s7b_engine_set_positions_host.argtypes = [vp, i32, vp, vp, vp, vp, vp]
    lib.s7b_engine_compute_positions_host.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.s7b_engine_set_positions_batch.argtypes = [vp, i32, vp, vp, vp, vp, vp, ctypes.POINTER(i64), vp]
    lib.s7b_engine_system_results.argtypes = [vp, vp, vp, vp]
    lib.s7b_engine_set_profiling.argtypes = [vp, ctypes.c_int]
    lib.s7b_engine_profile_count.argtypes = [vp]
    lib.s7b_engine_profile_entry.argtypes = [vp, ctypes.c_int, ctypes.c_char_p, sz,
                                             ctypes.POINTER(ctypes.c_double), ctypes.POINTER(i64)]
    lib.s7b_launch_count.argtypes = [ctypes.c_int]
    lib.s7b_launch_count.restype = i64
    lib.s7b_engine_graph_stats.argtypes = [vp, ctypes.POINTER(i64), ctypes.POINTER(i64)]
    lib.s7b_engine_stage_graph_stats.argtypes = [vp, ctypes.POINTER(i64), ctypes.POINTER(i64)]
    lib.s7b_engine_set_graph_host.argtypes = [vp, i32, i32, i64, vp, vp, vp, vp, vp]
    lib.s7b_engine_read_rows_host.argtypes = [vp, ctypes.c_char_p, ctypes.c_int, i32, i32, i32, vp, vp]
    lib.s7b_engine_write_rows_host.argtypes = [vp, ctypes.c_char_p, ctypes.c_int, i32, i32, i32, vp, vp]
    lib.s7b_engine_read_scalars_host.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double), vp]
    lib.s7b_conv_plan_create.argtypes = [i32, ctypes.POINTER(i32), i32, i32, ctypes.POINTER(vp)]
    lib.s7b_conv_plan_destroy.argtypes = [vp]
    lib.s7b_conv_plan_destroy.restype = None
    lib.s7b_conv_plan_dims.argtypes = [vp] + [ctypes.POINTER(i32)] * 4
    lib.s7b_conv_forward.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i64, vp, vp]
    lib.s7b_conv_backward.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i64, vp, vp, vp, vp, vp]
    _lib = lib
    return lib


def set_option(name: str, value: int) -> None:
    check(load_library().s7b_set_option(name.encode(), int(value)))


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError('sevenn_b200: ' + load_library().s7b_last_error().decode())


# ---- parameter preparation (numpy, float64 -> float32) ------------------------------------------
def _silu(z):
    return z / (1.0 + np.exp(-z))


def _dsilu(z):
    s = 1.0 / (1.0 + np.exp(-z))
    return s * (1.0 + z * (1.0 - s))


def radial_embedding(spec: ModelSpec, coeffs: np.ndarray, r: np.ndarray):
    """Bessel x envelope and its r-derivative, float64 (edge_embedding.py:101-103,125-132,150-160)."""
    r = np.asarray(r, dtype=np.float64)
    c = np.asarray(coeffs, dtype=np.float64)[None, :]
    rr = r[:, None]
    pre = 2.0 / spec.cutoff
    with np.errstate(divide='ignore', invalid='ignore'):
        bes = np.where(rr > 1e-12, pre * np.sin(c * rr) / rr, pre * c)
        dbes = np.where(rr > 1e-12, pre * (c * np.cos(c * rr) / rr - np.sin(c * rr) / rr ** 2), 0.0)
    if spec.cutoff_fn == 'XPLOR':
        on2, c2, r2 = spec.cutoff_on ** 2, spec.cutoff ** 2, r * r
        den = (c2 - on2) ** 3
        a, b = c2 - r2, c2 + 2 * r2 - 3 * on2
        env = np.where(r < spec.cutoff_on, 1.0, a * a * b / den)
        denv = np.where(r < spec.cutoff_on, 0.0, (-4 * r * a * b + 4 * r * a * a) / den)
    else:
        p = float(spec.poly_p)
        x = r / spec.cutoff
        env = 1 - (p + 1) * (p + 2) / 2 * x ** p + p * (p + 2) * x ** (p + 1) - p * (p + 1) / 2 * x ** (p + 2)
        denv = (-(p + 1) * (p + 2) / 2 * p * x ** (p - 1) + p * (p + 2) * (p + 1) * x ** p
                - p * (p + 1) / 2 * (p + 2) * x ** (p + 1)) / spec.cutoff
    return bes * env[:, None], dbes * env[:, None] + bes * denv[:, None]


def radial_weights(spec: ModelSpec, arrays: Dict[str, np.ndarray], t: int, r: np.ndarray):
    """w(r) [len(r), W] and dw/dr of layer t's radial MLP, float64."""
    emb, demb = radial_embedding(spec, arrays['bessel_coeffs'], r)
    n_mlp = len(spec.radial_hidden) + 1
    h, dh = emb, demb
    for j in range(n_mlp):
        W = arrays[f'{t}.mlp{j}'].astype(np.float64) / math.sqrt(arrays[f'{t}.mlp{j}'].shape[0])
        z, dz = h @ W, dh @ W
        if j < n_mlp - 1:
            h, dh = SILU_NORM * _silu(z), SILU_NORM * _dsilu(z) * dz
        else:
            h, dh = z, dz
    return h, dh


def radial_table(spec: ModelSpec, arrays: Dict[str, np.ndarray], t: int, knots: int) -> np.ndarray:
    """Cubic Hermite coefficients [knots, W, 4] on a uniform grid over [0, cutoff]:
    w(r) = a0 + s(a1 + s(a2 + s a3)), s = (r - r_k)/h."""
    h = spec.cutoff / knots
    r = np.arange(knots + 1, dtype=np.float64) * h
    f, df = radial_weights(spec, arrays, t, r)
    f0, f1, d0, d1 = f[:-1], f[1:], df[:-1] * h, df[1:] * h
    tab = np.stack([f0, d0, 3 * (f1 - f0) - (2 * d0 + d1), 2 * (f0 - f1) + d0 + d1], axis=-1)
    return np.ascontiguousarray(tab, dtype=np.float32)


def pack_table_pairs(tab: np.ndarray):
    """[knots, W, 4] -> the two device arrays a lane reads for its channel pair:
    ``table``   [knots, W/2, 4] fp32 {a0e, a0o, a1e, a1o}  (value and slope*h: need fp32)
    ``table23`` [knots, W/2, 4] fp16 {a2e, a2o, a3e, a3o}  (|a2| <~ 1e-3, |a3| <~ 1e-5 of |w| <~ 60:
    half precision leaves w unchanged at the fp32 rounding level and dw/dr at ~2e-7 relative rms),
    returned bit-cast to float32 [knots, W/2, 2] for upload.  Every coefficient arrives as an aligned
    (even, odd) pair for the channel-pair Horner evaluation; 24 instead of 32 bytes per pair."""
    K, W, _ = tab.shape
    pairs = tab.reshape(K, W // 2, 2, 4)                       # [k, pair, parity, coef]
    t01 = np.ascontiguousarray(pairs[..., 0:2].transpose(0, 1, 3, 2).reshape(K, W // 2, 4), dtype=np.float32)
    t23 = np.ascontiguousarray(pairs[..., 2:4].transpose(0, 1, 3, 2).reshape(K, W // 2, 4)).astype(np.float16)
    return t01, np.ascontiguousarray(t23).view(np.float32)


def default_table_knots(spec: ModelSpec) -> int:
    """A grid on which the XPLOR switching radius (a C1-only point) is a knot."""
    return 2000 if spec.cutoff_fn == 'XPLOR' else 2048


def prepare_params(spec: ModelSpec, arrays: Dict[str, np.ndarray], radial: str, knots: int):
    out: Dict[tuple, np.ndarray] = {}
    f64 = lambda a: np.asarray(a, dtype=np.float64)
    S = spec.num_species
    L0 = spec.layers[0]
    mul0 = L0.x_muls[0]
    h0 = f64(arrays['embed']).reshape(S, mul0) / math.sqrt(S)

    def lin_blocks(flat, in_muls, out_muls, n_l):
        """split an e3nn Linear weight (same-l blocks, i_in major) into per-l [K, N] / sqrt(K)."""
        blocks, off = [], 0
        for l in range(n_l):
            k, n = in_muls[l], out_muls[l]
            blocks.append(f64(flat[off:off + k * n]).reshape(k, n) / math.sqrt(k))
            off += k * n
        assert off == len(flat), (off, len(flat))
        return blocks

    def sc_species_blocks(flat, L):
        """split a 'nequip' self-connection weight (``FullyConnectedTensorProduct(x, S x0e, gate_in)``: blocks
        [K, S, N] per l) into per-l [S, K, N] / sqrt(K * S), e3nn's 'element' path normalisation"""
        blocks, off = [], 0
        for k, n in sc_blocks(L):
            blocks.append(f64(flat[off:off + k * S * n]).reshape(k, S, n).transpose(1, 0, 2) / math.sqrt(k * S))
            off += k * S * n
        return blocks

    nequip = spec.self_connection == 'nequip'
    for L in spec.layers:
        t = L.t
        n_lx, n_lg = len(L.x_muls), len(L.gate_muls)
        si1 = lin_blocks(arrays[f'{t}.si1'], L.x_muls, L.x_muls, n_lx)
        n_sc = min(n_lx, n_lg)
        check_sc_weight(L, spec.self_connection, S, np.size(arrays[f'{t}.sc']))
        if nequip:
            sc = sc_species_blocks(arrays[f'{t}.sc'], L)
        else:
            sc = lin_blocks(arrays[f'{t}.sc'], L.x_muls, L.gate_muls, n_sc)
        den = float(arrays[f'{t}.den'][0])
        si2 = [b / den for b in lin_blocks(arrays[f'{t}.si2'], L.mid_K, L.gate_muls, n_lg)]
        if t == 0:
            x0 = h0 @ si1[0]
            g0 = np.zeros((S, L.dim_gate))
            if nequip:      # h0 depends on the species only: the whole self-connection is a per-species row
                g0[:, :L.gate_muls[0]] = np.einsum('su,suw->sw', h0, sc[0])
            else:
                g0[:, :L.gate_muls[0]] = h0 @ sc[0]
            out[('embed_x0', -1)] = x0
            out[('embed_g0', -1)] = g0
        else:
            out[('si1', t)] = np.concatenate([b.ravel() for b in si1])
            out[('si1T', t)] = np.concatenate([b.T.ravel() for b in si1])
            if nequip:      # [species][l block][K][N], and its per-block transpose for the backward
                out[('sc_species', t)] = np.concatenate([b[s].ravel() for s in range(S) for b in sc])
                out[('scT_species', t)] = np.concatenate([b[s].T.ravel() for s in range(S) for b in sc])
            else:
                out[('sc', t)] = np.concatenate([b.ravel() for b in sc])
                out[('scT', t)] = np.concatenate([b.T.ravel() for b in sc])
        out[('si2', t)] = np.concatenate([b.ravel() for b in si2])
        out[('si2T', t)] = np.concatenate([b.T.ravel() for b in si2])
        if radial == 'table':
            out[('table', t)], out[('table23', t)] = pack_table_pairs(radial_table(spec, arrays, t, knots))
        else:
            for j in range(len(spec.radial_hidden) + 1):
                W = f64(arrays[f'{t}.mlp{j}'])
                W = W / math.sqrt(W.shape[0])
                out[(f'mlp{j}', t)] = W
                out[(f'mlp{j}T', t)] = W.T
    Lz = spec.layers[-1]
    r1 = f64(arrays['readout1']).reshape(Lz.out_muls[0], spec.readout_hidden) / math.sqrt(Lz.out_muls[0])
    r2 = f64(arrays['readout2']).reshape(spec.readout_hidden, 1) / math.sqrt(spec.readout_hidden)
    wr = (r1 @ r2).ravel()
    out[('readout', -1)] = wr
    out[('readout_lo', -1)] = wr - wr.astype(np.float32).astype(np.float64)     # residual of the fp32 rounding
    out[('scale', -1)] = f64(arrays['scale'])
    out[('shift', -1)] = f64(arrays['shift'])
    out[('bessel', -1)] = f64(arrays['bessel_coeffs'])
    return {k: np.ascontiguousarray(v, dtype=np.float32) for k, v in out.items()}


def model_desc(spec: ModelSpec, knots: int) -> S7bModelDesc:
    """The C struct ``S7bModelDesc`` (include/sevenn_b200.h) for a model spec."""
    d = S7bModelDesc()
    d.n_layers, d.lmax_filter, d.num_species, d.n_basis = spec.n_layers, spec.lmax_filter, spec.num_species, spec.n_basis
    d.cutoff, d.cutoff_fn = spec.cutoff, 0 if spec.cutoff_fn == 'XPLOR' else 1
    d.cutoff_on, d.poly_p = spec.cutoff_on, spec.poly_p
    if len(spec.radial_hidden) != 2:
        raise NotImplementedError('radial MLP must have two hidden layers')
    d.radial_hidden[0], d.radial_hidden[1] = spec.radial_hidden
    irreps = [list(L.x_muls) for L in spec.layers] + [list(spec.layers[-1].out_muls)]
    for t, muls in enumerate(irreps):
        d.n_l[t] = len(muls)
        for l, m in enumerate(muls):
            d.muls[t][l] = m
    d.table_knots = knots
    return d


def _host(a):
    """numpy view of a host array, or a host copy of a torch tensor on any device"""
    return a.detach().cpu().numpy() if hasattr(a, 'detach') else np.asarray(a)


class _DevView:
    """``__cuda_array_interface__`` view of an engine-owned device buffer."""

    def __init__(self, ptr: int, shape, typestr: str):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, data=(ptr, False),
                                             version=2, strides=None)


class B200Engine:
    """One model on one GPU.  ``radial``: 'table' (cubic-spline radial weights, default) or 'mlp'
    (the radial MLP evaluated exactly per edge with FP32 GEMM kernels)."""

    def __init__(self, meta: dict, arrays: Dict[str, np.ndarray], radial: str = 'table',
                 knots: Optional[int] = None, device: Optional[int] = None, atomic_virial: bool = False):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError('sevenn_b200 needs a CUDA device (sm_90a); there is no CPU path')
        self.torch = torch
        self.lib = load_library()
        self.spec = build_spec(meta)
        self.meta = meta
        self.device = torch.device('cuda', torch.cuda.current_device() if device is None else device)
        if radial not in ('table', 'mlp'):
            raise ValueError("radial must be 'table' or 'mlp'")
        self.radial = radial
        self.knots = (knots or default_table_knots(self.spec)) if radial == 'table' else 0
        spec = self.spec
        d = model_desc(spec, self.knots)
        self._h = ctypes.c_void_p()
        self.atomic_virial = bool(atomic_virial)
        with torch.cuda.device(self.device):
            check(self.lib.s7b_engine_create(ctypes.byref(d), ctypes.byref(self._h)))
            check(self.lib.s7b_engine_set_atomic_virial(self._h, 1 if atomic_virial else 0))
            for (name, t), arr in prepare_params(spec, arrays, radial, self.knots).items():
                check(self.lib.s7b_engine_set_param(self._h, name.encode(), t, arr.ctypes.data, arr.size))
        self._graph = None
        self.n_nodes = self.n_local = self.n_edges = 0

    def __del__(self):
        try:
            if getattr(self, '_h', None) is not None and self._h.value:
                self.lib.s7b_engine_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- graph ----------------------------------------------------------------------------------
    def set_graph(self, species, edge_index, edge_vec, n_local: Optional[int] = None):
        """species [n_nodes] species indices; edge_index [2,E] ([0] = centre, [1] = neighbour);
        edge_vec [E,3].  numpy or torch (any device).  Edges are sorted by centre here if needed."""
        torch = self.torch
        dev = self.device
        species = torch.as_tensor(species).to(dev, torch.int32).contiguous()
        ei = torch.as_tensor(edge_index).to(dev)
        ev = torch.as_tensor(edge_vec).to(dev, torch.float32)
        n_nodes = int(species.shape[0])
        n_local = n_nodes if n_local is None else int(n_local)
        E = int(ei.shape[1])
        dst, src = ei[0].long(), ei[1].long()
        perm = None
        if E > 1 and bool((dst[1:] < dst[:-1]).any()):
            perm = torch.argsort(dst, stable=True)
            dst, src, ev = dst[perm], src[perm], ev[perm]
        if E > 0 and (int(dst.max()) >= n_local or int(src.max()) >= n_nodes):
            raise ValueError('edge index out of range')
        rowptr = torch.zeros(n_local + 1, dtype=torch.int64, device=dev)
        if E > 0:
            rowptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n_local), 0)
        g = dict(species=species, rowptr=rowptr.to(torch.int32).contiguous(),
                 src=src.to(torch.int32).contiguous(), edge_vec=ev.contiguous(), perm=perm)
        self.set_graph_csr(g['species'], g['rowptr'], g['src'], g['edge_vec'], n_local)
        self._graph.update(perm=perm)
        return self._graph

    def set_graph_csr(self, species, rowptr, src, edge_vec, n_local: int):
        """Device int32/float32 tensors already in CSR-over-centres form (kept alive by the engine)."""
        self._graph = dict(species=species, rowptr=rowptr, src=src, edge_vec=edge_vec, perm=None)
        self.n_nodes, self.n_local, self.n_edges = int(species.shape[0]), int(n_local), int(src.shape[0])
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_set_graph(
                self._h, self.n_nodes, self.n_local, self.n_edges, species.data_ptr(),
                rowptr.data_ptr(), src.data_ptr(), edge_vec.data_ptr(), self._stream()))

    # ---- host-staged stage protocol (what examples/lammps/pair_e3gnn_b200_parallel.cpp calls) -----------------
    def set_graph_host(self, species, edge_centre, edge_neighbour, edge_vec, n_local: int):
        """graph with ghosts from host arrays: edges sorted by centre, centres < n_local (``s7b_engine_set_graph_host``)"""
        sp = np.ascontiguousarray(species, dtype=np.int32)
        c = np.ascontiguousarray(edge_centre, dtype=np.int32)
        nb = np.ascontiguousarray(edge_neighbour, dtype=np.int32)
        v = np.ascontiguousarray(edge_vec, dtype=np.float32)
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_set_graph_host(self._h, len(sp), int(n_local), len(c), sp.ctypes.data, c.ctypes.data,
                                                     nb.ctypes.data, v.ctypes.data, self._stream()))
        self._graph = dict(perm=None)
        self.n_nodes, self.n_local, self.n_edges = len(sp), int(n_local), len(c)
        return self

    def read_rows(self, name: str, layer: int, row_begin: int, n_rows: int, width: int) -> np.ndarray:
        out = np.empty((n_rows, width), dtype=np.float32)
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_read_rows_host(self._h, name.encode(), int(layer), int(row_begin), int(n_rows), int(width),
                                                     out.ctypes.data, self._stream()))
        return out

    def write_rows(self, name: str, layer: int, row_begin: int, rows: np.ndarray):
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_write_rows_host(self._h, name.encode(), int(layer), int(row_begin), rows.shape[0],
                                                      rows.shape[1], rows.ctypes.data, self._stream()))

    def read_scalars(self):
        """(energy, virial[6]) of the last BWD_END as host doubles"""
        e, v = ctypes.c_double(), (ctypes.c_double * 6)()
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_read_scalars_host(self._h, ctypes.byref(e), v, self._stream()))
        return float(e.value), np.array(list(v))

    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def set_interior(self, n_interior: int):
        """owned atoms [0, n_interior) have no ghost neighbour (split stages of the multi-GPU runner)"""
        check(self.lib.s7b_engine_set_interior(self._h, int(n_interior)))

    # ---- ghost-exchange pack / unpack kernels (C ABI s7b_gather_rows / s7b_scatter_add_rows) ----------
    def gather_rows(self, src, idx32, out):
        """out[i] = src[idx32[i]] (rows of a 2-D float32 tensor; idx32 int32 on the device)"""
        n = int(idx32.shape[0])
        if n:
            check(self.lib.s7b_gather_rows(src.data_ptr(), src.stride(0), idx32.data_ptr(), n, src.shape[1],
                                           out.data_ptr(), self._stream()))
        return out

    def scatter_add_rows(self, dst, idx32, rows):
        """dst[idx32[i]] += rows[i]; idx32 must hold unique indices"""
        n = int(idx32.shape[0])
        if n:
            check(self.lib.s7b_scatter_add_rows(dst.data_ptr(), dst.stride(0), idx32.data_ptr(), n, dst.shape[1],
                                                rows.data_ptr(), self._stream()))
        return dst

    # ---- execution --------------------------------------------------------------------------------
    def run_stage(self, stage: int, layer: int = 0):
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_run_stage(self._h, stage, layer, self._stream()))

    def compute(self):
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_compute(self._h, self._stream()))
        return self

    def buffer(self, name: str, layer: int = 0, dtype: str = 'f4', shape=None):
        """Zero-copy torch view of an engine buffer (valid until the next set_graph)."""
        n = ctypes.c_size_t()
        ptr = self.lib.s7b_engine_buffer(self._h, name.encode(), layer, ctypes.byref(n))
        if not ptr or n.value == 0:
            tdt = {'f4': self.torch.float32, 'f8': self.torch.float64, 'i4': self.torch.int32}[dtype]
            return self.torch.zeros(shape if shape is not None else (0,), dtype=tdt, device=self.device)
        shp = (n.value,) if shape is None else tuple(shape)
        assert int(np.prod(shp)) == n.value, (name, shp, n.value)
        return self.torch.as_tensor(_DevView(ptr, shp, '<' + dtype), device=self.device)

    def results(self) -> dict:
        """Energy (python float, from the device double), per-atom energies, forces, edge forces,
        virial (= -sum r (x) f; divide by the volume for 'inferred_stress')."""
        t = self.torch
        energy = self.buffer('energy', dtype='f8').clone()
        return dict(
            energy=energy,
            atomic_energy=self.buffer('atomic_energy', shape=(self.n_local,)).clone(),
            forces=self.buffer('forces', shape=(self.n_nodes, 3)).clone(),
            edge_force=self.buffer('edge_force', shape=(self.n_edges, 3)).clone() if self.n_edges else t.zeros(0, 3, device=self.device),
            virial=self.buffer('virial', dtype='f8').clone())

    def compute_host(self, species: np.ndarray, edge_centre: np.ndarray, edge_neighbour: np.ndarray,
                     edge_vec: np.ndarray):
        """Host-buffer entry (C ABI ``s7b_engine_compute_host``): numpy in, numpy out; edges must be
        sorted by centre.  Returns (energy, atomic_energy, forces, virial6)."""
        species = np.ascontiguousarray(species, dtype=np.int32)
        ec = np.ascontiguousarray(edge_centre, dtype=np.int32)
        en = np.ascontiguousarray(edge_neighbour, dtype=np.int32)
        ev = np.ascontiguousarray(edge_vec, dtype=np.float32)
        n, E = len(species), len(ec)
        energy = np.zeros(1, np.float64)
        virial = np.zeros(6, np.float64)
        ae = np.zeros(n, np.float32)
        forces = np.zeros((n, 3), np.float32)
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_compute_host(
                self._h, n, E, species.ctypes.data, ec.ctypes.data, en.ctypes.data, ev.ctypes.data,
                energy.ctypes.data, ae.ctypes.data, forces.ctypes.data, virial.ctypes.data, self._stream()))
        self._graph = None
        self.n_nodes = self.n_local = n
        self.n_edges = E
        return float(energy[0]), ae, forces, virial

    @staticmethod
    def _pos_args(species, positions, cell, pbc):
        sp = np.ascontiguousarray(species, dtype=np.int32)
        pos = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 3)
        c = np.zeros((3, 3)) if cell is None else np.ascontiguousarray(cell, dtype=np.float64).reshape(3, 3)
        pb = np.ascontiguousarray(np.broadcast_to(np.asarray(pbc, dtype=bool), (3,)).astype(np.int32))
        return sp, pos, np.ascontiguousarray(c), pb

    def set_positions(self, species, positions, cell, pbc):
        """Build the neighbour list / graph on the device from host positions (C ABI
        ``s7b_engine_set_positions_host``) and make it the current graph."""
        sp, pos, c, pb = self._pos_args(species, positions, cell, pbc)
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_set_positions_host(self._h, len(sp), sp.ctypes.data, pos.ctypes.data,
                                                         c.ctypes.data, pb.ctypes.data, self._stream()))
        self._graph = dict(perm=None)
        self.n_nodes = self.n_local = len(sp)
        n = ctypes.c_size_t()
        self.lib.s7b_engine_buffer(self._h, b'graph_src', 0, ctypes.byref(n))
        self.n_edges = int(n.value)
        return self

    def set_positions_batch(self, species, positions, atom_ptr, cells, pbc):
        """Neighbour lists of B structures built in one pass on the device, installed as one union graph (C ABI
        ``s7b_engine_set_positions_batch``).  species [n] (indices), positions [n,3], atom_ptr [B+1] (atoms of
        structure b: [atom_ptr[b], atom_ptr[b+1])), cells [B,3,3] (rows = lattice vectors, zeros where a structure
        has none), pbc broadcastable to [B,3]: torch tensors on any device, or numpy arrays.  Species and
        positions go to (or stay on) the device; atom_ptr, cells and pbc are read on the host."""
        torch = self.torch
        ap = np.ascontiguousarray(_host(atom_ptr), dtype=np.int32).ravel()
        B = len(ap) - 1
        if B < 1:
            raise ValueError('atom_ptr needs B + 1 >= 2 entries')
        c = np.ascontiguousarray(_host(cells), dtype=np.float64).reshape(B, 9)
        pb = np.ascontiguousarray(np.broadcast_to(np.asarray(_host(pbc), dtype=bool), (B, 3)).astype(np.int32))
        sp = torch.as_tensor(species).detach().to(self.device, torch.int32).contiguous().reshape(-1)
        pos = torch.as_tensor(positions).detach().to(self.device, torch.float64).contiguous().reshape(-1, 3)
        if sp.shape[0] != pos.shape[0] or sp.shape[0] != int(ap[-1]):
            raise ValueError(f'species ({sp.shape[0]}) and positions ({pos.shape[0]}) need atom_ptr[-1] = {int(ap[-1])} rows')
        ne = ctypes.c_int64()
        with torch.cuda.device(self.device):
            check(self.lib.s7b_engine_set_positions_batch(self._h, B, ap.ctypes.data, sp.data_ptr(), pos.data_ptr(),
                                                          c.ctypes.data, pb.ctypes.data, ctypes.byref(ne), self._stream()))
        self._graph = dict(perm=None, n_systems=B)
        self.n_nodes = self.n_local = int(ap[-1])
        self.n_edges = int(ne.value)
        return self

    def system_results(self):
        """(energy [B], virial [B,6]) float64 device tensors of the last ``compute`` on a graph from
        ``set_positions_batch``: fp64 sums of the per-atom energies, virial = -sum r (x) f per structure
        (xx,yy,zz,xy,yz,zx).  C ABI ``s7b_engine_system_results``."""
        torch = self.torch
        B = (self._graph or {}).get('n_systems', 0)
        energy = torch.empty(B, dtype=torch.float64, device=self.device)
        virial = torch.empty(B, 6, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.s7b_engine_system_results(self._h, energy.data_ptr(), virial.data_ptr(), self._stream()))
        return energy, virial

    def neighbor_rows(self, species, positions, cell, pbc, centres):
        """Device neighbour rows of the atoms `centres` (indices) against all atoms: torch views
        (rowptr [len(centres)+1] int32, src [E] int32 = indices into all atoms, edge_vec [E,3] float32),
        valid until the next neighbour-list call (C ABI ``s7b_engine_neighbor_rows_host``)."""
        sp, pos, c, pb = self._pos_args(species, positions, cell, pbc)
        cen = np.ascontiguousarray(centres, dtype=np.int32)
        ne = ctypes.c_int64()
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_neighbor_rows_host(self._h, len(sp), sp.ctypes.data, pos.ctypes.data, c.ctypes.data,
                                                         pb.ctypes.data, len(cen), cen.ctypes.data, ctypes.byref(ne), self._stream()))
        E = int(ne.value)
        return (self.buffer('nl_rowptr', dtype='i4', shape=(len(cen) + 1,)),
                self.buffer('nl_src', dtype='i4', shape=(E,)),
                self.buffer('nl_vec', shape=(E, 3)))

    def graph_arrays(self):
        """(rowptr, src, edge_vec) of the current graph as torch views."""
        return (self.buffer('graph_rowptr', dtype='i4', shape=(self.n_local + 1,)),
                self.buffer('graph_src', dtype='i4', shape=(self.n_edges,)),
                self.buffer('graph_edge_vec', shape=(self.n_edges, 3)))

    def compute_positions(self, species, positions, cell, pbc):
        """positions in -> (energy, atomic_energy, forces, virial6, n_edges): neighbour list, all stages
        and the copies back in one C-ABI call (``s7b_engine_compute_positions_host``)."""
        sp, pos, c, pb = self._pos_args(species, positions, cell, pbc)
        n = len(sp)
        energy, virial = np.zeros(1, np.float64), np.zeros(6, np.float64)
        ae, forces = np.zeros(n, np.float32), np.zeros((n, 3), np.float32)
        ne = ctypes.c_int64()
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_engine_compute_positions_host(
                self._h, n, sp.ctypes.data, pos.ctypes.data, c.ctypes.data, pb.ctypes.data, energy.ctypes.data,
                ae.ctypes.data, forces.ctypes.data, virial.ctypes.data, ctypes.byref(ne), self._stream()))
        self._graph = dict(perm=None)
        self.n_nodes = self.n_local = n
        self.n_edges = int(ne.value)
        return float(energy[0]), ae, forces, virial, int(ne.value)

    def set_profiling(self, enable: bool):
        check(self.lib.s7b_engine_set_profiling(self._h, 1 if enable else 0))

    def profile(self) -> dict:
        """{label: (total_ms, calls)} accumulated since set_profiling(True)."""
        out = {}
        for i in range(self.lib.s7b_engine_profile_count(self._h)):
            name = ctypes.create_string_buffer(96)
            ms, calls = ctypes.c_double(), ctypes.c_int64()
            check(self.lib.s7b_engine_profile_entry(self._h, i, name, 96, ctypes.byref(ms), ctypes.byref(calls)))
            out[name.value.decode()] = (ms.value, calls.value)
        return out

    def graph_stats(self):
        """(captures, replays) of the CUDA-graph path of ``compute``."""
        c, r = ctypes.c_int64(), ctypes.c_int64()
        check(self.lib.s7b_engine_graph_stats(self._h, ctypes.byref(c), ctypes.byref(r)))
        return int(c.value), int(r.value)

    def stage_graph_stats(self):
        """(captures, replays) of the per-stage CUDA graphs of ``run_stage`` (option ``stage_graphs``)."""
        c, r = ctypes.c_int64(), ctypes.c_int64()
        check(self.lib.s7b_engine_stage_graph_stats(self._h, ctypes.byref(c), ctypes.byref(r)))
        return int(c.value), int(r.value)

    def launch_count(self, reset: bool = False) -> int:
        return int(self.lib.s7b_launch_count(1 if reset else 0))
