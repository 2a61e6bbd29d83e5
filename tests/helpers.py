"""Shared helpers for tests (systems from tests/golden, graph building, oracle cache)."""
import functools
import json
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


@functools.lru_cache(maxsize=None)
def golden_vectors():
    return json.load(open(os.path.join(GOLDEN, 'reference_vectors.json')))


@functools.lru_cache(maxsize=None)
def model_weights(name):
    from sevenn_b200.checkpoint import load_weights
    return load_weights(os.path.join(ROOT, 'weights', f'{name}.npz'))


@functools.lru_cache(maxsize=None)
def oracle(name, dtype_name='float64'):
    import torch
    from oracle.oracle import Oracle
    meta, arrays = model_weights(name)
    return Oracle(meta, arrays, dtype=getattr(torch, dtype_name))


def system_graph(system, cutoff):
    from sevenn_b200.neighbors import build_graph
    pos = np.asarray(system['positions'], dtype=np.float64)
    cell = np.zeros((3, 3)) if system['cell'] is None else np.asarray(system['cell'], dtype=np.float64)
    ei, ev = build_graph(pos, cell, bool(system['pbc']), cutoff)
    vol = abs(np.linalg.det(cell)) if system['pbc'] else 0.0
    return ei, ev, vol


def species_of(meta, numbers):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(z)] for z in numbers], dtype=np.int64)


def stage_errors(engine, arrays, species, edge_index, edge_vec, ref=None):
    """Run ``engine`` stage by stage on a graph and compare every intermediate the fp64 oracle also produces:
    [(stage, max |engine - oracle|, max |oracle|)] in evaluation order -- x after self_interaction_1, mid / den,
    gate_in and the gate output h of every layer, then the atomic energies, edge forces and forces.  Engine
    buffers are in the channel-major layout, the oracle's in e3nn mul_ir order: the oracle side is permuted
    (spec.perm_cm_from_mulir / mid_perm_cm_from_mulir).  ``arrays`` are the weights the engine was built with
    (for the convolution denominators); ``ref`` an oracle ``forward(..., keep=True)`` result."""
    import torch
    from sevenn_b200 import engine as eng
    from sevenn_b200.spec import perm_cm_from_mulir
    if ref is None:
        ref = oracle(_model_of(engine)).forward(species, edge_index, edge_vec, keep=True)
    sv = ref['saved']
    engine.set_graph(species, edge_index, edge_vec)
    spec = engine.spec
    N, E = len(species), edge_index.shape[1]
    out = []

    def add(tag, got, want):
        got = got.detach().cpu().double().numpy().reshape(np.shape(want))
        want = np.asarray(want, dtype=np.float64)
        out.append((tag, float(np.abs(got - want).max()) if want.size else 0.0,
                    float(np.abs(want).max()) if want.size else 0.0))

    def sync():
        torch.cuda.synchronize()

    engine.run_stage(eng.STAGE_FWD_BEGIN)
    sync()
    for L in spec.layers:
        t = L.t
        add(f'layer {t} x', engine.buffer('x', t).reshape(N, -1), sv[f'{t}.x_si1'].numpy()[:, perm_cm_from_mulir(list(L.x_muls))])
        engine.run_stage(eng.STAGE_FWD_LAYER, t)
        sync()
        den = float(np.asarray(arrays[f'{t}.den']).ravel()[0])
        add(f'layer {t} mid', engine.buffer('mid', t).reshape(N, -1) / den, sv[f'{t}.mid'].numpy()[:, L.mid_perm_cm_from_mulir()])
        add(f'layer {t} gate_in', engine.buffer('gate_in', t).reshape(N, -1), sv[f'{t}.gate_in'].numpy()[:, perm_cm_from_mulir(list(L.gate_muls))])
        add(f'layer {t} h', engine.buffer('h', t).reshape(N, -1), sv[f'{t}.x_out'].numpy()[:, perm_cm_from_mulir(list(L.out_muls))])
    engine.run_stage(eng.STAGE_FWD_END)
    sync()
    add('atomic energy', engine.buffer('atomic_energy', shape=(N,)), ref['atomic_energy'].numpy())
    for t in range(spec.n_layers - 1, -1, -1):
        engine.run_stage(eng.STAGE_BWD_LAYER_A, t)
        if t > 0:
            engine.run_stage(eng.STAGE_BWD_LAYER_B, t)
    engine.run_stage(eng.STAGE_BWD_END)
    sync()
    perm = engine._graph['perm']
    want_fe = ref['edge_force'].numpy()
    if perm is not None:
        want_fe = want_fe[perm.cpu().numpy()]
    if E:
        add('edge force', engine.buffer('edge_force', shape=(E, 3)), want_fe)
    add('forces', engine.buffer('forces', shape=(N, 3)), ref['forces'].numpy())
    return out


def first_divergence(errors, rtol=1e-4, atol=1e-5):
    """The first stage of ``stage_errors`` whose error exceeds atol + rtol * (its reference scale), or None;
    fp32 intermediates of a correct engine sit near 1e-6 relative, a broken kernel far above."""
    for tag, err, scale in errors:
        if not err <= atol + rtol * scale:
            return tag
    return None


def format_stage_errors(errors):
    return '\n'.join(f'  {tag:20s} max|diff| {err:.3e}   ref scale {scale:.3e}' for tag, err, scale in errors)


def _model_of(engine):
    for name in ('sevennet_0', 'sevennet_l3i5'):
        if model_weights(name)[0] is engine.meta:
            return name
    raise ValueError('pass the oracle result (ref=) for an engine not built from a shipped model')
