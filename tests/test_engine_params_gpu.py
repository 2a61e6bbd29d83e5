"""s7b_engine_set_param refuses what the kernels cannot read: every parameter of SevenNet-0 (radial tables and the
exact radial MLP) and of the 'nequip' variant of synthetic model B one element short and one long, unknown names,
per-layer names outside [0, n_layers) and global names with a layer.  After all of them the engine computes what a
fresh engine computes."""
import os

import numpy as np
import pytest

from helpers import ROOT

pytestmark = pytest.mark.gpu

UNKNOWN = ['si1t', 'table_fw', '']


@pytest.fixture(scope='module', params=['sevennet_0-table', 'sevennet_0-mlp', 'B_nequip-table'])
def case(request, tmp_path_factory):
    """(meta, arrays, radial, prepared parameters {(name, layer): fp32 array}, engine)"""
    from sevenn_b200.engine import B200Engine, prepare_params
    model, radial = request.param.split('-')
    if model == 'sevennet_0':
        from sevenn_b200.checkpoint import load_weights
        meta, arrays = load_weights(os.path.join(ROOT, 'weights', 'sevennet_0.npz'))
    else:
        from synthetic_nequip import convert, write_nequip_checkpoint
        path = write_nequip_checkpoint(tmp_path_factory.mktemp('nequip_ckpt') / 'synthetic_B_nequip.pth', 'B', seed=11)
        meta, arrays = convert(path, 'B')
    eng = B200Engine(meta, arrays, radial=radial)
    return meta, arrays, radial, prepare_params(eng.spec, arrays, radial, eng.knots), eng


def _upload(eng, name, layer, arr):
    from sevenn_b200.engine import check
    arr = np.ascontiguousarray(arr, np.float32)
    check(eng.lib.s7b_engine_set_param(eng._h, name.encode(), int(layer), arr.ctypes.data, arr.size))


def _refusals(params, n_layers):
    """(name, layer, array, strings the error must contain) of every upload the engine must refuse.  The arrays hold
    seeded random values, not the model's, so that a refused call which still wrote the engine would change what
    it computes."""
    rng = np.random.RandomState(17)
    values = lambda n: rng.standard_normal(n).astype(np.float32)
    out = []
    for (name, t), arr in params.items():
        n = arr.size
        who = [f'parameter {name} '] + ([f'layer {t}:'] if t >= 0 else [])
        out += [(name, t, values(n - 1), who), (name, t, values(n + 1), who)]
        if t >= 0:
            out += [(name, bad, values(n), [f'parameter {name} ', f'layer {bad} ']) for bad in (-1, n_layers)]
        else:
            out.append((name, 0, values(n), ['layer 0:', f'parameter {name} ']))
    n = params[('si2', 0)].size
    out += [(name, 0, values(n), [f"unknown parameter '{name}'"]) for name in UNKNOWN]
    return out


def test_refused_uploads_name_the_parameter(case):
    _, _, _, params, eng = case
    for name, layer, arr, who in _refusals(params, eng.spec.n_layers):
        with pytest.raises(RuntimeError) as err:
            _upload(eng, name, layer, arr)
        for s in who:
            assert s in str(err.value), (name, layer, arr.size, str(err.value))


def test_refused_uploads_leave_the_engine_unchanged(case):
    """per-atom energies bit for bit; forces within what the float atomics of the force scatter vary between runs.
    That each call is refused is test_refused_uploads_name_the_parameter's; here only what the engine computes after
    them counts, so an upload that raises but still changed the engine fails here."""
    import torch
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import build_graph, diamond_si
    meta, arrays, radial, params, eng = case
    for name, layer, arr, _ in _refusals(params, eng.spec.n_layers):
        try:
            _upload(eng, name, layer, arr)
        except RuntimeError:
            pass
    pos, cell, _ = diamond_si(2, 2, 2, sigma=0.05, seed=5)
    ei, ev = build_graph(pos, cell, True, float(eng.spec.cutoff))
    species = np.random.RandomState(5).randint(0, eng.spec.num_species, size=len(pos))

    def run(e):
        e.set_graph(species, ei, ev)
        e.compute()
        torch.cuda.synchronize()
        r = e.results()
        return r['atomic_energy'].cpu().numpy(), r['forces'].cpu().numpy()

    ae, f = run(eng)
    ae_fresh, f_fresh = run(B200Engine(meta, arrays, radial=radial))
    assert np.array_equal(ae.view(np.uint32), ae_fresh.view(np.uint32))
    fs = max(1.0, float(np.abs(f_fresh).max()))
    assert float(np.abs(f - f_fresh).max()) <= 1e-5 * fs
