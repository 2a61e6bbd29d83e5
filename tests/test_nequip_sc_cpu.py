"""The species-wise ('nequip') self-connection on the CPU: checkpoint conversion, the fp64 oracle (pinned to the
already-pinned linear self-connection), the weight folds of prepare_params and the flat export."""
import struct

import numpy as np
import pytest
import torch

from nequip_oracle import nequip_oracle, species_linear
from synthetic_models import NUMBERS, convert as convert_linear, write_checkpoint
from synthetic_nequip import S, convert, nequip_checkpoint, write_nequip_checkpoint


def _mixed_si64(meta, seed=0):
    """64-atom rattled diamond cell with the atoms' species drawn from all S species"""
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, _ = diamond_si(2, 2, 2, sigma=0.05, seed=seed)
    ei, ev = build_graph(pos, cell, True, 5.0)
    sp = np.random.RandomState(seed).randint(0, S, size=len(pos))
    return sp, ei, ev


@pytest.mark.parametrize('arch', ['A', 'B'])
def test_equivalent_to_linear_self_connection(tmp_path, arch):
    """W_l[:, s, :] = sqrt(S) M_l for every s is the linear self-connection with weights M_l"""
    meta_l, arr_l = convert_linear(write_checkpoint(tmp_path / 'lin.pth', arch, seed=3), arch)
    meta_n, arr_n = convert(write_nequip_checkpoint(tmp_path / 'neq.pth', arch, seed=3, sc='from_linear'), arch)
    assert meta_l['self_connection'] == 'linear' and meta_n['self_connection'] == 'nequip'
    assert arr_n['1.sc'].size == S * arr_l['1.sc'].size
    # the file holds fp32(sqrt(S) M): compare against the linear model with M = that / sqrt(S) in fp64
    from sevenn_b200.spec import build_spec, sc_blocks
    for L in build_spec(meta_l).layers:
        parts, off = [], 0
        for k, n in sc_blocks(L):
            W = arr_n[f'{L.t}.sc'][off:off + k * S * n].astype(np.float64).reshape(k, S, n)
            assert np.all(W == W[:, :1, :])
            parts.append((W[:, 0, :] / np.sqrt(S)).ravel())
            off += k * S * n
        assert np.allclose(np.concatenate(parts), arr_l[f'{L.t}.sc'], rtol=1e-6, atol=0)
        arr_l[f'{L.t}.sc'] = np.concatenate(parts)
    sp, ei, ev = _mixed_si64(meta_l)
    ref = nequip_oracle(meta_l, arr_l).forward(sp, ei, ev)
    out = nequip_oracle(meta_n, arr_n).forward(sp, ei, ev)
    assert abs(float(out['energy']) - float(ref['energy'])) < 1e-10
    assert float((out['forces'] - ref['forces']).abs().max()) < 1e-10
    assert float((out['atomic_energy'] - ref['atomic_energy']).abs().max()) < 1e-10


def test_only_one_species_gets_a_self_connection(tmp_path):
    meta, arrays = convert(write_nequip_checkpoint(tmp_path / 'one.pth', 'A', seed=1, sc='one_species', only=4), 'A')
    from sevenn_b200.spec import build_spec
    spec = build_spec(meta)
    L = spec.layers[1]
    rng = np.random.RandomState(0)
    sp = torch.as_tensor(np.concatenate([np.arange(S), rng.randint(0, S, size=40)]))
    x = torch.as_tensor(rng.standard_normal((len(sp), L.dim_x)))
    from oracle.oracle import Oracle
    blocks = Oracle._blocks(L.x_muls)
    sc = species_linear(x, torch.as_tensor(arrays['1.sc'], dtype=torch.float64), blocks, list(L.gate_muls), sp, S)
    mine = (sp == 4).numpy()
    assert float(sc[~mine].abs().max()) == 0.0
    assert float(sc[mine].abs().min(dim=1).values.max()) > 0.0 and float(sc[mine].abs().max()) > 1e-2
    # the engine's per-species weights: only the slice of species 4 is non-zero
    from sevenn_b200.engine import default_table_knots, prepare_params
    P = prepare_params(spec, arrays, 'table', default_table_knots(spec))
    per = P[('sc_species', 1)].reshape(S, -1)
    assert np.count_nonzero(np.abs(per).sum(axis=1)) == 1 and np.abs(per[4]).sum() > 0


def test_relabelled_species_leave_energies_unchanged(tmp_path):
    meta, arrays = convert(write_nequip_checkpoint(tmp_path / 'r.pth', 'A', seed=2), 'A')
    sp, ei, ev = _mixed_si64(meta, seed=1)
    ref = nequip_oracle(meta, arrays).forward(sp, ei, ev)
    perm = np.random.RandomState(7).permutation(S)          # old species s -> new index perm[s]
    inv = np.argsort(perm)
    from sevenn_b200.spec import build_spec, sc_blocks
    spec = build_spec(meta)
    meta2 = dict(meta, type_map={z: int(perm[i]) for z, i in meta['type_map'].items()})
    arr2 = dict(arrays)
    arr2['embed'] = arrays['embed'].reshape(S, -1)[inv].ravel()
    arr2['shift'], arr2['scale'] = arrays['shift'][inv], arrays['scale'][inv]
    for L in spec.layers:
        parts, off = [], 0
        for k, n in sc_blocks(L):
            parts.append(arrays[f'{L.t}.sc'][off:off + k * S * n].reshape(k, S, n)[:, inv, :].ravel())
            off += k * S * n
        arr2[f'{L.t}.sc'] = np.concatenate(parts)
    out = nequip_oracle(meta2, arr2).forward(perm[sp], ei, ev)
    assert abs(float(out['energy']) - float(ref['energy'])) < 1e-10
    assert float((out['forces'] - ref['forces']).abs().max()) < 1e-10


def test_wrong_weight_size_names_the_layer(tmp_path):
    ck = nequip_checkpoint('A', seed=0)
    k = '2_self_connection_intro.fc_tensor_product.weight'
    ck['model_state_dict'][k] = ck['model_state_dict'][k][:-32]
    path = tmp_path / 'bad.pth'
    torch.save(ck, str(path))
    with pytest.raises(ValueError, match='layer 2'):
        convert(path, 'A')
    # a linear-SC weight under a nequip config: refused the same way
    ck = nequip_checkpoint('B', seed=0)
    k = '1_self_connection_intro.fc_tensor_product.weight'
    ck['model_state_dict'][k] = ck['model_state_dict'][k][:ck['model_state_dict'][k].numel() // S]
    torch.save(ck, str(path))
    with pytest.raises(ValueError, match='layer 1'):
        convert(path, 'B')


def test_parity_nequip_checkpoint_still_refused_with_is_parity(tmp_path):
    path = write_nequip_checkpoint(tmp_path / 'p.pth', 'A', parity=True)
    with pytest.raises(NotImplementedError, match='is_parity'):
        convert(path, 'A')


def test_unknown_self_connection_type_refused(tmp_path):
    ck = nequip_checkpoint('A')
    ck['config']['self_connection_type'] = 'other'
    torch.save(ck, str(tmp_path / 'o.pth'))
    with pytest.raises(NotImplementedError, match='self_connection_type'):
        convert(tmp_path / 'o.pth', 'A')


def test_saved_files_keep_the_type_and_old_files_default_to_linear(tmp_path):
    import os
    from sevenn_b200.checkpoint import load_weights, random_weights, save_weights
    from sevenn_b200.spec import build_spec, sc_numel
    meta, arrays = convert(write_nequip_checkpoint(tmp_path / 'n.pth', 'B'), 'B')
    save_weights(str(tmp_path / 'n.npz'), meta, arrays)
    m2, a2 = load_weights(str(tmp_path / 'n.npz'))
    assert build_spec(m2).self_connection == 'nequip'
    assert all(np.array_equal(a2[k], arrays[k]) for k in arrays)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    m0, _ = load_weights(os.path.join(root, 'weights', 'sevennet_0.npz'))
    assert 'self_connection' not in m0 and build_spec(m0).self_connection == 'linear'
    w = random_weights(m2, seed=0)
    spec = build_spec(m2)
    assert all(w[f'{L.t}.sc'].size == sc_numel(L, 'nequip', S) for L in spec.layers)


@pytest.mark.parametrize('arch', ['A', 'C'])
def test_embed_g0_fold_is_the_layer0_self_connection(tmp_path, arch):
    from sevenn_b200.engine import default_table_knots, prepare_params
    from sevenn_b200.spec import build_spec
    meta, arrays = convert(write_nequip_checkpoint(tmp_path / 'f.pth', arch, seed=5), arch)
    spec = build_spec(meta)
    L0 = spec.layers[0]
    P = prepare_params(spec, arrays, 'table', default_table_knots(spec))
    h0 = torch.as_tensor(arrays['embed'], dtype=torch.float64).reshape(S, -1) / np.sqrt(S)
    from oracle.oracle import Oracle
    ref = species_linear(h0, torch.as_tensor(arrays['0.sc'], dtype=torch.float64), Oracle._blocks(L0.x_muls),
                         list(L0.gate_muls), torch.arange(S), S).numpy()
    g0 = P[('embed_g0', -1)].astype(np.float64)
    assert g0.shape == (S, L0.dim_gate)
    assert np.allclose(g0, ref, rtol=1e-6, atol=1e-7 * np.abs(ref).max())
    assert not any(name in ('sc', 'scT') for name, _ in P)


def test_species_parameters_layout(tmp_path):
    from sevenn_b200.engine import prepare_params
    from sevenn_b200.spec import build_spec, sc_blocks
    meta, arrays = convert(write_nequip_checkpoint(tmp_path / 'l.pth', 'A', seed=6), 'A')
    spec = build_spec(meta)
    P = prepare_params(spec, arrays, 'mlp', 0)
    for L in spec.layers[1:]:
        blocks, off = [], 0
        for k, n in sc_blocks(L):
            blocks.append(arrays[f'{L.t}.sc'][off:off + k * S * n].astype(np.float64).reshape(k, S, n) / np.sqrt(k * S))
            off += k * S * n
        want = np.concatenate([b[:, s, :].ravel() for s in range(S) for b in blocks])
        wantT = np.concatenate([b[:, s, :].T.ravel() for s in range(S) for b in blocks])
        assert np.array_equal(P[('sc_species', L.t)], want.astype(np.float32))
        assert np.array_equal(P[('scT_species', L.t)], wantT.astype(np.float32))


def test_export_flat_writes_species_parameters(tmp_path):
    from sevenn_b200.export import export_flat
    meta, arrays = convert(write_nequip_checkpoint(tmp_path / 'e.pth', 'B'), 'B')
    path = str(tmp_path / 'm.s7b')
    export_flat(path, meta, arrays)
    from sevenn_b200.engine import S7bModelDesc
    import ctypes
    with open(path, 'rb') as f:
        assert f.read(8) == b'S7BMODEL' and struct.unpack('<i', f.read(4))[0] == 1
        f.read(ctypes.sizeof(S7bModelDesc))
        n_arrays, n_types = struct.unpack('<ii', f.read(8))
        f.read(8 * n_types)
        names = []
        for _ in range(n_arrays):
            name = f.read(32).rstrip(b'\0').decode()
            layer, numel = struct.unpack('<iq', f.read(12))
            f.read(4 * numel)
            names.append((name, layer, numel))
    T = len(meta['irreps_per_layer']) - 1
    for t in range(1, T):
        got = {n: k for n, l, k in names if l == t}
        assert 'sc_species' in got and 'scT_species' in got and 'sc' not in got and 'scT' not in got
        assert got['sc_species'] == got['scT_species'] and got['sc_species'] % S == 0
    assert len(NUMBERS) == S
