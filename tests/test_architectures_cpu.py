"""CPU checks for models other than SevenNet-0 / SevenNet-l3i5: synthetic reference checkpoints convert to the
expected specs, and every tensor-product kind generated for the new (lmax_filter, lmax_out) groups passes the
numpy-einsum forward / backward check and the packed-pair-vs-scalar check of the generated arithmetic."""
import ctypes
import importlib.util
import os
import re
import subprocess

import numpy as np
import pytest

from sevenn_b200.cg import tp_path_coefficients
from sevenn_b200.sh import spherical_harmonics
from synthetic_models import ARCHS, convert, irreps_per_layer, write_checkpoint

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'sevenn_b200', 'csrc')
F32P = ctypes.POINTER(ctypes.c_float)
OLD_KINDS = ([(l1, 2, 2) for l1 in range(3)] + [(l1, 2, 0) for l1 in range(3)]
             + [(l1, 3, 3) for l1 in range(4)] + [(l1, 3, 0) for l1 in range(4)])


def _gen_kernels():
    spec = importlib.util.spec_from_file_location('gen_kernels', os.path.join(CSRC, 'gen_kernels.py'))
    gk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gk)
    return gk


GK = _gen_kernels()
NEW_KINDS = [k for k in GK.KINDS if k not in OLD_KINDS]


def fp(a):
    return a.ctypes.data_as(F32P)


def ip(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))


def _expected_paths(l1, lf, lo):
    return sorted([(l2, l3) for l2 in range(lf + 1) for l3 in range(abs(l1 - l2), l1 + l2 + 1) if l3 <= lo],
                  key=lambda p: (p[1], p[0]))


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    """the C interface of tests/cpu_harness/tp_harness.cpp, instantiated for the new kinds of gen_kernels.KINDS"""
    src = open(os.path.join(ROOT, 'tests', 'cpu_harness', 'tp_harness.cpp')).read()
    src = src.replace('"../../sevenn_b200/csrc/generated/', '"' + os.path.join(CSRC, 'generated') + '/')
    kinds = ' '.join(f'X({a},{b},{c})' for a, b, c in NEW_KINDS)
    src, n = re.subn(r'#define FOR_KINDS\(X\)(?:[^\n]*\\\n)*[^\n]*\n', f'#define FOR_KINDS(X) {kinds}\n', src, count=1)
    assert n == 1
    d = tmp_path_factory.mktemp('arch_harness')
    cpp, so = d / 'tp_harness_new.cpp', d / 'libtp_harness_new.so'
    cpp.write_text(src)
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-shared', '-fPIC', str(cpp), '-o', str(so)])
    return ctypes.CDLL(str(so))


def test_every_group_is_generated():
    groups = {(lf, lo) for lf in (1, 2, 3) for lo in range(4)}
    assert set(GK.GROUPS) == groups
    for lf, lo in groups:
        assert os.path.exists(os.path.join(CSRC, f'conv_group_{lf}{lo}.cu'))
        for l1 in range(4):
            # every kind with a path is generated; a role without paths has no kind (and launches nothing)
            assert ((l1, lf, lo) in GK.KINDS) == bool(_expected_paths(l1, lf, lo)), (l1, lf, lo)
    assert GK.KINDS[:len(OLD_KINDS)] == OLD_KINDS       # the kinds of the two pretrained models come first, unchanged
    committed = open(os.path.join(CSRC, 'generated', 'tp_kinds.cuh')).read()
    for k in NEW_KINDS:
        assert GK.gen_kind(*k) in committed


@pytest.mark.parametrize('l1,lf,lo', NEW_KINDS)
def test_new_kind_forward_backward(lib, l1, lf, lo):
    npath, nacc = ctypes.c_int(), ctypes.c_int()
    l2s, l3s, offs = (np.zeros(16, np.int32) for _ in range(3))
    assert lib.tp_info(l1, lf, lo, ctypes.byref(npath), ctypes.byref(nacc), ip(l2s), ip(l3s), ip(offs)) == 0
    npath, nacc = npath.value, nacc.value
    expect = _expected_paths(l1, lf, lo)
    assert [(int(a), int(b)) for a, b in zip(l2s[:npath], l3s[:npath])] == expect
    assert list(offs[:npath]) == list(np.cumsum([0] + [2 * l3 + 1 for _, l3 in expect])[:-1])

    rng = np.random.RandomState(1000 + l1 * 100 + lf * 10 + lo)
    d1, ny = 2 * l1 + 1, (lf + 1) ** 2
    x = rng.normal(size=d1).astype(np.float32)
    Y = spherical_harmonics(lf, rng.normal(size=3)).astype(np.float32)
    w = rng.normal(size=npath).astype(np.float32)
    ga = rng.normal(size=nacc).astype(np.float32)
    acc0 = rng.normal(size=nacc).astype(np.float32)
    acc = acc0.copy()
    assert lib.tp_fwd(l1, lf, lo, fp(x), fp(Y), fp(w), fp(acc)) == 0
    ref = acc0.astype(np.float64).copy()
    dw_ref, dx_ref, dY_ref = np.zeros(npath), np.zeros(d1), np.zeros(ny)
    for p, (l2, l3) in enumerate(expect):
        c = tp_path_coefficients(l1, l2, l3)
        yb = Y[l2 * l2:(l2 + 1) ** 2].astype(np.float64)
        gab = ga[offs[p]:offs[p] + 2 * l3 + 1].astype(np.float64)
        s = np.einsum('ijk,i,j->k', c, x.astype(np.float64), yb)
        ref[offs[p]:offs[p] + 2 * l3 + 1] += w[p] * s
        dw_ref[p] = s @ gab
        dx_ref += w[p] * np.einsum('ijk,j,k->i', c, yb, gab)
        dY_ref[l2 * l2:(l2 + 1) ** 2] += w[p] * np.einsum('ijk,i,k->j', c, x.astype(np.float64), gab)
    assert np.allclose(acc, ref, atol=2e-5, rtol=1e-5)

    dw, dx = np.zeros(npath, np.float32), np.zeros(d1, np.float32)
    dY0 = rng.normal(size=ny).astype(np.float32)
    dY = dY0.copy()
    assert lib.tp_bwd(l1, lf, lo, fp(x), fp(Y), fp(w), fp(ga), fp(dw), fp(dx), fp(dY)) == 0
    assert np.allclose(dw, dw_ref, atol=2e-5, rtol=1e-5)
    assert np.allclose(dx, dx_ref, atol=2e-5, rtol=1e-5)
    dY_ref[0] = 0.0        # Y_0 is a constant: the kernels never produce dE/dY_0
    assert np.allclose(dY - dY0, dY_ref, atol=3e-5, rtol=1e-5)


@pytest.mark.parametrize('l1,lf,lo', NEW_KINDS)
def test_new_kind_packed_pair_matches_scalar(lib, l1, lf, lo):
    npath, nacc = ctypes.c_int(), ctypes.c_int()
    t = [np.zeros(16, np.int32) for _ in range(3)]
    assert lib.tp_info(l1, lf, lo, ctypes.byref(npath), ctypes.byref(nacc), ip(t[0]), ip(t[1]), ip(t[2])) == 0
    npath, nacc = npath.value, nacc.value
    rng = np.random.RandomState(70 + l1)
    d1, ny = 2 * l1 + 1, (lf + 1) ** 2
    Y = spherical_harmonics(lf, rng.normal(size=3)).astype(np.float32)
    x2, w2, ga2 = (rng.normal(size=(n, 2)).astype(np.float32) for n in (d1, npath, nacc))
    acc2 = np.zeros((nacc, 2), np.float32)
    dw2, dx2, dY2 = np.zeros((npath, 2), np.float32), np.zeros((d1, 2), np.float32), np.zeros((ny, 2), np.float32)
    assert lib.tp_fwd2(l1, lf, lo, fp(x2), fp(Y), fp(w2), fp(acc2)) == 0
    assert lib.tp_bwd2(l1, lf, lo, fp(x2), fp(Y), fp(w2), fp(ga2), fp(dw2), fp(dx2), fp(dY2)) == 0
    for h in range(2):
        x, w, ga = (np.ascontiguousarray(a[:, h]) for a in (x2, w2, ga2))
        acc = np.zeros(nacc, np.float32)
        dw, dx, dY = np.zeros(npath, np.float32), np.zeros(d1, np.float32), np.zeros(ny, np.float32)
        lib.tp_fwd(l1, lf, lo, fp(x), fp(Y), fp(w), fp(acc))
        lib.tp_bwd(l1, lf, lo, fp(x), fp(Y), fp(w), fp(ga), fp(dw), fp(dx), fp(dY))
        assert np.allclose(acc2[:, h], acc, atol=1e-6) and np.allclose(dw2[:, h], dw, atol=1e-6)
        assert np.allclose(dx2[:, h], dx, atol=1e-6) and np.allclose(dY2[:, h], dY, atol=1e-6)


@pytest.mark.parametrize('arch', sorted(ARCHS))
def test_synthetic_checkpoint_converts(tmp_path, arch):
    from sevenn_b200.spec import build_spec, irreps_dim, parse_even_irreps
    meta, arrays = convert(write_checkpoint(tmp_path / f'{arch}.pth', arch), arch)
    a = ARCHS[arch]
    assert meta['irreps_per_layer'] == irreps_per_layer(arch) and meta['lmax_filter'] == a['lmax_edge']
    spec = build_spec(meta)
    assert spec.n_layers == a['layers'] and spec.n_sh == (a['lmax_edge'] + 1) ** 2
    mid = parse_even_irreps(a['mid'])
    assert len(mid) == a['lmax_node'] + 1
    for L in spec.layers:
        assert L.dim_x == irreps_dim(list(L.x_muls))
        want = [(l1, l2, l3) for l1 in range(len(L.x_muls)) for l2 in range(a['lmax_edge'] + 1)
                for l3 in range(abs(l1 - l2), l1 + l2 + 1) if l3 < len(L.out_muls)]
        assert sorted((p.l1, p.l2, p.l3) for p in L.paths) == sorted(want)
        assert [p.l3 for p in L.paths] == sorted(p.l3 for p in L.paths)
        assert L.weight_numel == sum(L.x_muls[p.l1] for p in L.paths)
        assert arrays[f'{L.t}.mlp2'].shape == (64, L.weight_numel)
        assert L.mid_K == tuple(sum(L.x_muls[p.l1] for p in L.paths if p.l3 == l3) for l3 in range(len(L.out_muls)))
    # an energy of the right order on a small Si cell (fp64 oracle): the weights are scaled like a trained model
    from oracle.oracle import Oracle
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.05, seed=1)
    ei, ev = build_graph(pos, cell, True, 5.0)
    sp = np.array([spec.type_map[int(v)] for v in z])
    ref = Oracle(meta, arrays).forward(sp, ei, ev)
    assert 0.5 < abs(float(ref['energy'])) / len(z) < 50.0
    assert float(ref['forces'].abs().max()) < 100.0


def test_parity_checkpoint_still_refused(tmp_path):
    with pytest.raises(NotImplementedError, match='is_parity'):
        convert(write_checkpoint(tmp_path / 'p.pth', 'B', parity=True), 'B')
