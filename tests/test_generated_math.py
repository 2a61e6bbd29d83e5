"""CPU check of the GENERATED CUDA arithmetic (tensor-product bodies and spherical harmonics):
the same headers the kernels include are compiled with g++ and compared with numpy einsum over
the coupling tensors of sevenn_b200/cg.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from sevenn_b200.cg import tp_path_coefficients
from sevenn_b200.sh import spherical_harmonics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32P = ctypes.POINTER(ctypes.c_float)


def fp(a):
    return a.ctypes.data_as(F32P)


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    # regenerate into a scratch dir and make sure the committed headers are current
    src = os.path.join(ROOT, 'tests', 'cpu_harness', 'tp_harness.cpp')
    so = str(tmp_path_factory.mktemp('harness') / 'libtp_harness.so')
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-shared', '-fPIC', src, '-o', so])
    return ctypes.CDLL(so)


KINDS = ([(l1, 2, 2) for l1 in range(3)] + [(l1, 2, 0) for l1 in range(3)]
         + [(l1, 3, 3) for l1 in range(4)] + [(l1, 3, 0) for l1 in range(4)])


@pytest.mark.parametrize('l1,lf,lo', KINDS)
def test_tp_kind_forward_backward(lib, l1, lf, lo):
    npath, nacc = ctypes.c_int(), ctypes.c_int()
    l2s, l3s, offs = (np.zeros(16, np.int32) for _ in range(3))
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    assert lib.tp_info(l1, lf, lo, ctypes.byref(npath), ctypes.byref(nacc), ip(l2s), ip(l3s), ip(offs)) == 0
    npath, nacc = npath.value, nacc.value
    expect = sorted([(l2, l3) for l2 in range(lf + 1) for l3 in range(abs(l1 - l2), l1 + l2 + 1) if l3 <= lo],
                    key=lambda p: (p[1], p[0]))
    assert [(int(a), int(b)) for a, b in zip(l2s[:npath], l3s[:npath])] == expect

    rng = np.random.RandomState(l1 * 100 + lf * 10 + lo)
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


@pytest.mark.parametrize('l1,lf,lo', KINDS)
def test_tp_kind_packed_pair_instantiation_matches_scalar(lib, l1, lf, lo):
    """The V2 (two channels per lane on the GPU) instantiation of the generated code equals
    two independent scalar evaluations."""
    npath, nacc = ctypes.c_int(), ctypes.c_int()
    t = [np.zeros(16, np.int32) for _ in range(3)]
    ip = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_int))
    lib.tp_info(l1, lf, lo, ctypes.byref(npath), ctypes.byref(nacc), ip(t[0]), ip(t[1]), ip(t[2]))
    npath, nacc = npath.value, nacc.value
    rng = np.random.RandomState(7 + l1)
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


@pytest.mark.parametrize('lmax', [1, 2, 3])
def test_sh_eval_and_vjp(lib, lmax):
    rng = np.random.RandomState(lmax)
    ny = (lmax + 1) ** 2
    for _ in range(10):
        v = rng.normal(size=3)
        u = (v / np.linalg.norm(v)).astype(np.float32)
        Y = np.zeros(ny, np.float32)
        assert lib.sh_eval(lmax, ctypes.c_float(u[0]), ctypes.c_float(u[1]), ctypes.c_float(u[2]), fp(Y)) == 0
        assert np.allclose(Y, spherical_harmonics(lmax, u.astype(np.float64)), atol=3e-6)
        gY = rng.normal(size=ny).astype(np.float32)
        g = np.zeros(3, np.float32)
        assert lib.sh_vjp(lmax, ctypes.c_float(u[0]), ctypes.c_float(u[1]), ctypes.c_float(u[2]), fp(gY), fp(g)) == 0
        # finite differences of sum_j gY_j Y_j(v/|v|) w.r.t. v: tangential part of g, divided by |v| (=1)
        eps, num = 1e-5, np.zeros(3)
        for c in range(3):
            dp, dm = u.astype(np.float64).copy(), u.astype(np.float64).copy()
            dp[c] += eps
            dm[c] -= eps
            num[c] = (gY[1:].astype(np.float64) @ (spherical_harmonics(lmax, dp)[1:] - spherical_harmonics(lmax, dm)[1:])) / (2 * eps)
        ud = u.astype(np.float64)
        gt = g.astype(np.float64) - ud * (ud @ g.astype(np.float64))
        assert np.allclose(gt, num, atol=2e-4)


def test_generated_headers_are_current(tmp_path):
    """The committed generated/*.cuh must be what gen_kernels.py produces now."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('gen_kernels', os.path.join(ROOT, 'sevenn_b200', 'csrc', 'gen_kernels.py'))
    gk = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gk)
    committed = open(os.path.join(ROOT, 'sevenn_b200', 'csrc', 'generated', 'tp_kinds.cuh')).read()
    for k in gk.KINDS[:3]:
        assert gk.gen_kind(*k) in committed
