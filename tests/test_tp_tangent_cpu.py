"""CPU checks of the convolution's second order: the per-lane arithmetic of the second-order kernels
(sevenn_b200/csrc/tp_tangent.cuh, compiled with g++ like tests/test_generated_math.py does) against numpy over the
coupling tensors of sevenn_b200/cg.py, and the ctypes signature of s7b_conv_double_backward against the header."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from sevenn_b200.cg import tp_path_coefficients
from sevenn_b200.sh import spherical_harmonics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32P = ctypes.POINTER(ctypes.c_float)
KINDS = [(0, 1, 1), (1, 1, 1), (0, 1, 0), (1, 1, 0), (2, 1, 3), (3, 1, 3),
         (0, 2, 2), (1, 2, 2), (2, 2, 2), (0, 2, 0), (1, 2, 0), (2, 2, 0), (3, 2, 3),
         (0, 3, 3), (1, 3, 3), (2, 3, 3), (3, 3, 3), (0, 3, 0), (1, 3, 0), (2, 3, 0), (3, 3, 0), (2, 3, 1)]


def fp(a):
    return a.ctypes.data_as(F32P)


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    src = os.path.join(ROOT, 'tests', 'cpu_harness', 'tp_tangent_harness.cpp')
    so = str(tmp_path_factory.mktemp('harness') / 'libtp_tangent_harness.so')
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-shared', '-fPIC', src, '-o', so])
    return ctypes.CDLL(so)


def paths(l1, lf, lo):
    return sorted([(l2, l3) for l2 in range(lf + 1) for l3 in range(abs(l1 - l2), l1 + l2 + 1) if l3 <= lo],
                  key=lambda p: (p[1], p[0]))


def tp(l1, lf, lo, x, Y, w):
    """acc of TP(x, Y, w) in fp64 (Y[0] as given: the kernels' Y_0 = 1 is the caller's business)"""
    out = []
    for p, (l2, l3) in enumerate(paths(l1, lf, lo)):
        c = tp_path_coefficients(l1, l2, l3)
        out.append(w[p] * np.einsum('ijk,i,j->k', c, x, Y[l2 * l2:(l2 + 1) ** 2]))
    return np.concatenate(out)


def jac(f, v):
    """d f / d v of a function linear in v, by unit vectors (exact up to rounding)"""
    return np.stack([f(e) for e in np.eye(len(v))], axis=1)


@pytest.mark.parametrize('has', [1, 2, 4, 7])
@pytest.mark.parametrize('l1,lf,lo', KINDS)
def test_tangent_arithmetic(lib, l1, lf, lo, has):
    rng = np.random.RandomState(l1 * 100 + lf * 10 + lo + 1000 * has)
    d1, ny, npath = 2 * l1 + 1, (lf + 1) ** 2, len(paths(l1, lf, lo))
    x, tx = (rng.normal(size=d1).astype(np.float32) for _ in range(2))
    Y = spherical_harmonics(lf, rng.normal(size=3)).astype(np.float32)
    tY = rng.normal(size=ny).astype(np.float32)
    tY[0] = 123.0                    # the kernels never read Y_0 / tY_0: the tangent's l = 0 part is 0
    w, tw = (rng.normal(size=npath).astype(np.float32) for _ in range(2))
    nacc = len(tp(l1, lf, lo, x, Y, w))
    ga = rng.normal(size=nacc).astype(np.float32)
    hx, hY, hw = bool(has & 1), bool(has & 2), bool(has & 4)

    X, TX, W, TW, GA = (v.astype(np.float64) for v in (x, tx, w, tw, ga))
    Y1 = Y.astype(np.float64)
    Y1[0] = 1.0
    TY0 = tY.astype(np.float64)
    TY0[0] = 0.0
    T = lambda x_, y_, w_: tp(l1, lf, lo, x_, y_, w_)
    zero = lambda n: np.zeros(n)
    jvp_ref = (T(TX, Y1, W) if hx else 0) + (T(X, TY0, W) if hY else 0) + (T(X, Y1, TW) if hw else 0) + zero(nacc)
    dw_ref = zero(npath)
    dx_ref = zero(d1)
    dY_ref = zero(ny)
    if hx:
        dw_ref += jac(lambda e: T(TX, Y1, e), W).T @ GA
        dY_ref += jac(lambda e: T(TX, e, W), Y1).T @ GA
    if hY:
        dw_ref += jac(lambda e: T(X, TY0, e), W).T @ GA
        dx_ref += jac(lambda e: T(e, TY0, W), X).T @ GA
    if hw:
        dx_ref += jac(lambda e: T(e, Y1, TW), X).T @ GA
        dY_ref += jac(lambda e: T(X, e, TW), Y1).T @ GA

    acc0 = rng.normal(size=nacc).astype(np.float32)
    acc = acc0.copy()
    assert lib.tt_jvp(l1, lf, lo, has, fp(x), fp(Y), fp(w), fp(tx), fp(tY), fp(tw), fp(acc)) == 0
    assert np.allclose(acc, acc0 + jvp_ref, atol=1e-5, rtol=1e-5)

    dY0 = rng.normal(size=ny).astype(np.float32)
    for out in (7, 1, 2, 4):
        dw = np.full(npath, np.nan, np.float32)
        dx = np.full(d1, np.nan, np.float32)
        dY = dY0.copy()
        assert lib.tt_bwd(l1, lf, lo, has, out, fp(x), fp(Y), fp(w), fp(ga), fp(tx), fp(tY), fp(tw),
                          fp(dw), fp(dx), fp(dY)) == 0
        assert dY[0] == dY0[0]                        # dY[0] is never written
        if out & 1:
            assert np.allclose(dw, dw_ref, atol=1e-5, rtol=1e-5), (out, dw, dw_ref)
        if out & 2:
            assert np.allclose(dx, dx_ref, atol=1e-5, rtol=1e-5), (out, dx, dx_ref)
        if out & 4:
            assert np.allclose(dY[1:], dY0[1:] + dY_ref[1:], atol=1e-5, rtol=1e-5), (out, dY, dY_ref)
        else:
            assert np.array_equal(dY, dY0)            # a pass without dY leaves the accumulator alone


def test_double_backward_ctypes_signature():
    """The ctypes argtypes of s7b_conv_double_backward (sevenn_b200/engine.py) follow its declaration in
    include/sevenn_b200.h: pointers as void*, int32_t / int64_t as c_int32 / c_int64, in order."""
    lib_path = os.path.join(ROOT, 'sevenn_b200', 'lib', 'libsevenn_b200.so')
    if not os.path.exists(lib_path):
        import __graft_entry__
        __graft_entry__.build()
    header = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API\s+int\s+s7b_conv_double_backward\s*\(([^)]*)\)', header)
    assert m is not None
    params = [p.strip() for p in m.group(1).split(',')]
    assert len(params) == 18
    want = [ctypes.c_void_p if '*' in p else {'int32_t': ctypes.c_int32, 'int64_t': ctypes.c_int64}[p.split()[0]]
            for p in params]
    names = [re.findall(r'\w+', p)[-1] for p in params]
    assert names[10:13] == ['tan_x', 'tan_sh', 'tan_weight'] and names[13:17] == \
        ['grad_grad_out', 'grad_x', 'grad_sh', 'grad_weight']
    from sevenn_b200.engine import load_library
    assert load_library().s7b_conv_double_backward.argtypes == want
