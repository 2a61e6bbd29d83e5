"""CPU checks of the Hessian-vector product's per-edge arithmetic: the generated second-order harmonics SH2<L>, the
edge tangent and the edge backward tangent of sevenn_b200/csrc/hvp_math.cuh (compiled with g++ like
tests/test_tp_tangent_cpu.py does) against fp64 numpy, the forward-mode radial weights (engine.radial_weights_jet)
against fp64 differences of engine.radial_weights, and the ctypes signature of s7b_engine_hvp."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import sympy as sp

from sevenn_b200.sh import X, Y, Z, sh_polynomials

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32P = ctypes.POINTER(ctypes.c_float)


def fp(a):
    return np.ascontiguousarray(a, dtype=np.float32).ctypes.data_as(F32P)


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    src = os.path.join(ROOT, 'tests', 'cpu_harness', 'hvp_harness.cpp')
    so = str(tmp_path_factory.mktemp('harness') / 'libhvp_harness.so')
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-shared', '-fPIC', src, '-o', so])
    lib = ctypes.CDLL(so)
    lib.hv_edge_bwd_tangent.argtypes = [ctypes.c_int, F32P, F32P, F32P, F32P, ctypes.c_float, ctypes.c_float, F32P]
    lib.hv_radial_basis_jet.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_float,
                                        F32P, ctypes.c_int, F32P]
    return lib


_CACHE = {}


def sh64(L):
    """fp64 (Y(u), vjp(u, gY)) of the unconstrained polynomials the generated code restates"""
    if L not in _CACHE:
        polys = sh_polynomials(L)
        grad = [[sp.diff(p, v) for v in (X, Y, Z)] for p in polys]
        _CACHE[L] = (sp.lambdify((X, Y, Z), polys, 'numpy'), sp.lambdify((X, Y, Z), grad, 'numpy'))
    fY, fJ = _CACHE[L]
    Yv = lambda u: np.array([float(v) for v in fY(*u)])
    vjp = lambda u, gY: np.array([[float(c) for c in row] for row in fJ(*u)]).T @ gY
    return Yv, vjp


def unit(rng):
    u = rng.normal(size=3)
    return u / np.linalg.norm(u)


@pytest.mark.parametrize('L', [1, 2, 3])
def test_sh_hvp_against_differences_of_vjp(lib, L):
    """SH2<L>::hvp = d/dh vjp(u + h t, gY) at h = 0, by fp64 central differences with Richardson extrapolation"""
    rng = np.random.RandomState(L)
    _, vjp = sh64(L)
    ny = (L + 1) ** 2
    worst = 0.0
    for _ in range(20):
        u, t = unit(rng), rng.normal(size=3)
        gY = rng.normal(size=ny)
        gY[0] = 0.0
        d = lambda h: (vjp(u + h * t, gY) - vjp(u - h * t, gY)) / (2 * h)
        ref = (4 * d(1e-4) - d(2e-4)) / 3
        out = np.zeros(3, np.float32)
        assert lib.hv_sh_hvp(L, fp(u), fp(gY), fp(t), out.ctypes.data_as(F32P)) == 0
        scale = np.abs(gY).sum() * np.abs(t).sum() * 10 ** L
        worst = max(worst, np.abs(out - ref).max() / scale)
    assert worst < 1e-6, worst


def edge_geometry64(L, v):
    """fp64 (r, Y(v / r)) as the edge kernels define them"""
    Yv, _ = sh64(L)
    r = np.linalg.norm(v)
    return r, Yv(v / r)


EDGE_VECTORS = [np.array([1.3, -0.7, 2.1]), np.array([1e-4, 2e-4, -1.5e-4]), np.array([0.0, 0.0, 3e-3]),
                np.array([4.9, 0.3, 0.2]), np.array([5.5, -3.0, 1.0]), np.array([-2.0, 7.0, 0.5])]


@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('k', range(len(EDGE_VECTORS)))
def test_edge_tangent(lib, L, k):
    """(dr, dY) of edge_tangent<L> against fp64 central differences along dv, from r ~ 1e-4 to beyond the cutoff"""
    rng = np.random.RandomState(10 * L + k)
    v = EDGE_VECTORS[k]
    r = np.linalg.norm(v)
    dv = rng.normal(size=3) * r           # keep the step relative to the edge
    h = 1e-5
    (rp, Yp), (rm, Ym) = edge_geometry64(L, v + h * dv), edge_geometry64(L, v - h * dv)
    ref_r, ref_Y = (rp - rm) / (2 * h), (Yp - Ym) / (2 * h)
    dr = ctypes.c_float()
    dY = np.zeros((L + 1) ** 2, np.float32)
    assert lib.hv_edge_tangent(L, fp(v), fp(dv), ctypes.byref(dr), dY.ctypes.data_as(F32P)) == 0
    assert abs(dr.value - ref_r) < 1e-5 * r * np.linalg.norm(dv) / r + 1e-12
    assert dY[0] == 0.0
    assert np.abs(dY - ref_Y).max() < 1e-4 * np.abs(ref_Y).max() + 1e-6


@pytest.mark.parametrize('L', [1, 2, 3])
def test_edge_tangent_zero_vector(lib, L):
    """r = 0 has no direction: zeros, no NaN"""
    dr = ctypes.c_float()
    dY = np.full((L + 1) ** 2, np.nan, np.float32)
    assert lib.hv_edge_tangent(L, fp(np.zeros(3)), fp(np.ones(3)), ctypes.byref(dr), dY.ctypes.data_as(F32P)) == 0
    assert dr.value == 0.0 and np.all(dY == 0.0)


def edge_force64(L, v, gY, ar):
    """fp64 edge_bwd_kernel: f = ar u + (I - u u^T) vjp(u, gY) / r"""
    _, vjp = sh64(L)
    r = np.linalg.norm(v)
    u = v / r
    g = vjp(u, gY)
    return ar * u + (g - (g @ u) * u) / r


@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('k', range(len(EDGE_VECTORS)))
def test_edge_bwd_tangent(lib, L, k):
    """edge_bwd_tangent<L> = d/de f(v + e dv; gY + e dgY, ar + e dar) by fp64 central differences"""
    rng = np.random.RandomState(100 + 10 * L + k)
    v = EDGE_VECTORS[k]
    r = np.linalg.norm(v)
    ny = (L + 1) ** 2
    dv = rng.normal(size=3) * r
    gY, dgY = rng.normal(size=ny), rng.normal(size=ny)
    gY[0] = dgY[0] = 0.0
    ar, dar = rng.normal(), rng.normal()
    f = lambda e: edge_force64(L, v + e * dv, gY + e * dgY, ar + e * dar)
    h = 1e-6
    ref = (f(h) - f(-h)) / (2 * h)
    df = np.zeros(3, np.float32)
    assert lib.hv_edge_bwd_tangent(L, fp(v), fp(dv), fp(gY), fp(dgY), ar, dar, df.ctypes.data_as(F32P)) == 0
    scale = (abs(dar) + abs(ar) + np.abs(gY).sum() * 10 ** L / r + np.abs(dgY).sum() * 10 ** L / r)
    assert np.abs(df - ref).max() < 2e-6 * scale, (df, ref)


def _spec_arrays(cutoff_fn, cutoff=5.0, r_on=4.5, p=6, nb=8, seed=0):
    from sevenn_b200.spec import ModelSpec
    rng = np.random.RandomState(seed)
    spec = ModelSpec.__new__(ModelSpec)
    object.__setattr__(spec, 'cutoff', cutoff)
    object.__setattr__(spec, 'cutoff_fn', cutoff_fn)
    object.__setattr__(spec, 'cutoff_on', r_on)
    object.__setattr__(spec, 'poly_p', p)
    object.__setattr__(spec, 'radial_hidden', [16, 24])
    arrays = {'bessel_coeffs': np.arange(1, nb + 1) * np.pi / cutoff * (1 + rng.uniform(-0.05, 0.05, nb)),
              '0.mlp0': rng.normal(size=(nb, 16)), '0.mlp1': rng.normal(size=(16, 24)), '0.mlp2': rng.normal(size=(24, 32))}
    return spec, arrays


@pytest.mark.parametrize('cutoff_fn,p', [('XPLOR', 0), ('poly_cut', 6), ('poly_cut', 3)])
def test_radial_weights_jet(cutoff_fn, p):
    """w, w', w'' of the forward-mode restatement against engine.radial_weights (w, w') and fp64 central differences
    of its w' (w''), on both sides of r_on and up to the cutoff; zero from the cutoff on"""
    from sevenn_b200.engine import radial_weights, radial_weights_jet
    spec, arrays = _spec_arrays(cutoff_fn, p=p)
    r = np.concatenate([np.linspace(0.3, 4.45, 40), [4.47, 4.53], np.linspace(4.55, 4.97, 12)])
    w0, w1, w2 = radial_weights_jet(spec, arrays, 0, r)
    f, df = radial_weights(spec, arrays, 0, r)
    assert np.allclose(w0, f, rtol=1e-12, atol=1e-12 * np.abs(f).max())
    assert np.allclose(w1, df, rtol=1e-10, atol=1e-10 * np.abs(df).max())
    h = 1e-5
    d2 = (radial_weights(spec, arrays, 0, r + h)[1] - radial_weights(spec, arrays, 0, r - h)[1]) / (2 * h)
    assert np.abs(w2 - d2).max() < 1e-6 * np.abs(d2).max()
    beyond = radial_weights_jet(spec, arrays, 0, np.array([5.0, 5.2]))
    assert all(np.all(b == 0.0) for b in beyond)


@pytest.mark.parametrize('cutoff_fn,p', [('XPLOR', 0), ('poly_cut', 6), ('poly_cut', 3)])
def test_device_radial_basis_jet(lib, cutoff_fn, p):
    """the device's envelope x Bessel jet (hvp_math.cuh) against the numpy restatement's first MLP input"""
    spec, arrays = _spec_arrays(cutoff_fn, p=p)
    r = np.concatenate([[1e-3, 0.01, 0.1], np.linspace(0.3, 4.97, 60), [5.0, 5.4]]).astype(np.float32)
    fn = 0 if cutoff_fn == 'XPLOR' else 1
    for b, c in enumerate(arrays['bessel_coeffs']):
        out = np.zeros((len(r), 3), np.float32)
        lib.hv_radial_basis_jet(fn, spec.cutoff, spec.cutoff_on, p, float(c), fp(r), len(r), out.ctypes.data_as(F32P))
        # reference: one-hot MLP input picks basis b out of the numpy jet
        one = {'bessel_coeffs': arrays['bessel_coeffs'], '0.mlp0': np.eye(len(arrays['bessel_coeffs']))[:, [b]] * np.sqrt(8)}
        spec1 = spec.__class__.__new__(spec.__class__)
        for k in ('cutoff', 'cutoff_fn', 'cutoff_on', 'poly_p'):
            object.__setattr__(spec1, k, getattr(spec, k))
        object.__setattr__(spec1, 'radial_hidden', [])
        ref = np.stack([a[:, 0] for a in radial_weights_jet_nomlp(spec1, one, r.astype(np.float64))], axis=1)
        tol = 2e-5 * np.abs(ref).max(axis=0) + 1e-6
        assert np.all(np.abs(out - ref) <= tol), (b, np.abs(out - ref).max(axis=0), tol)


def radial_weights_jet_nomlp(spec, arrays, r):
    from sevenn_b200.engine import radial_weights_jet
    return radial_weights_jet(spec, arrays, 0, r)


def test_silu_n_jet(lib):
    from sevenn_b200.spec import SILU_NORM
    z = np.linspace(-8, 8, 101).astype(np.float32)
    out = np.zeros((len(z), 3), np.float32)
    lib.hv_silu_n_jet(fp(z), len(z), out.ctypes.data_as(F32P))
    s = lambda x: SILU_NORM * x / (1 + np.exp(-x))
    zz, h = z.astype(np.float64), 1e-4
    ref = np.stack([s(zz), (s(zz + h) - s(zz - h)) / (2 * h), (s(zz + h) - 2 * s(zz) + s(zz - h)) / h ** 2], axis=1)
    assert np.abs(out - ref).max() < 1e-5


def test_hvp_ctypes_signature():
    """The ctypes argtypes of s7b_engine_hvp (sevenn_b200/engine.py) follow its declaration in include/sevenn_b200.h"""
    lib_path = os.path.join(ROOT, 'sevenn_b200', 'lib', 'libsevenn_b200.so')
    if not os.path.exists(lib_path):
        import __graft_entry__
        __graft_entry__.build()
    header = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API\s+int\s+s7b_engine_hvp\s*\(([^)]*)\)', header)
    assert m is not None
    params = [p.strip() for p in m.group(1).split(',')]
    assert [re.findall(r'\w+', p)[-1] for p in params] == ['eng', 'd_v', 'd_out', 'stream']
    assert all('*' in p for p in params)
    from sevenn_b200.engine import load_library
    assert load_library().s7b_engine_hvp.argtypes == [ctypes.c_void_p] * 4
