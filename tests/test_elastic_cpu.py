"""CPU checks of the elastic-tensor path: the strain term of the Hessian-vector product's edge tangent
(sevenn_b200/csrc/hvp_math.cuh, compiled with g++ through tests/cpu_harness/elastic_harness.cpp) against fp64 numpy,
the assembly of sevenn_b200/elastic.py against a brute-force relaxed-ion tensor of a Morse-pair crystal, and the
ctypes signature of s7b_engine_hvp_strain."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.optimize

from sevenn_b200 import elastic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32P = ctypes.POINTER(ctypes.c_float)
F64P = ctypes.POINTER(ctypes.c_double)
I32P = ctypes.POINTER(ctypes.c_int)


def fp(a):
    return np.ascontiguousarray(a, dtype=np.float32).ctypes.data_as(F32P)


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    src = os.path.join(ROOT, 'tests', 'cpu_harness', 'elastic_harness.cpp')
    so = str(tmp_path_factory.mktemp('harness') / 'libelastic_harness.so')
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-shared', '-fPIC', src, '-o', so])
    lib = ctypes.CDLL(so)
    lib.hv_edge_strain_tangent.argtypes = [ctypes.c_int, F32P, F32P, F32P, F64P, F32P, F32P, F32P]
    lib.hv_structure_of.argtypes = [I32P, ctypes.c_int, ctypes.c_int]
    return lib


def sh_values(L):
    import sympy as sp
    from sevenn_b200.sh import X, Y, Z, sh_polynomials
    f = sp.lambdify((X, Y, Z), sh_polynomials(L), 'numpy')
    return lambda u: np.array([float(c) for c in f(*u)])


@pytest.mark.parametrize('L', [1, 2, 3])
@pytest.mark.parametrize('with_v', [False, True])
def test_edge_strain_tangent(lib, L, with_v):
    """(dvec, dr, dY) with a general (non-symmetric) strain, alone and with a position tangent, against fp64 central
    differences of the edge geometry along vec + h (eps . vec + vs - vc)"""
    rng = np.random.RandomState(7 * L + with_v)
    Yf = sh_values(L)
    for _ in range(10):
        v = rng.normal(size=3) * 2.0
        eps = rng.normal(size=(3, 3))
        vs, vc = rng.normal(size=3), rng.normal(size=3)
        dvec = eps @ v + ((vs.astype(np.float32) - vc.astype(np.float32)).astype(np.float64) if with_v else 0.0)
        geo = lambda w: (np.linalg.norm(w), Yf(w / np.linalg.norm(w)))
        h = 1e-5
        (rp, Yp), (rm, Ym) = geo(v + h * dvec), geo(v - h * dvec)
        dv = np.zeros(3, np.float32)
        dr = ctypes.c_float()
        dY = np.zeros((L + 1) ** 2, np.float32)
        e64 = np.ascontiguousarray(eps, dtype=np.float64)
        assert lib.hv_edge_strain_tangent(L, fp(v), fp(vs) if with_v else None, fp(vc), e64.ctypes.data_as(F64P),
                                          dv.ctypes.data_as(F32P), ctypes.byref(dr), dY.ctypes.data_as(F32P)) == 0
        assert np.abs(dv - dvec).max() < 1e-6 * np.abs(dvec).max()
        assert abs(dr.value - (rp - rm) / (2 * h)) < 1e-5 * np.linalg.norm(dvec)
        ref_Y = (Yp - Ym) / (2 * h)
        assert np.abs(dY - ref_Y).max() < 1e-4 * np.abs(ref_Y).max() + 1e-6


def test_no_strain_is_the_position_tangent(lib):
    """a null strain leaves dvec = vs - vc exactly (the arithmetic of the plain HVP)"""
    v, vs, vc = np.array([1.0, 2.0, -0.5]), np.array([0.3, -0.1, 0.7]), np.array([0.11, 0.2, -0.4])
    dv = np.zeros(3, np.float32)
    dr = ctypes.c_float()
    dY = np.zeros(16, np.float32)
    lib.hv_edge_strain_tangent(3, fp(v), fp(vs), fp(vc), None, dv.ctypes.data_as(F32P), ctypes.byref(dr),
                               dY.ctypes.data_as(F32P))
    assert np.array_equal(dv, vs.astype(np.float32) - vc.astype(np.float32))


def test_structure_of(lib):
    """the structure of every atom, with empty structures anywhere in the batch"""
    ap = np.array([0, 0, 3, 3, 3, 7, 8, 8], np.int32)
    B = len(ap) - 1
    for n in range(int(ap[-1])):
        b = lib.hv_structure_of(ap.ctypes.data_as(I32P), B, n)
        assert ap[b] <= n < ap[b + 1], (n, b)
    one = np.array([0, 5], np.int32)
    assert all(lib.hv_structure_of(one.ctypes.data_as(I32P), 1, n) == 0 for n in range(5))


def test_voigt_strains():
    eps = elastic.voigt_strains()
    assert np.array_equal(eps[0], np.diag([1.0, 0, 0])) and np.array_equal(eps[2], np.diag([0, 0, 1.0]))
    assert eps[3][1, 2] == eps[3][2, 1] == 0.5 and eps[4][0, 2] == eps[4][2, 0] == 0.5
    assert eps[5][0, 1] == eps[5][1, 0] == 0.5 and all(np.count_nonzero(e) in (1, 2) for e in eps)


# ---- a Morse-pair crystal with a two-atom basis, in the engine's conventions ---------------------------------------
# Directed edges (centre c, neighbour s, vec = x_s + shift - x_c) held fixed; E = 1/2 sum_e phi(|vec_e|);
# f_e = dE/dvec_e; F_c = sum_{e: centre c} f_e - sum_{e: neighbour c} f_e; W = -sum_e vec_e (x) f_e (xx,yy,zz,xy,yz,zx).
MORSE = dict(D=0.4, a=1.4, r0=2.6)


def _phi(r, d1=False):
    D, a, r0 = MORSE['D'], MORSE['a'], MORSE['r0']
    x = np.exp(-a * (r - r0))
    return 2 * D * a * (x - x * x) if d1 else D * (x * x - 2 * x)


class Morse:
    def __init__(self, cell, frac, rc):
        self.cell, self.x0 = np.asarray(cell, float), np.asarray(frac, float) @ np.asarray(cell, float)
        n = len(frac)
        c, s, vec = [], [], []
        rng3 = range(-3, 4)
        for i in range(n):
            for j in range(n):
                for a in rng3:
                    for b in rng3:
                        for k in rng3:
                            w = self.x0[j] + np.array([a, b, k]) @ self.cell - self.x0[i]
                            if 1e-9 < np.linalg.norm(w) < rc:
                                c.append(i), s.append(j), vec.append(w)
        self.c, self.s, self.vec0 = np.array(c), np.array(s), np.array(vec)
        self.n = n

    def vec(self, eps=None, u=None):
        v = self.vec0 if eps is None else self.vec0 @ (np.eye(3) + eps).T
        return v if u is None else v + u[self.s] - u[self.c]

    def forces_virial(self, vec):
        r = np.linalg.norm(vec, axis=1)
        f = 0.5 * _phi(r, True)[:, None] * vec / r[:, None]
        F = np.zeros((self.n, 3))
        np.add.at(F, self.c, f)
        np.add.at(F, self.s, -f)
        W = -np.array([(vec[:, 0] * f[:, 0]).sum(), (vec[:, 1] * f[:, 1]).sum(), (vec[:, 2] * f[:, 2]).sum(),
                       (vec[:, 0] * f[:, 1]).sum(), (vec[:, 1] * f[:, 2]).sum(), (vec[:, 2] * f[:, 0]).sum()])
        return F, W

    def relax(self, eps=None, u0=None):
        """positions of atoms 1.. with atom 0 fixed, at zero force, for the fixed edge list strained by eps"""
        def res(x):
            u = np.concatenate([np.zeros((1, 3)), x.reshape(-1, 3)])
            return self.forces_virial(self.vec(eps, u))[0][1:].ravel()
        x0 = np.zeros(3 * (self.n - 1)) if u0 is None else u0[1:].ravel()
        sol = scipy.optimize.root(res, x0, method='hybr', tol=1e-15)
        u = np.concatenate([np.zeros((1, 3)), sol.x.reshape(-1, 3)])
        assert np.abs(self.forces_virial(self.vec(eps, u))[0]).max() < 1e-11
        return u


def _richardson(g, h):
    d = lambda s: (g(s) - g(-s)) / (2 * s)
    return (4 * d(h) - d(2 * h)) / 3


def test_elastic_assembly_against_brute_force():
    """Relaxed-ion tensor of a triclinic Morse crystal with a two-atom basis: elastic.py assembles it from raw
    products of the kind the engine gives (out = H v + Lambda eps = -dF/ds and dW/ds along vec + s (eps . vec +
    v[s] - v[c]), here fp64 differences), and must match -d(W/V0)/de of the structure relaxed at every strain
    (scipy), differenced at +-d and +-2d, to 1e-6 relative.  This pins the Voigt factors, the sign of W and the
    translation projection."""
    cell = np.array([[3.1, 0.15, 0.2], [0.3, 3.3, 0.1], [0.25, 0.4, 3.5]])
    m = Morse(cell, [[0.0, 0.0, 0.0], [0.3, 0.35, 0.4]], rc=3.5)
    u_ref = m.relax()                                   # force-free reference: the formula assumes it
    m.vec0 = m.vec(None, u_ref)
    V0 = abs(np.linalg.det(cell))
    n = m.n

    def product(eps, v):
        def fw(s):
            F, W = m.forces_virial(m.vec(None if eps is None else s * eps, None if v is None else s * v))
            return np.concatenate([-F.ravel(), W])
        d = _richardson(fw, 1e-4)
        return d[:3 * n].reshape(n, 3), d[3 * n:]

    strains = elastic.voigt_strains()
    prods = [product(e, None) for e in strains]
    outs, dvir = np.stack([p[0] for p in prods]), np.stack([p[1] for p in prods])
    H = np.stack([product(None, np.eye(3 * n)[k].reshape(n, 3))[0].ravel() for k in range(3 * n)])
    lam = elastic.internal_strain(outs)
    assert np.abs(lam.reshape(n, 3, 6).sum(axis=0)).max() < 1e-8 * np.abs(lam).max()   # sum_i Lambda_i = 0
    assert np.abs(lam).max() > 1e-2                                                       # the basis does relax
    C0 = elastic.clamped_ion(dvir, V0)
    C = elastic.elastic_tensor(dvir, outs, V0, H)

    # brute force: relax at each strain, difference -W / V0 in Voigt order
    ref = np.zeros((6, 6))
    ref0 = np.zeros((6, 6))
    for k, e in enumerate(strains):
        sig = lambda d, relax=True: -elastic.virial_to_voigt(
            m.forces_virial(m.vec(d * e, m.relax(d * e) if relax else None))[1]) / V0
        ref[:, k] = _richardson(sig, 1e-3)
        ref0[:, k] = _richardson(lambda d: sig(d, False), 1e-3)
    err0 = np.abs(C0 - ref0).max() / np.abs(ref0).max()
    err = np.abs(C - ref).max() / np.abs(ref).max()
    print(f'Morse: max|C0| = {np.abs(ref0).max():.4e}, max|C| = {np.abs(ref).max():.4e} eV/A^3, '
          f'max|C0 - C0_ref| / max = {err0:.2e}, max|C - C_ref| / max = {err:.2e} (bound 1e-6), '
          f'max|C0 - C| / max = {np.abs(ref0 - ref).max() / np.abs(ref).max():.2e}')
    assert err0 < 1e-6 and err < 1e-6
    assert np.abs(ref0 - ref).max() > 0.1 * np.abs(ref).max()        # relaxation matters in this crystal


def test_relaxed_equals_clamped_without_internal_strain():
    """Lambda = 0 leaves C0; the translations of H are projected out (a singular H is fine)"""
    rng = np.random.RandomState(0)
    n = 3
    a = rng.normal(size=(3 * n, 3 * n))
    q = elastic.translation_complement(n)
    H = q @ (a @ a.T)[:3 * n - 3, :3 * n - 3] @ q.T
    assert np.abs(H.reshape(n, 3, 3 * n).sum(axis=0)).max() < 1e-10
    dvir = rng.normal(size=(6, 6))
    C0 = elastic.clamped_ion(dvir, 7.0)
    assert np.array_equal(elastic.elastic_tensor(dvir, np.zeros((6, n, 3)), 7.0, H), C0)
    assert np.allclose(elastic.pinv_hessian(H) @ H @ q, q, atol=1e-8)


def test_hvp_strain_ctypes_signature():
    """The ctypes argtypes of s7b_engine_hvp_strain (sevenn_b200/engine.py) follow include/sevenn_b200.h"""
    lib_path = os.path.join(ROOT, 'sevenn_b200', 'lib', 'libsevenn_b200.so')
    if not os.path.exists(lib_path):
        import __graft_entry__
        __graft_entry__.build()
    header = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API\s+int\s+s7b_engine_hvp_strain\s*\(([^)]*)\)', header)
    assert m is not None
    params = [p.strip() for p in m.group(1).split(',')]
    assert [re.findall(r'\w+', p)[-1] for p in params] == ['eng', 'd_v', 'd_strain', 'd_out', 'd_dvirial', 'stream']
    assert all('*' in p for p in params)
    assert 'double' in params[2] and 'double' in params[4] and 'float' in params[1] and 'float' in params[3]
    from sevenn_b200.engine import EXPORTS, load_library
    assert 's7b_engine_hvp_strain' in EXPORTS
    assert load_library().s7b_engine_hvp_strain.argtypes == [ctypes.c_void_p] * 6
