"""CPU checks of the D3 Hessian-vector product's arithmetic (sevenn_b200/csrc/d3_hvp_math.cuh, compiled with g++
through tests/cpu_harness/d3_hvp_harness.cpp): the damping, counting-function and reference-weight jets against fp64
numpy, the pair and strain tangent, the ctypes signature of s7b_d3_hvp_strain, and the bookkeeping of the summed
elastic assembly (network + D3) on a toy pair potential."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from oracle.d3_oracle import AU_TO_ANG, K1, K3, d3_params
from sevenn_b200 import elastic
from d3_cells import MIN_DIST

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F32P = ctypes.POINTER(ctypes.c_float)
F64P = ctypes.POINTER(ctypes.c_double)
RMIN, RMAX = MIN_DIST / AU_TO_ANG, np.sqrt(9000.0)        # bohr: the shortest fixture pair to the default vdW cutoff


def fp(a):
    return np.ascontiguousarray(a, dtype=np.float32).ctypes.data_as(F32P)


@pytest.fixture(scope='module')
def lib(tmp_path_factory):
    src = os.path.join(ROOT, 'tests', 'cpu_harness', 'd3_hvp_harness.cpp')
    so = str(tmp_path_factory.mktemp('harness') / 'libd3_hvp_harness.so')
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-shared', '-fPIC', src, '-o', so])
    lib = ctypes.CDLL(so)
    f, i, d = ctypes.c_float, ctypes.c_int, ctypes.c_double
    lib.d3h_damp_jet.argtypes = [i, F32P, i, f, f, f, f, f, f, f, f, F32P]
    lib.d3h_count_jet.argtypes = [F32P, i, f, f, F32P]
    lib.d3h_weight_jet.argtypes = [F32P, i, F32P, i, d, F64P]
    lib.d3h_pair_tangent.argtypes = [F64P, F64P, F64P, F32P, F32P]
    return lib


def _richardson(f, x, h):
    """d f / dx at x by Richardson-extrapolated central differences (f vectorised over x)"""
    d1 = (f(x + h) - f(x - h)) / (2 * h)
    d2 = (f(x + h / 2) - f(x - h / 2)) / h
    return (4 * d2 - d1) / 3


def _damp_fp64(damping, p, r0, par):
    """(g, g') of the oracle's damping functions in fp64 (oracle/d3_oracle.py), as functions of r (bohr)"""
    if damping == 1:
        R0 = par['a1'] * np.sqrt(p) + par['a2']
        g = lambda r: par['s6'] / (r ** 6 + R0 ** 6) + par['s8'] * p / (r ** 8 + R0 ** 8)
        g1 = lambda r: -(6 * par['s6'] * r ** 5 / (r ** 6 + R0 ** 6) ** 2 + 8 * par['s8'] * p * r ** 7 / (r ** 8 + R0 ** 8) ** 2)
    else:
        def parts(r):
            t6, t8 = (par['a1'] * r0 / r) ** par['alp6'], (par['a2'] * r0 / r) ** par['alp8']
            return t6, t8, 1 / (1 + 6 * t6), 1 / (1 + 6 * t8)

        def g(r):
            t6, t8, d6, d8 = parts(r)
            return par['s6'] * d6 / r ** 6 + 3 * par['s8'] * p * d8 / r ** 8

        def g1(r):
            t6, t8, d6, d8 = parts(r)
            return (par['s6'] * (-6 * d6 / r ** 7 + 6 * par['alp6'] * t6 * d6 ** 2 / r ** 7)
                    + 3 * par['s8'] * p * (-8 * d8 / r ** 9 + 6 * par['alp8'] * t8 * d8 ** 2 / r ** 9))
    return g, g1


def _functionals(damping):
    """every functional's parameters of one damping, as the engine sets them (d3.D3Engine)"""
    out = []
    for name, q in d3_params()['functionals'][damping].items():
        out.append((name, dict(s6=q['s6'], s8=q['s18'], a1=q['rs6'], a2=q['rs18'], alp6=q['alp'], alp8=q['alp'] + 2.0)))
    return out


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
def test_damping_jet(lib, damping):
    """(g, g', g'') of every functional, for the element pairs with the smallest and largest r2r4 products (and r0),
    from the shortest fixture pair to the vdW cutoff, against fp64: g and g' in closed form, g'' by Richardson
    differences of g'.  Bound per point: 2e-5 of the scale of the terms each derivative sums (the jet with |s6|, |s8|:
    |g|, |g'| + |g| / r, |g''| + |g'| / r + |g| / r^2)."""
    P = d3_params()
    z = np.array([1, 6, 9, 36, 55, 83]) - 1
    r = np.geomspace(RMIN, RMAX, 400)
    worst = 0.0
    for name, par in _functionals(damping):
        for zi in z:
            for zj in z:
                r42 = P['r2r4'][zi] * P['r2r4'][zj]
                r0 = P['r0ab'][zi, zj] / AU_TO_ANG
                p = 3 * r42 if damping == 'damp_bj' else r42
                # the kernel sees the float-rounded parameters: the fp64 reference takes them rounded alike
                f32 = lambda v: float(np.float32(v))
                parf = {k: f32(v) for k, v in par.items()}
                g, g1 = _damp_fp64(1 if damping == 'damp_bj' else 0, f32(p), f32(r0), parf)
                out = np.zeros(3 * len(r), np.float32)
                lib.d3h_damp_jet(1 if damping == 'damp_bj' else 0, fp(r), len(r), p, r0, par['s6'], par['s8'], par['a1'],
                                 par['a2'], par['alp6'], par['alp8'], out.ctypes.data_as(F32P))
                out = out.reshape(-1, 3).astype(np.float64)
                rr = r.astype(np.float32).astype(np.float64)
                ref = np.stack([g(rr), g1(rr), _richardson(g1, rr, 1e-4 * rr)], 1)
                # scale: the same jet with |s6|, |s8| (s8 < 0 in some functionals: g then crosses zero)
                ga, g1a = _damp_fp64(1 if damping == 'damp_bj' else 0, f32(p), f32(r0),
                                     dict(parf, s6=abs(parf['s6']), s8=abs(parf['s8'])))
                ab = np.abs(np.stack([ga(rr), g1a(rr), _richardson(g1a, rr, 1e-4 * rr)], 1))
                scale = [ab[:, 0], ab[:, 1] + ab[:, 0] / rr, ab[:, 2] + ab[:, 1] / rr + ab[:, 0] / rr ** 2]
                for k in range(3):
                    e = np.abs(out[:, k] - ref[:, k]) / scale[k]
                    worst = max(worst, float(e.max()))
                    assert e.max() < 2e-5, (name, zi + 1, zj + 1, k, e.max())
    print(f'{damping}: worst relative error over {len(_functionals(damping))} functionals = {worst:.2e}')


def test_count_jet(lib):
    """(f, f', f'') of the counting function for small and large covalent radius sums, from the shortest fixture pair
    to the CN cutoff, against fp64 closed form (f, f') and Richardson differences of f'"""
    P = d3_params()
    r = np.geomspace(RMIN, 40.0, 400)
    worst = 0.0
    for rc in (2 * P['rcov'].min(), P['rcov'].min() + P['rcov'].max(), 2 * P['rcov'].max()):
        rc = float(np.float32(rc))
        f = lambda x: 1.0 / (1.0 + np.exp(-K1 * (rc / x - 1.0)))
        f1 = lambda x: -K1 * rc * np.exp(-K1 * (rc / x - 1.0)) / (x * x * (1.0 + np.exp(-K1 * (rc / x - 1.0))) ** 2)
        rf = r.astype(np.float32).astype(np.float64)
        out = np.zeros(3 * len(r), np.float32)
        lib.d3h_count_jet(fp(rf ** 2), len(r), rc, K1, out.ctypes.data_as(F32P))
        out = out.reshape(-1, 3).astype(np.float64)
        ref = np.stack([f(rf), f1(rf), _richardson(f1, rf, 1e-5 * rf)], 1)
        scale = np.abs(ref[:, 2]) + np.abs(ref[:, 1]) * (K1 * rc / rf ** 2 + 2 / rf)
        for k in range(3):
            e = np.abs(out[:, k] - ref[:, k]) / (scale if k == 2 else np.abs(ref[:, k]).max())
            worst = max(worst, float(e.max()))
            assert e.max() < 1e-5, (rc, k, e.max())
    print(f'counting function: worst relative error = {worst:.2e}')


def _weights_fp64(cn, cnr):
    """W [k, m] of the oracle's Gaussian weights in fp64 (no fallback)"""
    w = np.exp(K3 * (cnr[None, :] - cn[:, None]) ** 2)
    return w / w.sum(1, keepdims=True)


@pytest.mark.parametrize('Z', [1, 6, 14, 29, 55, 83])
def test_weight_jet(lib, Z):
    """W, W', W'' of one atom across and beyond its reference coordination numbers against fp64: W in closed form,
    W' and W'' by Richardson differences; and into the D <= 1e-300 fallback, where W is one-hot and W' = W'' = 0"""
    P = d3_params()
    m = int(P['mxc'][Z - 1])
    cnref = P['cnref'][Z - 1].astype(np.float32)
    cnr = cnref[:m].astype(np.float64)
    cn = np.linspace(0.0, cnr.max() + 3.0, 301).astype(np.float32)
    out = np.zeros(15 * len(cn))
    lib.d3h_weight_jet(fp(cn), len(cn), fp(cnref), m, K3, out.ctypes.data_as(F64P))
    out = out.reshape(-1, 3, 5)
    c = cn.astype(np.float64)
    Wf = lambda x: _weights_fp64(x, cnr)
    ref = [Wf(c), _richardson(Wf, c, 1e-4), _richardson(lambda x: _richardson(Wf, x, 1e-4), c, 1e-3)]
    for k in range(3):
        e = np.abs(out[:, k, :m] - ref[k]).max() / max(np.abs(ref[k]).max(), 1e-12)
        # the squared distances (CN - CN_a)^2 are rounded to float, as in d3_weights_kernel: ~1e-7 relative in W
        assert e < (1e-6 if k < 2 else 1e-4), (Z, k, e)
        assert np.all(out[:, k, m:] == 0.0)
    # the fallback: far from every reference the weight sum underflows
    far = np.array([cnr.max() + 14.0, cnr.max() + 40.0], np.float32)
    out = np.zeros(15 * len(far))
    lib.d3h_weight_jet(fp(far), len(far), fp(cnref), m, K3, out.ctypes.data_as(F64P))
    out = out.reshape(-1, 3, 5)
    near = int(np.argmin(((cnref[:m] - far[0]) ** 2)))
    assert np.array_equal(out[:, 0], np.tile(np.eye(5)[near], (2, 1)))
    assert np.all(out[:, 1:] == 0.0)


@pytest.mark.parametrize('with_v,with_eps', [(True, False), (False, True), (True, True)])
def test_pair_tangent(lib, with_v, with_eps):
    """dvec = v_j - v_i + eps . vec, and (dr, du) against fp64 central differences of |vec| and vec / |vec| along it"""
    rng = np.random.RandomState(3 + 2 * with_v + with_eps)
    for _ in range(20):
        vec = rng.normal(size=3) * rng.uniform(RMIN, 30.0)
        vi, vj = rng.normal(size=3), rng.normal(size=3)
        eps = rng.normal(size=(3, 3))
        vec32 = vec.astype(np.float32).astype(np.float64)
        dvec = ((vj - vi) if with_v else 0.0) + (eps @ vec32 if with_eps else 0.0)
        zero = np.zeros(3)
        out = np.zeros(11, np.float32)
        e64 = np.ascontiguousarray(eps)
        lib.d3h_pair_tangent(np.ascontiguousarray(vi if with_v else zero).ctypes.data_as(F64P),
                             np.ascontiguousarray(vj if with_v else zero).ctypes.data_as(F64P),
                             e64.ctypes.data_as(F64P) if with_eps else None, fp(vec32), out.ctypes.data_as(F32P))
        assert np.abs(out[:3] - dvec).max() < 1e-6 * np.abs(dvec).max()
        h = 1e-6
        rp, rm = np.linalg.norm(vec32 + h * dvec), np.linalg.norm(vec32 - h * dvec)
        up, um = (vec32 + h * dvec) / rp, (vec32 - h * dvec) / rm
        assert abs(out[3] - np.linalg.norm(vec32)) < 1e-6 * np.linalg.norm(vec32)
        assert np.abs(out[4:7] - vec32 / np.linalg.norm(vec32)).max() < 1e-6
        assert abs(out[7] - (rp - rm) / (2 * h)) < 1e-5 * np.linalg.norm(dvec)
        du = (up - um) / (2 * h)
        assert np.abs(out[8:11] - du).max() < 1e-5 * np.linalg.norm(dvec) / np.linalg.norm(vec32)


def test_d3_hvp_strain_ctypes_signature():
    """The ctypes argtypes of s7b_d3_hvp_strain (sevenn_b200/engine.py) follow include/sevenn_b200.h"""
    lib_path = os.path.join(ROOT, 'sevenn_b200', 'lib', 'libsevenn_b200.so')
    if not os.path.exists(lib_path):
        import __graft_entry__
        __graft_entry__.build()
    header = open(os.path.join(ROOT, 'include', 'sevenn_b200.h')).read()
    m = re.search(r'S7B_API\s+int\s+s7b_d3_hvp_strain\s*\(([^)]*)\)', header)
    assert m is not None
    params = [p.strip() for p in m.group(1).split(',')]
    assert [re.findall(r'\w+', p)[-1] for p in params] == ['d3', 'd_v', 'd_strain', 'd_out', 'd_dvirial', 'stream']
    assert all('*' in p for p in params)
    assert all('double' in p for p in params[1:5])
    from sevenn_b200.engine import EXPORTS, load_library
    assert 's7b_d3_hvp_strain' in EXPORTS
    assert load_library().s7b_d3_hvp_strain.argtypes == [ctypes.c_void_p] * 6


# ---- summing two energies' second derivatives before the elastic assembly ------------------------------------------
# Two pair potentials A (Morse) and B (a soft r^-6 attraction) on one two-atom-basis crystal, with the bookkeeping of
# tests/test_elastic_cpu.py: fixed directed edges, E = 1/2 sum_e phi(|vec_e|), W = -sum_e vec_e (x) f_e.
def _toy():
    rng = np.random.RandomState(11)
    cell = np.array([[3.1, 0.2, -0.1], [0.3, 2.9, 0.15], [-0.2, 0.1, 3.3]])
    frac = np.array([[0.0, 0.0, 0.0], [0.47, 0.53, 0.49]]) + rng.normal(scale=0.02, size=(2, 3))
    pos = frac @ cell
    edges = []
    for c in range(2):
        for s in range(2):
            for t in np.array(np.meshgrid(*[np.arange(-2, 3)] * 3, indexing='ij')).reshape(3, -1).T:
                if c == s and not t.any():
                    continue
                if np.linalg.norm(pos[s] + t @ cell - pos[c]) < 5.0:
                    edges.append((c, s, t))
    return cell, pos, edges


PHIS = dict(A=(lambda r: 0.4 * (np.exp(-2.8 * (r - 2.6)) - 2 * np.exp(-1.4 * (r - 2.6)))),
            B=(lambda r: -6.0 / (r ** 6 + 8.0)))


def _energy(which, cell, pos, edges, strain=np.zeros((3, 3))):
    F = np.eye(3) + strain
    e = 0.0
    for c, s, t in edges:
        vec = (pos[s] + t @ cell - pos[c]) @ F.T
        e += 0.5 * sum(PHIS[w](np.linalg.norm(vec)) for w in which)
    return e


def _pieces(which, cell, pos, edges):
    """(dvirial [6, 6], outs [6, N, 3], V, H) of energy ``which`` in the layout ``elastic.elastic_tensor`` takes, from
    fp64 central differences of E(x + dx, e) in the displacements dx and the six Voigt strains e"""
    n, h = len(pos), 1e-4
    eps6 = elastic.voigt_strains()
    m = 3 * n + 6

    def E(z):
        return _energy(which, cell, pos + z[:3 * n].reshape(n, 3), edges, np.tensordot(z[3 * n:], eps6, 1))
    full = np.zeros((m, m))
    for a in range(m):
        for b in range(a, m):
            ea, eb = np.eye(m)[a] * h, np.eye(m)[b] * h
            full[a, b] = full[b, a] = (E(ea + eb) - E(ea - eb) - E(eb - ea) + E(-ea - eb)) / (4 * h * h)
    dvir = np.zeros((6, 6))
    for j in range(6):
        dvir[:, elastic.VIRIAL_TO_VOIGT[j]] = -full[3 * n + j, 3 * n:]        # row k: dW along strain k
    return dvir, full[:3 * n, 3 * n:].T.reshape(6, n, 3), abs(np.linalg.det(cell)), full[:3 * n, :3 * n]


def test_summed_pieces_assemble_the_sum():
    """Sum-then-assemble gives the relaxed-ion tensor of the summed energy; assemble-then-sum does not (the relaxed-
    ion tensor is not linear in (Lambda, H)), while the clamped-ion tensors do add."""
    cell, pos, edges = _toy()
    pa, pb, pab = _pieces('A', cell, pos, edges), _pieces('B', cell, pos, edges), _pieces('AB', cell, pos, edges)
    summed = [pa[0] + pb[0], pa[1] + pb[1], pa[2], pa[3] + pb[3]]
    C_ref = elastic.elastic_tensor(*pab)
    C_sum = elastic.elastic_tensor(*summed)
    C_wrong = elastic.elastic_tensor(*pa) + elastic.elastic_tensor(*pb)
    scale = np.abs(C_ref).max()
    print(f'toy: max|C| = {scale:.3e}, sum-then-assemble {np.abs(C_sum - C_ref).max() / scale:.1e}, '
          f'assemble-then-sum {np.abs(C_wrong - C_ref).max() / scale:.1e}')
    assert np.abs(C_sum - C_ref).max() < 1e-6 * scale
    assert np.abs(C_wrong - C_ref).max() > 1e-3 * scale
    C0 = lambda p: elastic.elastic_tensor(p[0], p[1], p[2])
    assert np.abs(C0(pa) + C0(pb) - C0(pab)).max() < 1e-6 * scale
