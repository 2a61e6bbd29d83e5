"""Second derivatives in strain (s7b_engine_hvp_strain, B200Engine.hvp_strain) and the elastic tensors built from them
(SevenNetCalculator.get_elastic_tensor, DeviceBatch.elastic_tensors) on the GPU.

Reference for the raw products: along edge_vec + s (eps . edge_vec + v[neighbour] - v[centre]) with the edge list held
fixed, out = -dF/ds and dvirial = dW/ds of the fp64 oracle's forces F and virial W, by central differences at h and
2h combined by Richardson extrapolation, with h kept below a fifth of every edge's distance from r_on and the cutoff
(as test_hvp_gpu.fd_hvp).  Bounds as test_hvp_gpu: 2e-4 (mlp radial mode) and 5e-4 (table mode) of the largest
reference element, for both outputs.  The observed errors are printed next to their bounds."""
import numpy as np
import pytest

from helpers import model_weights
from test_hvp_gpu import BOUND, CASES, _Atoms, _si, _species, _weights

pytestmark = pytest.mark.gpu

VIRIAL_PAIRS = ((0, 0), (1, 1), (2, 2), (0, 1), (1, 2), (2, 0))   # the virial's order xx,yy,zz,xy,yz,zx


def _full(w6):
    """symmetric 3x3 of a virial 6-vector"""
    w = np.zeros((3, 3))
    for k, (a, b) in enumerate(VIRIAL_PAIRS):
        w[a, b] = w[b, a] = w6[k]
    return w


def _six(m):
    return np.array([m[a, b] for a, b in VIRIAL_PAIRS])


def _oracle(meta, arrays):
    import torch
    from oracle.oracle import Oracle
    from nequip_oracle import nequip_oracle
    from sevenn_b200.spec import build_spec
    make = nequip_oracle if build_spec(meta).self_connection == 'nequip' else Oracle
    return make(meta, arrays, dtype=torch.float64, device='cuda' if torch.cuda.is_available() else 'cpu')


def _margin(meta, ev):
    """distance of the nearest edge from a kink of the radial weights' derivatives (the cutoff; r_on for XPLOR)"""
    from sevenn_b200.spec import build_spec
    spec = build_spec(meta)
    r = np.linalg.norm(np.asarray(ev, np.float64), axis=1)
    kinks = [spec.cutoff] + ([spec.cutoff_on] if spec.cutoff_fn == 'XPLOR' else [])
    return min(np.abs(r - k).min() for k in kinks)


def fd_strain(meta, arrays, species, ei, ev, v, eps):
    """(-dF/ds [n, 3], dW/ds [6]) of the fp64 oracle along edge_vec + s (eps . edge_vec + v[nb] - v[centre])"""
    o = _oracle(meta, arrays)
    ev = np.asarray(ev, np.float64)
    dvec = np.zeros_like(ev)
    if v is not None:
        dvec += v[ei[1]] - v[ei[0]]
    if eps is not None:
        dvec += ev @ np.asarray(eps, np.float64).T
    h = min(1e-3, _margin(meta, ev) / (5 * 2 * np.linalg.norm(dvec, axis=1).max()))

    def fw(s):
        out = o.forward(species, ei, ev + s * dvec)
        return np.concatenate([-out['forces'].cpu().numpy().ravel(), out['virial'].detach().cpu().numpy()])

    d = lambda s: (fw(s) - fw(-s)) / (2 * s)
    r = (4 * d(h) - d(2 * h)) / 3
    return r[:-6].reshape(-1, 3), r[-6:]


def _triclinic(meta, seed=11):
    """rattled two-species (Si, Ge) diamond cell under a triclinic shear: non-zero forces and stress"""
    from sevenn_b200.neighbors import build_graph, diamond_si
    from sevenn_b200.spec import build_spec
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.0)
    shear = np.array([[1.0, 0.06, -0.04], [0.03, 0.98, 0.05], [-0.05, 0.02, 1.03]])
    pos, cell = pos @ shear, cell @ shear
    pos = pos + np.random.RandomState(seed).normal(scale=0.08, size=pos.shape)
    z = z.copy()
    z[::2] = 32
    ei, ev = build_graph(pos, cell, True, build_spec(meta).cutoff)
    return pos, cell, z, ei, ev


def _strain(rng, scale=0.3):
    return rng.normal(size=(3, 3)) * scale


STRAIN_CASES = CASES + [('sevennet_0', 'table', 'triclinic'), ('sevennet_0', 'mlp', 'triclinic')]


@pytest.mark.parametrize('case,radial,system', STRAIN_CASES)
def test_hvp_strain_against_fp64_differences(case, radial, system, tmp_path):
    """out and dvirial of hvp_strain for a strain alone, a position tangent alone and both together"""
    from sevenn_b200.engine import B200Engine
    import torch
    meta, arrays = _weights(case, str(tmp_path))
    if system == 'si64':
        species, ei, ev = _si(meta)
    elif system == 'cluster':
        species, ei, ev = _si(meta, n=1, periodic=False)
    else:
        _, _, z, ei, ev = _triclinic(meta)
        species = _species(meta, z)
    rng = np.random.RandomState(sum(map(ord, case + radial + system)) + 1)
    n = len(species)
    v, eps = rng.normal(size=(n, 3)), _strain(rng)
    e = B200Engine(meta, arrays, radial=radial)
    e.set_graph(species, ei, ev)
    e.compute()
    for tag, vv, ee in (('strain', None, eps), ('positions', v, None), ('both', v, eps)):
        out, dw = e.hvp_strain(vv, None if ee is None else ee[None])
        torch.cuda.synchronize()
        out, dw = out.double().cpu().numpy(), dw.cpu().numpy()[0]
        ref_out, ref_dw = fd_strain(meta, arrays, species, ei, ev, vv, ee)
        err_o = np.abs(out - ref_out).max() / np.abs(ref_out).max()
        err_w = np.abs(dw - ref_dw).max() / np.abs(ref_dw).max()
        print(f'hvp_strain {case} {radial} {system} [{tag}]: max|out| = {np.abs(ref_out).max():.3e}, err {err_o:.2e}; '
              f'max|dW| = {np.abs(ref_dw).max():.3e}, err {err_w:.2e} (bound {BOUND[radial]:.0e})')
        assert err_o < BOUND[radial] and err_w < BOUND[radial], tag


@pytest.fixture(scope='module')
def tri():
    """SevenNet-0 table-mode engine after a compute on the rattled triclinic cell"""
    from sevenn_b200.engine import B200Engine
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z, ei, ev = _triclinic(meta)
    e = B200Engine(meta, arrays)
    e.set_graph(_species(meta, z), ei, ev)
    e.compute()
    return e


def test_mixed_symmetry(tri):
    """v . (out along Voigt strain j) = -(dvirial along v)_j + sum_i F_i . (e_j v_i): the virial tangent against the
    force path.  out differentiates along (I + s e_j) r + t v, -W_j = dE/de_j along (I + s e_j)(r + t v); the two
    mixed derivatives differ by sum_e f_e . (e_j dvec_e) = -sum_i F_i . (e_j v_i), which vanishes at a force-free
    structure (this cell is rattled)."""
    from sevenn_b200 import elastic
    rng = np.random.RandomState(3)
    v = rng.normal(size=(tri.n_nodes, 3))
    F = tri.results()['forces'].double().cpu().numpy()
    _, dwv = tri.hvp_strain(v, None)
    dwv = elastic.virial_to_voigt(dwv.cpu().numpy()[0])
    for j, eps in enumerate(elastic.voigt_strains()):
        out = tri.hvp_strain(None, eps[None])[0].double().cpu().numpy()
        a, b = float((v * out).sum()), -float(dwv[j]) + float((F * (v @ eps.T)).sum())
        scale = np.abs(v).sum() * np.abs(out).max()
        print(f'mixed symmetry, Voigt {j}: v.(Lambda e_j) = {a:.6e}, -dW(v)_j + F.(e_j v) = {b:.6e}, |diff| / scale = '
              f'{abs(a - b) / scale:.2e} (bound 1e-5)')
        assert abs(a - b) < 1e-5 * scale


def test_rotation(tri):
    """an antisymmetric strain is a rotation: out = -omega F, dW = omega W - W omega"""
    r = tri.results()
    F, W = r['forces'].double().cpu().numpy(), _full(r['virial'].cpu().numpy())
    assert np.abs(F).max() > 0.1
    om = np.array([[0.0, 0.3, -0.2], [-0.3, 0.0, 0.5], [0.2, -0.5, 0.0]])
    out, dw = tri.hvp_strain(None, om[None])
    out, dw = out.double().cpu().numpy(), dw.cpu().numpy()[0]
    ref_o, ref_w = -F @ om.T, _six(om @ W - W @ om)
    err_o = np.abs(out - ref_o).max() / np.abs(ref_o).max()
    err_w = np.abs(dw - ref_w).max() / np.abs(ref_w).max()
    print(f'rotation: max|omega F| = {np.abs(ref_o).max():.3e}, err {err_o:.2e}; max|omega W - W omega| = '
          f'{np.abs(ref_w).max():.3e}, err {err_w:.2e} (bound 1e-5)')
    assert err_o < 1e-5 and err_w < 1e-5


# ---- physics on diamond Si ------------------------------------------------------------------------------------------
def _diamond(a, primitive=False):
    if primitive:
        cell = 0.5 * a * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]])
        return np.array([[0.0, 0.0, 0.0], [0.25 * a] * 3]), cell, np.array([14, 14])
    from sevenn_b200.neighbors import diamond_si
    return diamond_si(1, 1, 1, a=a, sigma=0.0)


@pytest.fixture(scope='module')
def si_relaxed():
    """(calculator, a0) with a0 the zero-pressure lattice constant of diamond Si for SevenNet-0 (secant search on the
    pressure of the 8-atom cubic cell)"""
    from sevenn_b200.calculator import SevenNetCalculator
    calc = SevenNetCalculator('7net-0')

    def pressure(a):
        calc.calculate(_Atoms(*_diamond(a)))
        return -float(np.mean(calc.results['stress'][:3]))

    a = [5.40, 5.46]
    p = [pressure(x) for x in a]
    for _ in range(20):
        a.append(a[-1] - p[-1] * (a[-1] - a[-2]) / (p[-1] - p[-2]))
        p.append(pressure(a[-1]))
        if abs(p[-1]) < 1e-6 or abs(a[-1] - a[-2]) < 1e-9:
            break
    print(f'SevenNet-0 Si: a0 = {a[-1]:.6f} A, pressure {p[-1]:.2e} eV/A^3')
    assert abs(p[-1]) < 1e-5
    return calc, a[-1]


def test_si_cubic_elastic_constants(si_relaxed):
    from sevenn_b200.spec import build_spec
    from sevenn_b200.neighbors import build_graph
    calc, a0 = si_relaxed
    atoms = _Atoms(*_diamond(a0))
    calc.calculate(atoms)
    before = {k: np.copy(v) for k, v in calc.results.items()}
    C0 = calc.get_elastic_tensor(atoms, relaxed=False)
    C = calc.get_elastic_tensor(atoms)
    assert all(np.array_equal(before[k], calc.results[k]) for k in before)
    assert C.shape == (6, 6) and C.dtype == np.float64
    m = np.abs(C0).max()
    sym = np.abs(C0 - C0.T).max() / m
    print(f'Si a0 = {a0:.5f}: C0 [GPa] =\n{np.round(C0 / 0.006241509, 2)}\nC [GPa] =\n{np.round(C / 0.006241509, 2)}\n'
          f'max|C0 - C0^T| / max|C0| = {sym:.2e} (bound 1e-4)')
    assert sym < 1e-4
    for T, tag in ((C0, 'C0'), (C, 'C')):
        d, od = np.diag(T), T[:3, :3][~np.eye(3, dtype=bool)]
        cub = [np.ptp(d[:3]), np.ptp(od), np.ptp(d[3:]), np.abs(T[:3, 3:]).max(), np.abs(T[3:, :3]).max(),
               np.abs(T[3:, 3:] - np.diag(d[3:])).max()]
        print(f'{tag} cubic relations: {np.round(np.array(cub) / m, 7)} of max (bound 1e-3)')
        assert max(cub) < 1e-3 * m, tag
    print(f'relaxation: dC11 = {(C[0, 0] - C0[0, 0]) / m:.2e}, dC12 = {(C[0, 1] - C0[0, 1]) / m:.2e} of max (bound '
          f'1e-3), C44 {C0[3, 3]:.4f} -> {C[3, 3]:.4f} eV/A^3')
    assert abs(C[0, 0] - C0[0, 0]) < 1e-3 * m and abs(C[0, 1] - C0[0, 1]) < 1e-3 * m
    assert C[3, 3] < C0[3, 3] - 1e-2 * m
    # bulk modulus: V d2E/dV2 of the fp64 oracle's energies under a uniform scaling of the edge vectors
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = _diamond(a0)
    ei, ev = build_graph(pos, cell, True, build_spec(meta).cutoff)
    ev = ev.astype(np.float64)
    o = _oracle(meta, arrays)
    E = lambda s: float(o.forward(_species(meta, z), ei, ev * (1 + s))['energy'])
    h = min(1e-3, _margin(meta, ev) / (10 * np.linalg.norm(ev, axis=1).max()))
    d1 = lambda s: (E(s) - E(-s)) / (2 * s)
    d2 = lambda s: (E(s) - 2 * E(0.0) + E(-s)) / (s * s)
    e1, e2 = (4 * d1(h) - d1(2 * h)) / 3, (4 * d2(h) - d2(2 * h)) / 3
    V0 = abs(np.linalg.det(cell))
    bulk = (e2 - 2 * e1) / (9 * V0)          # V = V0 (1 + s)^3: V d2E/dV2 = (E'' - 2 E') / (9 V0)
    kc = (C[0, 0] + 2 * C[0, 1]) / 3
    print(f'bulk modulus: (C11 + 2 C12) / 3 = {kc:.6f}, V d2E/dV2 = {bulk:.6f} eV/A^3, rel diff '
          f'{abs(kc - bulk) / bulk:.2e} (bound 1e-3; step {h:.1e})')
    assert abs(kc - bulk) < 1e-3 * bulk


def test_relaxed_ion_brute_force():
    """get_elastic_tensor(relaxed=True) of the 2-atom primitive diamond cell (self-image edges, moved by strain only)
    against -d(W/V0)/de of the fp64 oracle with the second atom relaxed (scipy) at each strain +-d, +-2d, edge list
    fixed, Richardson-extrapolated; bound 1e-3 of max|C|.  a = 5.40 A keeps every edge well away from r_on."""
    import scipy.optimize
    from sevenn_b200 import elastic
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import build_graph
    from sevenn_b200.spec import build_spec
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = _diamond(5.40, primitive=True)
    ei, ev = build_graph(pos, cell, True, build_spec(meta).cutoff)
    ev = ev.astype(np.float64)
    assert (ei[0] == ei[1]).any()
    species = _species(meta, z)
    V0 = abs(np.linalg.det(cell))
    o = _oracle(meta, arrays)

    def run(eps, u1):
        u = np.stack([np.zeros(3), u1])
        return o.forward(species, ei, ev @ (np.eye(3) + eps).T + u[ei[1]] - u[ei[0]])

    def sigma(eps):
        sol = scipy.optimize.root(lambda x: run(eps, x)['forces'].cpu().numpy()[1], np.zeros(3), method='hybr',
                                  tol=1e-14)
        out = run(eps, sol.x)
        assert np.abs(out['forces'].cpu().numpy()).max() < 1e-9
        return -elastic.virial_to_voigt(out['virial'].detach().cpu().numpy()) / V0

    d = min(1e-3, _margin(meta, ev) / (10 * np.linalg.norm(ev, axis=1).max()))
    ref = np.zeros((6, 6))
    for k, e in enumerate(elastic.voigt_strains()):
        g = lambda s: (sigma(s * e) - sigma(-s * e)) / (2 * s)
        ref[:, k] = (4 * g(d) - g(2 * d)) / 3
    C = SevenNetCalculator('7net-0').get_elastic_tensor(_Atoms(pos, cell, z))
    err = np.abs(C - ref).max() / np.abs(ref).max()
    print(f'relaxed-ion brute force (step {d:.1e}): max|C| = {np.abs(ref).max():.4f} eV/A^3, '
          f'max|C - C_ref| / max = {err:.2e} (bound 1e-3)')
    assert err < 1e-3


# ---- batches --------------------------------------------------------------------------------------------------------
def _batch_structs():
    p2, c2, z2 = _diamond(5.40, primitive=True)
    p8, c8, z8 = _diamond(5.45)
    shear = np.array([[1.0, 0.04, 0.0], [0.0, 1.0, 0.03], [0.02, 0.0, 1.0]])
    p3, c3, z3 = _diamond(5.43)
    return [(p2, c2, z2), (p8, c8, z8), (p3 @ shear, c3 @ shear, z3)]


def test_batch_elastic_tensors():
    """DeviceBatch.elastic_tensors of three different cells equals get_elastic_tensor per structure"""
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.calculator import SevenNetCalculator
    structs = _batch_structs()
    calc = SevenNetCalculator('7net-0')
    ref = np.stack([calc.get_elastic_tensor(_Atoms(*s)) for s in structs])
    ref0 = np.stack([calc.get_elastic_tensor(_Atoms(*s), relaxed=False) for s in structs])
    args = (np.concatenate([z for _, _, z in structs]), np.concatenate([p for p, _, _ in structs]),
            np.stack([c for _, c, _ in structs]), True,
            np.concatenate([np.full(len(z), b) for b, (_, _, z) in enumerate(structs)]))
    db = DeviceBatch(calc.engine)
    for relaxed, want in ((True, ref), (False, ref0)):
        got = db.elastic_tensors(*args, relaxed=relaxed)
        assert got.shape == (3, 6, 6)
        err = np.abs(got - want).max() / np.abs(want).max()
        print(f'batch elastic tensors (relaxed={relaxed}): max|batch - single| / max = {err:.2e} (bound 1e-5)')
        assert err < 1e-5


def test_batch_strain_products():
    """a union-graph hvp_strain with a different strain and tangent per structure equals the single-structure products"""
    import torch
    from sevenn_b200.engine import B200Engine
    meta, arrays = model_weights('sevennet_0')
    structs = [(p + np.random.RandomState(b).normal(scale=0.05, size=p.shape), c, z)
               for b, (p, c, z) in enumerate(_batch_structs())]
    rng = np.random.RandomState(9)
    vs = [rng.normal(size=(len(p), 3)) for p, _, _ in structs]
    eps = rng.normal(size=(3, 3, 3)) * 0.3
    e = B200Engine(meta, arrays)
    singles, dws = [], []
    for (p, c, z), v, ep in zip(structs, vs, eps):
        e.set_positions(_species(meta, z), p, c, True)
        e.compute()
        o, d = e.hvp_strain(v, ep[None])
        singles.append(o.double().cpu().numpy())
        dws.append(d.cpu().numpy()[0])
    ap = np.cumsum([0] + [len(p) for p, _, _ in structs])
    e.set_positions_batch(np.concatenate([_species(meta, z) for _, _, z in structs]),
                          np.concatenate([p for p, _, _ in structs]), ap, np.stack([c for _, c, _ in structs]), True)
    e.compute()
    ob, db = e.hvp_strain(np.concatenate(vs), eps)
    torch.cuda.synchronize()
    ref_o, ref_w = np.concatenate(singles), np.stack(dws)
    err_o = np.abs(ob.double().cpu().numpy() - ref_o).max() / np.abs(ref_o).max()
    err_w = np.abs(db.cpu().numpy() - ref_w).max() / np.abs(ref_w).max()
    print(f'batch hvp_strain: out err {err_o:.2e}, dvirial err {err_w:.2e} of max (bound 1e-5)')
    assert db.shape == (3, 6) and err_o < 1e-5 and err_w < 1e-5


# ---- refusals and side effects --------------------------------------------------------------------------------------
def test_refusals():
    import torch
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.engine import B200Engine, check
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z, ei, ev = _triclinic(meta)
    species = _species(meta, z)
    n = len(species)
    e = B200Engine(meta, arrays)
    e.set_graph(species, ei, ev)
    with pytest.raises(RuntimeError, match='s7b_engine_hvp_strain needs an s7b_engine_compute'):
        e.hvp_strain(None, np.eye(3)[None])
    e.compute()
    with pytest.raises(ValueError, match='v has'):
        e.hvp_strain(np.ones((n + 1, 3)))
    with pytest.raises(ValueError, match='strain has'):
        e.hvp_strain(None, np.eye(3)[None].repeat(2, 0))
    keep = ei[0] < n - 2
    e.set_graph(species, ei[:, keep], ev[keep], n_local=n - 2)
    e.compute()
    with pytest.raises(RuntimeError, match='ghost'):
        e.hvp_strain(None, np.eye(3)[None])
    t = B200Engine(meta, arrays)          # table mode, radial MLP never uploaded: the C ABI refuses
    t.set_graph(species, ei, ev)
    t.compute()
    out = torch.empty(n, 3, device=t.device)
    eps = torch.eye(3, dtype=torch.float64, device=t.device)
    with pytest.raises(RuntimeError, match='mlp0 of layer 0 is missing'):
        check(t.lib.s7b_engine_hvp_strain(t._h, None, eps.data_ptr(), out.data_ptr(), None, t._stream()))
    calc = SevenNetCalculator('7net-0')

    class Slab(_Atoms):
        def get_pbc(self):
            return np.array([True, True, False])

    with pytest.raises(ValueError, match='periodic'):
        calc.get_elastic_tensor(Slab(pos, cell, z))
    with pytest.raises(ValueError, match='periodic'):
        calc.get_elastic_tensor(_Atoms(pos, np.zeros((3, 3)), z))
    with pytest.raises(ValueError, match='periodic'):
        DeviceBatch(calc.engine).elastic_tensors(z, pos, cell[None], [True, False, True], np.zeros(n, np.int64))
    # no edges: zero-filled outputs
    e.set_graph(species[:3], np.zeros((2, 0), np.int64), np.zeros((0, 3), np.float32))
    e.compute()
    o, d = e.hvp_strain(np.ones((3, 3)), np.eye(3)[None])
    assert bool((o == 0).all()) and bool((d == 0).all())


def test_no_strain_matches_hvp(tri):
    """hvp_strain(v, None) is hvp(v) to the force scatter's atomic rounding; hvp_strain(None, None) is zero"""
    rng = np.random.RandomState(2)
    v = rng.normal(size=(tri.n_nodes, 3))
    a = tri.hvp(v).double().cpu().numpy()
    b = tri.hvp_strain(v, None)[0].double().cpu().numpy()
    print(f'hvp_strain(v, None) vs hvp(v): max|diff| / max = {np.abs(a - b).max() / np.abs(a).max():.2e}')
    assert np.allclose(b, a, rtol=1e-6, atol=1e-6 * np.abs(a).max())
    o, d = tri.hvp_strain()
    assert bool((o == 0).all()) and bool((d == 0).all())


def test_compute_unchanged_by_hvp_strain():
    import torch
    from sevenn_b200.engine import B200Engine
    meta, arrays = model_weights('sevennet_0')
    _, _, z, ei, ev = _triclinic(meta)
    e = B200Engine(meta, arrays)
    e.set_graph(_species(meta, z), ei, ev)

    def step():
        e.compute()
        torch.cuda.synchronize()
        r = e.results()
        return {k: r[k].cpu().numpy() for k in ('energy', 'forces', 'virial')}

    r1 = step()
    e.hvp_strain(np.ones((len(z), 3)), np.eye(3)[None])
    r2 = step()
    for k in r1:
        print(f'{k}: max|after hvp_strain - before| = {np.abs(r2[k] - r1[k]).max():.2e}')
        assert np.allclose(r2[k], r1[k], rtol=1e-6, atol=1e-6 * np.abs(r1[k]).max()), k
