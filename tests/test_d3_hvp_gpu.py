"""The D3 Hessian-vector product (s7b_d3_hvp_strain, D3Engine / D3Batch.hvp_strain) and what is built on it
(D3Calculator / SevenNetD3Calculator.get_hessian and get_elastic_tensor, DeviceBatch.elastic_tensors with d3) against
the fp64 D3 oracle (oracle/d3_oracle.py, mimic_fp32=False: the smooth function; the GPU holds CN as a float for the
weights, so differences of its own forces would be a step function)."""
import numpy as np
import pytest

import d3_cells
from test_d3_batch_gpu import _Atoms

pytestmark = pytest.mark.gpu

AU = 0.52917726
KW = dict(vdw_cutoff=2500.0, cn_cutoff=900.0)        # reduced cutoffs (bohr^2): the oracle enumerates all pairs
BOUND = 1e-4


def _nacl():
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.08, seed=12)
    return z, pos, cell, (True, True, True)


def _system(name):
    """(numbers, positions, cell, pbc) as evaluated: a structure without a cell gets D3Calculator's generated cell"""
    if name == 'nacl':
        return _nacl()
    z, pos, cell, pbc = d3_cells.FIXTURES[name]()
    if np.asarray(cell).sum() == 0:
        rc = np.sqrt(max(KW['vdw_cutoff'], KW['cn_cutoff'])) * AU
        cell = np.eye(3) * (pos.max(0) - pos.min(0) + rc + 1.0)
        pbc = (True, True, True)
    return z, pos, cell, pbc


def _margin(pos, cell, pbc, kw=KW):
    """min over all pairs (any image) of | r - rc | for both cutoffs (Angstrom), and the largest pair distance
    inside a cutoff: a step that moves no pair distance by more than the margin crosses no cutoff"""
    from oracle.d3_oracle import _translations
    lat = np.asarray(cell, dtype=np.float64)
    frac = np.asarray(pos, dtype=np.float64) @ np.linalg.inv(lat)
    x = (frac - np.floor(frac)) @ lat                   # wrapped, as the oracle and the kernels do
    out = np.inf
    for c2 in (kw['vdw_cutoff'], kw['cn_cutoff']):
        rc = np.sqrt(c2) * AU
        tau, _ = _translations(lat / AU, np.sqrt(c2) + 2.0, pbc)
        tau = tau * AU
        for i in range(len(x)):
            d = x[None, :, :] - x[i][None, None, :] + tau[:, None, :]
            r = np.linalg.norm(d, axis=-1).ravel()
            out = min(out, float(np.abs(r[r > 0] - rc).min()))
    return out, np.sqrt(max(kw['vdw_cutoff'], kw['cn_cutoff'])) * AU


def _oracle(z, pos, cell, pbc, damping, kw=KW):
    from oracle.d3_oracle import d3_reference
    return d3_reference(z, pos, cell, pbc, damping=damping, functional='pbe', mimic_fp32=False, **kw)


def _six(s):
    return np.array([s[0, 0], s[1, 1], s[2, 2], s[0, 1], s[1, 2], s[2, 0]])


def _fd(z, pos, cell, pbc, damping, v, eps, kw=KW):
    """(-dF/ds, dW/ds) along r -> (I + s eps)(r) + s v of the oracle, Richardson-extrapolated central differences,
    with a step that crosses no cutoff"""
    margin, rc = _margin(pos, cell, pbc, kw)
    reach = 2 * np.abs(v).max() + np.linalg.norm(eps, 2) * rc
    h = min(1e-3, margin / (4 * reach)) if reach > 0 else 1e-3

    def at(s):
        F = np.eye(3) + s * eps
        o = _oracle(z, pos @ F.T + s * v, cell @ F.T, pbc, damping, kw)
        return o['forces'], _six(o['sigma'])

    def d(s):
        (fp, wp), (fm, wm) = at(s), at(-s)
        return -(fp - fm) / (2 * s), (wp - wm) / (2 * s)
    (a1, b1), (a2, b2) = d(h), d(h / 2)
    return (4 * a2 - a1) / 3, (4 * b2 - b1) / 3, h, margin


def _engine(damping, kw=KW):
    from sevenn_b200.d3 import D3Engine
    return D3Engine(damping, 'pbe', **kw)


def _forward(eng, z, pos, cell, pbc):
    eng.set_system(z, pos, cell, pbc)
    for s in (1, 2, 3):
        eng.run_stage(s)


SYSTEMS = ['sheared', 'rotated', 'slab', 'wire', 'compressed_cs', 'species16', 'molecule', 'nacl']


@pytest.mark.parametrize('tangent', ['v', 'eps', 'both'])
@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('system', SYSTEMS)
def test_hvp_strain_against_fp64_differences(system, damping, tangent):
    z, pos, cell, pbc = _system(system)
    rng = np.random.RandomState(SYSTEMS.index(system) * 6 + 3 * (damping == 'damp_zero') + ['v', 'eps', 'both'].index(tangent))
    v = rng.normal(size=pos.shape) if tangent != 'eps' else np.zeros(pos.shape)
    v /= max(np.abs(v).max(), 1e-300) if tangent != 'eps' else 1.0
    eps = rng.normal(size=(3, 3)) * 0.5 if tangent != 'v' else np.zeros((3, 3))
    eng = _engine(damping)
    _forward(eng, z, pos, cell, pbc)
    out, dw = eng.hvp_strain(v if tangent != 'eps' else None, eps[None] if tangent != 'v' else None)
    out, dw = out.cpu().numpy(), dw.cpu().numpy()[0]
    ref_o, ref_w, h, margin = _fd(z, pos, cell, pbc, damping, v, eps)
    eo = np.abs(out - ref_o).max() / np.abs(ref_o).max()
    ew = np.abs(dw - ref_w).max() / np.abs(ref_w).max()
    print(f'{system} {damping} {tangent}: max|out| = {np.abs(ref_o).max():.3e} eV/A, err {eo:.2e}; max|dW| = '
          f'{np.abs(ref_w).max():.3e} eV, err {ew:.2e} (bound {BOUND:.0e}; step {h:.1e}, cutoff margin {margin:.1e} A)')
    assert eo < BOUND and ew < BOUND


def test_mixed_identity():
    """v . (Lambda e_j) = -dW_j(v) + sum_i F_i . (e_j v_i), as for the network (DESIGN §8.1)"""
    from sevenn_b200 import elastic
    z, pos, cell, pbc = _nacl()
    eng = _engine('damp_bj')
    E, F, _ = eng.compute(z, pos, cell, pbc)
    rng = np.random.RandomState(3)
    v = rng.normal(size=pos.shape)
    dwv = elastic.virial_to_voigt(eng.hvp_strain(v, None)[1].cpu().numpy()[0])
    for j, eps in enumerate(elastic.voigt_strains()):
        out = eng.hvp_strain(None, eps[None])[0].cpu().numpy()
        a, b = float((v * out).sum()), -float(dwv[j]) + float((F * (v @ eps.T)).sum())
        scale = np.abs(v).sum() * np.abs(out).max()
        print(f'mixed identity, Voigt {j}: {a:.6e} vs {b:.6e}, |diff| / scale = {abs(a - b) / scale:.2e} (bound 1e-5)')
        assert abs(a - b) < 1e-5 * scale


def test_hessian_symmetric_and_translation_invariant():
    from sevenn_b200.d3 import D3Calculator
    z, pos, cell, pbc = _nacl()
    atoms = _Atoms(z, pos, cell, pbc)
    H = D3Calculator('damp_bj', 'pbe').get_hessian(atoms)
    m = np.abs(H).max()
    sym = np.abs(H - H.T).max() / m
    rows = np.abs(H.reshape(3 * len(z), len(z), 3).sum(1)).max() / m
    print(f'D3 Hessian, 64-atom NaCl, default cutoffs: max|H| = {m:.3e} eV/A^2, asymmetry {sym:.2e}, row sums {rows:.2e}')
    assert H.shape == (3 * len(z), 3 * len(z)) and sym < 1e-5 and rows < 1e-5


def test_molecule_hessian_leaves_atoms():
    """a structure without a cell: the generated cell, and atoms is not modified"""
    from sevenn_b200.d3 import D3Calculator
    z, pos, cell, pbc = d3_cells.molecule()
    atoms = _Atoms(z, pos, cell, pbc)
    H = D3Calculator('damp_zero', 'pbe', **KW).get_hessian(atoms)
    assert np.array_equal(atoms.cell, np.zeros((3, 3))) and not atoms.pbc.any()
    assert np.abs(H - H.T).max() < 1e-5 * np.abs(H).max()


def test_nacl_clamped_ion_cubic_and_scaling():
    """D3-only C0 of perfect rock-salt NaCl is cubic, and V sum_{i,j<=3} C0_ij = f'' + f' for f(s) = E((1 + s) r) of the
    oracle's energies.  This holds exactly at any pre-stress: W(s) is the virial of the scaled cell and
    tr W(s) = -(1 + s) f'(s), so the tangent of tr W along eps = I, -V sum C0_ij, is -f'(0) - f''(0)."""
    from sevenn_b200.d3 import D3Calculator
    from sevenn_b200.neighbors import rocksalt_nacl
    kw = dict(vdw_cutoff=2000.0, cn_cutoff=900.0)
    pos, cell, z = rocksalt_nacl(1, 1, 1, sigma=0.0)
    C0 = D3Calculator('damp_bj', 'pbe', **kw).get_elastic_tensor(_Atoms(z, pos, cell, True), relaxed=False)
    m = np.abs(C0).max()
    d, od = np.diag(C0), C0[:3, :3][~np.eye(3, dtype=bool)]
    cub = [np.ptp(d[:3]), np.ptp(od), np.ptp(d[3:]), np.abs(C0[:3, 3:]).max(), np.abs(C0[3:, :3]).max(),
           np.abs(C0[3:, 3:] - np.diag(d[3:])).max()]
    margin, rc = _margin(pos, cell, (True,) * 3, kw)
    h = min(1e-3, margin / (4 * rc))
    E = lambda s: _oracle(z, pos * (1 + s), cell * (1 + s), (True,) * 3, 'damp_bj', kw)['energy']
    d1 = lambda s: (E(s) - E(-s)) / (2 * s)
    d2 = lambda s: (E(s) - 2 * E(0.0) + E(-s)) / (s * s)
    f1, f2 = (4 * d1(h / 2) - d1(h)) / 3, (4 * d2(h / 2) - d2(h)) / 3
    ref = f2 + f1
    V = abs(np.linalg.det(cell))
    got = V * C0[:3, :3].sum()
    print(f'NaCl D3 C0 [eV/A^3] =\n{np.round(C0, 6)}\ncubic relations {np.round(np.array(cub) / m, 8)} of max; '
          f'V sum C0_ij = {got:.6e}, f\'\' + f\' = {f2:.6e} + {f1:.6e} eV, rel diff {abs(got - ref) / abs(ref):.2e} '
          f'(step {h:.1e})')
    assert max(cub) < 1e-5 * m
    assert abs(got - ref) < 1e-4 * abs(ref)


def test_sevennet_d3_hessian_is_the_sum():
    from sevenn_b200.d3 import SevenNetD3Calculator
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.05, seed=2)
    atoms = _Atoms(z, pos, cell, True)
    calc = SevenNetD3Calculator('7net-0', device='cuda')
    H = calc.get_hessian(atoms)
    ref = calc.sevennet_calc.get_hessian(atoms) + calc.d3_calc.get_hessian(atoms)
    assert H.dtype == np.float64 and np.abs(H - ref).max() < 1e-6 * np.abs(ref).max()


def test_relaxed_ion_brute_force():
    """SevenNetD3Calculator.get_elastic_tensor of the 2-atom primitive Si cell against -d(W/V0)/de of the network
    oracle (edge list fixed) plus the D3 oracle, the second atom relaxed by scipy at each strain; bound 1e-3 of max|C|"""
    import scipy.optimize
    from sevenn_b200 import elastic
    from sevenn_b200.d3 import SevenNetD3Calculator
    from sevenn_b200.neighbors import build_graph
    from sevenn_b200.spec import build_spec
    from test_elastic_gpu import _diamond, _margin as _nn_margin, _oracle as _nn_oracle
    from test_hvp_gpu import _species
    from helpers import model_weights
    kw = dict(vdw_cutoff=1600.0, cn_cutoff=625.0)
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = _diamond(5.40, primitive=True)
    ei, ev = build_graph(pos, cell, True, build_spec(meta).cutoff)
    ev = ev.astype(np.float64)
    species = _species(meta, z)
    V0 = abs(np.linalg.det(cell))
    o = _nn_oracle(meta, arrays)

    def run(eps, u1):
        u = np.stack([np.zeros(3), u1])
        F = np.eye(3) + eps
        nn = o.forward(species, ei, ev @ F.T + u[ei[1]] - u[ei[0]])
        d3 = _oracle(z, pos @ F.T + u, cell @ F.T, (True,) * 3, 'damp_bj', kw)
        return nn['forces'].cpu().numpy() + d3['forces'], nn['virial'].detach().cpu().numpy() + _six(d3['sigma'])

    def sigma(eps):
        sol = scipy.optimize.root(lambda x: run(eps, x)[0][1], np.zeros(3), method='hybr', tol=1e-14)
        f, w = run(eps, sol.x)
        assert np.abs(f).max() < 1e-9
        return -elastic.virial_to_voigt(w) / V0

    m3, rc = _margin(pos, cell, (True,) * 3, kw)
    d = min(1e-3, _nn_margin(meta, ev) / (10 * np.linalg.norm(ev, axis=1).max()), m3 / (10 * rc))
    ref = np.zeros((6, 6))
    for k, e in enumerate(elastic.voigt_strains()):
        g = lambda s: (sigma(s * e) - sigma(-s * e)) / (2 * s)
        ref[:, k] = (4 * g(d) - g(2 * d)) / 3
    C = SevenNetD3Calculator('7net-0', device='cuda', **kw).get_elastic_tensor(_Atoms(z, pos, cell, True))
    err = np.abs(C - ref).max() / np.abs(ref).max()
    print(f'network + D3 relaxed-ion brute force (step {d:.1e}): max|C| = {np.abs(ref).max():.4f} eV/A^3, '
          f'max|C - C_ref| / max = {err:.2e} (bound 1e-3)')
    assert err < 1e-3


def _batch_structs():
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    out = []
    for fn, seed in [(diamond_si, 1), (rocksalt_nacl, 2), (diamond_si, 3)]:
        pos, cell, z = fn(1, 1, 1, sigma=0.04, seed=seed)
        cell = cell @ (np.eye(3) + 0.02 * np.random.RandomState(seed).normal(size=(3, 3))).T
        out.append((z, pos, cell, (True, True, True)))
    return out


def test_batch_members_equal_alone():
    """each member's D3Batch.hvp_strain output equals the structure alone, bit for bit"""
    import torch
    from sevenn_b200.d3 import D3Batch
    structs = _batch_structs()
    d3b = D3Batch('damp_bj', 'pbe', **KW)
    ap = np.cumsum([0] + [len(s[0]) for s in structs])
    cat = lambda k: np.concatenate([s[k] for s in structs])
    cells = np.stack([s[2] for s in structs])
    rng = np.random.RandomState(5)
    v = rng.normal(size=(int(ap[-1]), 3))
    eps = rng.normal(size=(len(structs), 3, 3))
    d3b.compute(torch.as_tensor(cat(0)), torch.as_tensor(cat(1)), cells, True, atom_ptr=ap)
    out, dw = d3b.hvp_strain(v, eps)
    out, dw = out.cpu().numpy(), dw.cpu().numpy()
    for b, s in enumerate(structs):
        alone = D3Batch('damp_bj', 'pbe', **KW)
        alone.compute(torch.as_tensor(s[0]), torch.as_tensor(s[1]), s[2][None], True)
        o1, w1 = alone.hvp_strain(v[ap[b]:ap[b + 1]], eps[b][None])
        assert np.array_equal(out[ap[b]:ap[b + 1]], o1.cpu().numpy()) and np.array_equal(dw[b], w1.cpu().numpy()[0])


def test_batch_elastic_tensors_with_d3():
    """DeviceBatch.elastic_tensors(d3=...) equals per-structure SevenNetD3Calculator.get_elastic_tensor to 1e-5"""
    import torch
    from sevenn_b200.batch import SevenNetD3Model
    from sevenn_b200.d3 import SevenNetD3Calculator

    class State:
        pass
    structs = _batch_structs()
    st = State()
    st.atomic_numbers = torch.as_tensor(np.concatenate([s[0] for s in structs]))
    st.positions = torch.as_tensor(np.concatenate([s[1] for s in structs]))
    st.row_vector_cell = torch.as_tensor(np.stack([s[2] for s in structs]))
    st.pbc = True
    st.system_idx = torch.as_tensor(np.repeat(np.arange(len(structs)), [len(s[0]) for s in structs]))
    model = SevenNetD3Model('7net-0', device='cuda', **KW)
    calc = SevenNetD3Calculator('7net-0', device='cuda', **KW)
    for relaxed in (True, False):
        C = model.elastic_tensors(st, relaxed=relaxed)
        ref = np.stack([calc.get_elastic_tensor(_Atoms(*s), relaxed=relaxed) for s in structs])
        err = np.abs(C - ref).max() / np.abs(ref).max()
        print(f'batch elastic tensors with D3 (relaxed={relaxed}): max|C - C_alone| / max = {err:.2e} (bound 1e-5)')
        assert err < 1e-5


def test_refusals_zero_atoms_and_no_side_effects():
    import torch
    from sevenn_b200.d3 import D3Batch
    z, pos, cell, pbc = _nacl()
    eng = _engine('damp_bj')
    with pytest.raises(RuntimeError, match='no system'):
        eng.hvp_strain(None, None)
    eng.set_system(z, pos, cell, pbc)
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.hvp_strain(np.zeros(pos.shape))
    eng.run_stage(1)
    eng.run_stage(2)
    eng.run_stage(3, 0, eng.n // 2)                   # a partial range
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.hvp_strain(np.zeros(pos.shape))
    for s in (1, 2, 3):
        eng.run_stage(s)
    before = eng.results()
    v = np.random.RandomState(0).normal(size=pos.shape)
    out1 = eng.hvp_strain(v, np.eye(3)[None])
    after = eng.results()
    assert before[0] == after[0] and np.array_equal(before[1], after[1]) and np.array_equal(before[2], after[2])
    out2 = eng.hvp_strain(v, np.eye(3)[None])
    assert all(torch.equal(a, b) for a, b in zip(out1, out2))            # deterministic
    with pytest.raises(ValueError, match='expected'):
        eng.hvp_strain(np.zeros((3, 3)))
    with pytest.raises(ValueError, match='expected'):
        eng.hvp_strain(None, np.zeros((2, 3, 3)))
    o, w = eng.hvp_strain(None, None)
    assert not o.any() and not w.any()
    eng.set_system(z, pos, cell, pbc)                 # a new set-up
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.hvp_strain(v)
    # zero atoms: an empty batch member and an all-empty batch zero-fill
    d3b = D3Batch('damp_bj', 'pbe', **KW)
    d3b.compute(torch.zeros(0, dtype=torch.int32), torch.zeros(0, 3), cell[None], True, atom_ptr=[0, 0])
    o, w = d3b.hvp_strain(None, np.eye(3)[None])
    assert o.shape == (0, 3) and w.shape == (1, 6) and not w.any()
    with pytest.raises(RuntimeError, match='no batch'):
        D3Batch('damp_bj', 'pbe', **KW).hvp_strain(None, None)
