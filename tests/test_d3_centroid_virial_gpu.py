"""D3's per-atom centroid virial (s7b_d3_centroid_virial, D3Engine.centroid_virial / D3Batch.centroid_virials) and what
is built on it (D3Calculator / SevenNetD3Calculator.get_centroid_virials, DeviceBatch.centroid_virials with d3,
SevenNetD3Model.centroid_virials).

Reference: the fp64 restatement of tests/d3_centroid_reference.py, which tests/test_d3_centroid_virial_cpu.py checks
against the one-hot columns of the fp64 flux recursion.  Bound: max|Wc - Wc_ref| / sum_i |Wc_i,ref| < 1e-4, as for the
D3 Hessian-vector product and heat flux.  At the default cutoffs the rows are checked against independent GPU paths:
the virial of the forward and D3Engine.heat_flux.  The observed errors are printed."""
import numpy as np
import pytest

import d3_cells
from d3_centroid_reference import centroid_virials, pairwise_split

pytestmark = pytest.mark.gpu

AU = 0.52917726
KW = dict(vdw_cutoff=2500.0, cn_cutoff=900.0)        # reduced cutoffs (bohr^2) for the fp64 reference
BOUND = 1e-4


def _nacl(seed=12):
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.08, seed=seed)
    return z, pos, cell, (True, True, True)


def _si(nrep=1, seed=3):
    """rattled, sheared diamond Si: CN ~4 lies between silicon's references, so the CN part is not zero"""
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(nrep, nrep, nrep, sigma=0.08, seed=seed)
    return z, pos, cell @ (np.eye(3) + 0.03 * np.array([[0, 1, 0], [0, 0, -1], [1, 0, 0]])).T, (True, True, True)


def _system(name, kw=KW):
    """(numbers, positions, cell, pbc) as evaluated: a structure without a cell gets D3Calculator's generated cell"""
    if name == 'nacl':
        return _nacl()
    z, pos, cell, pbc = d3_cells.FIXTURES[name]()
    if np.asarray(cell).sum() == 0:
        rc = np.sqrt(max(kw['vdw_cutoff'], kw['cn_cutoff'])) * AU
        cell = np.eye(3) * (pos.max(0) - pos.min(0) + rc + 1.0)
        pbc = (True, True, True)
    return z, pos, cell, pbc


def _engine(damping, kw=KW):
    from sevenn_b200.d3 import D3Engine
    return D3Engine(damping, 'pbe', **kw)


def _forward(eng, z, pos, cell, pbc):
    eng.set_system(z, pos, cell, pbc)
    for s in (1, 2, 3):
        eng.run_stage(s)


def _wc(eng, z, pos, cell, pbc):
    _forward(eng, z, pos, cell, pbc)
    return eng.centroid_virial().cpu().numpy()


def _w3(w6):
    """[6] virial (xx,yy,zz,xy,yz,zx) -> 3x3"""
    xx, yy, zz, xy, yz, zx = w6
    return np.array([[xx, xy, zx], [xy, yy, yz], [zx, yz, zz]])


SYSTEMS = ['molecule', 'sheared', 'rotated', 'slab', 'wire', 'compressed_cs', 'species16', 'nacl']


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('system', SYSTEMS)
def test_against_fp64_reference(system, damping):
    z, pos, cell, pbc = _system(system)
    W = _wc(_engine(damping), z, pos, cell, pbc)
    ref, _, cnp = centroid_virials(z, pos, cell, pbc, damping, **KW, parts=True)
    err = np.abs(W - ref).max() / np.abs(ref).sum()
    print(f'{system} {damping}: max|Wc - Wc_ref| / sum|Wc_ref| = {err:.2e} (bound {BOUND:.0e}); '
          f'CN part max {np.abs(cnp).max():.2e} of max|Wc| {np.abs(ref).max():.2e} eV')
    assert W.shape == (len(z), 3, 3) and W.dtype == np.float64
    assert err < BOUND


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
def test_sum_is_the_virial_and_contraction_is_the_flux_at_default_cutoffs(damping):
    """sum_i Wc_i = D3Batch.compute's virial, sum_i Wc_i v_i = D3Engine.heat_flux(v)'s J_pot, self images included"""
    import torch
    from sevenn_b200.d3 import D3Batch
    rng = np.random.RandomState(1 + (damping == 'damp_zero'))
    for name in ('nacl', 'si', 'sheared', 'compressed_cs'):
        z, pos, cell, pbc = _si() if name == 'si' else _system(name)
        d3b = D3Batch(damping, 'pbe')
        out = d3b.compute(torch.as_tensor(z), torch.as_tensor(pos), cell[None], pbc)
        W = d3b.centroid_virials().cpu().numpy()
        vir = _w3(out['virial'].cpu().numpy()[0])
        ev = np.abs(W.sum(0) - vir).max() / np.abs(vir).max()
        v = rng.normal(size=pos.shape)
        jpot = d3b.heat_flux(v)[0].cpu().numpy()[0]
        J = np.einsum('iab,ib->a', W, v)
        scale = np.abs(W * v[:, None, :]).sum()
        ej = np.abs(J - jpot).max() / scale
        print(f'{name} {damping}, default cutoffs: max|sum Wc - W| / max|W| = {ev:.1e}; '
              f'max|sum Wc v - J_pot| / sum|Wc_i v_i| = {ej:.1e}')
        assert ev < 1e-5 and ej < 1e-5


def test_one_hot_flux_columns_at_default_cutoffs():
    """on an 8-atom cell, column b of Wc_i is D3Engine.heat_flux's J_pot for the velocity e_(i,b)"""
    z, pos, cell, pbc = _si()
    eng = _engine('damp_bj', {})
    W = _wc(eng, z, pos, cell, pbc)
    cols = np.zeros_like(W)
    for i in range(len(z)):
        for b in range(3):
            v = np.zeros(pos.shape)
            v[i, b] = 1.0
            cols[i, :, b] = eng.heat_flux(v)[0].cpu().numpy()[0]
    err = np.abs(W - cols).max() / np.abs(W).sum()
    print(f'8-atom Si, default cutoffs: max|Wc - flux columns| / sum|Wc| = {err:.1e}')
    assert err < 1e-5


def test_invariances():
    """at the default cutoffs: wrapping an atom changes nothing, Wc(R r) = R Wc R^T, a 2x2x2 supercell tiles the rows"""
    from scipy.spatial.transform import Rotation
    z, pos, cell, pbc = _si(2, seed=21)
    eng = _engine('damp_bj', {})
    W = _wc(eng, z, pos, cell, pbc)
    scale = np.abs(W).max()
    p2 = pos.copy()
    p2[5] += cell[0] - cell[2]
    Ww = _wc(eng, z, p2, cell, pbc)
    print(f'wrap: max|dWc| / max|Wc| = {np.abs(Ww - W).max() / scale:.1e}')
    assert np.abs(Ww - W).max() < 1e-5 * scale
    Rm = Rotation.from_euler('zyx', [0.3, -0.7, 1.1]).as_matrix()
    Wr = _wc(eng, z, pos @ Rm.T, cell @ Rm.T, pbc)
    er = np.abs(Wr - Rm @ W @ Rm.T).max() / scale
    print(f'rotation: max|Wc(R r) - R Wc R^T| / max|Wc| = {er:.1e}')
    assert er < 1e-4
    shifts = np.array([[i, j, k] for i in range(2) for j in range(2) for k in range(2)]) @ cell
    ps = (pos[None] + shifts[:, None]).reshape(-1, 3)
    Ws = _wc(eng, np.tile(z, 8), ps, 2 * cell, pbc)
    es = np.abs(Ws - np.tile(W, (8, 1, 1))).max() / scale
    print(f'supercell: max|Wc_super - tiled Wc| / max|Wc| = {es:.1e}')
    assert es < 1e-4


def _batch_structs():
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    out = []
    for fn, seed in [(diamond_si, 1), (rocksalt_nacl, 2), (diamond_si, 3)]:
        pos, cell, z = fn(1, 1, 1, sigma=0.04, seed=seed)
        cell = cell @ (np.eye(3) + 0.02 * np.random.RandomState(seed).normal(size=(3, 3))).T
        out.append((z, pos, cell, (True, True, True)))
    return out


def test_batch_members_equal_alone():
    """each member's rows of D3Batch.centroid_virials equal the structure alone, bit for bit"""
    import torch
    from sevenn_b200.d3 import D3Batch
    structs = _batch_structs() + [_system('slab')]
    d3b = D3Batch('damp_bj', 'pbe', **KW)
    ap = np.cumsum([0] + [len(s[0]) for s in structs])
    cat = lambda k: np.concatenate([s[k] for s in structs])
    d3b.compute(torch.as_tensor(cat(0)), torch.as_tensor(cat(1)), np.stack([s[2] for s in structs]),
                np.array([s[3] for s in structs]), atom_ptr=ap)
    W = d3b.centroid_virials().cpu().numpy()
    for b, s in enumerate(structs):
        alone = D3Batch('damp_bj', 'pbe', **KW)
        alone.compute(torch.as_tensor(s[0]), torch.as_tensor(s[1]), s[2][None], s[3])
        W1 = alone.centroid_virials().cpu().numpy()
        print(f'structure {b}: max|Wc batch - alone| = {np.abs(W[ap[b]:ap[b + 1]] - W1).max():.1e}')
        assert np.array_equal(W[ap[b]:ap[b + 1]], W1)


def test_nothing_else_changes_and_refusals():
    import torch
    from sevenn_b200.d3 import D3Batch
    z, pos, cell, pbc = _si(2)
    eng = _engine('damp_bj')
    v = np.random.RandomState(0).normal(size=pos.shape)
    with pytest.raises(RuntimeError, match='no system'):
        eng.centroid_virial()
    eng.set_system(z, pos, cell, pbc)
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.centroid_virial()
    eng.run_stage(1)
    eng.run_stage(2)
    eng.run_stage(3, 0, eng.n // 2)                   # a partial range
    names = ('cn', 'dc6i', 'eatom', 'force', 'energy', 'sigma')
    partial = eng.results(), [eng.buffer(k).clone() for k in names]
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.centroid_virial()
    assert all(torch.equal(a, b) for a, b in zip(partial[1], [eng.buffer(k) for k in names]))
    for s in (1, 2, 3):
        eng.run_stage(s)
    snap = lambda: (eng.results(), [eng.buffer(k).clone() for k in names], eng.hvp_strain(v, np.eye(3)[None]),
                    eng.heat_flux(v))
    before = snap()
    W1 = eng.centroid_virial()
    after = snap()
    assert before[0][0] == after[0][0] and all(np.array_equal(a, b) for a, b in zip(before[0][1:], after[0][1:]))
    for k in (1, 2, 3):
        assert all(torch.equal(a, b) for a, b in zip(before[k], after[k]))
    assert torch.equal(W1, eng.centroid_virial())                     # deterministic
    eng.set_system(z, pos, cell, pbc)                 # a new set-up
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.centroid_virial()
    # zero atoms: nothing to launch, an empty result
    d3b = D3Batch('damp_bj', 'pbe', **KW)
    d3b.compute(torch.zeros(0, dtype=torch.int32), torch.zeros(0, 3), cell[None], True, atom_ptr=[0, 0])
    assert d3b.centroid_virials().shape == (0, 3, 3)
    with pytest.raises(RuntimeError, match='no batch'):
        D3Batch('damp_bj', 'pbe', **KW).centroid_virials()


@pytest.mark.parametrize('name', ['nacl', 'sheared'])
def test_negative_control_pairwise_split(name):
    """the forward's per-atom rows spair + schain (fp64 reference) against Wc: they sum to the same virial but are
    not the centroid virial where CN varies.  In rock salt the C6 weights are one-hot (CN far above the references of
    Na and Cl), dC6/dCN = 0, D3 is a pair potential there and the split is exact."""
    z, pos, cell, pbc = _system(name)
    W = _wc(_engine('damp_bj'), z, pos, cell, pbc)
    split = pairwise_split(z, pos, cell, pbc, 'damp_bj', **KW)
    d = np.abs(split - W).max() / np.abs(W).max()
    print(f'{name}: max|pairwise split - Wc| / max|Wc| = {d:.2e}')
    if name == 'sheared':
        assert d > 1e-2
    else:
        assert d < 1e-4


class _Atoms:
    """the part of ase.Atoms the calculators use"""

    def __init__(self, numbers, positions, cell, pbc):
        self.numbers, self.positions = np.asarray(numbers), np.asarray(positions, dtype=np.float64)
        self.cell, self.pbc = np.asarray(cell, dtype=np.float64), np.broadcast_to(np.asarray(pbc, dtype=bool), (3,))

    def get_cell(self):
        return self.cell

    def get_pbc(self):
        return self.pbc

    def get_positions(self):
        return self.positions

    def get_atomic_numbers(self):
        return self.numbers

    def set_cell(self, cell):
        self.cell = np.asarray(cell, dtype=np.float64)

    def set_pbc(self, pbc):
        self.pbc = np.asarray(pbc, dtype=bool)


def test_sevennet_d3_calculator_is_the_sum():
    """network + D3 in fp64; the steps of calculate are reused and results are not touched"""
    from sevenn_b200.d3 import SevenNetD3Calculator
    z, pos, cell, pbc = _si(2, seed=5)
    atoms = _Atoms(z, pos, cell, pbc)
    calc = SevenNetD3Calculator('7net-0', device='cuda', **KW)
    calc.calculate(atoms)
    before = {k: np.copy(x) for k, x in calc.results.items()}
    calls = []
    forward = calc.d3_calc._forward
    calc.d3_calc._forward = lambda a: (calls.append(1), forward(a))
    stats = calc.sevennet_calc.engine.graph_stats()
    W = calc.get_centroid_virials(atoms)
    assert not calls and calc.sevennet_calc.engine.graph_stats() == stats, 'get_centroid_virials reran a step'
    assert all(np.array_equal(before[k], calc.results[k]) for k in before)
    net = calc.sevennet_calc.engine.centroid_virial().cpu().numpy()
    d3 = calc.d3_calc.engine.centroid_virial().cpu().numpy()
    assert W.shape == (len(z), 3, 3) and W.dtype == np.float64
    # the network's pass scatters with fp32 atomics, so a second call of it differs in the last bits (DESIGN.md §8.5)
    en = np.abs(W - (net + d3)).max() / np.abs(W).max()
    print(f'SevenNet-0 + D3: max|Wc - (network + D3)| / max|Wc| = {en:.1e} (network rerun)')
    assert en < 1e-5
    ref = _wc(_engine('damp_bj'), z, pos, cell, pbc)
    print(f'SevenNet-0 + D3: max|Wc_D3| {np.abs(d3).max():.3e}, max|Wc_net| {np.abs(net).max():.3e} eV; '
          f'D3 part against a fresh engine: {np.abs(d3 - ref).max():.1e}')
    assert np.array_equal(d3, ref)
    atoms2 = _Atoms(z, pos + 0.01, cell, pbc)
    assert np.isfinite(calc.get_centroid_virials(atoms2)).all() and calls


def test_d3_calculator_molecule_leaves_atoms():
    """a structure without a cell: the generated cell, and atoms is not modified"""
    from sevenn_b200.d3 import D3Calculator
    z, pos, cell, pbc = d3_cells.molecule()
    atoms = _Atoms(z, pos, cell, pbc)
    W = D3Calculator('damp_zero', 'pbe', **KW).get_centroid_virials(atoms)
    assert np.array_equal(atoms.cell, np.zeros((3, 3))) and not atoms.pbc.any()
    ref = centroid_virials(*_system('molecule'), 'damp_zero', **KW)
    assert np.abs(W - ref).max() < BOUND * np.abs(ref).sum()


def test_device_batch_with_d3_equals_calculator():
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
    ap = np.cumsum([0] + [len(s[0]) for s in structs])
    W = model.centroid_virials(st).cpu().numpy()
    ref = np.concatenate([calc.get_centroid_virials(_Atoms(*s)) for s in structs])
    err = np.abs(W - ref).max() / np.abs(ref).max()
    print(f'batch centroid virials with D3: max|Wc - Wc_alone| / max = {err:.1e}')
    assert W.shape == (int(ap[-1]), 3, 3) and err < 1e-6
    # without d3 the rows are the network's alone, as before
    net = model._batch.centroid_virials().cpu().numpy()
    en = np.abs(W - (net + model.d3.centroid_virials().cpu().numpy())).max() / np.abs(W).max()
    print(f'batch: max|Wc - (network + D3)| / max|Wc| = {en:.1e} (network rerun)')
    assert en < 1e-5
    # a D3Batch whose last compute was on other structures is refused
    model.d3.compute(st.atomic_numbers[:ap[1]], st.positions[:ap[1]], structs[0][2][None], True)
    with pytest.raises(ValueError, match='atom_ptr'):
        model._batch.centroid_virials(d3=model.d3)
