"""The D3 heat flux (s7b_d3_heat_flux, D3Engine / D3Batch.heat_flux) and what is built on it
(D3Calculator / SevenNetD3Calculator.get_heat_flux, DeviceBatch.heat_flux with d3, SevenNetD3Model.heat_flux).

Reference: the fp64 recursion of tests/d3_flux_reference.py on the periodic cell, which tests/test_d3_heat_flux_cpu.py
checks against Richardson differences of the oracle's atomic energies.  Bound: |J - J_ref| / sum_j |R_j,ref| < 1e-4,
R_j the per-atom terms, as for the D3 Hessian-vector product.  The observed errors are printed."""
import numpy as np
import pytest

import d3_cells
from d3_flux_reference import recursion_flux

pytestmark = pytest.mark.gpu

AU = 0.52917726
KW = dict(vdw_cutoff=2500.0, cn_cutoff=900.0)        # reduced cutoffs (bohr^2) for the fp64 reference
BOUND = 1e-4
MASS = {1: 1.008, 2: 4.0026, 6: 12.011, 11: 22.99, 14: 28.0855, 17: 35.45}


def _nacl(seed=12):
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.08, seed=seed)
    return z, pos, cell, (True, True, True)


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


def _flux(eng, z, pos, cell, pbc, v):
    _forward(eng, z, pos, cell, pbc)
    jpot, ju = eng.heat_flux(v)
    return jpot.cpu().numpy()[0], ju.cpu().numpy()[0]


def _w3(w6):
    """[6] virial (xx,yy,zz,xy,yz,zx) -> 3x3"""
    xx, yy, zz, xy, yz, zx = w6
    return np.array([[xx, xy, zx], [xy, yy, yz], [zx, yz, zz]])


SYSTEMS = ['molecule', 'sheared', 'rotated', 'slab', 'wire', 'compressed_cs', 'species16', 'nacl']


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
@pytest.mark.parametrize('system', SYSTEMS)
def test_against_fp64_recursion(system, damping):
    z, pos, cell, pbc = _system(system)
    rng = np.random.RandomState(SYSTEMS.index(system) * 2 + (damping == 'damp_zero'))
    v = rng.normal(size=pos.shape)
    eng = _engine(damping)
    jpot, ju = _flux(eng, z, pos, cell, pbc, v)
    ref, R, U = recursion_flux(z, pos, cell, pbc, v, damping, **KW)
    scale = np.abs(R).sum()
    err = np.abs(jpot - ref).max() / scale
    Ug = eng.atomic_energies().cpu().numpy()
    eu = np.abs(Ug - U).max() / np.abs(U).max()
    ju_ref = (U[:, None] * v).sum(0)
    eju = np.abs(ju - ju_ref).max() / np.abs(U[:, None] * v).sum()
    print(f'{system} {damping}: J_pot = {jpot}, ref {ref}, err / sum|R_j| = {err:.2e} (bound {BOUND:.0e}); '
          f'U err {eu:.1e}, sum U v err {eju:.1e}')
    assert err < BOUND and eu < BOUND and eju < BOUND


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
def test_uniform_velocity_is_virial_times_c_at_default_cutoffs(damping):
    """sum_i dU_j/dr_i = 0 leaves J_pot = W c, against D3Batch.compute's virial; self images included"""
    import torch
    from sevenn_b200.d3 import D3Batch
    c = np.array([0.3, -1.1, 0.7])
    for name in ('nacl', 'sheared', 'compressed_cs'):
        z, pos, cell, pbc = _system(name)
        d3b = D3Batch(damping, 'pbe')
        out = d3b.compute(torch.as_tensor(z), torch.as_tensor(pos), cell[None], pbc)
        jpot, _ = d3b.heat_flux(np.tile(c, (len(z), 1)))
        W = _w3(out['virial'].cpu().numpy()[0])
        J = jpot.cpu().numpy()[0]
        err = np.abs(J - W @ c).max() / (np.abs(W).max() * np.abs(c).max())
        print(f'{name} {damping}, default cutoffs: J_pot = {J}, W c = {W @ c}, err / (max|W| max|c|) = {err:.1e}')
        assert err < 1e-5


def test_invariances():
    """at the default cutoffs: wrapping an atom changes nothing, rotation is covariant, a 2x2x2 supercell gives 8 J"""
    from scipy.spatial.transform import Rotation
    z, pos, cell, pbc = _nacl(21)
    v = np.random.RandomState(10).normal(size=pos.shape)
    eng = _engine('damp_bj', {})
    J, ju = _flux(eng, z, pos, cell, pbc, v)
    scale = np.abs(J).max()
    p2 = pos.copy()
    p2[5] += cell[0] - cell[2]
    Jw, juw = _flux(eng, z, p2, cell, pbc, v)
    print(f'wrap: {np.abs(Jw - J).max() / scale:.1e}')
    assert np.abs(Jw - J).max() < 1e-5 * scale and np.abs(juw - ju).max() < 1e-5 * np.abs(ju).max()
    Rm = Rotation.from_euler('zyx', [0.3, -0.7, 1.1]).as_matrix()
    Jr, _ = _flux(eng, z, pos @ Rm.T, cell @ Rm.T, pbc, v @ Rm.T)
    print(f'rotation: {np.abs(Jr - Rm @ J).max() / scale:.1e}')
    assert np.abs(Jr - Rm @ J).max() < 1e-4 * scale
    shifts = np.array([[i, j, k] for i in range(2) for j in range(2) for k in range(2)]) @ cell
    ps = (pos[None] + shifts[:, None]).reshape(-1, 3)
    Js, jus = _flux(eng, np.tile(z, 8), ps, 2 * cell, pbc, np.tile(v, (8, 1)))
    print(f'supercell: {np.abs(Js - 8 * J).max() / (8 * scale):.1e}')
    assert np.abs(Js - 8 * J).max() < 1e-4 * 8 * scale and np.abs(jus - 8 * ju).max() < 1e-5 * 8 * np.abs(ju).max()


def _batch_structs():
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    out = []
    for fn, seed in [(diamond_si, 1), (rocksalt_nacl, 2), (diamond_si, 3)]:
        pos, cell, z = fn(1, 1, 1, sigma=0.04, seed=seed)
        cell = cell @ (np.eye(3) + 0.02 * np.random.RandomState(seed).normal(size=(3, 3))).T
        out.append((z, pos, cell, (True, True, True)))
    return out


def test_batch_members_equal_alone():
    """each member's D3Batch.heat_flux equals the structure alone, bit for bit"""
    import torch
    from sevenn_b200.d3 import D3Batch
    structs = _batch_structs() + [_system('slab')]
    d3b = D3Batch('damp_bj', 'pbe', **KW)
    ap = np.cumsum([0] + [len(s[0]) for s in structs])
    cat = lambda k: np.concatenate([s[k] for s in structs])
    v = np.random.RandomState(5).normal(size=(int(ap[-1]), 3))
    d3b.compute(torch.as_tensor(cat(0)), torch.as_tensor(cat(1)), np.stack([s[2] for s in structs]),
                np.array([s[3] for s in structs]), atom_ptr=ap)
    jp, ju = (t.cpu().numpy() for t in d3b.heat_flux(v))
    for b, s in enumerate(structs):
        alone = D3Batch('damp_bj', 'pbe', **KW)
        alone.compute(torch.as_tensor(s[0]), torch.as_tensor(s[1]), s[2][None], s[3])
        jp1, ju1 = (t.cpu().numpy()[0] for t in alone.heat_flux(v[ap[b]:ap[b + 1]]))
        print(f'structure {b}: J_pot batch {jp[b]} alone {jp1}')
        assert np.array_equal(jp[b], jp1) and np.array_equal(ju[b], ju1)


def test_nothing_else_changes_and_refusals():
    import torch
    from sevenn_b200.d3 import D3Batch
    z, pos, cell, pbc = _nacl()
    eng = _engine('damp_bj')
    v = np.random.RandomState(0).normal(size=pos.shape)
    with pytest.raises(RuntimeError, match='no system'):
        eng.heat_flux(np.zeros((0, 3)))
    eng.set_system(z, pos, cell, pbc)
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.heat_flux(v)
    eng.run_stage(1)
    eng.run_stage(2)
    eng.run_stage(3, 0, eng.n // 2)                   # a partial range
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.heat_flux(v)
    for s in (1, 2, 3):
        eng.run_stage(s)
    names = ('cn', 'dc6i', 'eatom', 'force', 'energy', 'sigma')
    before = eng.results(), [eng.buffer(k).clone() for k in names], eng.hvp_strain(v, np.eye(3)[None])
    f1 = eng.heat_flux(v)
    after = eng.results(), [eng.buffer(k).clone() for k in names], eng.hvp_strain(v, np.eye(3)[None])
    assert before[0][0] == after[0][0] and all(np.array_equal(a, b) for a, b in zip(before[0][1:], after[0][1:]))
    assert all(torch.equal(a, b) for a, b in zip(before[1], after[1]))
    assert all(torch.equal(a, b) for a, b in zip(before[2], after[2]))
    f2 = eng.heat_flux(v)
    assert all(torch.equal(a, b) for a, b in zip(f1, f2))            # deterministic
    with pytest.raises(ValueError, match='expected'):
        eng.heat_flux(np.zeros((3, 3)))
    with pytest.raises(ValueError, match='expected'):
        eng.heat_flux(np.zeros((3, len(z))))
    eng.set_system(z, pos, cell, pbc)                 # a new set-up
    with pytest.raises(RuntimeError, match='stages 1, 2 and 3'):
        eng.heat_flux(v)
    # zero atoms: an all-empty batch zero-fills
    d3b = D3Batch('damp_bj', 'pbe', **KW)
    d3b.compute(torch.zeros(0, dtype=torch.int32), torch.zeros(0, 3), cell[None], True, atom_ptr=[0, 0])
    jp, ju = d3b.heat_flux(np.zeros((0, 3)))
    assert jp.shape == (1, 3) and not jp.any() and not ju.any()
    with pytest.raises(RuntimeError, match='no batch'):
        D3Batch('damp_bj', 'pbe', **KW).heat_flux(np.zeros((0, 3)))


class _Atoms:
    """the part of ase.Atoms the calculators and get_heat_flux use"""

    def __init__(self, numbers, positions, cell, pbc, v):
        self.numbers, self.positions = np.asarray(numbers), np.asarray(positions, dtype=np.float64)
        self.cell, self.pbc = np.asarray(cell, dtype=np.float64), np.broadcast_to(np.asarray(pbc, dtype=bool), (3,))
        self.v = np.asarray(v, dtype=np.float64)

    def get_cell(self):
        return self.cell

    def get_pbc(self):
        return self.pbc

    def get_positions(self):
        return self.positions

    def get_atomic_numbers(self):
        return self.numbers

    def get_velocities(self):
        return self.v

    def get_masses(self):
        return np.array([MASS[int(a)] for a in self.numbers])

    def set_cell(self, cell):
        self.cell = np.asarray(cell, dtype=np.float64)

    def set_pbc(self, pbc):
        self.pbc = np.asarray(pbc, dtype=bool)


def _kinetic(atoms):
    v, m = atoms.get_velocities(), atoms.get_masses()
    return ((0.5 * m * (v * v).sum(1))[:, None] * v).sum(0)


def test_sevennet_d3_calculator_is_the_sum():
    """network (J_pot + sum U v) + D3 (J_pot + sum U v) + the kinetic part once; the steps of calculate are reused
    and results are not touched"""
    from sevenn_b200.d3 import SevenNetD3Calculator
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.05, seed=3)
    atoms = _Atoms(z, pos, cell, True, np.random.RandomState(4).normal(size=pos.shape) * 0.05)
    calc = SevenNetD3Calculator('7net-0', device='cuda', **KW)
    calc.calculate(atoms)
    before = {k: np.copy(x) for k, x in calc.results.items()}
    calls = []
    forward = calc.d3_calc._forward
    calc.d3_calc._forward = lambda a: (calls.append(1), forward(a))
    stats = calc.sevennet_calc.engine.graph_stats()
    J = calc.get_heat_flux(atoms)
    assert not calls and calc.sevennet_calc.engine.graph_stats() == stats, 'get_heat_flux reran a step'
    assert all(np.array_equal(before[k], calc.results[k]) for k in before)
    net = calc.sevennet_calc.get_heat_flux(atoms)                 # its J_pot + sum U v + the kinetic part
    eng = _engine('damp_bj')
    jp, ju = _flux(eng, z, pos, cell, (True,) * 3, atoms.get_velocities())
    ref = net + jp + ju
    err = np.abs(J - ref).max() / np.abs(ref).max()
    print(f'SevenNet-0 + D3: J = {J}, network {net}, D3 J_pot {jp}, D3 sum U v {ju}, kinetic {_kinetic(atoms)}; '
          f'err {err:.1e}')
    assert J.shape == (3,) and J.dtype == np.float64 and err < 1e-6
    jpot = calc.get_heat_flux(atoms, convective=False)
    ref_pot = calc.sevennet_calc.get_heat_flux(atoms, convective=False) + jp
    assert np.abs(jpot - ref_pot).max() < 1e-6 * np.abs(ref_pot).max()
    assert not calls
    atoms2 = _Atoms(z, pos + 0.01, cell, True, atoms.get_velocities())
    assert np.isfinite(calc.get_heat_flux(atoms2)).all() and calls


def test_d3_calculator_molecule_leaves_atoms():
    """a structure without a cell: the generated cell, and atoms is not modified"""
    from sevenn_b200.d3 import D3Calculator
    z, pos, cell, pbc = d3_cells.molecule()
    v = np.random.RandomState(8).normal(size=pos.shape)
    atoms = _Atoms(z, pos, cell, pbc, v)
    J = D3Calculator('damp_zero', 'pbe', **KW).get_heat_flux(atoms, convective=False)
    assert np.array_equal(atoms.cell, np.zeros((3, 3))) and not atoms.pbc.any()
    ref, R, _ = recursion_flux(*_system('molecule'), v, 'damp_zero', **KW)
    assert np.abs(J - ref).max() < BOUND * np.abs(R).sum()


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
    st.masses = torch.as_tensor([MASS[int(a)] for a in st.atomic_numbers])
    v = np.random.RandomState(9).normal(size=(len(st.atomic_numbers), 3)) * 0.05
    model = SevenNetD3Model('7net-0', device='cuda', **KW)
    calc = SevenNetD3Calculator('7net-0', device='cuda', **KW)
    ap = np.cumsum([0] + [len(s[0]) for s in structs])
    for convective in (True, False):
        J = model.heat_flux(st, v, convective=convective).cpu().numpy()
        ref = np.stack([calc.get_heat_flux(_Atoms(*s, v[ap[b]:ap[b + 1]]), convective=convective)
                        for b, s in enumerate(structs)])
        err = np.abs(J - ref).max() / np.abs(ref).max()
        print(f'batch heat flux with D3 (convective={convective}): max|J - J_alone| / max = {err:.1e}')
        assert err < 1e-6
    # a D3Batch whose last compute was on other structures is refused
    model.d3.compute(st.atomic_numbers[:ap[1]], st.positions[:ap[1]], structs[0][2][None], True)
    with pytest.raises(ValueError, match='atom_ptr'):
        model._batch.heat_flux(v, st.masses, d3=model.d3)
