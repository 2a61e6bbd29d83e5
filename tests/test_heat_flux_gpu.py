"""The engine's heat flux (s7b_engine_heat_flux, B200Engine.heat_flux, DeviceBatch.heat_flux,
SevenNetCalculator.get_heat_flux) on the GPU.

Reference: tests/flux_reference.py, fp64 central differences of the oracle's atomic energies (Richardson), on the
unfolded cluster of a periodic cell.  Bound: |J_engine - J_ref| / sum_j |J_j,ref|, J_j the per-atom contributions
r_j dU_j(v) - dU_j(r v) of the reference, which do not cancel; 2e-4 in the 'mlp' radial mode and 5e-4 in 'table'
mode (whose forward runs on the tables while the tangent pass evaluates the radial MLP), as for the Hessian-vector
product.  The observed errors are printed."""
import os

import numpy as np
import pytest

from flux_reference import make_oracle, reference_flux, unfold, n_layers
from helpers import model_weights

pytestmark = pytest.mark.gpu

BOUND = {'mlp': 2e-4, 'table': 5e-4}


def _species(meta, z):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z], dtype=np.int32)


def _synthetic(arch, tmp):
    from synthetic_models import convert, write_checkpoint
    return convert(write_checkpoint(os.path.join(tmp, f'flux_{arch}.pth'), arch, seed=17), arch)


def _weights(case, tmp):
    return _synthetic(case[6:], tmp) if case.startswith('synth_') else model_weights(case)


def engine_flux(meta, arrays, radial, species, pos, cell, pbc, v):
    from sevenn_b200.engine import B200Engine
    e = B200Engine(meta, arrays, radial=radial)
    e.set_positions(species, pos, cell, pbc)
    e.compute()
    jpot, ju = e.heat_flux(v)
    return e, jpot[0].cpu().numpy(), ju[0].cpu().numpy()


def _primitive_si(a=5.431):
    cell = 0.5 * a * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]])
    pos = np.array([[0.0, 0.0, 0.0], [0.25 * a, 0.25 * a, 0.25 * a]]) + np.array([[0.0, 0.0, 0.0], [0.03, -0.05, 0.02]])
    return pos, cell, np.array([14, 14])


def _check(case, radial, species, pos, cell, periodic, v, tmp):
    import torch
    from sevenn_b200.spec import build_spec
    meta, arrays = _weights(case, tmp)
    spec = build_spec(meta)
    o = make_oracle(meta, arrays, 'cuda')
    if periodic:
        cpos, parent = unfold(pos, cell, n_layers(meta) * spec.cutoff + 1.0)
        ref, per = reference_flux(o, spec, species[parent], cpos, v[parent], n_cell=len(pos))
    else:
        cpos = pos
        ref, per = reference_flux(o, spec, species, pos, v)
    _, got, _ = engine_flux(meta, arrays, radial, species, pos, cell if periodic else np.zeros((3, 3)),
                            np.array([periodic] * 3), v)
    torch.cuda.synchronize()
    scale = np.abs(per).sum()
    err = np.abs(got - ref).max() / scale
    print(f'flux {case} {radial} {"periodic" if periodic else "cluster"}: {len(cpos)} atoms in the reference, '
          f'J_ref = {ref}, J = {got}, err / sum|J_j| = {err:.2e} (bound {BOUND[radial]:.0e})')
    assert err < BOUND[radial]


@pytest.mark.parametrize('case', ['sevennet_0', 'sevennet_l3i5'])
@pytest.mark.parametrize('radial', ['table', 'mlp'])
def test_cluster_against_reference(case, radial, tmp_path):
    from sevenn_b200.neighbors import diamond_si
    meta, _ = _weights(case, str(tmp_path))
    pos, _, z = diamond_si(1, 1, 1, sigma=0.08, seed=7)
    v = np.random.RandomState(3).normal(size=pos.shape)
    _check(case, radial, _species(meta, z), pos, None, False, v, str(tmp_path))


@pytest.mark.parametrize('arch,radial', [('A', 'table'), ('B', 'mlp'), ('C', 'table'), ('D', 'mlp')])
def test_periodic_synthetic_against_unfolded_reference(arch, radial, tmp_path):
    from sevenn_b200.neighbors import diamond_si
    from synthetic_models import NUMBERS
    meta, _ = _weights('synth_' + arch, str(tmp_path))
    pos, cell, _ = diamond_si(1, 1, 1, sigma=0.08, seed=9)
    z = np.array([NUMBERS[i % 3] for i in range(len(pos))])
    v = np.random.RandomState(4).normal(size=pos.shape)
    _check('synth_' + arch, radial, _species(meta, z), pos, cell, True, v, str(tmp_path))


def test_sevennet0_primitive_si_against_unfolded_reference(tmp_path):
    """2-atom Si: the reference runs on the ~25 A unfolded cluster"""
    meta, _ = model_weights('sevennet_0')
    pos, cell, z = _primitive_si()
    v = np.random.RandomState(5).normal(size=pos.shape)
    _check('sevennet_0', 'table', _species(meta, z), pos, cell, True, v, str(tmp_path))


@pytest.fixture(scope='module')
def si64():
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    return meta, arrays, _species(meta, z), pos, cell


def test_uniform_velocity_is_virial_times_c(si64):
    meta, arrays, species, pos, cell = si64
    c = np.array([0.4, -0.9, 1.3])
    e, J, _ = engine_flux(meta, arrays, 'table', species, pos, cell, np.ones(3, bool), np.tile(c, (len(pos), 1)))
    w = e.buffer('virial', dtype='f8', shape=(6,)).cpu().numpy()
    W = np.array([[w[0], w[3], w[5]], [w[3], w[1], w[4]], [w[5], w[4], w[2]]])
    err = np.abs(J - W @ c).max() / np.abs(W @ c).max()
    print(f'uniform c: J_pot = {J}, W c = {W @ c}, rel err {err:.1e}')
    assert err < 1e-5


def _edge_pairwise(e, v):
    """-sum_e vec_e (f_e . v_src(e)) = sum_k W_k v_k from the engine's own edges and edge forces"""
    _, src, ev = e.graph_arrays()
    src = src.long().cpu().numpy()
    ev = ev.double().cpu().numpy()
    f = e.buffer('edge_force', shape=(e.n_edges, 3)).double().cpu().numpy()
    return -(ev * (f * v[src]).sum(1, keepdims=True)).sum(0), np.abs(ev * (f * v[src]).sum(1, keepdims=True)).sum()


def test_one_layer_is_the_atomic_virial_form(tmp_path):
    from synthetic_models import convert, layered, write_checkpoint
    from sevenn_b200.neighbors import diamond_si
    arch = layered('flux_one_layer', 2, 2, ['32x0e', '32x0e'])
    meta, arrays = convert(write_checkpoint(os.path.join(str(tmp_path), 'f1.pth'), arch, seed=11), arch)
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    v = np.random.RandomState(6).normal(size=pos.shape)
    e, J, _ = engine_flux(meta, arrays, 'mlp', _species(meta, z), pos, cell, np.ones(3, bool), v)
    pair, scale = _edge_pairwise(e, v)
    err = np.abs(J - pair).max() / scale
    print(f'one layer: J_pot = {J}, pairwise {pair}, err / sum|terms| = {err:.1e}')
    assert err < 1e-5


def test_negative_control_pairwise_form_is_wrong_for_sevennet0(si64):
    """the atomic-virial contraction sum_k W_k v_k misses the many-body flux of a 5-layer model"""
    meta, arrays, species, pos, cell = si64
    v = np.random.RandomState(8).normal(size=pos.shape)
    e, J, _ = engine_flux(meta, arrays, 'table', species, pos, cell, np.ones(3, bool), v)
    pair, scale = _edge_pairwise(e, v)
    gap = np.abs(J - pair).max() / scale
    print(f'SevenNet-0 Si64: J_pot = {J}, sum_k W_k v_k = {pair}, |diff| / sum|terms| = {gap:.2e}')
    assert gap > 10 * BOUND['table']


def test_invariances(si64):
    import torch
    meta, arrays, species, pos, cell = si64
    rng = np.random.RandomState(10)
    v = rng.normal(size=pos.shape)
    pbc = np.ones(3, bool)
    _, J, _ = engine_flux(meta, arrays, 'table', species, pos, cell, pbc, v)
    scale = np.abs(J).max()
    # wrapping an atom by a lattice vector
    p2 = pos.copy()
    p2[5] += cell[0] - cell[2]
    _, Jw, _ = engine_flux(meta, arrays, 'table', species, p2, cell, pbc, v)
    print(f'wrap: {np.abs(Jw - J).max() / scale:.1e}')
    assert np.abs(Jw - J).max() < 1e-5 * scale
    # rotation of positions, cell and v
    from scipy.spatial.transform import Rotation
    Rm = Rotation.from_euler('zyx', [0.3, -0.7, 1.1]).as_matrix()
    _, Jr, _ = engine_flux(meta, arrays, 'table', species, pos @ Rm.T, cell @ Rm.T, pbc, v @ Rm.T)
    print(f'rotation: {np.abs(Jr - Rm @ J).max() / scale:.1e}')
    assert np.abs(Jr - Rm @ J).max() < 1e-4 * scale
    # 2x2x2 supercell with tiled velocities
    shifts = np.array([[i, j, k] for i in range(2) for j in range(2) for k in range(2)]) @ cell
    ps = (pos[None] + shifts[:, None]).reshape(-1, 3)
    _, Js, _ = engine_flux(meta, arrays, 'table', np.tile(species, 8), ps, 2 * cell, pbc, np.tile(v, (8, 1)))
    print(f'supercell: {np.abs(Js - 8 * J).max() / (8 * scale):.1e}')
    assert np.abs(Js - 8 * J).max() < 1e-4 * 8 * scale
    torch.cuda.synchronize()


def test_batch_members_equal_single_structures_bitwise():
    import torch
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = model_weights('sevennet_0')
    systems = [diamond_si(1, 1, 1, sigma=0.05, seed=s) for s in (1, 2)] + [diamond_si(2, 1, 1, sigma=0.05, seed=3)]
    rng = np.random.RandomState(12)
    vs = [rng.normal(size=p.shape) for p, _, _ in systems]
    ms = [np.full(len(p), 28.0855) for p, _, _ in systems]
    e = B200Engine(meta, arrays, radial='table')
    b = DeviceBatch(e)
    numbers = np.concatenate([z for _, _, z in systems])
    positions = np.concatenate([p for p, _, _ in systems])
    cells = np.stack([c for _, c, _ in systems])
    sidx = np.concatenate([np.full(len(p), i) for i, (p, _, _) in enumerate(systems)])
    b.compute(numbers, positions, cells, np.ones(3, bool), sidx)
    Jb = b.heat_flux(np.concatenate(vs), np.concatenate(ms)).cpu().numpy()
    jpot_b, _ = e.heat_flux(np.concatenate(vs))
    jpot_b = jpot_b.cpu().numpy()
    for i, (p, c, z) in enumerate(systems):
        b.compute(z, p, c[None], np.ones(3, bool), np.zeros(len(p)))
        Ji = b.heat_flux(vs[i], ms[i]).cpu().numpy()
        jpot_i = e.heat_flux(vs[i])[0].cpu().numpy()
        print(f'structure {i}: J_pot batch {jpot_b[i]} alone {jpot_i[0]}')
        assert np.array_equal(jpot_b[i], jpot_i[0])
        assert np.array_equal(Jb[i], Ji[0])
    torch.cuda.synchronize()


def test_no_edges_gives_zero_jpot():
    from sevenn_b200.engine import B200Engine
    meta, arrays = model_weights('sevennet_0')
    pos = np.array([[0.0, 0.0, 0.0], [20.0, 0.0, 0.0]])
    e = B200Engine(meta, arrays, radial='table')
    e.set_positions(_species(meta, [14, 14]), pos, np.zeros((3, 3)), np.zeros(3, bool))
    e.compute()
    assert e.n_edges == 0
    v = np.array([[1.0, 2.0, 3.0], [-1.0, 0.5, 0.0]])
    jpot, ju = e.heat_flux(v)
    assert np.array_equal(jpot.cpu().numpy(), np.zeros((1, 3)))
    U = e.buffer('atomic_energy_f64', dtype='f8', shape=(2,)).cpu().numpy()
    assert np.allclose(ju.cpu().numpy()[0], (U[:, None] * v.astype(np.float32)).sum(0), rtol=1e-12)


def test_refusals():
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import build_graph, diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.05, seed=1)
    species = _species(meta, z)
    e = B200Engine(meta, arrays, radial='table')
    ei, ev = build_graph(pos, cell, True, 5.0)
    e.set_graph(species, ei, ev)
    v = np.zeros((len(pos), 3))
    with pytest.raises(RuntimeError, match='needs an s7b_engine_compute'):
        e.heat_flux(v)
    e.compute()
    with pytest.raises(ValueError):
        e.heat_flux(np.zeros((len(pos) + 1, 3)))
    with pytest.raises(ValueError):
        e.heat_flux(np.zeros((3, len(pos))))
    e.heat_flux(v)
    e.set_graph(species, ei[:, ei[0] < 6], ev[ei[0] < 6], n_local=6)      # atoms 6, 7 are ghosts
    e.compute()
    with pytest.raises(RuntimeError, match='ghost'):
        e.heat_flux(v)


class _Atoms:
    def __init__(self, pos, cell, z, v):
        self.pos, self.cell, self.z, self.v = pos, cell, z, v

    def get_positions(self):
        return self.pos

    def get_cell(self):
        return self.cell

    def get_pbc(self):
        return np.array([True] * 3)

    def get_atomic_numbers(self):
        return self.z

    def get_velocities(self):
        return self.v

    def get_masses(self):
        return np.full(len(self.z), 28.0855)


def test_calculator_reuses_the_step_and_leaves_results():
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    v = np.random.RandomState(13).normal(size=pos.shape) * 0.05
    atoms = _Atoms(pos, cell, z, v)
    calc = SevenNetCalculator('7net-0')
    calc.calculate(atoms)
    before = {k: np.copy(x) for k, x in calc.results.items()}
    stats = calc.engine.graph_stats()
    J = calc.get_heat_flux(atoms)
    assert calc.engine.graph_stats() == stats, 'get_heat_flux after a calculation on the same atoms ran a step'
    assert all(np.array_equal(before[k], calc.results[k]) for k in before)
    jpot = calc.get_heat_flux(atoms, convective=False)
    U = before['energies']
    conv = ((U + 0.5 * 28.0855 * (v * v).sum(1))[:, None] * v).sum(0)
    print(f'calculator: J = {J}, J_pot = {jpot}, J_conv = {conv}')
    assert J.shape == (3,) and J.dtype == np.float64
    assert np.allclose(J - jpot, conv, rtol=1e-5, atol=1e-6 * np.abs(conv).max())
    atoms2 = _Atoms(pos + 0.01, cell, z, v)
    J2 = calc.get_heat_flux(atoms2)
    assert calc.engine.graph_stats() != stats
    assert np.isfinite(J2).all()


def test_nothing_else_changes(si64):
    """compute after a flux pass matches compute before it, and the Hessian-vector product likewise.  The force
    scatter adds with float atomics, so two computes in a row already differ in their last bits; the bound is that
    run-to-run difference or 1e-6 of the largest value, whichever is larger."""
    import torch
    from sevenn_b200.engine import B200Engine
    meta, arrays, species, pos, cell = si64
    e = B200Engine(meta, arrays, radial='table')
    e.set_positions(species, pos, cell, np.ones(3, bool))
    u = np.random.RandomState(14).normal(size=pos.shape)

    def run():
        e.compute()
        out = (e.buffer('energy', dtype='f8', shape=(1,)).clone(), e.buffer('forces', shape=(len(pos), 3)).clone())
        return out + (e.hvp(u),)

    a, b = run(), run()
    e.heat_flux(u)
    c = run()
    for x, y, z_ in zip(a, b, c):
        run_to_run = (x - y).abs().max().item()
        bound = max(run_to_run, 1e-6 * x.abs().max().item())
        print(f'after a flux pass: max diff {(x - z_).abs().max().item():.2e}, run to run {run_to_run:.2e}')
        assert (x - z_).abs().max().item() <= bound, 'a flux pass changed a later compute or HVP'
    torch.cuda.synchronize()
