"""The engine's per-atom centroid virial (s7b_engine_centroid_virial, B200Engine.centroid_virial,
DeviceBatch.centroid_virials, SevenNetCalculator.get_centroid_virials) on the GPU.

Reference: tests/centroid_reference.py, four fp64 reverse passes of the oracle with per-atom weighted atomic energies,
on the unfolded cluster of a periodic cell.  Bound: max |Wc_engine - Wc_ref| / sum_i sum_ab |Wc_i,ab,ref|; 2e-4 in
the 'mlp' radial mode and 5e-4 in 'table' mode (whose forward runs on the tables while this pass evaluates the radial
MLP), as for the heat flux.  Also against the engine's own forward-mode heat flux, an independent CUDA path, and the
identities of DESIGN.md §8.5.  The observed errors are printed."""
import os

import numpy as np
import pytest

from centroid_reference import reference_centroid_cell
from flux_reference import make_oracle
from helpers import model_weights

pytestmark = pytest.mark.gpu

BOUND = {'mlp': 2e-4, 'table': 5e-4}


def _species(meta, z):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z], dtype=np.int32)


def _synthetic(arch, tmp):
    from synthetic_models import convert, write_checkpoint
    return convert(write_checkpoint(os.path.join(tmp, f'wc_{arch}.pth'), arch, seed=17), arch)


def _weights(case, tmp):
    return _synthetic(case[6:], tmp) if case.startswith('synth_') else model_weights(case)


def engine_wc(meta, arrays, radial, species, pos, cell, pbc, **kw):
    from sevenn_b200.engine import B200Engine
    e = B200Engine(meta, arrays, radial=radial, **kw)
    e.set_positions(species, pos, cell, pbc)
    e.compute()
    return e, e.centroid_virial().cpu().numpy()


def _primitive_si(a=5.431):
    cell = 0.5 * a * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]])
    pos = np.array([[0.0, 0.0, 0.0], [0.25 * a, 0.25 * a, 0.25 * a]]) + np.array([[0.0, 0.0, 0.0], [0.03, -0.05, 0.02]])
    return pos, cell, np.array([14, 14])


def _check(case, radial, species, pos, cell, periodic, tmp):
    import torch
    from sevenn_b200.spec import build_spec
    meta, arrays = _weights(case, tmp)
    spec = build_spec(meta)
    o = make_oracle(meta, arrays, 'cuda')
    ref = reference_centroid_cell(o, spec, species, pos, cell if periodic else None)
    _, got = engine_wc(meta, arrays, radial, species, pos, cell if periodic else np.zeros((3, 3)),
                       np.array([periodic] * 3))
    torch.cuda.synchronize()
    err = np.abs(got - ref).max() / np.abs(ref).sum()
    print(f'centroid {case} {radial} {"periodic" if periodic else "cluster"}: err / sum|Wc| = {err:.2e} '
          f'(bound {BOUND[radial]:.0e})')
    assert err < BOUND[radial]


@pytest.mark.parametrize('case', ['sevennet_0', 'sevennet_l3i5'])
@pytest.mark.parametrize('radial', ['table', 'mlp'])
def test_cluster_against_reference(case, radial, tmp_path):
    from sevenn_b200.neighbors import diamond_si
    meta, _ = _weights(case, str(tmp_path))
    pos, _, z = diamond_si(1, 1, 1, sigma=0.08, seed=7)
    _check(case, radial, _species(meta, z), pos, None, False, str(tmp_path))


@pytest.mark.parametrize('arch,radial', [('A', 'table'), ('B', 'mlp'), ('C', 'table'), ('D', 'mlp')])
def test_periodic_synthetic_against_unfolded_reference(arch, radial, tmp_path):
    from sevenn_b200.neighbors import diamond_si
    from synthetic_models import NUMBERS
    meta, _ = _weights('synth_' + arch, str(tmp_path))
    pos, cell, _ = diamond_si(1, 1, 1, sigma=0.08, seed=9)
    z = np.array([NUMBERS[i % 3] for i in range(len(pos))])
    _check('synth_' + arch, radial, _species(meta, z), pos, cell, True, str(tmp_path))


def test_sevennet0_primitive_si_against_unfolded_reference(tmp_path):
    """2-atom Si: the reference runs on the ~25 A unfolded cluster"""
    meta, _ = model_weights('sevennet_0')
    pos, cell, z = _primitive_si()
    _check('sevennet_0', 'table', _species(meta, z), pos, cell, True, str(tmp_path))


@pytest.fixture(scope='module')
def si64():
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    return meta, arrays, _species(meta, z), pos, cell


@pytest.mark.parametrize('cells', [(1, 1, 1), (2, 2, 2)])
def test_columns_equal_the_forward_mode_flux(cells):
    """Wc column by column from 3N one-hot-velocity heat_flux calls (8 atoms), and sum_i Wc_i v_i = J_pot for random
    v (8 and 64 atoms)"""
    import torch
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = diamond_si(*cells, sigma=0.05, seed=6)
    n = len(pos)
    e, Wc = engine_wc(meta, arrays, 'table', _species(meta, z), pos, cell, np.ones(3, bool))
    scale = np.abs(Wc).sum()
    if n <= 8:
        cols = np.zeros((n, 3, 3))
        for i in range(n):
            for b in range(3):
                v = np.zeros((n, 3))
                v[i, b] = 1.0
                cols[i, :, b] = e.heat_flux(v)[0][0].cpu().numpy()
        err = np.abs(cols - Wc).max() / scale
        print(f'{n} atoms: one-hot heat flux columns vs reverse pass: err / sum|Wc| = {err:.1e}')
        assert err < 1e-5
    for seed in range(3):
        v = np.random.RandomState(20 + seed).normal(size=pos.shape)
        J = e.heat_flux(v)[0][0].cpu().numpy()
        Jc = np.einsum('iab,ib->a', Wc, v.astype(np.float32).astype(np.float64))
        err = np.abs(J - Jc).max() / np.abs(Wc * np.abs(v)[:, None, :]).sum()
        print(f'{n} atoms, random v: J_pot = {J}, sum Wc v = {Jc}, err / sum|terms| = {err:.1e}')
        assert err < 1e-5
    torch.cuda.synchronize()


def test_sum_is_the_virial(si64):
    meta, arrays, species, pos, cell = si64
    e, Wc = engine_wc(meta, arrays, 'table', species, pos, cell, np.ones(3, bool))
    w = e.buffer('virial', dtype='f8', shape=(6,)).cpu().numpy()
    W = np.array([[w[0], w[3], w[5]], [w[3], w[1], w[4]], [w[5], w[4], w[2]]])
    err = np.abs(Wc.sum(0) - W).max() / np.abs(Wc).sum()
    asym = np.abs(Wc - Wc.transpose(0, 2, 1)).max() / np.abs(Wc).max()
    print(f'sum_i Wc_i = {Wc.sum(0).tolist()}, W = {W.tolist()}, err / sum|Wc| = {err:.1e}, '
          f'per-atom asymmetry {asym:.1e}')
    assert err < 1e-5
    assert asym > 1e-3


def _pairwise(e):
    """-sum_{e: neighbour k} vec_e (x) f_e per atom k, from the engine's own edges and edge forces"""
    _, src, ev = e.graph_arrays()
    src = src.long().cpu().numpy()
    ev = ev.double().cpu().numpy()
    f = e.buffer('edge_force', shape=(e.n_edges, 3)).double().cpu().numpy()
    out = np.zeros((e.n_nodes, 3, 3))
    np.add.at(out, src, -ev[:, :, None] * f[:, None, :])
    return out


def test_one_layer_is_the_atomic_virial(tmp_path):
    from synthetic_models import convert, layered, write_checkpoint
    from sevenn_b200.neighbors import diamond_si
    arch = layered('wc_one_layer', 2, 2, ['32x0e', '32x0e'])
    meta, arrays = convert(write_checkpoint(os.path.join(str(tmp_path), 'w1.pth'), arch, seed=11), arch)
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    e, Wc = engine_wc(meta, arrays, 'mlp', _species(meta, z), pos, cell, np.ones(3, bool), atomic_virial=True)
    av = e.buffer('atomic_virial', shape=(len(pos), 6)).double().cpu().numpy()
    rows = np.stack([Wc[:, 0, 0], Wc[:, 1, 1], Wc[:, 2, 2], Wc[:, 0, 1], Wc[:, 1, 2], Wc[:, 2, 0]], 1)
    scale = np.abs(Wc).sum()
    err = np.abs(Wc - _pairwise(e)).max() / scale
    err_av = np.abs(rows - av).max() / scale
    print(f'one layer: |Wc - pairwise| / sum|Wc| = {err:.1e}, |rows - atomic_virial| / sum|Wc| = {err_av:.1e}')
    assert err < 1e-6 and err_av < 1e-6


def test_negative_control_atomic_virial_differs_for_sevennet0(si64):
    """the pairwise split differs from the centroid virial for a 5-layer model"""
    meta, arrays, species, pos, cell = si64
    e, Wc = engine_wc(meta, arrays, 'table', species, pos, cell, np.ones(3, bool))
    gap = np.abs(Wc - _pairwise(e)).max() / np.abs(Wc).sum()
    print(f'SevenNet-0 Si64: max |Wc - pairwise| / sum|Wc| = {gap:.2e}')
    assert gap > BOUND['table']


def test_invariances(si64):
    import torch
    meta, arrays, species, pos, cell = si64
    pbc = np.ones(3, bool)
    _, Wc = engine_wc(meta, arrays, 'table', species, pos, cell, pbc)
    scale = np.abs(Wc).max()
    # wrapping an atom by a lattice vector
    p2 = pos.copy()
    p2[5] += cell[0] - cell[2]
    _, Ww = engine_wc(meta, arrays, 'table', species, p2, cell, pbc)
    print(f'wrap: {np.abs(Ww - Wc).max() / scale:.1e}')
    assert np.abs(Ww - Wc).max() < 1e-5 * scale
    # rotation: Wc(R r) = R Wc R^T
    from scipy.spatial.transform import Rotation
    Rm = Rotation.from_euler('zyx', [0.3, -0.7, 1.1]).as_matrix()
    _, Wr = engine_wc(meta, arrays, 'table', species, pos @ Rm.T, cell @ Rm.T, pbc)
    rot = np.einsum('ab,ibc,dc->iad', Rm, Wc, Rm)
    print(f'rotation: {np.abs(Wr - rot).max() / scale:.1e}')
    assert np.abs(Wr - rot).max() < 1e-4 * scale
    # 2x2x2 supercell tiles the values
    shifts = np.array([[i, j, k] for i in range(2) for j in range(2) for k in range(2)]) @ cell
    ps = (pos[None] + shifts[:, None]).reshape(-1, 3)
    _, Ws = engine_wc(meta, arrays, 'table', np.tile(species, 8), ps, 2 * cell, pbc)
    print(f'supercell: {np.abs(Ws - np.tile(Wc, (8, 1, 1))).max() / scale:.1e}')
    assert np.abs(Ws - np.tile(Wc, (8, 1, 1))).max() < 1e-4 * scale
    torch.cuda.synchronize()


def test_batch_members_equal_single_structures():
    """within the tolerance of the fp32 atomics of the scatter (the per-edge sums of a role spread over two CTAs)"""
    import torch
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = model_weights('sevennet_0')
    systems = [diamond_si(1, 1, 1, sigma=0.05, seed=s) for s in (1, 2)] + [diamond_si(2, 1, 1, sigma=0.05, seed=3)]
    e = B200Engine(meta, arrays, radial='table')
    b = DeviceBatch(e)
    numbers = np.concatenate([z for _, _, z in systems])
    positions = np.concatenate([p for p, _, _ in systems])
    cells = np.stack([c for _, c, _ in systems])
    sidx = np.concatenate([np.full(len(p), i) for i, (p, _, _) in enumerate(systems)])
    b.compute(numbers, positions, cells, np.ones(3, bool), sidx)
    Wb = b.centroid_virials().cpu().numpy()
    off = 0
    for i, (p, c, z) in enumerate(systems):
        b.compute(z, p, c[None], np.ones(3, bool), np.zeros(len(p)))
        Wi = b.centroid_virials().cpu().numpy()
        err = np.abs(Wb[off:off + len(p)] - Wi).max() / np.abs(Wi).max()
        print(f'structure {i}: max |batch - alone| / max |Wc| = {err:.1e}')
        assert err < 1e-5
        off += len(p)
    torch.cuda.synchronize()


def test_no_edges_gives_zeros():
    from sevenn_b200.engine import B200Engine
    meta, arrays = model_weights('sevennet_0')
    pos = np.array([[0.0, 0.0, 0.0], [20.0, 0.0, 0.0]])
    e = B200Engine(meta, arrays, radial='table')
    e.set_positions(_species(meta, [14, 14]), pos, np.zeros((3, 3)), np.zeros(3, bool))
    e.compute()
    assert e.n_edges == 0
    assert np.array_equal(e.centroid_virial().cpu().numpy(), np.zeros((2, 3, 3)))


def test_refusals():
    import torch
    from sevenn_b200.engine import B200Engine, check
    from sevenn_b200.neighbors import build_graph, diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = diamond_si(1, 1, 1, sigma=0.05, seed=1)
    species = _species(meta, z)
    e = B200Engine(meta, arrays, radial='table')
    ei, ev = build_graph(pos, cell, True, 5.0)
    e.set_graph(species, ei, ev)
    with pytest.raises(RuntimeError, match='needs an s7b_engine_compute'):
        e.centroid_virial()
    e.compute()
    e.centroid_virial()
    e.set_graph(species, ei[:, ei[0] < 6], ev[ei[0] < 6], n_local=6)      # atoms 6, 7 are ghosts
    e.compute()
    with pytest.raises(RuntimeError, match='ghost'):
        e.centroid_virial()
    # a table-mode engine without its radial MLP (the C ABI directly, Python uploads it on the first call)
    t = B200Engine(meta, arrays)
    t.set_graph(species, ei, ev)
    t.compute()
    out = torch.empty(len(pos), 9, dtype=torch.float64, device=t.device)
    with pytest.raises(RuntimeError, match='mlp0 of layer 0 is missing'):
        check(t.lib.s7b_engine_centroid_virial(t._h, out.data_ptr(), t._stream()))
    host = np.zeros((len(pos), 9))
    with pytest.raises(RuntimeError, match='mlp0 of layer 0 is missing'):
        check(t.lib.s7b_engine_centroid_virial_host(t._h, host.ctypes.data, t._stream()))


def test_host_variant_equals_device(si64):
    meta, arrays, species, pos, cell = si64
    e, Wc = engine_wc(meta, arrays, 'table', species, pos, cell, np.ones(3, bool))
    from sevenn_b200.engine import check
    host = np.zeros((len(pos), 9))
    check(e.lib.s7b_engine_centroid_virial_host(e._h, host.ctypes.data, e._stream()))
    err = np.abs(host.reshape(-1, 3, 3) - Wc).max() / np.abs(Wc).max()
    print(f'host variant vs device: {err:.1e}')
    assert err < 1e-5


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
    Wc = calc.get_centroid_virials(atoms)
    assert calc.engine.graph_stats() == stats, 'get_centroid_virials after a calculation on the same atoms ran a step'
    assert all(np.array_equal(before[k], calc.results[k]) for k in before)
    assert Wc.shape == (len(pos), 3, 3) and Wc.dtype == np.float64
    jpot = calc.get_heat_flux(atoms, convective=False)
    Jc = np.einsum('iab,ib->a', Wc, v.astype(np.float32).astype(np.float64))
    print(f'calculator: J_pot = {jpot}, sum Wc v = {Jc}')
    assert np.abs(jpot - Jc).max() < 1e-5 * np.abs(Wc * np.abs(v)[:, None, :]).sum()
    W2 = calc.get_centroid_virials(_Atoms(pos + 0.01, cell, z, v))
    assert calc.engine.graph_stats() != stats
    assert np.isfinite(W2).all()


def test_nothing_else_changes(si64):
    """compute, HVP and heat flux after a centroid pass match those before it, within the run-to-run difference of
    two computes (float atomics in the force scatter) or 1e-6 of the largest value, whichever is larger"""
    import torch
    from sevenn_b200.engine import B200Engine
    meta, arrays, species, pos, cell = si64
    e = B200Engine(meta, arrays, radial='table')
    e.set_positions(species, pos, cell, np.ones(3, bool))
    u = np.random.RandomState(14).normal(size=pos.shape)

    def run():
        e.compute()
        out = (e.buffer('energy', dtype='f8', shape=(1,)).clone(), e.buffer('forces', shape=(len(pos), 3)).clone())
        return out + (e.hvp(u), e.heat_flux(u)[0])

    a, b = run(), run()
    e.centroid_virial()
    c = run()
    for x, y, z_ in zip(a, b, c):
        run_to_run = (x - y).abs().max().item()
        bound = max(run_to_run, 1e-6 * x.abs().max().item())
        print(f'after a centroid pass: max diff {(x - z_).abs().max().item():.2e}, run to run {run_to_run:.2e}')
        assert (x - z_).abs().max().item() <= bound, 'a centroid pass changed a later compute, HVP or flux'
    torch.cuda.synchronize()


def test_lammps_heat_flux_of_cvatom_equals_the_engine_flux(tmp_path):
    """tests/mock_lammps_centroid/harness_centroid.cpp built with -DREAL_ENGINE: the serial pair style with an exported
    SevenNet-0 file on a 32-atom Si cluster; compute heat/flux's contraction sum_i cvatom_i v_i equals
    s7b_engine_heat_flux's J_pot for the same velocities.  The table-mode file carries the radial MLP
    (export_flat(..., radial_mlp=True)); without it the style refuses with a message naming the option."""
    import subprocess
    from helpers import ROOT
    from sevenn_b200.export import export_flat
    mock, ex = os.path.join(ROOT, 'tests', 'mock_lammps_centroid'), os.path.join(ROOT, 'examples', 'lammps')
    lib_dir = os.path.join(ROOT, 'sevenn_b200', 'lib')
    cuda = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    exe = str(tmp_path / 'harness_centroid_real')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-DREAL_ENGINE', '-I', mock, '-I', ex, '-I', os.path.join(cuda, 'include'),
                           os.path.join(mock, 'harness_centroid.cpp'), os.path.join(ex, 'pair_e3gnn_b200.cpp'), '-o', exe,
                           f'-L{lib_dir}', '-lsevenn_b200', f'-Wl,-rpath,{lib_dir}', f'-L{os.path.join(cuda, "lib64")}',
                           '-lcudart', f'-Wl,-rpath,{os.path.join(cuda, "lib64")}'])
    meta, arrays = model_weights('sevennet_0')
    model = str(tmp_path / 'sevennet_0.s7b')
    export_flat(model, meta, arrays, radial_mlp=True)
    p = subprocess.run([exe, model], capture_output=True, text=True, timeout=300)
    print(p.stdout)
    assert p.returncode == 0 and p.stdout.strip().endswith('OK'), p.stdout + p.stderr
