"""GPU parity tests (run on an H100 with `pytest -m gpu`): the CUDA engine, called through
the C ABI (ctypes), against (a) the reference's own golden vectors and (b) the fp64 CPU oracle
on the same inputs.

Tolerances (BASELINE.json north_star): energies within 1e-4 eV, forces within 1e-3 eV/A.  The
tests use much tighter bounds where fp32 allows: 2e-5 eV on small-cell energies, 5e-5 eV/A on forces.
"""
import numpy as np
import pytest

from helpers import golden_vectors, model_weights, oracle, species_of, system_graph

pytestmark = pytest.mark.gpu

E_TOL, F_TOL = 2e-5, 5e-5


@pytest.fixture(scope='module')
def engines():
    from sevenn_b200.engine import B200Engine
    cache = {}

    def get(name, radial):
        key = (name, radial)
        if key not in cache:
            meta, arrays = model_weights(name)
            cache[key] = B200Engine(meta, arrays, radial=radial)
        return cache[key]
    return get


def run_engine(e, species, ei, ev):
    import torch
    e.set_graph(species, ei, ev)
    e.compute()
    torch.cuda.synchronize()
    r = e.results()
    return dict(energy=float(r['energy'].cpu()[0]), atomic_energy=r['atomic_energy'].cpu().numpy(),
                forces=r['forces'].cpu().numpy(), virial=r['virial'].cpu().numpy(),
                edge_force=r['edge_force'].cpu().numpy(), perm=e._graph['perm'])


@pytest.mark.parametrize('case', sorted(golden_vectors().keys()))
@pytest.mark.parametrize('radial', ['table', 'mlp'])
def test_reference_golden_vectors(engines, case, radial):
    g = golden_vectors()[case]
    meta, _ = model_weights(g['model'])
    e = engines(g['model'], radial)
    ei, ev, vol = system_graph(g['system'], e.spec.cutoff)
    sp = species_of(meta, g['system']['numbers'])
    out = run_engine(e, sp, ei, ev)
    ref = oracle(g['model']).forward(sp, ei, ev, volume=vol)
    # (a) the reference's golden numbers, with the reference's own tolerances (floored at fp32 noise)
    tol = g['atol']
    assert abs(out['energy'] - g['energy']) <= max(tol['energy'], 2e-5)
    assert np.allclose(out['forces'], g['forces'], atol=max(tol['forces'], 3e-5), rtol=0)
    if 'energies' in g:
        assert np.allclose(out['atomic_energy'], g['energies'], atol=max(tol['energies'], 1e-5), rtol=0)
    if 'inferred_stress' in g:
        assert np.allclose(out['virial'] / vol, g['inferred_stress'], atol=max(tol['stress'], 1e-5), rtol=0)
    if 'ase_stress' in g:
        assert np.allclose(-(out['virial'] / vol)[[0, 1, 2, 4, 5, 3]], g['ase_stress'], atol=max(tol['stress'], 1e-5), rtol=0)
    # (b) the fp64 oracle on the same graph
    assert abs(out['energy'] - float(ref['energy'])) <= E_TOL
    assert np.allclose(out['atomic_energy'], ref['atomic_energy'].numpy(), atol=E_TOL, rtol=0)
    assert np.allclose(out['forces'], ref['forces'].numpy(), atol=F_TOL, rtol=0)
    assert np.allclose(out['virial'], ref['virial'].numpy(), atol=2e-4, rtol=1e-5)


@pytest.mark.parametrize('name', ['sevennet_0', 'sevennet_l3i5'])
@pytest.mark.parametrize('radial', ['table', 'mlp'])
def test_si64_against_oracle(engines, name, radial):
    """BASELINE.json configs[0]: 64-atom Si cell, energy+force vs the reference path."""
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, z = diamond_si(2, 2, 2)
    ei, ev = build_graph(pos, cell, True, 5.0)
    meta, _ = model_weights(name)
    sp = species_of(meta, z)
    out = run_engine(engines(name, radial), sp, ei, ev)
    ref = oracle(name).forward(sp, ei, ev, volume=abs(np.linalg.det(cell)))
    assert abs(out['energy'] - float(ref['energy'])) <= 1e-4
    assert np.allclose(out['atomic_energy'], ref['atomic_energy'].numpy(), atol=E_TOL, rtol=0)
    assert np.allclose(out['forces'], ref['forces'].numpy(), atol=F_TOL, rtol=0)
    want_fe = ref['edge_force'].numpy()
    if out['perm'] is not None:
        want_fe = want_fe[out['perm'].cpu().numpy()]
    assert np.allclose(out['edge_force'], want_fe, atol=2e-5, rtol=0)
    assert np.allclose(out['virial'], ref['virial'].numpy(), atol=5e-4, rtol=1e-5)


def test_table_and_exact_mlp_radial_agree(engines):
    """The cubic-spline radial tables reproduce the exact per-edge MLP to fp32 noise."""
    from sevenn_b200.neighbors import build_graph, rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.1, seed=3)
    ei, ev = build_graph(pos, cell, True, 5.0)
    meta, _ = model_weights('sevennet_0')
    sp = species_of(meta, z)
    a = run_engine(engines('sevennet_0', 'table'), sp, ei, ev)
    b = run_engine(engines('sevennet_0', 'mlp'), sp, ei, ev)
    assert abs(a['energy'] - b['energy']) < 2e-5
    assert np.allclose(a['forces'], b['forces'], atol=2e-5, rtol=0)


def test_host_buffer_entry_matches_device_entry(engines):
    """s7b_engine_compute_host (H2D + compute + D2H) == set_graph/compute on device tensors."""
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, z = diamond_si(2, 2, 3, seed=5)
    ei, ev = build_graph(pos, cell, True, 5.0)
    meta, _ = model_weights('sevennet_0')
    sp = species_of(meta, z)
    e = engines('sevennet_0', 'table')
    a = run_engine(e, sp, ei, ev)
    energy, ae, forces, virial = e.compute_host(sp, ei[0], ei[1], ev)
    assert abs(energy - a['energy']) < 1e-6
    assert np.allclose(ae, a['atomic_energy'], atol=1e-6)
    assert np.allclose(forces, a['forces'], atol=2e-6)      # RED.ADD order differs between runs
    assert np.allclose(virial, a['virial'], atol=1e-5)


def test_host_entry_rejects_unsorted_edges(engines):
    e = engines('sevennet_0', 'table')
    sp = np.zeros(3, np.int32)
    with pytest.raises(RuntimeError, match='sorted by centre'):
        e.compute_host(sp, np.array([1, 0]), np.array([0, 1]), np.ones((2, 3), np.float32))
    with pytest.raises(RuntimeError, match='out of range'):
        e.compute_host(sp, np.array([0, 1]), np.array([1, 7]), np.ones((2, 3), np.float32))


def test_full_size_properties_12k_atoms(engines):
    """BASELINE.json configs[1] size (12 000 atoms, 336 000 edges): size-independent properties.
    * net force vanishes (Newton's third law of the edge-force scatter)
    * replicating a perturbed 64-atom cell 5x5x... is not available, so periodic extensivity is
      checked on a replicated 3x3x3 block instead (same local environments -> same energies)
    * a deterministic checksum: atomic energies sum to the total energy."""
    from sevenn_b200.neighbors import build_graph, diamond_si
    meta, _ = model_weights('sevennet_0')
    e = engines('sevennet_0', 'table')
    pos, cell, z = diamond_si(10, 10, 15)
    ei, ev = build_graph(pos, cell, True, 5.0)
    assert len(pos) == 12000 and ei.shape[1] == 336000
    out = run_engine(e, species_of(meta, z), ei, ev)
    assert np.abs(out['forces'].sum(0)).max() < 2e-3
    assert abs(out['atomic_energy'].astype(np.float64).sum() - out['energy']) < 1e-6 * 12000
    assert np.isfinite(out['forces']).all()
    # extensivity: tile the perturbed 64-atom cell 2x2x2 -> identical environments, 8x the energy
    p1, c1, z1 = diamond_si(2, 2, 2)
    shifts = np.array([[i, j, k] for i in range(2) for j in range(2) for k in range(2)], dtype=float)
    p8 = np.concatenate([p1 + s @ c1 for s in shifts])
    z8 = np.tile(z1, 8)
    ei1, ev1 = build_graph(p1, c1, True, 5.0)
    ei8, ev8 = build_graph(p8, 2 * c1, True, 5.0)
    o1 = run_engine(e, species_of(meta, z1), ei1, ev1)
    o8 = run_engine(e, species_of(meta, z8), ei8, ev8)
    assert abs(o8['energy'] - 8 * o1['energy']) < 2e-4
    assert np.allclose(o8['forces'][:64], o1['forces'], atol=2e-5)


def test_forces_are_energy_gradient_finite_difference(engines):
    """dE/dx by central differences of the engine's own energy (fp64 accumulated) vs its forces."""
    from sevenn_b200.neighbors import build_graph, rocksalt_nacl
    meta, _ = model_weights('sevennet_0')
    e = engines('sevennet_0', 'table')
    pos, cell, z = rocksalt_nacl(1, 1, 1, sigma=0.08, seed=11)
    sp = species_of(meta, z)
    ei, ev = build_graph(pos, cell, True, 5.0)
    f = run_engine(e, sp, ei, ev)['forces']
    h = 2e-3
    for (i, c) in [(0, 0), (3, 1), (5, 2)]:
        ep = []
        for s in (+1, -1):
            p = pos.copy()
            p[i, c] += s * h
            ei2, ev2 = build_graph(p, cell, True, 5.0)
            ep.append(run_engine(e, sp, ei2, ev2)['energy'])
        fd = -(ep[0] - ep[1]) / (2 * h)
        assert abs(fd - f[i, c]) < 5e-3, (i, c, fd, f[i, c])


def test_calculator_surface(engines):
    """SevenNetCalculator-compatible results on the reference's rattled NaCl case
    (tests/unit_tests/test_calculator.py:56-84)."""
    from sevenn_b200.calculator import SevenNetCalculator
    g = golden_vectors()['7net0_nacl_rattled']

    class Atoms:
        def __init__(s, sysd):
            s.sysd = sysd
        def get_positions(s): return np.array(s.sysd['positions'])
        def get_cell(s): return np.array(s.sysd['cell'])
        def get_pbc(s): return np.array([True] * 3)
        def get_atomic_numbers(s): return np.array(s.sysd['numbers'])

    calc = SevenNetCalculator('7net-0', device='cuda')
    res = calc.calculate(Atoms(g['system']))
    assert abs(res['energy'] - g['energy']) < 2e-5 and res['free_energy'] == res['energy']
    assert np.allclose(res['forces'], g['forces'], atol=3e-5)
    assert np.allclose(res['energies'], g['energies'], atol=1e-5)
    assert np.allclose(res['stress'], g['ase_stress'], atol=1e-5)
    assert res['num_edges'] == 58


def test_atomic_virial_matches_oracle():
    """compute_atomic_virial=True: 'stresses' = per-atom virial (force_output.py:198-214), and it sums to
    the total virial."""
    from sevenn_b200.calculator import SevenNetCalculator
    g = golden_vectors()['7net0_hfo2_0']

    class Atoms:
        def get_positions(s): return np.array(g['system']['positions'])
        def get_cell(s): return np.array(g['system']['cell'])
        def get_pbc(s): return np.array([True] * 3)
        def get_atomic_numbers(s): return np.array(g['system']['numbers'])

    calc = SevenNetCalculator('7net-0', device='cuda', compute_atomic_virial=True)
    res = calc.calculate(Atoms())
    meta, _ = model_weights('sevennet_0')
    ei, ev, vol = system_graph(g['system'], 5.0)
    ref = oracle('sevennet_0').forward(species_of(meta, g['system']['numbers']), ei, ev, volume=vol)
    assert np.allclose(res['stresses'], ref['atomic_virial'].numpy(), atol=5e-5)
    assert np.allclose(res['stresses'].sum(0) / vol, -res['stress'][[0, 1, 2, 5, 3, 4]], atol=1e-6)
    assert np.allclose(res['energies'], g['energies'], atol=2e-5) and np.allclose(res['forces'], g['forces'], atol=3e-5)
