"""Device neighbour list (csrc/neighbor.cuh) vs the numpy builders (which restate the reference's
matscipy/ASE semantics and are themselves pinned on the CPU to the edge counts the reference's tests hold and to a
direct enumeration of the definition, tests/test_host_logic.py): identical directed edge multisets, for large / tiny / triclinic / non-periodic
/ slab systems; and the positions-in entry point vs the graph-in entry point."""
import numpy as np
import pytest

from helpers import golden_vectors, model_weights, species_of

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def eng():
    from sevenn_b200.engine import B200Engine
    meta, arrays = model_weights('sevennet_0')
    return B200Engine(meta, arrays)


def _canonical(dst, src, vec):
    """edges sorted by (centre, neighbour, coarse vector) -> arrays that can be compared with a tolerance"""
    vec = np.asarray(vec, dtype=np.float64)
    q = np.rint(vec * 20).astype(np.int64)                 # 0.05 A buckets only order images of one pair
    o = np.lexsort((q[:, 2], q[:, 1], q[:, 0], src, dst))
    return np.asarray(dst)[o], np.asarray(src)[o], vec[o]


def _check(eng, pos, cell, pbc, z):
    from sevenn_b200.neighbors import neighbor_list_brute, neighbor_list_cells
    meta, _ = model_weights('sevennet_0')
    sp = species_of(meta, z)
    eng.set_positions(sp, pos, cell, pbc)
    rowptr, src, vec = (t.cpu().numpy() for t in eng.graph_arrays())
    pb = np.broadcast_to(np.asarray(pbc, dtype=bool), (3,))
    if len(pos) > 400 and pb.all():
        ei, ev = neighbor_list_cells(pos, cell, 5.0)
    else:
        c = np.zeros((3, 3)) if cell is None else np.asarray(cell, dtype=float)
        ei, ev, _ = neighbor_list_brute(pos, c, pb, 5.0)
    assert len(src) == ei.shape[1]
    assert (np.diff(rowptr) >= 0).all() and rowptr[-1] == len(src)
    dst = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
    d1, s1, v1 = _canonical(dst, src, vec)
    d2, s2, v2 = _canonical(ei[0], ei[1], ev)
    assert (d1 == d2).all() and (s1 == s2).all()
    assert np.allclose(v1, v2, atol=2e-6)                   # device: double differences stored as float
    return sp


def test_nl_large_orthorhombic(eng):
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(6, 5, 4, seed=3)
    _check(eng, pos, cell, True, z)


def test_nl_positions_outside_cell_are_wrapped(eng):
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(3, 3, 3, seed=1)
    shift = np.random.RandomState(0).randint(-2, 3, size=(len(pos), 3)).astype(float) @ cell
    from sevenn_b200.neighbors import neighbor_list_brute
    meta, _ = model_weights('sevennet_0')
    eng.set_positions(species_of(meta, z), pos + shift, cell, True)
    n_shifted = eng.n_edges
    eng.set_positions(species_of(meta, z), pos, cell, True)
    assert eng.n_edges == n_shifted == 216 * 28


@pytest.mark.parametrize('case', ['7net0_nacl', '7net0_hfo2_0', '7net0_h2o', '7net0_three_o', '7net0_single_o'])
def test_nl_golden_systems(eng, case):
    g = golden_vectors()[case]['system']
    _check(eng, np.array(g['positions'], dtype=float), g['cell'], bool(g['pbc']), g['numbers'])


def test_nl_slab_mixed_pbc(eng):
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 1, sigma=0.05, seed=2)
    cell = cell.copy()
    cell[2, 2] = 30.0                      # vacuum, non-periodic along c
    _check(eng, pos, cell, [True, True, False], z)


def test_positions_entry_matches_graph_entry(eng):
    import torch
    from sevenn_b200.neighbors import build_graph, rocksalt_nacl
    meta, _ = model_weights('sevennet_0')
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.08, seed=5)
    sp = species_of(meta, z)
    energy, ae, forces, virial, n_edges = eng.compute_positions(sp, pos, cell, True)
    ei, ev = build_graph(pos, cell, True, 5.0)
    eng.set_graph(sp, ei, ev)
    eng.compute()
    torch.cuda.synchronize()
    r = eng.results()
    assert n_edges == ei.shape[1]
    assert abs(energy - float(r['energy'].cpu()[0])) < 2e-5      # different neighbour order within rows
    assert np.allclose(forces, r['forces'].cpu().numpy(), atol=2e-5)
    assert np.allclose(virial, r['virial'].cpu().numpy(), atol=2e-4)


@pytest.mark.parametrize('fixture', ['dense', 'tiny_cell', 'many_species'])
def test_nl_adversarial_fixtures(eng, fixture):
    """rows of 85 neighbours (dense), a triclinic cell smaller than the cutoff (tiny_cell: many images of a
    pair and of the atom itself), every species (tests/graphs.py)"""
    import graphs
    g = graphs.fixture(fixture, 'sevennet_0')
    _check(eng, g.positions, g.cell, g.pbc, g.numbers)
