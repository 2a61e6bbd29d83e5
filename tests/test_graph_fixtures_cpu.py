"""The adversarial graphs of tests/graphs.py have the property each of them exists for (CPU only): if a builder
changes, the GPU comparisons in test_adversarial_graphs_gpu.py, test_conv_op_gpu.py and test_neighbor_gpu.py
must not quietly stop reaching the kernel branch they were written for."""
import numpy as np
import pytest

import graphs
from helpers import model_weights

MODELS = ['sevennet_0', 'sevennet_l3i5']


def _check_common(g):
    n, E = len(g.species), g.edge_index.shape[1]
    assert g.edge_index.shape == (2, E) and g.edge_vec.shape == (E, 3)
    if E:
        assert (np.diff(g.edge_index[0]) >= 0).all()                     # sorted by centre
        assert g.edge_index.min() >= 0 and g.edge_index.max() < n
        r = np.linalg.norm(g.edge_vec, axis=1)
        assert r.max() < graphs.CUTOFF and r.min() > 0.0
        # edge_vec = r_j - r_i + shift, the shift a lattice vector of the cell (zero when not periodic)
        d = g.edge_vec - (g.positions[g.edge_index[1]] - g.positions[g.edge_index[0]])
        if any(g.pbc):
            s = d @ np.linalg.inv(g.cell)
            assert np.allclose(s, np.rint(s), atol=1e-9)
        else:
            assert np.abs(d).max() < 1e-12


@pytest.mark.parametrize('name', graphs.FIXTURES)
def test_fixture_is_a_valid_graph(name):
    g = graphs.fixture(name, 'sevennet_0')
    _check_common(g)
    assert g.species.shape == g.numbers.shape == (len(g.positions),)


def test_dense_rows_are_longer_than_two_record_fetches():
    d = graphs.degrees(graphs.fixture('dense', 'sevennet_0'))
    assert d.min() >= 75 and len(d) == 256


def test_hub_has_a_long_row_next_to_empty_rows():
    g = graphs.fixture('hub', 'sevennet_0')
    d = graphs.degrees(g)
    assert d[0] >= 150 and 150 <= d.max() <= 300
    assert d[1] == 0 and d[3] == 0 and d[-1] == 0                  # node 1 shares a 2-node warp with the hub
    r = np.linalg.norm(g.positions[1:][d[1:] > 0], axis=1)
    assert r.min() >= 1.0 and r.max() <= 4.95
    p = g.positions[d > 0]
    pair = np.linalg.norm(p[:, None] - p[None], axis=-1) + np.eye(len(p)) * 9
    assert pair.min() >= 0.8


def test_ragged_hits_every_refill_boundary_also_in_adjacent_nodes():
    d = graphs.degrees(graphs.fixture('ragged', 'sevennet_0'))
    for m in graphs.RAGGED_LENGTHS:
        assert (d == m).any(), m
    adj = set(zip(d[:-1].tolist(), d[1:].tolist()))
    assert (0, 65) in adj and (65, 0) in adj and (1, 64) in adj and (16, 17) in adj and (32, 33) in adj
    # both 16-lane halves of a warp: an even node followed by an odd one with a very different length
    pairs = {(int(d[i]), int(d[i + 1])) for i in range(0, len(d) - 1, 2)}
    assert any(a == 0 and b >= 64 for a, b in pairs) and any(a >= 64 and b == 0 for a, b in pairs)


def test_isolated_atoms_at_start_middle_and_end():
    d = graphs.degrees(graphs.fixture('isolated', 'sevennet_0'))
    n = len(d)
    assert n % 2 == 1
    assert d[0] == 0 and d[n // 2] == 0 and d[-1] == 0
    assert (d > 0).sum() == n - 3


@pytest.mark.parametrize('n', graphs.SIZES)
def test_sizes(n):
    g = graphs.fixture(f'sizes_{n}', 'sevennet_0')
    assert len(g.species) == n
    if n > 1:
        assert graphs.degrees(g).max() > 0


@pytest.mark.parametrize('model', MODELS)
def test_many_species_covers_every_species(model):
    meta, _ = model_weights(model)
    g = graphs.fixture('many_species', model)
    from sevenn_b200.spec import build_spec
    assert set(g.species.tolist()) == set(range(build_spec(meta).num_species))


@pytest.mark.parametrize('model', MODELS)
def test_radial_edges_reach_the_ends_of_the_table(model):
    from sevenn_b200.engine import default_table_knots
    from sevenn_b200.spec import build_spec
    meta, _ = model_weights(model)
    knots = default_table_knots(build_spec(meta))
    g = graphs.fixture('radial_edges', model)
    r = np.linalg.norm(g.edge_vec, axis=1)
    for t in graphs.radial_targets(knots):
        assert np.abs(r - t).min() < 1e-9, t
    r32 = np.linalg.norm(g.edge_vec.astype(np.float32), axis=1)          # what the engine sees
    assert r.max() < graphs.CUTOFF and r32.max() < np.float32(graphs.CUTOFF)
    h = graphs.CUTOFF / knots
    assert (r32 > graphs.CUTOFF - h).sum() >= 6                         # the last table interval, 3 pairs
    assert (r < 2 * h).sum() == 0 and (r < 0.4).sum() == 4               # first intervals: 0.2 and 0.35 A


def test_tiny_cell_sees_periodic_images():
    g = graphs.fixture('tiny_cell', 'sevennet_0')
    heights = abs(np.linalg.det(g.cell)) / np.linalg.norm(np.cross(g.cell[[1, 2, 0]], g.cell[[2, 0, 1]]), axis=1)
    assert heights.max() < graphs.CUTOFF and all(g.pbc)
    i, j = g.edge_index
    assert ((i == 0) & (j == 1)).sum() >= 3                             # one pair in several images
    assert ((i == 0) & (j == 0)).sum() >= 2 and ((i == 1) & (j == 1)).sum() >= 2    # own images
