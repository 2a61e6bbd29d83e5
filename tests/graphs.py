"""Deterministic adversarial graphs for comparing the engine with the fp64 oracle (CPU only, numpy).

Each builder returns a ``Graph``: the first six fields are what the engine and the oracle consume
(species indices, edge_index [2, E] with [0] = centre, edge_vec [E, 3] = r_j - r_i + shift, volume, cell, pbc);
``positions`` and ``numbers`` are kept so that the device neighbour list can be run on the same system.
Every graph is built for a model's ``type_map`` (``meta``), and exists for one property the kernels have to
survive; tests/test_graph_fixtures_cpu.py asserts that property, so a fixture cannot silently lose it.

  dense         compressed fcc (256 atoms, a = 2.8 A): every row longer than 2 x 32 and 4 x 16 edges
  hub           one centre atom with 150-300 neighbours on shells next to isolated atoms (long and empty rows
                in the same warp)
  ragged        rows of 0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65 edges: every edge-record refill boundary
  isolated      atoms without edges at index 0, in the middle and last; odd n
  sizes_<n>     n-atom clusters of perturbed Si / NaCl / HfO2 across the 64-row, 128-row and 8-node tiles
  many_species  every species of the model, rattled
  radial_edges  edge lengths at the ends of the radial table: 0.2 and 0.35 A, a knot, and just below the cutoff
  tiny_cell     triclinic periodic cell smaller than the cutoff (many images of a pair, self images)
"""
from __future__ import annotations

import functools
from typing import NamedTuple

import numpy as np

from sevenn_b200.neighbors import diamond_si, neighbor_list_brute, rocksalt_nacl

CUTOFF = 5.0
RAGGED_LENGTHS = (0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65)
SIZES = (1, 2, 3, 7, 9, 63, 64, 65, 127, 129)
FIXTURES = ('dense', 'hub', 'ragged', 'isolated', 'many_species', 'radial_edges', 'tiny_cell') + \
    tuple(f'sizes_{n}' for n in SIZES)


class Graph(NamedTuple):
    species: np.ndarray        # [n] species indices of the model
    edge_index: np.ndarray     # [2, E] int64, sorted by centre
    edge_vec: np.ndarray       # [E, 3] float64
    volume: float              # 0 for a non-periodic system
    cell: np.ndarray           # [3, 3] (zeros when non-periodic)
    pbc: tuple
    positions: np.ndarray      # [n, 3]
    numbers: np.ndarray        # [n] atomic numbers


def _species(meta, numbers):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(z)] for z in numbers], dtype=np.int64)


def _graph(meta, pos, numbers, cell=None, pbc=False):
    pos = np.asarray(pos, dtype=np.float64)
    pbc3 = tuple(bool(b) for b in np.broadcast_to(np.asarray(pbc, dtype=bool), (3,)))
    c = np.zeros((3, 3)) if cell is None else np.asarray(cell, dtype=np.float64)
    ei, ev, _ = neighbor_list_brute(pos, c, pbc3, CUTOFF)
    vol = abs(np.linalg.det(c)) if all(pbc3) else 0.0
    return Graph(_species(meta, numbers), ei, ev, vol, c, pbc3, pos, np.asarray(numbers, dtype=np.int64))


def degrees(g: Graph) -> np.ndarray:
    return np.bincount(g.edge_index[0], minlength=len(g.species))


def dense(meta) -> Graph:
    fcc = np.array([[0, 0, 0], [0, .5, .5], [.5, 0, .5], [.5, .5, 0]])
    a, nc = 2.8, 4
    grid = np.stack(np.meshgrid(*[np.arange(nc)] * 3, indexing='ij'), -1).reshape(-1, 3)
    pos = ((grid[:, None, :] + fcc[None]) * a).reshape(-1, 3)
    pos = pos + np.random.RandomState(1).normal(scale=0.04, size=pos.shape)
    z = np.where(np.arange(len(pos)) % 3 == 0, 14, 6)          # SiC-like mix
    return _graph(meta, pos, z, np.eye(3) * a * nc, True)


def _shell_points(radius, n, rng):
    """n points on a sphere (golden-angle spiral), randomly rotated"""
    i = np.arange(n) + 0.5
    phi = np.arccos(1 - 2 * i / n)
    th = np.pi * (1 + 5 ** 0.5) * i
    p = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1) * radius
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    return p @ q


def hub(meta) -> Graph:
    """atom 0: an Hf hub with 166 H neighbours on shells of radius 2.2, 3.6 and 4.9 A (pair distances >= 1.3 A;
    heavier shell atoms this close drive the model to forces of 1e2 - 1e6 eV/A); atoms 1, 3 and the last:
    isolated, far away, so that the hub and an empty row share a warp"""
    rng = np.random.RandomState(7)
    shell = np.concatenate([_shell_points(r, n, rng) for r, n in ((2.2, 16), (3.6, 50), (4.9, 100))])
    far = np.array([[40.0, 0, 0], [0, 40.0, 0], [0, 0, 40.0]])
    pos = np.concatenate([[[0.0, 0, 0]], far[:1], shell[:1], far[1:2], shell[1:], far[2:]])
    z = np.full(len(pos), 1)
    z[0] = 72
    z[[1, 3, len(pos) - 1]] = 8
    return _graph(meta, pos, z)


def ragged(meta) -> Graph:
    """Rows cut from the full neighbour list of a dense periodic simple-cubic crystal (every atom has > 65
    neighbours) to the lengths of RAGGED_LENGTHS, in ascending, descending and alternating (0, 65, 1, 64, ...)
    order so that every length also sits next to very different ones.  Not symmetric: the engine and the
    oracle evaluate any directed graph."""
    a, nc = 1.6, 5
    grid = np.stack(np.meshgrid(*[np.arange(nc)] * 3, indexing='ij'), -1).reshape(-1, 3).astype(float)
    pos = grid * a + np.random.RandomState(3).normal(scale=0.05, size=grid.shape)
    cell = np.eye(3) * a * nc
    z = np.where(np.arange(len(pos)) % 2 == 0, 11, 17)
    full = _graph(meta, pos, z, cell, True)
    L = list(RAGGED_LENGTHS)
    alt = [v for pair in zip(L, L[::-1]) for v in pair]
    seq = L + L[::-1] + alt
    want = [seq[i % len(seq)] for i in range(len(pos))]
    rowptr = np.concatenate([[0], np.cumsum(degrees(full))])
    rng = np.random.RandomState(5)
    keep = []
    for i, m in enumerate(want):
        row = np.arange(rowptr[i], rowptr[i + 1])
        keep.append(np.sort(rng.choice(row, size=m, replace=False)))
    keep = np.concatenate(keep).astype(np.int64)
    return full._replace(edge_index=full.edge_index[:, keep], edge_vec=full.edge_vec[keep])


def isolated(meta) -> Graph:
    """a 20-atom HfO2 cluster plus three atoms far away, placed at index 0, in the middle and last (n = 23)"""
    pos, z = _fluorite_hfo2(2)
    c = pos.mean(0)
    order = np.argsort(np.linalg.norm(pos - c, axis=1), kind='stable')[:20]
    cl_pos, cl_z = pos[order], z[order]
    far = np.array([[-60.0, 0, 0], [0, -60.0, 0], [0, 0, -60.0]])
    n = 23
    slots = [0, n // 2, n - 1]
    P, Z = np.zeros((n, 3)), np.zeros(n, dtype=np.int64)
    rest = [i for i in range(n) if i not in slots]
    P[slots], Z[slots] = far, [8, 72, 8]
    P[rest], Z[rest] = cl_pos, cl_z
    return _graph(meta, P, Z)


def _fluorite_hfo2(nc, a=5.07, sigma=0.05, seed=0):
    fcc = np.array([[0, 0, 0], [0, .5, .5], [.5, 0, .5], [.5, .5, 0]])
    o = np.array([[x, y, zz] for x in (.25, .75) for y in (.25, .75) for zz in (.25, .75)])
    basis = np.concatenate([fcc, o])
    zb = np.array([72] * 4 + [8] * 8)
    grid = np.stack(np.meshgrid(*[np.arange(nc)] * 3, indexing='ij'), -1).reshape(-1, 3)
    pos = ((grid[:, None, :] + basis[None]) * a).reshape(-1, 3)
    pos = pos + np.random.RandomState(seed).normal(scale=sigma, size=pos.shape)
    return pos, np.tile(zb, len(grid))


def sizes(meta, n) -> Graph:
    """the n atoms nearest the centre of a perturbed Si, NaCl or HfO2 crystal (chosen by n), non-periodic"""
    k = SIZES.index(n) % 3
    if k == 0:
        pos, _, z = diamond_si(3, 3, 3, seed=n)
    elif k == 1:
        pos, _, z = rocksalt_nacl(3, 3, 3, seed=n)
    else:
        pos, z = _fluorite_hfo2(3, seed=n)
    c = pos.mean(0) + 0.1
    order = np.argsort(np.linalg.norm(pos - c, axis=1), kind='stable')[:n]
    return _graph(meta, pos[order], z[order])


def many_species(meta) -> Graph:
    """every atomic number of the model's type_map (plus random repeats) on a rattled 5 x 5 x 4 simple-cubic
    lattice, a = 2.5 A, periodic"""
    rng = np.random.RandomState(11)
    zs = np.array(sorted(int(k) for k in meta['type_map']))
    n = 100
    z = np.concatenate([zs, rng.choice(zs, size=n - len(zs))])
    rng.shuffle(z)
    grid = np.stack(np.meshgrid(np.arange(5), np.arange(5), np.arange(4), indexing='ij'), -1).reshape(-1, 3)
    a = 2.5
    pos = grid * a + rng.normal(scale=0.1, size=grid.shape)
    return _graph(meta, pos, z, np.diag([5 * a, 5 * a, 4 * a]), True)


def radial_targets(knots):
    """pair distances at the ends of the radial table (h = cutoff / knots, the engine's table spacing)"""
    h = CUTOFF / knots
    return np.array([0.2, 0.35, 1000 * h, CUTOFF - h / 2, CUTOFF - 1e-4, CUTOFF - 1e-6])


def radial_edges(meta) -> Graph:
    """one isolated dimer per target distance (both directions), dimers 30 A apart, random orientations.  The
    two short pairs are H-H (an Si-O pair at 0.2 A drives the models to 1e8 - 1e12 eV), the others Si-O."""
    from sevenn_b200.engine import default_table_knots
    from sevenn_b200.spec import build_spec
    rng = np.random.RandomState(13)
    pos, z = [], []
    for i, r in enumerate(radial_targets(default_table_knots(build_spec(meta)))):
        u = rng.normal(size=3)
        u /= np.linalg.norm(u)
        c = np.array([30.0 * i, 0, 0])
        pos += [c, c + r * u]
        z += [1, 1] if r < 1.0 else [14, 8]
    return _graph(meta, np.array(pos), z)


def tiny_cell(meta) -> Graph:
    """two atoms in a triclinic cell with all heights below the cutoff"""
    cell = np.array([[2.7, 0.0, 0.0], [0.8, 2.5, 0.0], [0.6, 0.9, 2.6]])
    pos = np.array([[0.1, 0.2, 0.05], [1.9, 1.5, 1.3]])
    return _graph(meta, pos, [14, 6], cell, True)


def build(name: str, meta) -> Graph:
    if name.startswith('sizes_'):
        return sizes(meta, int(name.split('_')[1]))
    return globals()[name](meta)


@functools.lru_cache(maxsize=None)
def fixture(name: str, model: str) -> Graph:
    """``build`` for one of the shipped models (cached)"""
    from helpers import model_weights
    meta, _ = model_weights(model)
    return build(name, meta)
