"""Deterministic D3 test systems for comparing the D3 kernels with the fp64 oracle (CPU only, numpy).

Each builder returns ``(numbers, positions [n,3] A, cell rows [3,3] A, pbc)`` from a fixed seed and keeps every
pair of atoms (all periodic images included) at least ``MIN_DIST`` apart, so that no result rests on an
accidental r -> 0.  Every system exists for one property the kernels have to survive at the default cutoffs
(9000 / 1600 bohr^2); tests/test_d3_cells_cpu.py asserts that property, so a fixture cannot silently lose it.

  sheared        strongly sheared triclinic cell (one obtuse angle), >= 2 cell-list bins in every direction,
                 atoms given outside [0,1) in fractional coordinates and some exactly on cell faces
  rotated        ``sheared`` under a generic rotation: the cell is not in the LAMMPS (lower-triangular) frame
  slab           pbc (T,T,F); the non-periodic extent spans 4 bins
  wire           pbc (T,F,F); the non-periodic extents span 3 bins each
  compressed_cs  8 Cs + 3 H + He in a 5.75 A cell: reference-weight sums D < 1e-300 (one-hot fallback),
                 1e-300 < D < 1e-99, and atom pairs on both sides of D_i D_j = 1e-99, none near a threshold
  species16      16 elements: H, heavy elements, and every count 1..5 of C6 reference points (mxc)
  nacl_large     4 800-atom rocksalt NaCl (atom-range splits only; too large for the oracle)
  molecule       cell-less organic-like cluster with negative coordinates, pbc (F,F,F)

``LAMMPS_FRAME`` lists the systems whose cell rows are lower-triangular, which the reference's compiled D3
accepts as they are (tools/make_d3_golden.py).
"""
from __future__ import annotations

import functools

import numpy as np

from sevenn_b200.neighbors import rocksalt_nacl

MIN_DIST = 1.0            # A, every fixture
ORACLE_FIXTURES = ('sheared', 'rotated', 'slab', 'wire', 'compressed_cs', 'species16')
LAMMPS_FRAME = ('sheared', 'slab', 'compressed_cs', 'species16')
SPECIES16 = (1, 2, 6, 7, 8, 11, 14, 16, 26, 29, 35, 50, 54, 74, 82, 83)
AU_TO_ANG = 0.52917726
# (fixture, damping, functional) stored from the reference's compiled D3 by tools/make_d3_golden.py.  bpbe / bmk
# hold the largest s18 (bmk also the largest zero-damping rs6), ssb the smallest BJ s18 and rs6,
# slater-dirac-exchange the smallest zero-damping s18 and rs18, pwb6k the largest BJ rs18, o-lyp the smallest
# zero-damping rs6, wb97m the largest BJ rs6 and b2gp-plyp the smallest zero-damping s6.
GOLDEN_CASES = (('sheared', 'damp_bj', 'bpbe'), ('sheared', 'damp_zero', 'bmk'),
                ('slab', 'damp_bj', 'ssb'), ('slab', 'damp_zero', 'slater-dirac-exchange'),
                ('compressed_cs', 'damp_bj', 'pwb6k'), ('compressed_cs', 'damp_zero', 'o-lyp'),
                ('species16', 'damp_bj', 'wb97m'), ('species16', 'damp_zero', 'b2gp-plyp'))


def golden_key(fixture, damping, functional):
    return f'{fixture}_{damping}_{functional}'


def _images(cell, pbc, reach=2):
    rng = [np.arange(-reach, reach + 1) if p else np.zeros(1, dtype=int) for p in pbc]
    g = np.stack(np.meshgrid(*rng, indexing='ij'), -1).reshape(-1, 3)
    return g @ np.asarray(cell, dtype=np.float64)


def min_distance(positions, cell, pbc, reach=2):
    """Shortest distance between two atoms, or an atom and another image of itself (images up to +-reach cells)."""
    pos = np.asarray(positions, dtype=np.float64)
    tau = _images(cell, pbc, reach)
    best = np.inf
    for i in range(len(pos)):
        d = pos[None, :, :] - pos[i] + tau[:, None, :]
        r = np.sqrt((d ** 2).sum(-1))
        r[np.all(tau == 0, axis=1), i] = np.inf
        best = min(best, r.min())
    return best


def _place(rng, n, cell, pbc, sample, dmin, first=()):
    """``first`` and then points from sample(rng), each kept only if it is >= dmin from all earlier ones and their
    images, up to n points."""
    tau = _images(cell, pbc)
    pts = list(first)
    while len(pts) < n:
        p = sample(rng)
        if pts:
            d = np.asarray(pts)[None, :, :] - p + tau[:, None, :]
            if (d ** 2).sum(-1).min() < dmin * dmin:
                continue
        if any(pbc) and np.sqrt((tau[np.any(tau != 0, axis=1)] ** 2).sum(-1)).min() < dmin:
            raise ValueError('cell shorter than the minimum distance')
        pts.append(p)
    return np.asarray(pts)


SHEARED_CELL = np.array([[15.0, 0.0, 0.0], [-8.0, 13.0, 0.0], [5.0, -4.0, 13.0]])


@functools.lru_cache(maxsize=None)
def _sheared():
    rng = np.random.RandomState(101)
    cell = SHEARED_CELL
    faces = np.array([[0.0, 0.3, 0.7], [0.5, 1.0, 0.2], [0.25, 0.6, 0.0], [1.0, 0.0, 1.0]]) @ cell   # faces, a corner
    frac = _place(rng, 100, cell, (True,) * 3, lambda r: r.uniform(0, 1, 3) @ cell, 1.6, faces) @ np.linalg.inv(cell)
    frac += rng.randint(-2, 3, size=frac.shape)                      # given outside [0,1): wrapping is exercised
    z = rng.choice([1, 6, 8, 14, 29], size=len(frac))
    return z, frac @ cell, cell, (True, True, True)


def sheared():
    z, pos, cell, pbc = _sheared()
    return z.copy(), pos.copy(), cell.copy(), pbc


def rotation():
    """A generic proper rotation (fixed seed)."""
    q, r = np.linalg.qr(np.random.RandomState(0).normal(size=(3, 3)))
    q = q * np.sign(np.diag(r))[None, :]
    return q if np.linalg.det(q) > 0 else -q


def rotated():
    z, pos, cell, pbc = sheared()
    R = rotation()
    return z, pos @ R.T, cell @ R.T, pbc


def slab():
    rng = np.random.RandomState(202)
    cell = np.array([[13.0, 0.0, 0.0], [3.0, 12.5, 0.0], [0.0, 0.0, 26.0]])
    pbc = (True, True, False)
    pos = _place(rng, 110, cell, pbc, lambda r: r.uniform(0, 1, 3) * [1, 1, 0] @ cell + [0, 0, r.uniform(3.0, 23.0)], 1.7)
    pos[:, :2] += rng.randint(-1, 2, size=(len(pos), 1)) * cell[0, :2]         # outside the cell in x only
    z = rng.choice([8, 13, 14, 1], size=len(pos))
    return z, pos, cell, pbc


def wire():
    rng = np.random.RandomState(303)
    cell = np.diag([12.6, 21.0, 21.0])
    pbc = (True, False, False)

    def sample(r):
        while True:
            yz = r.uniform(-7.5, 7.5, 2)
            if (yz ** 2).sum() < 7.5 ** 2:
                return np.array([r.uniform(-12.6, 25.2), 10.5 + yz[0], 10.5 + yz[1]])
    pos = _place(rng, 90, cell, pbc, sample, 1.6)
    z = rng.choice([6, 1, 7, 16], size=len(pos))
    return z, pos, cell, pbc


def compressed_cs():
    rng = np.random.RandomState(5)
    cell = np.array([[5.75, 0.0, 0.0], [0.4, 5.75, 0.0], [-0.3, 0.5, 5.75]])
    z = np.array([55] * 8 + [1] * 3 + [2])
    pos = _place(rng, len(z), cell, (True,) * 3, lambda r: r.uniform(0, 1, 3) @ cell, 1.25)
    return z, pos, cell, (True, True, True)


def species16():
    rng = np.random.RandomState(404)
    cell = np.array([[11.0, 0.0, 0.0], [2.0, 10.5, 0.0], [-1.5, 1.0, 11.5]])
    z = np.repeat(np.array(SPECIES16), 4)
    rng.shuffle(z)
    pos = _place(rng, len(z), cell, (True,) * 3, lambda r: r.uniform(0, 1, 3) @ cell, 2.0)
    return z, pos, cell, (True, True, True)


def nacl_large():
    pos, cell, z = rocksalt_nacl(10, 10, 6, sigma=0.05, seed=5)
    return z, pos, cell, (True, True, True)


def molecule():
    """No cell: D3Calculator generates one.  Centred on the origin, so about half the coordinates are negative."""
    rng = np.random.RandomState(505)

    def sample(r):
        while True:
            p = r.uniform(-4.5, 4.5, 3)
            if (p ** 2).sum() < 4.5 ** 2:
                return p
    pos = _place(rng, 30, np.zeros((3, 3)), (False,) * 3, sample, 1.1)
    z = rng.choice([1, 6, 7, 8], size=len(pos))
    return z, pos, np.zeros((3, 3)), (False, False, False)


FIXTURES = dict(sheared=sheared, rotated=rotated, slab=slab, wire=wire, compressed_cs=compressed_cs,
                species16=species16, nacl_large=nacl_large, molecule=molecule)


# ---- restated host and oracle rules the CPU test checks the fixtures against ------------------------
def cell_list_bins(cell):
    """Bins per direction as ``s7b_d3_set_system`` (csrc/d3.cu) picks them: floor(height / 6 A), 1..128,
    height = distance between the lattice planes spanned by the other two vectors."""
    inv = np.linalg.inv(np.asarray(cell, dtype=np.float64) / AU_TO_ANG)
    height = 1.0 / np.sqrt((inv ** 2).sum(0))
    return np.clip(np.floor(height / (6.0 / AU_TO_ANG)).astype(int), 1, 128)


def log_weight_sums(numbers, cn):
    """ln D_i, D_i = sum_a exp(K3 (CN_ref[a] - CN_i)^2) over the atom's mxc references, from the oracle's
    (float-rounded) coordination numbers with the oracle's arithmetic, evaluated in log space so that sums far
    below the double range stay finite."""
    from oracle.d3_oracle import K3, d3_params
    P = d3_params()
    zz = np.asarray(numbers, dtype=np.int64) - 1
    cnr = P['cnref'][zz].astype(np.float32).astype(np.float64)
    valid = np.arange(5)[None, :] < P['mxc'][zz][:, None]
    e = np.where(valid, K3 * ((cnr - np.asarray(cn)[:, None]) ** 2).astype(np.float32).astype(np.float64), -np.inf)
    m = e.max(1)
    return m + np.log(np.exp(e - m[:, None]).sum(1))
