"""Each D3 test system of tests/d3_cells.py keeps the property it exists for (CPU only)."""
import numpy as np
import pytest

import d3_cells as C


@pytest.mark.parametrize('fixture', sorted(C.FIXTURES))
def test_deterministic_and_minimum_distance(fixture):
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    z2, pos2, cell2, pbc2 = C.FIXTURES[fixture]()
    assert np.array_equal(z, z2) and np.array_equal(pos, pos2) and np.array_equal(cell, cell2) and pbc == pbc2
    assert len(z) == len(pos) and pos.shape[1] == 3 and len(pbc) == 3
    # nacl_large: a 56 x 56 x 34 A cell, images beyond the first shell are far
    reach = 1 if fixture == 'nacl_large' else 2
    assert C.min_distance(pos, cell, pbc, reach) >= C.MIN_DIST


def _frac(pos, cell):
    return pos @ np.linalg.inv(cell)


def _angles(cell):
    a, b, c = cell
    cos = lambda u, v: np.dot(u, v) / np.linalg.norm(u) / np.linalg.norm(v)  # noqa: E731
    return np.degrees(np.arccos([cos(b, c), cos(a, c), cos(a, b)]))


def test_sheared():
    z, pos, cell, pbc = C.sheared()
    assert 80 <= len(z) <= 150 and all(pbc)
    ang = _angles(cell)
    assert (ang > 90.0).sum() >= 1 and np.abs(ang - 90.0).max() > 25.0          # strongly sheared, one angle obtuse
    # the bin rule of s7b_d3_set_system, restated: >= 2 bins per direction means the sweep's image shifts
    # s0..s2 at q < 0 and q >= nb are taken inside the cell list, not only across a one-bin cell
    assert (C.cell_list_bins(cell) >= 2).all()
    f = _frac(pos, cell)
    assert ((f < 0) | (f >= 1)).any(axis=1).mean() > 0.5                          # most atoms are given outside
    assert (np.abs(f - np.round(f)) < 1e-12).any(axis=1).sum() >= 4                # and some on cell faces


def test_rotated():
    z0, pos0, cell0, _ = C.sheared()
    z, pos, cell, pbc = C.rotated()
    R = C.rotation()
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-14) and np.linalg.det(R) > 0
    assert np.abs(R).min() > 0.15 and np.abs(R).max() < 0.9                       # generic: no axis or plane kept
    assert np.abs(np.triu(cell, 1)).max() > 1.0                                    # not the LAMMPS frame
    assert np.array_equal(z, z0) and np.allclose(pos, pos0 @ R.T) and np.allclose(cell, cell0 @ R.T)


@pytest.mark.parametrize('fixture,want_pbc', [('slab', (True, True, False)), ('wire', (True, False, False))])
def test_partly_periodic(fixture, want_pbc):
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    assert pbc == want_pbc
    nb = C.cell_list_bins(cell)
    f = _frac(pos, cell)
    for a in range(3):
        if pbc[a]:
            assert nb[a] >= 2
        else:
            # the atoms lie inside the cell (the kernels wrap every direction, as the reference does) and occupy
            # at least 3 bins, so the search radius capped at nb - 1 bins is what limits the sweep
            assert (f[:, a] > 0).all() and (f[:, a] < 1).all()
            assert nb[a] >= 3 and len(np.unique(np.floor(f[:, a] * nb[a]))) >= 3


def test_compressed_cs_weight_regimes():
    """Weight sums from the oracle's float-rounded CN with the oracle's arithmetic (log space): some atoms below
    1e-300 (the kernel's one-hot fallback), some between 1e-300 and 1e-99, and atom pairs on both sides of the
    reference's D_i D_j = 1e-99 branch, none within 1 % (in log) of either threshold, so that a float-vs-double
    decision cannot flip."""
    from oracle.d3_oracle import d3_reference
    z, pos, cell, pbc = C.compressed_cs()
    assert (z == 55).mean() >= 2 / 3
    cn = d3_reference(z, pos, cell, pbc, mimic_fp32=True)['cn']
    ld = C.log_weight_sums(z, cn)
    lo, hi = np.log(1e-300), np.log(1e-99)
    assert (ld < lo).sum() >= 4
    assert ((ld > lo) & (ld < hi)).sum() >= 1
    den = ld[:, None] + ld[None, :]
    assert (den > hi).sum() >= 2 and (den < hi).sum() >= 2
    assert np.abs(den - hi).min() > 0.01 * abs(hi)
    assert np.abs(ld - lo).min() > 0.01 * abs(lo)


def test_species16():
    from oracle.d3_oracle import d3_params
    z, pos, cell, pbc = C.species16()
    uniq = np.unique(z)
    assert len(uniq) == 16 and 1 in uniq and (uniq >= 50).sum() >= 4
    assert set(d3_params()['mxc'][uniq - 1].tolist()) == {1, 2, 3, 4, 5}


def test_nacl_large():
    z, pos, cell, pbc = C.nacl_large()
    assert len(z) >= 4800 and all(pbc)


def test_molecule():
    z, pos, cell, pbc = C.molecule()
    assert not any(pbc) and not cell.any() and (pos < 0).any(axis=0).all()


def test_golden_cases():
    """The systems stored from the reference are in its (LAMMPS, lower-triangular) frame, and each functional holds
    the smallest or largest value of s6, s18, rs6 or rs18 of its damping."""
    from oracle.d3_oracle import d3_params
    F = d3_params()['functionals']
    for fixture, damping, functional in C.GOLDEN_CASES:
        assert fixture in C.LAMMPS_FRAME
        assert np.array_equal(np.triu(C.FIXTURES[fixture]()[2], 1), np.zeros((3, 3)))
        ext = [k for k in ('s6', 's18', 'rs6', 'rs18')
               if F[damping][functional][k] in (min(p[k] for p in F[damping].values()), max(p[k] for p in F[damping].values()))]
        assert ext, (damping, functional)
