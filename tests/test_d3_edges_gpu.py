"""The D3 kernels (csrc/d3_kernels.cuh) at the default cutoffs (9000 / 1600 bohr^2) on the systems of
tests/d3_cells.py: against the fp64 oracle (oracle/d3_oracle.py) for both dampings and the functionals that hold
the extremes of the functional table, against stored outputs of the reference's compiled D3, under a rotation of
the frame, through split atom ranges (the multi-GPU stage interface run on one GPU), and through one engine
reused across systems.  Negative controls show that the bounds resolve sub-percent errors in each of the three
kernel passes.

Bounds: those of tests/test_d3_gpu.py::test_matches_fp64_oracle (energy 2e-6 relative; forces and sigma 2e-5
of the largest component), with cn and dc6i (-dE/dCN) at 2e-6 and 2e-5 of their largest value.

Worst measured error per fixture over both dampings and all functionals of ``functionals()`` (rotated: pbe
only), as a fraction of the largest value of each quantity (the energy: relative), on an H100 80GB HBM3 with a
400 W power limit.  The forces and sigma vary in the last digit between runs (fp64 atomics in the block sums).

  fixture         cn       dc6i     energy   forces   sigma
  sheared         1.5e-07  1.2e-06  2.8e-07  1.1e-06  6.1e-07
  rotated         1.5e-07  8.1e-07  1.8e-07  4.9e-07  2.7e-07
  slab            1.7e-07  1.8e-06  2.2e-07  1.6e-06  7.1e-07
  wire            1.5e-07  1.1e-06  5.2e-07  1.2e-06  8.2e-07
  compressed_cs   1.8e-07  1.8e-06  4.1e-07  2.1e-06  6.9e-07   (dc6i against 1e-12 hartree, see DC6I_SCALE)
  species16       9.7e-08  7.0e-07  3.9e-07  1.5e-06  8.4e-07

Against the reference's stored outputs: energy <= 1.5e-6, forces <= 6.2e-6 eV/A, stress <= 1.7e-6 of its
largest component.  Rotation: energy 2e-16, forces <= 8.3e-8, sigma <= 1.8e-8.
"""
import os
import threading

import numpy as np
import pytest

import d3_cells as C

pytestmark = pytest.mark.gpu

BOUNDS = dict(cn=2e-6, dc6i=2e-5, energy=2e-6, forces=2e-5, sigma=2e-5)
# compressed_cs: every atom with a pair above the D_i D_j = 1e-99 branch has one dominant reference weight, so
# its -dE/dCN is ~1e-19 hartree, the rounding residue of a cancellation on both sides (kernel and oracle).  Its
# dc6i is measured against 1e-12 hartree instead, below which it moves no force by 1e-8 eV/A.
DC6I_SCALE = dict(compressed_cs=1e-12)


def functionals(damping):
    """pbe and, for each of s6, s18, rs6, rs18, the functionals with its smallest and largest value
    (first by name on ties)."""
    from oracle.d3_oracle import d3_params
    F = d3_params()['functionals'][damping]
    names = sorted(F)
    out = {'pbe'}
    for k in ('s6', 's18', 'rs6', 'rs18'):
        v = np.array([F[n][k] for n in names])
        out |= {names[int(v.argmin())], names[int(v.argmax())]}
    return sorted(out)


def _sigma6(s):
    return np.array([s[0, 0], s[1, 1], s[2, 2], s[0, 1], s[0, 2], s[1, 2]])


def _sigma33(s6):
    xx, yy, zz, xy, xz, yz = s6
    return np.array([[xx, xy, xz], [xy, yy, yz], [xz, yz, zz]])


def run_engine(eng, z, pos, cell, pbc):
    """energy, forces, sigma6 and the per-atom cn / dc6i of one evaluation, in the caller's atom order."""
    e, f, s = eng.compute(z, pos, cell, pbc)
    order = eng.buffer('order', dtype='i4').cpu().numpy()
    cn, dc = np.empty(len(z)), np.empty(len(z))
    cn[order] = eng.buffer('cn').cpu().numpy()
    dc[order] = eng.buffer('dc6i').cpu().numpy()
    return dict(energy=e, forces=f, sigma=s, cn=cn, dc6i=dc)


def errors(out, ref, dc6i_scale=0.0):
    """error of each quantity relative to the largest value of the reference (energy: relative)"""
    def rel(a, b, floor=1e-300):
        return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), floor))
    return dict(cn=rel(out['cn'], ref['cn']), dc6i=rel(out['dc6i'], ref['dc6i'], dc6i_scale),
                energy=abs(out['energy'] / ref['energy'] - 1.0), forces=rel(out['forces'], ref['forces']),
                sigma=rel(out['sigma'], _sigma6(ref['sigma'])))


def first_divergence(err, bounds=BOUNDS):
    """the first quantity, in the order of the passes that produce it, whose error exceeds its bound"""
    for k in ('cn', 'dc6i', 'energy', 'forces', 'sigma'):
        if not err[k] <= bounds[k]:
            return k
    return None


def _oracle(fixture, damping, functional):
    from oracle.d3_oracle import d3_reference
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    return d3_reference(z, pos, cell, pbc, damping=damping, functional=functional)


@pytest.mark.parametrize('fixture', C.ORACLE_FIXTURES)
def test_matches_fp64_oracle_default_cutoffs(fixture):
    from sevenn_b200.d3 import D3Engine
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    worst = dict.fromkeys(BOUNDS, 0.0)
    fails = []
    for damping in ('damp_bj', 'damp_zero'):
        # the rotated cell is the sheared one in another frame: pbe only (its extremes run on `sheared`)
        for functional in (['pbe'] if fixture == 'rotated' else functionals(damping)):
            out = run_engine(D3Engine(damping, functional), z, pos, cell, pbc)
            err = errors(out, _oracle(fixture, damping, functional), DC6I_SCALE.get(fixture, 0.0))
            worst = {k: max(worst[k], err[k]) for k in worst}
            bad = first_divergence(err)
            if bad is not None:
                fails.append(f'{damping}/{functional}: {bad} diverges first ({err[bad]:.2e} > {BOUNDS[bad]:.0e}); '
                             + ', '.join(f'{k} {v:.2e}' for k, v in err.items()))
    print(f'\nD3 {fixture:14s} ' + ' '.join(f'{k} {v:.1e}' for k, v in worst.items()))
    assert not fails, '\n'.join(fails)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'd3_compiled_reference.npz')


@pytest.mark.parametrize('fixture,damping,functional', C.GOLDEN_CASES)
def test_matches_compiled_reference(fixture, damping, functional):
    """Stored outputs of the reference's own D3 (tools/make_d3_golden.py); bounds of
    tests/test_d3_gpu.py::test_matches_compiled_reference (the reference sums lattice images in fp32)."""
    from sevenn_b200.d3 import D3Engine
    g = np.load(GOLDEN)
    k = C.golden_key(fixture, damping, functional)
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    assert np.array_equal(pos, g[k + '_positions'])          # the stored values belong to these inputs
    e_ref, f_ref, s_ref = float(g[k + '_energy']), g[k + '_forces'], g[k + '_stress']
    e, f, s = D3Engine(damping, functional).compute(z, pos, cell, pbc)
    print(f'\nD3 reference {k}: energy {abs(e / e_ref - 1.0):.1e}, forces {np.abs(f - f_ref).max():.1e} eV/A '
          f'(max {np.abs(f_ref).max():.1e}), stress {np.abs(s - s_ref).max() / np.abs(s_ref).max():.1e}')
    assert abs(e / e_ref - 1.0) < 1e-4
    assert np.abs(f - f_ref).max() < 2e-6 + 1e-4 * np.abs(f_ref).max()
    assert np.abs(s - s_ref).max() < 2e-4 * np.abs(s_ref).max()


def test_rotation_covariance():
    """forces and virial come back in the caller's frame: rotating the system rotates F and sigma"""
    from sevenn_b200.d3 import D3Engine
    R = C.rotation()
    for damping in ('damp_bj', 'damp_zero'):
        e0, f0, s0 = D3Engine(damping).compute(*C.sheared())
        e1, f1, s1 = D3Engine(damping).compute(*C.rotated())
        f_rot = f0 @ R.T
        s_rot = R @ _sigma33(s0) @ R.T
        de = abs(e1 / e0 - 1.0)
        df = np.abs(f1 - f_rot).max() / np.abs(f_rot).max()
        ds = np.abs(_sigma33(s1) - s_rot).max() / np.abs(s_rot).max()
        print(f'\nD3 rotation {damping}: energy {de:.1e}, forces {df:.1e}, sigma {ds:.1e}')
        assert de < BOUNDS['energy'] and df < BOUNDS['forces'] and ds < BOUNDS['sigma'], (damping, de, df, ds)


def test_species_limit():
    """16 species are evaluated (test_matches_fp64_oracle_default_cutoffs[species16]); a 17th is refused with the
    library's error.  16 is the size of the per-warp V table in shared memory (kD3MaxTypes)."""
    from sevenn_b200.d3 import D3Engine
    z, pos, cell, pbc = C.species16()
    z[0] = 3                                                       # Li is not among the 16
    assert len(set(z.tolist())) == 17
    eng = D3Engine()
    with pytest.raises(RuntimeError, match=r'1\.\.16 atom types are supported'):
        eng.compute(z, pos, cell, pbc)


# ---- split atom ranges --------------------------------------------------------------------------
def _sorted_state(eng):
    return {k: eng.buffer(k).clone() for k in ('cn', 'dc6i', 'force')}


def _assert_same(state, ref, energy, sigma, e_ref, s_ref, what):
    import torch
    for k in ('cn', 'dc6i', 'force'):
        assert torch.equal(state[k], ref[k]), f'{what}: {k} is not bit-identical to the unsplit run'
    assert abs(energy / e_ref - 1.0) <= 1e-13, (what, energy, e_ref)
    assert np.abs(np.asarray(sigma) - s_ref).max() <= 1e-13 * np.abs(s_ref).max(), (what, sigma, s_ref)


class _FakeGroup:
    """torch.distributed's collectives for `world` threads on one GPU: each thread is one rank."""

    def __init__(self, world):
        self.world = world
        self.barrier = threading.Barrier(world, timeout=120)
        self.slots = [None] * world
        self.local = threading.local()

    def get_world_size(self, group=None):
        return self.world

    def get_rank(self, group=None):
        return self.local.rank

    def _exchange(self, t):
        import torch
        self.slots[self.local.rank] = t.clone()
        torch.cuda.synchronize()
        self.barrier.wait()
        vals = list(self.slots)
        self.barrier.wait()
        return vals

    def all_gather_into_tensor(self, out, inp, group=None):
        import torch
        out.copy_(torch.cat(self._exchange(inp)))
        torch.cuda.synchronize()

    def all_reduce(self, t, group=None):
        import torch
        vals = self._exchange(t)
        acc = vals[0].clone()
        for v in vals[1:]:
            acc += v
        t.copy_(acc)
        torch.cuda.synchronize()


@pytest.mark.parametrize('fixture,world', [('sheared', 2), ('sheared', 3), ('sheared', 5), ('compressed_cs', 5),
                                           ('nacl_large', 2), ('nacl_large', 3), ('nacl_large', 5)])
def test_distributed_d3_split_ranges(fixture, world, monkeypatch):
    """``distributed_d3`` unchanged, `world` ranks as threads with one D3Engine each.  compressed_cs has 12 atoms:
    with 5 ranks the chunk is 3 and the last rank's range is empty."""
    import torch
    import torch.distributed as dist
    from sevenn_b200.d3 import D3Engine, distributed_d3
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    base = D3Engine()
    e_ref, f_ref, s_ref = base.compute(z, pos, cell, pbc)
    ref = _sorted_state(base)
    fake = _FakeGroup(world)
    for name in ('get_world_size', 'get_rank', 'all_gather_into_tensor', 'all_reduce'):
        monkeypatch.setattr(dist, name, getattr(fake, name), raising=False)
    engines = [D3Engine() for _ in range(world)]
    results, errs = [None] * world, []

    def rank_main(r):
        try:
            fake.local.rank = r
            results[r] = distributed_d3(engines[r], z, pos, cell, pbc)
        except BaseException as ex:   # noqa: BLE001
            errs.append(ex)
            fake.barrier.abort()

    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errs:
        raise errs[0]
    torch.cuda.synchronize()
    n = len(z)
    chunk = (n + world - 1) // world
    if fixture == 'compressed_cs':
        assert min((world - 1) * chunk, n) == n                     # the last rank's range is empty
    for r in range(world):
        e, f, s = results[r]
        _assert_same(_sorted_state(engines[r]), ref, e, s, e_ref, s_ref, f'rank {r} of {world}')
        assert np.array_equal(f, f_ref)


def _split_ranges(n):
    cuts = sorted({0, 1, 2, 7, 18, n // 3, n // 3 + 5, n - 1, n})
    return [(a, b) for a, b in zip([0] + cuts, cuts) if a <= b] + [(n // 2, n // 2)]


@pytest.mark.parametrize('fixture', ['sheared', 'nacl_large'])
def test_run_stage_split_ranges(fixture):
    """Every stage called over ranges of 1 atom, of sizes that are not multiples of the 4 warps per block, and
    empty ones, as the ranks of distributed_d3 call it, on one engine.  Stage 2 zeroes the forces, energy and
    sigma before it adds its range, so each range's stage-2 output is collected before the next call, and
    restored before stage 3 adds the chain-rule terms."""
    import torch
    from sevenn_b200.d3 import D3Engine
    z, pos, cell, pbc = C.FIXTURES[fixture]()
    base = D3Engine()
    e_ref, f_ref, s_ref = base.compute(z, pos, cell, pbc)
    ref = _sorted_state(base)
    n = len(z)
    ranges = _split_ranges(n)
    assert sum(b - a for a, b in ranges) == n and any(a == b for a, b in ranges)
    assert any((b - a) % 4 for a, b in ranges) and any(b - a == 1 for a, b in ranges)
    eng = D3Engine().set_system(z, pos, cell, pbc)
    for a, b in ranges:
        eng.run_stage(1, a, b)
    force = torch.zeros_like(eng.buffer('force', shape=(n, 3)))
    energy, sigma = 0.0, torch.zeros(6, dtype=torch.float64, device=force.device)
    for a, b in ranges:
        eng.run_stage(2, a, b)
        force[a:b] = eng.buffer('force', shape=(n, 3))[a:b]
        energy += float(eng.buffer('energy')[0])
        sigma += eng.buffer('sigma')
    eng.buffer('force', shape=(n, 3)).copy_(force)
    eng.buffer('energy').fill_(energy)
    eng.buffer('sigma').copy_(sigma)
    for a, b in ranges:
        eng.run_stage(3, a, b)
    e, f, s = eng.results()
    _assert_same(_sorted_state(eng), ref, e, s, e_ref, s_ref, f'{fixture} ranges {ranges}')
    assert np.array_equal(f, f_ref)


def test_engine_reuse_across_systems():
    """One engine, in sequence: nacl_large, a small NaCl cell (same species order: parameters are kept, buffers
    are not reallocated, fewer bins), compressed_cs (new species), the small cell with Cl listed first (same
    species, other type order), nacl_large again.  Each result equals that of a fresh engine bit for bit."""
    from sevenn_b200.d3 import D3Engine
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.05, seed=3)
    perm = np.argsort(z != 17, kind='stable')                       # Cl first
    systems = [('nacl_large', C.nacl_large()), ('nacl_small', (z, pos, cell, (True,) * 3)),
               ('compressed_cs', C.compressed_cs()), ('nacl_small_cl_first', (z[perm], pos[perm], cell, (True,) * 3)),
               ('nacl_large', C.nacl_large())]
    eng = D3Engine()
    for name, (zz, pp, cc, pb) in systems:
        got = run_engine(eng, zz, pp, cc, pb)
        want = run_engine(D3Engine(), zz, pp, cc, pb)
        assert np.array_equal(got['forces'], want['forces']), name
        assert np.array_equal(got['cn'], want['cn']), name
        assert abs(got['energy'] / want['energy'] - 1.0) <= 1e-13, name


class _Molecule:
    """the part of ase.Atoms D3Calculator uses (ASE is optional)"""

    def __init__(self, numbers, positions):
        self.numbers, self.positions = np.asarray(numbers), np.asarray(positions, dtype=np.float64)
        self.cell, self.pbc = np.zeros((3, 3)), np.zeros(3, dtype=bool)

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


def test_cell_less_molecule():
    """A molecule without a cell goes through D3Calculator's generated cell; negative coordinates wrap into it.
    The result is that of the isolated molecule: the oracle with pbc (F,F,F)."""
    from oracle.d3_oracle import d3_reference
    from sevenn_b200.d3 import D3Calculator
    z, pos, _, _ = C.molecule()
    assert (pos < 0).any()
    try:
        from ase import Atoms
        atoms = Atoms(numbers=z, positions=pos)
    except ImportError:
        atoms = _Molecule(z, pos)
    res = D3Calculator().calculate(atoms)
    inside = pos - pos.min(0) + 1.0                                 # the oracle wraps in every direction
    ref = d3_reference(z, inside, np.diag(inside.max(0) + 1.0), (False, False, False))
    vol = abs(np.linalg.det(np.asarray(atoms.get_cell(), dtype=np.float64)))
    s = ref['sigma']
    stress = -np.array([s[0, 0], s[1, 1], s[2, 2], s[1, 2], s[0, 2], s[0, 1]]) / vol
    de = abs(res['energy'] / ref['energy'] - 1.0)
    df = np.abs(res['forces'] - ref['forces']).max() / np.abs(ref['forces']).max()
    ds = np.abs(res['stress'] - stress).max() / np.abs(stress).max()
    print(f'\nD3 molecule: energy {de:.1e}, forces {df:.1e}, stress {ds:.1e}')
    assert de < BOUNDS['energy'] and df < BOUNDS['forces'] and ds < BOUNDS['sigma'], (de, df, ds)


# ---- negative controls ------------------------------------------------------------------------
def _tables(numbers):
    from sevenn_b200.d3 import d3_tables
    T = d3_tables()
    zz = np.array(list(dict.fromkeys(np.asarray(numbers).tolist()))) - 1
    f8 = lambda a: np.ascontiguousarray(a, dtype=np.float64)  # noqa: E731
    return dict(rcov=f8(T['rcov'][zz]), r2r4=f8(T['r2r4'][zz]), r0=f8(T['r0ab'][np.ix_(zz, zz)]),
                c6=f8(T['c6ref'][np.ix_(zz, zz)]), cr=f8(T['cnref'][zz]),
                mxc=np.ascontiguousarray(T['mxc'][zz], dtype=np.int32))


@pytest.mark.parametrize('perturbation,diverges', [('rcov', 'cn'), ('s8', 'dc6i'), ('no_stage3', 'forces')])
def test_negative_controls(perturbation, diverges):
    """On `sheared` (BJ, pbe), where the kernels pass: one species' rcov x 1.005 (pass 1), s8 x 1.01 (pass 2) and
    a skipped stage 3 must each fail the comparison with the unperturbed oracle, first at the quantity the
    perturbed pass produces."""
    from sevenn_b200.d3 import D3Engine
    from sevenn_b200.engine import check
    z, pos, cell, pbc = C.sheared()
    eng = D3Engine('damp_bj', 'pbe')
    eng.set_system(z, pos, cell, pbc)
    if perturbation == 'rcov':
        t = _tables(z)
        t['rcov'][1] *= 1.005
        check(eng.lib.s7b_d3_set_params(eng._h, len(t['rcov']), t['rcov'].ctypes.data, t['r2r4'].ctypes.data,
                                        t['r0'].ctypes.data, t['c6'].ctypes.data, t['cr'].ctypes.data,
                                        t['mxc'].ctypes.data))
    elif perturbation == 's8':
        p = eng.par
        check(eng.lib.s7b_d3_set_damping(eng._h, eng.damping, p['s6'], p['s8'] * 1.01, p['a1'], p['a2'], p['alp6'],
                                         p['alp8'], eng.rthr, eng.cnthr))
    for stage in ((1, 2) if perturbation == 'no_stage3' else (1, 2, 3)):
        eng.run_stage(stage)
    e, f, s = eng.results()
    order = eng.buffer('order', dtype='i4').cpu().numpy()
    cn, dc = np.empty(len(z)), np.empty(len(z))
    cn[order] = eng.buffer('cn').cpu().numpy()
    dc[order] = eng.buffer('dc6i').cpu().numpy()
    err = errors(dict(energy=e, forces=f, sigma=s, cn=cn, dc6i=dc), _oracle('sheared', 'damp_bj', 'pbe'))
    print(f'\nD3 negative control {perturbation}: ' + ', '.join(f'{k} {v:.1e}' for k, v in err.items()))
    assert first_divergence(err) == diverges, err
