"""D3's heat flux and per-atom centroid virial on the distributed partial-range driver (s7b_d3_centroid_pass,
s7b_d3_heat_flux_pass / _sums; sevenn_b200.d3.distributed_d3_centroid_virials / distributed_d3_heat_flux; DESIGN.md
§8.8), and DistributedRunner.heat_flux(..., d3=).

Ranks run as threads on one GPU with the stand-in collectives of test_d3_edges_gpu.py.  Every pass is one warp per
atom with a fixed order, so each rank's rows and flux must equal the one-GPU call's bit for bit, at world 1, 2, 3 and
5, on cells with and without a CN part (`sheared`, `molecule`, `species16` against rock-salt `nacl_large`, whose
weights are one-hot), partly periodic (`slab`) and with an empty range (`compressed_cs`, 12 atoms, world 5)."""
import os
import threading

import numpy as np
import pytest

import d3_cells as C
from test_d3_edges_gpu import _FakeGroup

pytestmark = pytest.mark.gpu

AU = 0.52917726
FIXTURES = ['sheared', 'compressed_cs', 'molecule', 'slab', 'species16', 'nacl_large']
WORLDS = (1, 2, 3, 5)
FORWARD = ('cn', 'dc6i', 'eatom', 'force', 'energy', 'sigma')


def _system(name):
    """(numbers, positions, cell, pbc) as evaluated at the default cutoffs: a structure without a cell gets
    D3Calculator's generated cell"""
    z, pos, cell, pbc = C.FIXTURES[name]()
    if np.asarray(cell).sum() == 0:
        cell = np.eye(3) * (pos.max(0) - pos.min(0) + np.sqrt(9000.0) * AU + 1.0)
        pbc = (True, True, True)
    return z, pos, cell, pbc


def _snapshot(eng):
    return [eng.buffer(k).clone() for k in FORWARD]


def _same(a, b):
    import torch
    return all(torch.equal(x, y) for x, y in zip(a, b))


def _run_ranks(world, fn, monkeypatch):
    """fn(rank) on `world` threads, each one rank of a _FakeGroup; returns the per-rank results"""
    import torch
    import torch.distributed as dist
    fake = _FakeGroup(world)
    for name in ('get_world_size', 'get_rank', 'all_gather_into_tensor', 'all_reduce'):
        monkeypatch.setattr(dist, name, getattr(fake, name), raising=False)
    results, errs = [None] * world, []

    def rank_main(r):
        try:
            fake.local.rank = r
            results[r] = fn(r)
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
    return results


@pytest.mark.parametrize('fixture', FIXTURES)
def test_ranks_equal_one_gpu_bitwise(fixture, monkeypatch):
    import torch
    from sevenn_b200.d3 import (D3Engine, distributed_d3, distributed_d3_centroid_virials,
                                distributed_d3_heat_flux)
    z, pos, cell, pbc = _system(fixture)
    n = len(z)
    v = np.random.RandomState(11).normal(size=(n, 3))
    for damping in ('damp_bj', 'damp_zero'):
        one = D3Engine(damping)
        e_ref, f_ref, s_ref = one.compute(z, pos, cell, pbc)
        wc_ref = one.centroid_virial()
        jpot_ref, ju_ref = one.heat_flux(v)
        for world in WORLDS:
            chunk = (n + world - 1) // world
            if fixture == 'compressed_cs' and world == 5:
                assert min(4 * chunk, n) == n                            # the last rank's range is empty
            engines = [D3Engine(damping) for _ in range(world)]

            def rank(r):
                eng = engines[r]
                res = distributed_d3(eng, z, pos, cell, pbc)
                before = _snapshot(eng)
                wc = distributed_d3_centroid_virials(eng)
                jpot, ju = distributed_d3_heat_flux(eng, v)
                wc2 = distributed_d3_centroid_virials(eng)               # after a flux: unchanged
                return res, before, _snapshot(eng), eng.results(), wc, jpot, ju, wc2

            for r, (res, before, after, res2, wc, jpot, ju, wc2) in enumerate(_run_ranks(world, rank, monkeypatch)):
                what = f'{fixture} {damping} rank {r} of {world}'
                assert torch.equal(wc, wc_ref), f'{what}: centroid virial'
                assert torch.equal(wc2, wc_ref), f'{what}: centroid virial after a flux'
                assert torch.equal(jpot, jpot_ref[0]) and torch.equal(ju, ju_ref[0]), f'{what}: heat flux'
                assert _same(before, after), f'{what}: a forward buffer changed'
                assert res[0] == res2[0] and np.array_equal(res[1], res2[1]) and np.array_equal(res[2], res2[2]), what
                assert np.array_equal(res[1], f_ref), what                # distributed_d3 itself is unchanged
        print(f'\n{fixture} {damping}: ranks {WORLDS} equal one GPU bit for bit, max |Wc| '
              f'{float(wc_ref.abs().max()):.3e} eV, J_pot {jpot_ref[0].cpu().numpy()}')


def _refused(eng, call, match):
    """call() must raise the library's refusal and leave every forward buffer and exchanged record as it was"""
    names = FORWARD + ('ct_nb', 'fx_nb', 'ct_out', 'fx_out')
    dt = dict(ct_nb='f4', fx_nb='f4')
    before = [eng.buffer(k, dtype=dt.get(k, 'f8')).clone() for k in names]
    with pytest.raises(RuntimeError, match=match):
        call()
    after = [eng.buffer(k, dtype=dt.get(k, 'f8')).clone() for k in names]
    assert _same(before, after), f'a refused call changed a buffer ({match})'


def test_refusals_change_nothing():
    import torch
    from sevenn_b200.d3 import D3Engine
    from sevenn_b200.engine import check
    z, pos, cell, pbc = _system('sheared')
    n = len(z)
    eng = D3Engine('damp_bj')
    lib, h = eng.lib, eng._h
    v = torch.as_tensor(np.random.RandomState(2).normal(size=(n, 3)), device=eng.device)
    jp = torch.zeros(1, 3, dtype=torch.float64, device=eng.device)
    ju = torch.zeros_like(jp)
    st = eng._stream

    def ct(p, a, b):
        return lambda: check(lib.s7b_d3_centroid_pass(h, p, a, b, st()))

    def fx(p, a, b):
        return lambda: check(lib.s7b_d3_heat_flux_pass(h, p, v.data_ptr(), a, b, st()))

    sums = lambda: check(lib.s7b_d3_heat_flux_sums(h, jp.data_ptr(), ju.data_ptr(), st()))   # noqa: E731
    # a first full round allocates every buffer the refusals are checked against
    eng.compute(z, pos, cell, pbc)
    for call in (ct(1, 0, n), ct(2, 0, n), fx(1, 0, n), fx(2, 0, n), sums):
        call()
    lo, hi = n // 3, 2 * n // 3
    eng.set_system(z, pos, cell, pbc)
    _refused(eng, ct(1, lo, hi), 'stages 1, 2 and 3 run in order over one atom range')          # no forward
    for s in (1, 2):
        eng.run_stage(s, lo, hi)
    _refused(eng, fx(1, lo, hi), 'stages 1, 2 and 3 run in order over one atom range')          # stage 3 missing
    eng.run_stage(3, lo, hi)
    _refused(eng, ct(1, lo, hi + 1), r'not inside the forward\'s range')                       # outside the range
    _refused(eng, fx(1, lo - 1, hi), r'not inside the forward\'s range')
    _refused(eng, ct(1, hi, lo), r'not inside the forward\'s range')
    _refused(eng, ct(2, lo, hi), 'pass 2 needs pass 1')                                         # pass 2 before 1
    _refused(eng, sums, 'sums need flux pass 2')                                                # sums before 2
    ct(1, lo, hi)()
    _refused(eng, fx(2, lo, hi), 'pass 2 needs pass 1')                                         # the other kind
    _refused(eng, ct(2, lo, hi + 1), r'not inside the forward\'s range')
    _refused(eng, ct(3, lo, hi), 'passes 1 and 2')
    fx(1, lo, lo + 5)()
    _refused(eng, fx(2, lo, lo + 6), 'pass 2 needs pass 1 over a range containing')
    _refused(eng, sums, 'sums need flux pass 2')                                                # after pass 1 only
    fx(2, lo + 1, lo + 5)()
    sums()
    _refused(eng, lambda: eng.centroid_virial(), r'all atoms \[0, n\)')                         # one-shot: refused
    _refused(eng, lambda: eng.heat_flux(v), r'all atoms \[0, n\)')
    eng.run_stage(1, lo, hi)                                                                    # a forward stage
    _refused(eng, ct(2, lo, hi), 'stages 1, 2 and 3')
    for s in (2, 3):
        eng.run_stage(s, lo, hi)
    _refused(eng, ct(2, lo, hi), 'pass 2 needs pass 1')
    _refused(eng, sums, 'sums need flux pass 2')
    ct(1, lo, hi)()
    eng._set_damping()                                                                          # set_damping
    _refused(eng, ct(2, lo, hi), 'stages 1, 2 and 3')
    _refused(eng, ct(1, lo, hi), 'stages 1, 2 and 3')
    for s in (1, 2, 3):
        eng.run_stage(s, lo, hi)
    fx(1, lo, hi)()
    fx(2, lo, hi)()
    eng.set_system(z, pos, cell, pbc)                                                           # set_system
    _refused(eng, fx(1, lo, hi), 'stages 1, 2 and 3')
    _refused(eng, sums, 'sums need flux pass 2')
    # a full-range forward is the range [0, n): the passes accept it, and the one-shot calls still work after them
    for s in (1, 2, 3):
        eng.run_stage(s)
    ct(1, 0, n)()
    ct(2, 0, n)()
    one = D3Engine('damp_bj')
    one.compute(z, pos, cell, pbc)
    assert torch.equal(eng.centroid_virial(), one.centroid_virial())


# ---- DistributedRunner with D3 over NCCL ------------------------------------------------------------------------
SI_MASS = 28.0855


def _si_cell():
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(4, 3, 3, sigma=0.05, seed=2)
    return z, pos, cell


def _runner_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    from helpers import model_weights, species_of
    from sevenn_b200.d3 import D3Engine, distributed_d3
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.parallel import DistributedRunner, brick_decompose
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        meta, arrays = model_weights('sevennet_0')
        z, pos, cell = _si_cell()
        part = brick_decompose(pos, cell, species_of(meta, z).astype(np.int32), (world, 1, 1), rank, 5.0)
        run = DistributedRunner(B200Engine(meta, arrays, device=rank), part)
        run.compute()
        d3 = D3Engine(device=rank)
        distributed_d3(d3, z, pos, cell, (True,) * 3)
        v = np.random.RandomState(9).normal(size=pos.shape) * 0.05
        j = run.heat_flux(v, np.full(len(pos), SI_MASS), d3=d3).cpu().numpy()
        jp = run.heat_flux(v, convective=False, d3=d3).cpu().numpy()
        run.close()
        q.put((rank, j, jp))
    finally:
        dist.destroy_process_group()


class _Atoms:
    """the part of ase.Atoms the calculators and get_heat_flux use"""

    def __init__(self, numbers, positions, cell, v):
        self.numbers, self.positions, self.cell, self.v = numbers, positions, cell, v

    def get_cell(self):
        return self.cell

    def get_pbc(self):
        return np.array([True] * 3)

    def get_positions(self):
        return self.positions

    def get_atomic_numbers(self):
        return self.numbers

    def get_velocities(self):
        return self.v

    def get_masses(self):
        return np.full(len(self.numbers), SI_MASS)


def test_distributed_runner_with_d3_over_nccl():
    """DistributedRunner.heat_flux(..., d3=) on two GPUs against SevenNetD3Calculator.get_heat_flux of the whole cell"""
    import socket
    import torch
    import torch.multiprocessing as mp
    from sevenn_b200.d3 import SevenNetD3Calculator
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    z, pos, cell = _si_cell()
    v = np.random.RandomState(9).normal(size=pos.shape) * 0.05
    atoms = _Atoms(z, pos, cell, v)
    calc = SevenNetD3Calculator('7net-0', device='cuda')
    j_ref = calc.get_heat_flux(atoms)
    jp_ref = calc.get_heat_flux(atoms, convective=False)
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_runner_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=300) for _ in range(2)]
        for p in procs:
            p.join(timeout=120)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    for _, j, jp in res:
        print(f'runner + D3: J {j} vs {j_ref}, J_pot {jp} vs {jp_ref}')
        assert np.abs(j - j_ref).max() < 1e-5 * np.abs(j_ref).max()
        assert np.abs(jp - jp_ref).max() < 1e-5 * np.abs(jp_ref).max()
    assert np.array_equal(res[0][1], res[1][1])
