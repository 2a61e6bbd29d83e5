"""D3 of a batch of structures in one pass (``d3.D3Batch``, C ABI ``s7b_d3_set_system_batch``) against the same
structures evaluated alone by ``D3Engine``, at the default cutoffs (9000 / 1600 bohr^2), for both dampings with pbe.

The mixed batch holds every system of tests/d3_cells.py that the oracle tests use plus the cell-less molecule, three
rattled 64-atom NaCl cells, a one-atom cell and an empty structure.  A batch member's per-atom cn, dc6i and forces
are those of the structure alone bit for bit: same wrap (rounded as the host loop of the single-structure set-up),
same grid, same bin order, same arithmetic.  Energy and virial are per-structure fixed-order sums of per-atom terms,
compared at 1e-12 relative.  ``SevenNetD3Model`` is checked against ``SevenNetD3Calculator`` on each structure alone
with the bounds of tests/test_batch_device_gpu.py, and against ``SevenNetModel`` + ``D3Batch`` (energies exactly).
"""
import types

import numpy as np
import pytest

import d3_cells as C

pytestmark = pytest.mark.gpu

MIXED = ('sheared', 'rotated', 'slab', 'wire', 'compressed_cs', 'species16', 'molecule')
AU_TO_ANG = 0.52917726


def nacl(seed, reps=(2, 2, 2)):
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(*reps, sigma=0.05, seed=seed)
    return z, pos, cell, (True, True, True)


def one_atom():
    return np.array([8]), np.array([[0.3, -0.2, 7.4]]), np.diag([7.0, 7.5, 6.5]), (True, True, True)


def empty():
    return np.zeros(0, dtype=np.int64), np.zeros((0, 3)), np.zeros((3, 3)), (False, False, False)


def mixed():
    return [C.FIXTURES[k]() for k in MIXED] + [nacl(s) for s in (11, 12, 13)] + [one_atom(), empty()]


def _arrays(structs):
    counts = [len(s[0]) for s in structs]
    z = np.concatenate([np.asarray(s[0], dtype=np.int64) for s in structs])
    pos = np.concatenate([np.asarray(s[1], dtype=np.float64).reshape(-1, 3) for s in structs])
    cells = np.stack([np.asarray(s[2], dtype=np.float64) for s in structs])
    pbc = np.array([np.broadcast_to(s[3], (3,)) for s in structs], dtype=bool)
    return z, pos, cells, pbc, np.repeat(np.arange(len(structs)), counts), np.concatenate([[0], np.cumsum(counts)])


def run_batch(d3b, structs, cells=None):
    """per-structure energy / virial and per-atom forces / cn / dc6i (caller's order) of one batched evaluation"""
    import torch
    z, pos, c, pbc, si, ap = _arrays(structs)
    out = d3b.compute(torch.tensor(z, device='cuda'), torch.tensor(pos, device='cuda'), c if cells is None else cells,
                      pbc, system_idx=torch.tensor(si, device='cuda'))
    eng = d3b.engine
    order = eng.buffer('order', dtype='i4').cpu().numpy()
    cn, dc = np.empty(len(z)), np.empty(len(z))
    cn[order] = eng.buffer('cn').cpu().numpy()
    dc[order] = eng.buffer('dc6i').cpu().numpy()
    return dict(energy=out['energy'].cpu().numpy(), virial=out['virial'].cpu().numpy(),
                forces=out['forces'].cpu().numpy(), cn=cn, dc6i=dc, ap=ap, cells=d3b.cells.copy())


def generated_cell(pos, rthr=9000.0, cnthr=1600.0):
    """D3Calculator's cell for a structure without one"""
    return np.eye(3) * (pos.max(axis=0) - pos.min(axis=0) + np.sqrt(max(rthr, cnthr)) * AU_TO_ANG + 1.0)


def run_alone(eng, s):
    z, pos, cell, pbc = s
    if np.all(np.asarray(cell) == 0):
        cell, pbc = generated_cell(np.asarray(pos, dtype=np.float64)), (True, True, True)
    e, f, sg = eng.compute(z, pos, cell, pbc)
    order = eng.buffer('order', dtype='i4').cpu().numpy()
    cn, dc = np.empty(len(z)), np.empty(len(z))
    cn[order] = eng.buffer('cn').cpu().numpy()
    dc[order] = eng.buffer('dc6i').cpu().numpy()
    virial = np.array([sg[0], sg[1], sg[2], sg[3], sg[5], sg[4]])       # xx,yy,zz,xy,yz,zx
    return dict(energy=e, virial=virial, forces=f, cn=cn, dc6i=dc, cell=cell)


def check_members(got, structs, eng, members=None):
    ap = got['ap']
    for b in (range(len(structs)) if members is None else members):
        a0, a1 = ap[b], ap[b + 1]
        if a1 == a0:
            assert got['energy'][b] == 0.0 and not got['virial'][b].any(), b
            continue
        want = run_alone(eng, structs[b])
        for k in ('cn', 'dc6i', 'forces'):
            assert np.array_equal(got[k][a0:a1], want[k]), (b, k)
        assert abs(got['energy'][b] / want['energy'] - 1.0) <= 1e-12, b
        assert np.abs(got['virial'][b] - want['virial']).max() <= 1e-12 * np.abs(want['virial']).max(), b
        assert np.array_equal(got['cells'][b], want['cell']), b


@pytest.mark.parametrize('damping', ['damp_bj', 'damp_zero'])
def test_members_match_structures_alone(damping):
    from sevenn_b200.d3 import D3Batch, D3Engine
    structs = mixed()
    got = run_batch(D3Batch(damping, 'pbe'), structs)
    check_members(got, structs, D3Engine(damping, 'pbe'))


def test_element_union_above_16():
    from sevenn_b200.d3 import D3Batch, D3Engine
    structs = [C.species16(), C.compressed_cs(), nacl(21)]
    assert len(set(np.concatenate([s[0] for s in structs]).tolist())) > 16
    got = run_batch(D3Batch(), structs)
    check_members(got, structs, D3Engine())


def test_type_words_are_table_rows_and_local_ranks():
    """Every sorted atom's type word: Z - 1 in the low byte, the rank of Z among the sorted distinct atomic numbers of
    its own structure above it; after a single-structure set-up, the type index"""
    from sevenn_b200.d3 import D3Batch
    structs = mixed() + [C.species16(), C.compressed_cs()]
    d3b = D3Batch()
    got = run_batch(d3b, structs)
    ap = got['ap']
    z = np.concatenate([np.asarray(s[0], dtype=np.int64) for s in structs])
    want = np.empty(len(z), dtype=np.int64)
    for b in range(len(structs)):
        zb = z[ap[b]:ap[b + 1]]
        want[ap[b]:ap[b + 1]] = (zb - 1) | (np.searchsorted(np.unique(zb), zb) << 8)
    order = d3b.engine.buffer('order', dtype='i4').cpu().numpy()
    words = np.empty(len(z), dtype=np.int64)
    words[order] = d3b.engine.buffer('type', dtype='i4').cpu().numpy()
    assert np.array_equal(words, want)
    eng = d3b.engine                                                      # the same handle, one structure
    zs, pos, cell, pbc = C.species16()
    eng.set_system(zs, pos, cell, pbc)
    lut = {zz: k for k, zz in enumerate(dict.fromkeys(zs.tolist()))}
    words = np.empty(len(zs), dtype=np.int64)
    words[eng.buffer('order', dtype='i4').cpu().numpy()] = eng.buffer('type', dtype='i4').cpu().numpy()
    assert np.array_equal(words, [lut[int(a)] for a in zs])


def _rerun(d3b, B, n):
    """the three stages and the results of the handle's current system, run again"""
    import torch
    from sevenn_b200.engine import check
    eng = d3b.engine
    e = torch.empty(B, dtype=torch.float64, device='cuda')
    f = torch.empty(n, 3, dtype=torch.float64, device='cuda')
    v = torch.empty(B, 6, dtype=torch.float64, device='cuda')
    for stage in (1, 2, 3):
        check(eng.lib.s7b_d3_run_stage(eng._h, stage, 0, n, eng._stream()))
    check(eng.lib.s7b_d3_system_results(eng._h, e.data_ptr(), f.data_ptr(), v.data_ptr(), eng._stream()))
    return e.cpu().numpy(), f.cpu().numpy(), v.cpu().numpy()


def test_refusals_name_the_structure_and_keep_the_previous_system():
    from sevenn_b200.d3 import D3Batch
    structs = [nacl(31), C.compressed_cs(), one_atom()]
    d3b = D3Batch()
    first = run_batch(d3b, structs)
    B, n = len(structs), int(first['ap'][-1])
    z17, pos17, cell17, pbc17 = C.species16()
    z17 = z17.copy()
    z17[0] = 3                                                            # Li: a 17th element
    bad_z = one_atom()
    bad_z = (np.array([0]),) + bad_z[1:]
    singular = nacl(32)
    singular = singular[:2] + (np.diag([11.28, 11.28, 0.0]),) + singular[3:]
    for case, where, msg in (([nacl(31), (z17, pos17, cell17, pbc17)], 1, 'more than 16 elements'),
                             ([one_atom(), nacl(33), bad_z], 2, 'atomic number outside 1..94'),
                             ([singular, one_atom()], 0, 'singular cell')):
        with pytest.raises(RuntimeError, match=f'structure {where} .*{msg}'):
            run_batch(d3b, case)
        e, f, v = _rerun(d3b, B, n)
        assert np.array_equal(e, first['energy']) and np.array_equal(f, first['forces'])
        assert np.array_equal(v, first['virial'])


def test_order_and_repetition_do_not_change_bits():
    from sevenn_b200.d3 import D3Batch
    structs = mixed()
    d3b = D3Batch()
    ref = run_batch(d3b, structs)
    B = len(structs)
    perm = list(range(B))[::-1] + [3, 0]                                  # reversed, then wire and sheared again
    got = run_batch(d3b, [structs[b] for b in perm])
    for k, b in enumerate(perm):
        assert got['energy'][k] == ref['energy'][b] and np.array_equal(got['virial'][k], ref['virial'][b]), b
        assert np.array_equal(got['forces'][got['ap'][k]:got['ap'][k + 1]], ref['forces'][ref['ap'][b]:ref['ap'][b + 1]]), b


def test_swapped_cells_change_those_two_members_only():
    from sevenn_b200.d3 import D3Batch
    structs = [nacl(41), C.sheared(), nacl(42), C.slab(), one_atom()]
    d3b = D3Batch()
    ref = run_batch(d3b, structs)
    _, _, cells, _, _, _ = _arrays(structs)
    cells[[1, 3]] = cells[[3, 1]]
    got = run_batch(d3b, structs, cells=cells)
    ap = ref['ap']
    for b in range(len(structs)):
        same = got['energy'][b] == ref['energy'][b] and np.array_equal(got['forces'][ap[b]:ap[b + 1]], ref['forces'][ap[b]:ap[b + 1]])
        assert same == (b not in (1, 3)), b


def _kernel_names(fn):
    """names of the kernels fn runs, without cub's radix sort (whose passes follow the key range and n, not B)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted(ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA
                  and 'emcpy' not in ev.name and 'emset' not in ev.name and 'cub' not in ev.name)


def test_scale_512_cells():
    import torch
    from sevenn_b200.d3 import D3Batch, D3Engine
    structs = [nacl(1000 + b) for b in range(512)]
    d3b = D3Batch()
    got = run_batch(d3b, structs)
    check_members(got, structs, D3Engine(), members=[0, 1, 137, 255, 256, 400, 510, 511])
    launches = {}
    for B in (2, 512):
        z, pos, cells, pbc, si, ap = _arrays(structs[:B])
        zt, pt = torch.tensor(z, device='cuda'), torch.tensor(pos, device='cuda')
        d3b.compute(zt, pt, cells, pbc, atom_ptr=ap)                      # warm
        launches[B] = _kernel_names(lambda: d3b.compute(zt, pt, cells, pbc, atom_ptr=ap))
    assert launches[2] == launches[512] and len(launches[2]) >= 8, launches


class _Atoms:
    """the part of ase.Atoms the calculators use (ASE is optional)"""

    def __init__(self, numbers, positions, cell, pbc):
        self.numbers, self.positions = np.asarray(numbers), np.asarray(positions, dtype=np.float64)
        self.cell, self.pbc = np.asarray(cell, dtype=np.float64), np.broadcast_to(np.asarray(pbc, dtype=bool), (3,))

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


@pytest.mark.parametrize('pos_dtype,device', [('float32', 'cuda'), ('float64', 'cuda'), ('float32', 'cpu'), ('float64', 'cpu')])
def test_sevennet_d3_model(pos_dtype, device):
    import torch
    from sevenn_b200.batch import DeviceBatch, SevenNetD3Model
    from sevenn_b200.d3 import D3Batch, SevenNetD3Calculator
    from sevenn_b200.neighbors import diamond_si
    structs = [nacl(51), nacl(52, (2, 2, 1))]
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=53)
    structs.append((z, pos, cell, (True, True, True)))
    z, pos, cells, pbc, si, ap = _arrays(structs)
    dt = getattr(torch, pos_dtype)
    state = types.SimpleNamespace(positions=torch.tensor(pos, dtype=dt, device=device),
                                  row_vector_cell=torch.tensor(cells, device=device),
                                  pbc=torch.tensor(pbc, device=device), atomic_numbers=torch.tensor(z, device=device),
                                  system_idx=torch.tensor(si, device=device))
    model = SevenNetD3Model('7net-0', device='cuda')
    out = model(state)
    # the network's batch + D3Batch: the D3 terms and both energies are deterministic, the network's fp32 forces are
    # not bit-reproducible between two evaluations, so forces and stress are compared at float32 resolution
    net = DeviceBatch(model.engine).compute(state.atomic_numbers, state.positions, cells, state.pbc, state.system_idx)
    d3 = D3Batch(device=model.device.index).compute(state.atomic_numbers, state.positions, cells, state.pbc, atom_ptr=ap)
    assert torch.equal(d3['energy'], model.d3.compute(state.atomic_numbers, state.positions, cells, state.pbc,
                                                      system_idx=state.system_idx)['energy'])
    assert torch.equal(out['energy'], (net['energy'] + d3['energy']).float())
    assert torch.allclose(out['forces'], (net['forces'].double() + d3['forces']).float(), rtol=0, atol=1e-6)
    assert torch.allclose(out['stress'], model._stress(net['virial'] + d3['virial'], cells).float(), rtol=1e-5, atol=1e-8)
    # each structure against SevenNetD3Calculator on that structure alone
    calc = SevenNetD3Calculator('7net-0', device='cuda')
    e, f, st = out['energy'].double().cpu().numpy(), out['forces'].double().cpu().numpy(), out['stress'].double().cpu().numpy()
    for b, (zz, pp, cc, pb) in enumerate(structs):
        pp = torch.tensor(pp, dtype=dt).double().numpy()                 # what the batch was given
        r = calc.calculate(_Atoms(zz, pp, cc, pb))
        assert abs(e[b] - r['energy']) <= 2e-5 * max(1.0, abs(r['energy'])), b
        assert np.allclose(f[ap[b]:ap[b + 1]], r['forces'], atol=2e-5), b
        s = r['stress']                                                   # Voigt xx,yy,zz,yz,xz,xy
        full = np.array([[s[0], s[5], s[4]], [s[5], s[1], s[3]], [s[4], s[3], s[2]]])
        assert np.allclose(st[b], full, atol=2e-5), b
