"""Batches evaluated from device-resident arrays: the batched device neighbour list
(``s7b_engine_set_positions_batch``), the per-structure fp64 energy / virial (``s7b_engine_system_results``),
``batch.DeviceBatch`` and the TorchSim-shaped ``SevenNetModel`` built on them, against every structure built
and evaluated alone through the single-structure positions-in path."""
import types

import numpy as np
import pytest

import d3_cells
import graphs
from helpers import golden_vectors, model_weights, species_of

pytestmark = pytest.mark.gpu

MODEL = 'sevennet_0'
# per-atom energies and the CSR are bit-identical (same grid, same stable sort, same forward kernels); the
# backward adds edge contributions with fp32 RED.ADD in a run-dependent order, so forces and the virial are
# compared with a bound of a few fp32 roundings of the largest term a row sums (~100 edges of |f| <= max|F|)
F_RTOL = 1e-5
V_RTOL = 1e-5
# the structure energy is an fp64 sum of the same fp64 per-atom energies in another order: ~n * 1e-16 * |E|
E_ATOL = 1e-9


@pytest.fixture(scope='module')
def meta():
    return model_weights(MODEL)[0]


@pytest.fixture(scope='module')
def eng():
    from sevenn_b200.engine import B200Engine
    return B200Engine(*model_weights(MODEL))


def _struct(name, numbers, pos, cell, pbc):
    return dict(name=name, numbers=np.asarray(numbers, dtype=np.int64).reshape(-1),
                positions=np.asarray(pos, dtype=np.float64).reshape(-1, 3),
                cell=np.zeros((3, 3)) if cell is None else np.asarray(cell, dtype=np.float64),
                pbc=tuple(bool(b) for b in np.broadcast_to(np.asarray(pbc, dtype=bool), (3,))))


def _golden(key):
    s = golden_vectors()[key]['system']
    return _struct(key, s['numbers'], s['positions'], s['cell'], bool(s['pbc']))


def _graph_fixture(name):
    g = graphs.fixture(name, MODEL)
    return _struct(name, g.numbers, g.positions, g.cell, g.pbc)


def _empty(name):
    return _struct(name, [], np.zeros((0, 3)), np.eye(3) * 10.0, True)


def mixed_batch():
    """triclinic, molecular (no cell), one-atom, tiny, dense, every-species, slab and wire members, plus empty
    structures in the middle and at the end"""
    return [_golden('7net0_nacl_rattled'), _golden('7net0_hfo2_0'), _golden('7net0_hfo2_1'), _golden('7net0_h2o'),
            _golden('7net0_single_o'), _graph_fixture('tiny_cell'), _empty('empty_mid'), _graph_fixture('isolated'),
            _graph_fixture('dense'), _graph_fixture('many_species'), _graph_fixture('radial_edges'),
            _struct('slab', *d3_cells.slab()), _struct('wire', *d3_cells.wire()),
            _struct('lone_si', [14], [[0.3, 0.2, 0.1]], np.eye(3) * 12.0, True), _empty('empty_end')]


def si_cells(count, seed0, reps=(2, 2, 2)):
    from sevenn_b200.neighbors import diamond_si
    out = []
    for k in range(count):
        pos, cell, z = diamond_si(*reps, sigma=0.08, seed=seed0 + k)
        out.append(_struct(f'si{reps}_{seed0 + k}', z, pos, cell, True))
    return out


def _arrays(structs):
    counts = [len(s['numbers']) for s in structs]
    return dict(numbers=np.concatenate([s['numbers'] for s in structs]),
                positions=np.concatenate([s['positions'] for s in structs]),
                atom_ptr=np.concatenate([[0], np.cumsum(counts)]).astype(np.int32),
                cells=np.stack([s['cell'] for s in structs]),
                pbc=np.array([s['pbc'] for s in structs]),
                system_idx=np.repeat(np.arange(len(structs)), counts))


def _set_batch(eng, meta, structs, cells=None):
    import torch
    a = _arrays(structs)
    pos = torch.tensor(a['positions'], device='cuda')
    eng.set_positions_batch(species_of(meta, a['numbers']), pos, a['atom_ptr'], a['cells'] if cells is None else cells,
                            a['pbc'])
    return a


def _csr(eng):
    return tuple(t.cpu().numpy().copy() for t in eng.graph_arrays())


def _alone_csr(eng, meta, s):
    eng.set_positions(species_of(meta, s['numbers']), s['positions'], s['cell'], s['pbc'])
    return _csr(eng)


def _concat(parts):
    rowptr, src, vec, a, e = [np.zeros(1, np.int32)], [], [], 0, 0
    for rp, s, v in parts:
        rowptr.append(rp[1:] + e)
        src.append(s + a)
        vec.append(v.reshape(-1, 3))
        a += len(rp) - 1
        e += len(s)
    return np.concatenate(rowptr), np.concatenate(src), np.concatenate(vec)


def _same_csr(got, want):
    return (got[0].shape == want[0].shape and np.array_equal(got[0], want[0]) and got[1].shape == want[1].shape
            and np.array_equal(got[1], want[1]) and np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32)))


def test_batch_csr_is_the_concatenation_of_structures_alone(eng, meta):
    structs = mixed_batch()
    want = _concat([_alone_csr(eng, meta, s) for s in structs])
    a = _set_batch(eng, meta, structs)
    got = _csr(eng)
    assert eng.n_nodes == a['atom_ptr'][-1] and eng.n_edges == len(want[1])
    assert _same_csr(got, want), [s['name'] for s in structs]
    # negative control: the rattled NaCl and the first HfO2 frame exchange cells -> different graphs
    cells = _arrays(structs)['cells'].copy()
    cells[[0, 1]] = cells[[1, 0]]
    _set_batch(eng, meta, structs, cells=cells)
    assert not _same_csr(_csr(eng), want)


def _canonical(dst, src, vec):
    vec = np.asarray(vec, dtype=np.float64)
    q = np.rint(vec * 20).astype(np.int64)                 # 0.05 A buckets only order images of one pair
    o = np.lexsort((q[:, 2], q[:, 1], q[:, 0], src, dst))
    return np.asarray(dst)[o], np.asarray(src)[o], vec[o]


def test_batch_rows_match_brute_force_edge_sets(eng, meta):
    from sevenn_b200.neighbors import neighbor_list_brute
    structs = mixed_batch()
    a = _set_batch(eng, meta, structs)
    rowptr, src, vec = _csr(eng)
    for b, s in enumerate(structs):
        if s['name'] not in ('7net0_h2o', 'tiny_cell', 'slab', 'wire', 'lone_si', '7net0_hfo2_1'):
            continue
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        e0, e1 = rowptr[a0], rowptr[a1]
        dst = np.repeat(np.arange(a1 - a0), np.diff(rowptr[a0:a1 + 1]))
        pos = s['positions']
        if any(s['pbc']):                # the brute-force images reach one cell: wrap atoms given outside it
            frac = pos @ np.linalg.inv(s['cell'])
            frac[:, list(s['pbc'])] -= np.floor(frac[:, list(s['pbc'])])
            pos = frac @ s['cell']
        ei, ev, _ = neighbor_list_brute(pos, s['cell'], s['pbc'], 5.0)
        assert e1 - e0 == ei.shape[1], s['name']
        d1, s1, v1 = _canonical(dst, src[e0:e1] - a0, vec[e0:e1])
        d2, s2, v2 = _canonical(ei[0], ei[1], ev)
        assert (d1 == d2).all() and (s1 == s2).all(), s['name']
        assert np.allclose(v1, v2, atol=2e-6), s['name']       # double differences stored as float


def _alone_results(eng, meta, s):
    e, ae, f, v, _ = eng.compute_positions(species_of(meta, s['numbers']), s['positions'], s['cell'], s['pbc'])
    ae64 = eng.buffer('atomic_energy_f64', dtype='f8', shape=(len(ae),)).cpu().numpy().copy()
    return e, ae, ae64, f, v


def _batch_results(eng, structs):
    import torch
    from sevenn_b200.batch import DeviceBatch
    a = _arrays(structs)
    out = DeviceBatch(eng).compute(a['numbers'], torch.tensor(a['positions'], device='cuda'), a['cells'], a['pbc'],
                                   torch.tensor(a['system_idx'], device='cuda'))
    ae64 = eng.buffer('atomic_energy_f64', dtype='f8', shape=(eng.n_local,)).cpu().numpy().copy()
    res = {k: (v.cpu().numpy() if hasattr(v, 'cpu') else v) for k, v in out.items()}
    res['ae64'] = ae64
    return a, res


def _check_against_alone(eng, meta, structs, a, res, which):
    for b in which:
        s = structs[b]
        if len(s['numbers']) == 0:
            continue
        e, ae, ae64, f, v = _alone_results(eng, meta, s)
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        assert np.array_equal(res['atomic_energy'][a0:a1].view(np.uint32), ae.view(np.uint32)), s['name']
        assert np.array_equal(res['ae64'][a0:a1].view(np.uint64), ae64.view(np.uint64)), s['name']
        assert abs(res['energy'][b] - e) <= E_ATOL, (s['name'], res['energy'][b] - e)
        fs = max(1.0, float(np.abs(f).max())) if len(f) else 1.0
        assert np.abs(res['forces'][a0:a1] - f).max(initial=0.0) <= F_RTOL * fs, s['name']
        vs = max(1.0, float(np.abs(v).max()))
        assert np.abs(res['virial'][b] - v).max() <= V_RTOL * vs, (s['name'], res['virial'][b], v)


def test_per_structure_results_match_structures_alone(eng, meta):
    structs = mixed_batch()
    a, res = _batch_results(eng, structs)
    assert res['energy'].dtype == np.float64 and res['virial'].shape == (len(structs), 6)
    _check_against_alone(eng, meta, structs, a, res, range(len(structs)))
    # empty structures: exactly zero energy and virial
    for b, s in enumerate(structs):
        if s['name'].startswith('empty'):
            assert res['energy'][b] == 0.0 and not res['virial'][b].any()


def test_order_and_repetition_do_not_change_bits(eng, meta):
    structs = mixed_batch()
    a, r1 = _batch_results(eng, structs)
    _, r2 = _batch_results(eng, structs)
    assert np.array_equal(r1['energy'].view(np.uint64), r2['energy'].view(np.uint64))     # fixed summation order
    rev = structs[::-1]
    ar, r3 = _batch_results(eng, rev)
    B = len(structs)
    for b in range(B):
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        c0, c1 = ar['atom_ptr'][B - 1 - b], ar['atom_ptr'][B - b]
        assert np.array_equal(r1['atomic_energy'][a0:a1].view(np.uint32), r3['atomic_energy'][c0:c1].view(np.uint32))
        assert np.array_equal(r1['ae64'][a0:a1].view(np.uint64), r3['ae64'][c0:c1].view(np.uint64))


def test_scale_520_structures(eng, meta):
    """512 rattled 64-atom Si cells and 8 cells of 1 000 atoms in one batch; a random sample checked against the
    structures alone, and the launches of the build do not depend on B"""
    structs = si_cells(512, 1000) + si_cells(8, 5000, reps=(5, 5, 5))
    order = np.random.RandomState(7).permutation(len(structs))
    structs = [structs[i] for i in order]
    a, res = _batch_results(eng, structs)
    assert res['energy'].shape == (520,)
    sample = np.random.RandomState(11).choice(len(structs), 16, replace=False)
    big = [b for b in range(len(structs)) if len(structs[b]['numbers']) == 1000][:2]
    _check_against_alone(eng, meta, structs, a, res, sorted(set(sample.tolist()) | set(big)))

    def build_launches(ss):
        _set_batch(eng, meta, ss)                  # sizes the buffers, so that both timed builds reuse them
        eng.launch_count(reset=True)
        _set_batch(eng, meta, ss)
        return eng.launch_count()
    assert build_launches(structs[:2]) == build_launches(structs)


def _state(structs, pos_dtype='float32', device='cuda', pbc=True):
    import torch
    a = _arrays(structs)
    return types.SimpleNamespace(
        positions=torch.tensor(a['positions'], dtype=getattr(torch, pos_dtype), device=device),
        row_vector_cell=torch.tensor(a['cells'], dtype=getattr(torch, pos_dtype), device=device),
        pbc=torch.tensor(pbc, device=device) if not isinstance(pbc, bool) else pbc,
        atomic_numbers=torch.tensor(a['numbers'], device=device),
        system_idx=torch.tensor(a['system_idx'], device=device))


def test_sevennet_model_replays_the_captured_step(meta):
    import torch
    from sevenn_b200.batch import SevenNetModel
    model = SevenNetModel('7net-0', device='cuda')
    structs = si_cells(64, 300)
    state = _state(structs, 'float64')
    model(state)
    n_edges0 = model.engine.n_edges
    c0, r0 = model.engine.graph_stats()
    g = torch.Generator(device='cuda').manual_seed(5)
    state.positions = state.positions + 0.02 * torch.randn(state.positions.shape, generator=g, device='cuda',
                                                         dtype=torch.float64)
    out = model(state)
    torch.cuda.synchronize()
    assert model.engine.n_edges != n_edges0          # the neighbour count drifted ...
    assert model.engine.graph_stats() == (c0, r0 + 1)   # ... inside the headroom: no new capture, one more replay
    moved = [dict(s, positions=p) for s, p in zip(structs, np.split(state.positions.cpu().numpy(), 64))]
    a = _arrays(moved)
    res = dict(energy=out['energy'].double().cpu().numpy(), forces=out['forces'].cpu().numpy())
    for b in (0, 17, 63):
        e, ae, _, f, _ = _alone_results(model.engine, meta, moved[b])
        assert abs(res['energy'][b] - e) <= 1e-5 * max(1.0, abs(e))     # float32 energy out
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        assert np.abs(res['forces'][a0:a1] - f).max() <= F_RTOL * max(1.0, float(np.abs(f).max()))


@pytest.mark.parametrize('pos_dtype,device,pbc', [('float32', 'cuda', True), ('float64', 'cuda', [True, True, True]),
                                                  ('float32', 'cpu', True)])
def test_torchsim_adapter_matches_batched_evaluator_and_golden(eng, pos_dtype, device, pbc):
    import torch
    from sevenn_b200.batch import BatchedEvaluator, SevenNetModel
    keys = ['7net0_nacl_rattled', '7net0_hfo2_0', '7net0_hfo2_1']
    structs = [_golden(k) for k in keys]
    model = SevenNetModel('7net-0', device='cuda')
    out = model(_state(structs, pos_dtype, device, pbc))
    e, f, st = (out[k].cpu().numpy() for k in ('energy', 'forces', 'stress'))
    rnd = lambda x: x.astype(getattr(np, pos_dtype)).astype(np.float64)     # what the model is given
    rounded = [dict(numbers=s['numbers'], cell=rnd(s['cell']), pbc=True, positions=rnd(s['positions'])) for s in structs]
    ev = BatchedEvaluator(eng)
    ref = ev.split(ev.compute(rounded))
    a = 0
    for b, (k, r) in enumerate(zip(keys, ref)):
        g = golden_vectors()[k]
        n = len(r['forces'])
        # BatchedEvaluator sums fp32 per-atom energies; the model returns float32 energies of the fp64 sum
        assert abs(e[b] - r['energy']) < 2e-5 * max(1.0, abs(r['energy'])), k
        assert np.allclose(f[a:a + n], r['forces'], atol=2e-5), k
        assert abs(e[b] - g['energy']) < max(g['atol']['energy'], 1e-4), k     # the reference's own numbers
        assert np.allclose(f[a:a + n], g['forces'], atol=2e-4), k
        assert np.allclose(st[b], st[b].T)
        a += n
    v = golden_vectors()['7net0_nacl_rattled']['ase_stress']   # ASE Voigt (xx,yy,zz,yz,xz,xy)
    full = np.array([[v[0], v[5], v[4]], [v[5], v[1], v[3]], [v[4], v[3], v[2]]])
    assert np.allclose(st[0], full, atol=2e-5)


def test_errors_leave_the_current_graph_alone(eng, meta):
    import torch
    from sevenn_b200.batch import DeviceBatch
    structs = [_golden('7net0_nacl_rattled'), _golden('7net0_hfo2_0')]
    _set_batch(eng, meta, structs)
    before, n_before = _csr(eng), (eng.n_nodes, eng.n_edges)
    a = _arrays(structs)
    db = DeviceBatch(eng)
    pos = torch.tensor(a['positions'], device='cuda')
    z = a['numbers'].copy()
    z[3] = 118
    with pytest.raises(ValueError, match='118'):
        db.set_batch(z, pos, a['cells'], a['pbc'], a['system_idx'])
    with pytest.raises(ValueError, match='sorted'):
        db.set_batch(a['numbers'], pos, a['cells'], a['pbc'], a['system_idx'][::-1].copy())
    cells = a['cells'].copy()
    cells[1, 1] = cells[1, 0]                          # two equal lattice vectors, periodic
    with pytest.raises(RuntimeError, match=r'singular cell \(structure 1\)'):
        db.set_batch(a['numbers'], pos, cells, a['pbc'], a['system_idx'])
    n = a['atom_ptr'][-1]
    bad = np.array([0, n, 1, n], dtype=np.int32)       # decreasing, same total
    with pytest.raises(RuntimeError, match='non-decreasing'):
        eng.set_positions_batch(species_of(meta, a['numbers']), pos, bad, np.concatenate([a['cells'], a['cells'][:1]]),
                                True)
    assert (eng.n_nodes, eng.n_edges) == n_before and _same_csr(_csr(eng), before)
    eng.compute_positions(species_of(meta, structs[0]['numbers']), structs[0]['positions'], structs[0]['cell'], True)
    with pytest.raises(RuntimeError, match='set_positions_batch'):
        eng.system_results()
