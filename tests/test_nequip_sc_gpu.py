"""The species-wise ('nequip') self-connection on the GPU: the species-segmented linear (C ABI s7b_species_linear)
against numpy fp64, and models with it (synthetic architectures A, B and C = SevenNet-0 widths, tests/
synthetic_nequip.py) against the fp64 oracle through every public interface.  Bounds are those of
test_architectures_gpu.py."""
import ctypes
import os
import struct
import subprocess
import types

import numpy as np
import pytest

from helpers import ROOT, first_divergence, format_stage_errors, stage_errors
from nequip_oracle import nequip_oracle
from synthetic_models import convert as convert_linear, write_checkpoint
from synthetic_nequip import S, convert, write_nequip_checkpoint

pytestmark = pytest.mark.gpu


# ---- s7b_species_linear against numpy -------------------------------------------------------------------------
def _species_linear(A, species, n_species, a_K, c_N, W, C0=None, accumulate=False):
    """A [n, sum (2l+1) K_l] (cm layout), W [S][l] blocks [K_l, N_l] -> C [n, sum (2l+1) N_l] from the GPU"""
    import torch
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    n_l = len(a_K)
    a_off = np.cumsum([0] + [(2 * l + 1) * k for l, k in enumerate(a_K)]).astype(np.int32)
    c_off = np.cumsum([0] + [(2 * l + 1) * k for l, k in enumerate(c_N)]).astype(np.int32)
    dA, dC = int(a_off[-1]), int(c_off[-1])
    flat = np.ascontiguousarray(np.concatenate([W[s][l].ravel() for s in range(n_species) for l in range(n_l)]), np.float32)
    At = torch.tensor(A, dtype=torch.float32, device='cuda').reshape(-1, dA).contiguous()
    Ct = (torch.zeros(len(species), dC, device='cuda') if C0 is None else torch.tensor(C0, dtype=torch.float32, device='cuda')).contiguous()
    sp = torch.tensor(np.asarray(species, np.int32), device='cuda')
    i32 = lambda v: np.ascontiguousarray(v, np.int32)
    ao, ak, co, cn = i32(a_off[:-1]), i32(a_K), i32(c_off[:-1]), i32(c_N)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.s7b_species_linear(At.data_ptr(), dA, len(species), sp.data_ptr(), n_species, n_l, ao.ctypes.data, ak.ctypes.data,
                                 flat.ctypes.data, Ct.data_ptr(), dC, co.ctypes.data, cn.ctypes.data, int(accumulate), st))
    torch.cuda.synchronize()
    return Ct.cpu().numpy(), a_off, c_off


def _reference(A, species, a_K, c_N, W, a_off, c_off, C0=None):
    n = len(species)
    C = np.zeros((n, int(c_off[-1]))) if C0 is None else C0.astype(np.float64).copy()
    bound = np.zeros_like(C)
    for l, (K, N) in enumerate(zip(a_K, c_N)):
        d = 2 * l + 1
        Ab = A[:, a_off[l]:a_off[l + 1]].reshape(n, d, K).astype(np.float64)
        Wn = np.stack([W[s][l] for s in species]).astype(np.float64)          # [n, K, N]
        C[:, c_off[l]:c_off[l + 1]] += np.einsum('nik,nkj->nij', Ab, Wn).reshape(n, d * N)
        bound[:, c_off[l]:c_off[l + 1]] = np.einsum('nik,nkj->nij', np.abs(Ab), np.abs(Wn)).reshape(n, d * N)
    return C, bound


def _species_of(case, n, n_species, rng):
    if case == 'mixed':
        return rng.randint(0, n_species, size=n)
    if case == 'all_one':                 # every atom of the last species: the others have none
        return np.full(n, n_species - 1)
    # S >= 3: species 0 has no atom, species 1 exactly one, the rest random; S = 2: species 0 exactly one
    if n_species == 1:
        return np.zeros(n, int)
    if n_species == 2:
        sp = np.ones(n, int)
        sp[n // 2] = 0
        return sp
    sp = rng.randint(2, n_species, size=n)
    sp[n // 2] = 1
    return sp


@pytest.mark.parametrize('case', ['mixed', 'all_one', 'empty_and_single'])
@pytest.mark.parametrize('n_species', [1, 2, 7, 89])
@pytest.mark.parametrize('width', [32, 96, 256, 1024])
def test_species_linear_against_numpy(width, n_species, case):
    rng = np.random.RandomState(width + n_species)
    n = 131 if width < 1024 else 70
    a_K, c_N = [width, 32, 64], [64, width, 32]
    W = [[rng.standard_normal((k, m)).astype(np.float32) / np.sqrt(k) for k, m in zip(a_K, c_N)] for _ in range(n_species)]
    sp = _species_of(case, n, n_species, rng)
    A = rng.standard_normal((n, sum((2 * l + 1) * k for l, k in enumerate(a_K)))).astype(np.float32)
    C, a_off, c_off = _species_linear(A, sp, n_species, a_K, c_N, W)
    ref, bound = _reference(A, sp, a_K, c_N, W, a_off, c_off)
    assert np.all(np.abs(C - ref) <= 2e-6 * bound + 1e-7), float(np.abs(C - ref).max())
    # accumulate onto C0
    C0 = rng.standard_normal(C.shape).astype(np.float32)
    Cacc, _, _ = _species_linear(A, sp, n_species, a_K, c_N, W, C0=C0, accumulate=True)
    ref_acc, _ = _reference(A, sp, a_K, c_N, W, a_off, c_off, C0=C0)
    assert np.all(np.abs(Cacc - ref_acc) <= 2e-6 * bound + 1e-6), float(np.abs(Cacc - ref_acc).max())
    # the transposed form (the backward's sc^T: blocks [N, K], A in the output layout)
    WT = [[w.T.copy() for w in Ws] for Ws in W]
    B = rng.standard_normal((n, C.shape[1])).astype(np.float32)
    CT, b_off, d_off = _species_linear(B, sp, n_species, c_N, a_K, WT)
    refT, boundT = _reference(B, sp, c_N, a_K, WT, b_off, d_off)
    assert np.all(np.abs(CT - refT) <= 2e-6 * boundT + 1e-7), float(np.abs(CT - refT).max())
    # a row's result does not depend on the other rows: the first 37 rows alone give the same bits; and reruns agree
    C37, _, _ = _species_linear(A[:37], sp[:37], n_species, a_K, c_N, W)
    assert np.array_equal(C37.view(np.uint32), C[:37].view(np.uint32))
    C2, _, _ = _species_linear(A, sp, n_species, a_K, c_N, W)
    assert np.array_equal(C2.view(np.uint32), C.view(np.uint32))


def test_species_linear_no_rows_and_bad_shapes():
    from sevenn_b200.engine import check, load_library
    rng = np.random.RandomState(0)
    W = [[rng.standard_normal((32, 32)).astype(np.float32)] for _ in range(3)]
    C, _, _ = _species_linear(np.zeros((0, 32), np.float32), np.zeros(0, int), 3, [32], [32], W)
    assert C.shape == (0, 32)
    lib = load_library()
    i32 = lambda v: np.ascontiguousarray(v, np.int32)
    z, k = i32([0]), i32([30])
    w = np.zeros(3 * 30 * 30, np.float32)
    with pytest.raises(RuntimeError, match='multiples of 4'):
        import torch
        buf = torch.zeros(8, 32, device='cuda')
        sp = torch.zeros(8, dtype=torch.int32, device='cuda')
        check(lib.s7b_species_linear(buf.data_ptr(), 32, 8, sp.data_ptr(), 3, 1, z.ctypes.data, k.ctypes.data, w.ctypes.data,
                                     buf.data_ptr(), 32, z.ctypes.data, k.ctypes.data, 0, None))


# ---- models ----------------------------------------------------------------------------------------------------
ARCHS = ['A', 'B', 'C']


@pytest.fixture(scope='module')
def models(tmp_path_factory):
    d = tmp_path_factory.mktemp('nequip_ckpt')
    out = {}
    for i, arch in enumerate(ARCHS):
        path = write_nequip_checkpoint(d / f'synthetic_{arch}_nequip.pth', arch, seed=10 + i)
        out[arch] = (path,) + convert(path, arch)
    return out


@pytest.fixture(scope='module')
def engines(models):
    from sevenn_b200.engine import B200Engine
    cache = {}

    def get(arch):
        if arch not in cache:
            cache[arch] = B200Engine(models[arch][1], models[arch][2], radial='table')
        return cache[arch]
    return get


def _mixed_si64(seed=4):
    """64-atom rattled diamond cell with species drawn from all S species"""
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, _ = diamond_si(2, 2, 2, sigma=0.05, seed=seed)
    ei, ev = build_graph(pos, cell, True, 5.0)
    return np.random.RandomState(seed).randint(0, S, size=len(pos)), ei, ev, abs(np.linalg.det(cell))


def _run(e, species, ei, ev):
    import torch
    e.set_graph(species, ei, ev)
    e.compute()
    torch.cuda.synchronize()
    r = e.results()
    return dict(energy=float(r['energy'].cpu()[0]), atomic_energy=r['atomic_energy'].cpu().numpy(),
                forces=r['forces'].cpu().numpy(), virial=r['virial'].cpu().numpy())


def _check(out, ref, n_atoms):
    f_ref = ref['forces'].numpy()
    fs = max(1.0, float(np.abs(f_ref).max()) / 5.0)
    es = max(1.0, float(np.abs(ref['atomic_energy'].numpy()).max()) / 10.0)
    assert abs(out['energy'] - float(ref['energy'])) <= 1e-4 * es * max(1.0, n_atoms / 64.0)
    assert np.allclose(out['atomic_energy'], ref['atomic_energy'].numpy(), atol=2e-5 * es, rtol=0)
    assert np.allclose(out['forces'], f_ref, atol=5e-5 * fs, rtol=0), float(np.abs(out['forces'] - f_ref).max())
    assert np.allclose(out['virial'], ref['virial'].numpy(), atol=5e-4 * fs, rtol=1e-5)


@pytest.mark.parametrize('system', ['si64', 'tiny_cell', 'hub'])
@pytest.mark.parametrize('arch', ARCHS)
def test_against_oracle(models, engines, arch, system):
    import graphs
    _, meta, arrays = models[arch]
    if system == 'si64':
        sp, ei, ev, vol = _mixed_si64()
    else:
        g = graphs.build(system, meta)
        sp, ei, ev, vol = g.species, g.edge_index, g.edge_vec, g.volume
    out = _run(engines(arch), sp, ei, ev)
    ref = nequip_oracle(meta, arrays).forward(sp, ei, ev, volume=vol)
    _check(out, ref, len(sp))


@pytest.mark.parametrize('arch', ARCHS)
def test_stage_errors_per_layer(models, engines, arch):
    _, meta, arrays = models[arch]
    sp, ei, ev, _ = _mixed_si64(seed=6)
    ref = nequip_oracle(meta, arrays).forward(sp, ei, ev, keep=True)
    errs = stage_errors(engines(arch), arrays, sp, ei, ev, ref=ref)
    assert first_divergence(errs) is None, format_stage_errors(errs)


@pytest.mark.parametrize('arch', ['A', 'C'])
def test_equivalent_to_linear_engine(tmp_path, arch):
    """the sqrt(S) M checkpoint on the species path against the linear-SC engine with M"""
    from sevenn_b200.engine import B200Engine
    meta_l, arr_l = convert_linear(write_checkpoint(tmp_path / 'l.pth', arch, seed=3), arch)
    meta_n, arr_n = convert(write_nequip_checkpoint(tmp_path / 'n.pth', arch, seed=3, sc='from_linear'), arch)
    sp, ei, ev, _ = _mixed_si64(seed=8)
    a = _run(B200Engine(meta_l, arr_l), sp, ei, ev)
    b = _run(B200Engine(meta_n, arr_n), sp, ei, ev)
    fs = max(1.0, float(np.abs(a['forces']).max()) / 5.0)
    assert abs(a['energy'] - b['energy']) <= 1e-4
    assert np.allclose(a['atomic_energy'], b['atomic_energy'], atol=2e-5, rtol=0)
    assert np.allclose(a['forces'], b['forces'], atol=5e-5 * fs, rtol=0)


def _structs(meta):
    import graphs
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    out = []
    for i, reps in enumerate([(1, 1, 1), (2, 1, 1), (2, 2, 1)]):
        pos, cell, z = diamond_si(*reps, sigma=0.05, seed=i)
        out.append(dict(numbers=z, positions=pos, cell=cell, pbc=(True, True, True)))
    pos, cell, z = rocksalt_nacl(1, 1, 2, sigma=0.1, seed=3)
    out.append(dict(numbers=z, positions=pos, cell=cell, pbc=(True, True, True)))
    g = graphs.build('tiny_cell', meta)
    out.append(dict(numbers=g.numbers, positions=g.positions, cell=g.cell, pbc=g.pbc))
    g = graphs.build('isolated', meta)
    out.append(dict(numbers=g.numbers, positions=g.positions, cell=g.cell, pbc=g.pbc))
    return out


def _flat(structs):
    return dict(numbers=np.concatenate([s['numbers'] for s in structs]),
                positions=np.concatenate([s['positions'] for s in structs]),
                cells=np.stack([s['cell'] for s in structs]),
                pbc=np.array([s['pbc'] for s in structs]),
                system_idx=np.concatenate([np.full(len(s['numbers']), b) for b, s in enumerate(structs)]),
                atom_ptr=np.cumsum([0] + [len(s['numbers']) for s in structs]))


def test_device_batch_members_and_replay_with_new_species(models):
    """every member equals the structure alone, bit for bit per atom; a second call with the same sizes but other
    species replays the captured step and equals a fresh engine"""
    import torch
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.engine import B200Engine
    from synthetic_models import NUMBERS
    _, meta, arrays = models['A']
    eng = B200Engine(meta, arrays)
    structs = _structs(meta)
    a = _flat(structs)
    rng = np.random.RandomState(3)
    numbers = np.array(NUMBERS)[rng.randint(0, S, size=len(a['numbers']))]     # every species, mixed
    pos = torch.tensor(a['positions'], device='cuda')
    si = torch.tensor(a['system_idx'], device='cuda')
    res = DeviceBatch(eng).compute(numbers, pos, a['cells'], a['pbc'], si)
    ae_b = res['atomic_energy'].cpu().numpy()
    tm = eng.spec.type_map
    for b, s in enumerate(structs):
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        sp = np.array([tm[int(z)] for z in numbers[a0:a1]], dtype=np.int32)
        e, ae, f, v, _ = eng.compute_positions(sp, s['positions'], s['cell'], s['pbc'])
        assert np.array_equal(ae_b[a0:a1].view(np.uint32), np.asarray(ae, np.float32).view(np.uint32)), b
        assert abs(float(res['energy'][b]) - e) <= 1e-9 * max(1.0, abs(e))
        fs = max(1.0, float(np.abs(f).max()))
        assert np.abs(res['forces'][a0:a1].cpu().numpy() - f).max(initial=0.0) <= 1e-5 * fs

    eng2 = B200Engine(meta, arrays)
    db = DeviceBatch(eng2)
    db.compute(numbers, pos, a['cells'], a['pbc'], si)
    c0, r0 = eng2.graph_stats()
    numbers2 = np.array(NUMBERS)[rng.randint(0, S, size=len(numbers))]
    assert (numbers2 != numbers).any()
    out = db.compute(numbers2, pos, a['cells'], a['pbc'], si)
    torch.cuda.synchronize()
    assert eng2.graph_stats() == (c0, r0 + 1)                    # replayed, not re-captured
    fresh = DeviceBatch(B200Engine(meta, arrays)).compute(numbers2, pos, a['cells'], a['pbc'], si)
    assert np.array_equal(out['atomic_energy'].cpu().numpy().view(np.uint32), fresh['atomic_energy'].cpu().numpy().view(np.uint32))
    fs = max(1.0, float(fresh['forces'].abs().max()))
    assert float((out['forces'] - fresh['forces']).abs().max()) <= 1e-5 * fs
    # and the replayed result is the model's: the oracle on one member
    o = nequip_oracle(meta, arrays)
    from sevenn_b200.neighbors import build_graph
    b = 2
    a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
    ei, ev = build_graph(a['positions'][a0:a1], a['cells'][b], True, 5.0)
    ref = o.forward(np.array([tm[int(z)] for z in numbers2[a0:a1]]), ei, ev)
    assert abs(float(out['energy'][b]) - float(ref['energy'])) <= 1e-4


def test_sevennet_model(models):
    import torch
    from sevenn_b200.batch import SevenNetModel
    from sevenn_b200.neighbors import build_graph
    _, meta, arrays = models['B']
    model = SevenNetModel((meta, arrays), device='cuda')
    structs = _structs(meta)[:4]
    a = _flat(structs)
    state = types.SimpleNamespace(
        positions=torch.tensor(a['positions'], device='cuda'), row_vector_cell=torch.tensor(a['cells'], device='cuda'),
        pbc=True, atomic_numbers=torch.tensor(a['numbers'], device='cuda'),
        system_idx=torch.tensor(a['system_idx'], device='cuda'))
    out = model(state)
    torch.cuda.synchronize()
    o = nequip_oracle(meta, arrays)
    for b in (0, 3):
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        ei, ev = build_graph(a['positions'][a0:a1], a['cells'][b], True, 5.0)
        ref = o.forward(np.array([model.type_map[int(z)] for z in a['numbers'][a0:a1]]), ei, ev)
        assert abs(float(out['energy'][b]) - float(ref['energy'])) <= 1e-4
        fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
        assert np.allclose(out['forces'][a0:a1].cpu().numpy(), ref['forces'].numpy(), atol=5e-5 * fs, rtol=0)


def _split_sequence(eng, T):
    from sevenn_b200 import engine as E
    eng.run_stage(E.STAGE_FWD_BEGIN)
    for t in range(T):
        if t == 0:
            eng.run_stage(E.STAGE_FWD_LAYER_A, t)
        else:
            eng.run_stage(E.STAGE_FWD_CONV_INTERIOR, t)
            eng.run_stage(E.STAGE_FWD_LAYER_A2, t)
        eng.run_stage(E.STAGE_FWD_LAYER_SC, t)
    eng.run_stage(E.STAGE_FWD_END)
    for t in range(T - 1, -1, -1):
        if t == 0:
            eng.run_stage(E.STAGE_BWD_LAYER_A, t)
            continue
        eng.run_stage(E.STAGE_BWD_LAYER_A1, t)
        eng.run_stage(E.STAGE_BWD_LAYER_A2, t)
        eng.run_stage(E.STAGE_BWD_LAYER_B1, t)
        eng.run_stage(E.STAGE_BWD_LAYER_B2, t)
    eng.run_stage(E.STAGE_BWD_END)


def _results(eng):
    return {k: v.cpu().numpy().copy() for k, v in eng.results().items() if hasattr(v, 'cpu')}


def _same(split, full):
    assert np.array_equal(split['atomic_energy'].view(np.uint32), full['atomic_energy'].view(np.uint32))
    fs = max(1.0, float(np.abs(full['forces']).max()))
    assert np.abs(split['forces'] - full['forces']).max() <= 1e-5 * fs
    vs = max(1.0, float(np.abs(full['virial']).max()))
    assert np.abs(split['virial'] - full['virial']).max() <= 1e-5 * vs


def test_split_stages_and_stage_graphs(models):
    """the interior / boundary split stages against s7b_engine_compute, directly and as per-stage CUDA graphs;
    replayed stage graphs with new species in the same buffer equal a fresh engine"""
    import torch
    from sevenn_b200.engine import B200Engine, set_option
    from sevenn_b200.neighbors import diamond_si
    _, meta, arrays = models['A']
    eng = B200Engine(meta, arrays)
    pos, cell, _ = diamond_si(3, 2, 2, sigma=0.05, seed=2)
    rng = np.random.RandomState(1)
    sp = rng.randint(0, S, size=len(pos)).astype(np.int32)
    T = eng.spec.n_layers

    def full(species):
        e = B200Engine(meta, arrays)
        e.set_positions(species, pos, cell, True)
        e.compute()
        torch.cuda.synchronize()
        return _results(e)

    ref = full(sp)
    eng.set_positions(sp, pos, cell, True)
    eng.set_interior(len(pos) // 3)
    _split_sequence(eng, T)
    torch.cuda.synchronize()
    _same(_results(eng), ref)
    try:
        set_option('stage_graphs', 1)
        for _ in range(2):
            _split_sequence(eng, T)
        torch.cuda.synchronize()
        _same(_results(eng), ref)
        captures, replays = eng.stage_graph_stats()
        assert captures > 0 and replays >= captures
        sp2 = rng.randint(0, S, size=len(pos)).astype(np.int32)
        eng.set_positions(sp2, pos, cell, True)
        eng.set_interior(len(pos) // 3)
        _split_sequence(eng, T)
        torch.cuda.synchronize()
        assert eng.stage_graph_stats()[0] == captures                  # replayed with the new species
        _same(_results(eng), full(sp2))
    finally:
        set_option('stage_graphs', 0)


class _Atoms:
    def __init__(self, numbers, positions, cell, pbc):
        self.numbers, self.positions, self.cell, self.pbc = numbers, positions, cell, pbc

    def get_positions(self):
        return self.positions

    def get_cell(self):
        return self.cell

    def get_pbc(self):
        return np.asarray(self.pbc)

    def get_atomic_numbers(self):
        return self.numbers


def test_calculator_from_nequip_checkpoint(models):
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import build_graph, rocksalt_nacl
    path, meta, arrays = models['C']
    calc = SevenNetCalculator(model=path)
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.1, seed=1)
    calc.calculate(_Atoms(z, pos, cell, (True, True, True)))
    ei, ev = build_graph(pos, cell, True, 5.0)
    sp = np.array([calc.type_map[int(a)] for a in z])
    ref = nequip_oracle(meta, arrays).forward(sp, ei, ev, volume=abs(np.linalg.det(cell)))
    out = dict(energy=calc.results['energy'], atomic_energy=calc.results['energies'], forces=calc.results['forces'],
               virial=ref['virial'].numpy())
    _check(out, ref, len(z))


def test_export_flat_and_cpp_host(models, tmp_path):
    from sevenn_b200.export import export_flat
    from sevenn_b200.neighbors import build_graph, diamond_si
    from synthetic_models import NUMBERS
    _, meta, arrays = models['A']
    exe = str(tmp_path / 'host_entry')
    lib_dir = os.path.join(ROOT, 'sevenn_b200', 'lib')
    subprocess.check_call(['g++', '-O1', '-std=c++17', os.path.join(ROOT, 'examples', 'host_entry.cpp'), '-o', exe,
                           f'-L{lib_dir}', '-lsevenn_b200', f'-Wl,-rpath,{lib_dir}'])
    model = str(tmp_path / 'synthetic_A_nequip.s7b')
    export_flat(model, meta, arrays)
    pos, cell, _ = diamond_si(2, 2, 2, sigma=0.05, seed=9)
    z = np.array(NUMBERS, np.int32)[np.random.RandomState(9).randint(0, S, size=len(pos))]
    ei, ev = build_graph(pos, cell, True, 5.0)
    path = str(tmp_path / 'graph.bin')
    with open(path, 'wb') as f:
        f.write(struct.pack('<iq', len(z), ei.shape[1]))
        f.write(z.tobytes() + ei[0].astype(np.int32).tobytes() + ei[1].astype(np.int32).tobytes()
                + ev.astype(np.float32).tobytes())
    out = subprocess.run([exe, model, path], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    lines = out.stdout.strip().splitlines()
    energy = float(lines[0])
    forces = np.array([[float(v) for v in l.split()] for l in lines[1:1 + len(z)]])
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    ref = nequip_oracle(meta, arrays).forward(np.array([tm[int(a)] for a in z]), ei, ev)
    fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
    assert abs(energy - float(ref['energy'])) < 1e-4
    assert np.allclose(forces, ref['forces'].numpy(), atol=5e-5 * fs)


def test_engine_refuses_mixed_or_missized_self_connection(models):
    from sevenn_b200.engine import B200Engine, check
    _, meta, arrays = models['B']
    eng = B200Engine(meta, arrays)
    w = np.zeros(10, np.float32)
    with pytest.raises(RuntimeError, match='layer 1.*sc_species'):
        check(eng.lib.s7b_engine_set_param(eng._h, b'sc_species', 1, w.ctypes.data, w.size))
    with pytest.raises(RuntimeError, match='cannot both be set'):
        check(eng.lib.s7b_engine_set_param(eng._h, b'sc', 1, w.ctypes.data, w.size))
