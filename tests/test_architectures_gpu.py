"""Models other than SevenNet-0 / SevenNet-l3i5 on the GPU: the synthetic architectures A-D of
tests/synthetic_models.py (other widths, lmax_edge != lmax_node, lmax 1) through every public interface, and the
convolution plug-in at every (lmax_filter, lmax_out) group and width, all against the fp64 oracle.

Bounds are those test_engine_gpu.py uses for SevenNet-0 on the 64-atom Si cell (energy 1e-4 eV, per-atom energy
2e-5 eV, forces 5e-5 eV/A, virial 5e-4 eV + 1e-5 relative), widened in proportion to the size of the reference
quantity where the synthetic model's forces or energies are larger than SevenNet-0's (|F| ~ 5 eV/A)."""
import os
import struct
import subprocess
import types

import numpy as np
import pytest

import graphs
from helpers import ROOT, first_divergence, format_stage_errors, oracle, stage_errors
from synthetic_models import ARCHS, convert, write_checkpoint

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def models(tmp_path_factory):
    """arch -> (checkpoint path, meta, arrays), converted from the reference checkpoint layout"""
    d = tmp_path_factory.mktemp('arch_ckpt')
    out = {}
    for i, arch in enumerate(sorted(ARCHS)):
        path = write_checkpoint(d / f'synthetic_{arch}.pth', arch, seed=i)
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


def _oracle(meta, arrays):
    import torch
    from oracle.oracle import Oracle
    return Oracle(meta, arrays, dtype=torch.float64)


def _si64(meta):
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    ei, ev = build_graph(pos, cell, True, 5.0)
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z]), ei, ev, abs(np.linalg.det(cell))


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
@pytest.mark.parametrize('arch', sorted(ARCHS))
def test_against_oracle(models, engines, arch, system):
    _, meta, arrays = models[arch]
    if system == 'si64':
        sp, ei, ev, vol = _si64(meta)
    else:
        g = graphs.build(system, meta)         # triclinic cell below the cutoff / non-periodic hub with empty rows
        sp, ei, ev, vol = g.species, g.edge_index, g.edge_vec, g.volume
    out = _run(engines(arch), sp, ei, ev)
    ref = _oracle(meta, arrays).forward(sp, ei, ev, volume=vol)
    _check(out, ref, len(sp))


def test_stage_errors_per_layer(models, engines):
    _, meta, arrays = models['C']
    sp, ei, ev, _ = _si64(meta)
    ref = _oracle(meta, arrays).forward(sp, ei, ev, keep=True)
    errs = stage_errors(engines('C'), arrays, sp, ei, ev, ref=ref)
    assert first_divergence(errs) is None, format_stage_errors(errs)


# ---- the convolution plug-in ----------------------------------------------------------------------------------
WIDTHS = (32, 64, 96, 128, 256)
GROUPS = [(lf, lo) for lf in (1, 2, 3) for lo in range(4)]


def _plugin_case(lf, lo, k):
    """x irreps l = 0..3 with widths drawn from WIDTHS (a different draw per group and k)"""
    rng = np.random.RandomState(10 * lf + lo + 100 * k)
    return [int(v) for v in rng.choice(WIDTHS, size=4)]


def _plugin_compare(x_muls, lf, lo, deg, seed):
    import torch
    from sevenn_b200.conv_op import B200Convolution
    from sevenn_b200.sh import spherical_harmonics
    from sevenn_b200.spec import build_layer
    from sevenn_b200.cg import tp_path_coefficients
    L = build_layer(0, x_muls, [32] * (lo + 1), lf)
    o = oracle('sevennet_0')
    for p in L.paths:        # coupling tensors of the paths SevenNet-0 does not have
        o.cg.setdefault((p.l1, p.l2, p.l3), torch.as_tensor(tp_path_coefficients(p.l1, p.l2, p.l3), dtype=o.dtype))
    rng = np.random.RandomState(seed)
    n, E = len(deg), int(deg.sum())
    dst = np.repeat(np.arange(n), deg)[rng.permutation(E)]
    src = rng.randint(0, n, size=E)
    x = rng.normal(size=(n, L.dim_x))
    sh = spherical_harmonics(lf, rng.normal(size=(E, 3)))
    w = rng.normal(size=(E, L.weight_numel))
    gout = rng.normal(size=(n, L.dim_mid))
    fan = max(np.bincount(dst).max(), np.bincount(src).max())
    g = max(1.0, np.sqrt(fan / 12.0))

    irr = lambda muls: '+'.join(f'{m}x{l}e' for l, m in enumerate(muls))
    mid = '+'.join(f'{p.mul}x{p.l3}e' for p in L.paths)
    inst = [(p.l1, p.l2, p.slot, 'uvu', True) for p in L.paths]
    conv = B200Convolution(irr(x_muls), irr([1] * (lf + 1)), mid, inst, shared_weights=False,
                           internal_weights=False).cuda()
    xt, sht, wt = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (x, sh, w))
    msg = o.tensor_product(L, xt[torch.as_tensor(src)], sht, wt)
    ref = torch.zeros(n, L.dim_mid, dtype=torch.float64).index_add_(0, torch.as_tensor(dst), msg)
    (ref * torch.as_tensor(gout)).sum().backward()
    xc, shc, wc = (torch.tensor(a, dtype=torch.float32, device='cuda', requires_grad=True) for a in (x, sh, w))
    out = conv(xc, shc, wc, torch.as_tensor(src, device='cuda', dtype=torch.int32),
               torch.as_tensor(dst, device='cuda', dtype=torch.int32))
    assert np.allclose(out.detach().cpu().numpy(), ref.detach().numpy(), atol=2e-4 * g, rtol=1e-5)
    (out * torch.as_tensor(gout, device='cuda', dtype=torch.float32)).sum().backward()
    assert np.allclose(xc.grad.cpu().numpy(), xt.grad.numpy(), atol=5e-4 * g, rtol=1e-4)
    assert np.allclose(wc.grad.cpu().numpy(), wt.grad.numpy(), atol=5e-4, rtol=1e-4)
    gsh_ref = sht.grad.numpy().copy()
    gsh_ref[:, 0] = 0.0
    assert np.allclose(shc.grad.cpu().numpy(), gsh_ref, atol=2e-3 * g, rtol=1e-4)


@pytest.mark.parametrize('k', [0, 1])
@pytest.mark.parametrize('lf,lo', GROUPS)
def test_plugin_every_group(lf, lo, k):
    rng = np.random.RandomState(k)
    deg = rng.randint(0, 24, size=41)
    deg[-1] = 0
    _plugin_compare(_plugin_case(lf, lo, k), lf, lo, deg, seed=lf * 10 + lo)


@pytest.mark.parametrize('pattern', ['ragged', 'hub'])
@pytest.mark.parametrize('x_muls,lf,lo', [([256, 96, 64, 32], 3, 3), ([96, 32, 96], 1, 2), ([64, 256], 2, 1)])
def test_plugin_row_lengths(x_muls, lf, lo, pattern):
    deg = graphs.degrees(graphs.fixture(pattern, 'sevennet_0'))
    _plugin_compare(x_muls, lf, lo, deg, seed=len(deg))


# ---- batches, split stages, checkpoint files --------------------------------------------------------------------
def _structs(meta):
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


def test_device_batch_matches_structures_alone(models, engines):
    import torch
    from sevenn_b200.batch import DeviceBatch
    _, meta, _ = models['B']
    eng = engines('B')
    structs = _structs(meta)
    a = _flat(structs)
    res = DeviceBatch(eng).compute(a['numbers'], torch.tensor(a['positions'], device='cuda'), a['cells'], a['pbc'],
                                   torch.tensor(a['system_idx'], device='cuda'))
    ae_b = res['atomic_energy'].cpu().numpy()
    tm = eng.spec.type_map
    for b, s in enumerate(structs):
        sp = np.array([tm[int(z)] for z in s['numbers']], dtype=np.int32)
        e, ae, f, v, _ = eng.compute_positions(sp, s['positions'], s['cell'], s['pbc'])
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        assert np.array_equal(ae_b[a0:a1].view(np.uint32), np.asarray(ae, np.float32).view(np.uint32)), b
        assert abs(float(res['energy'][b]) - e) <= 1e-9 * max(1.0, abs(e))
        fs = max(1.0, float(np.abs(f).max()))
        assert np.abs(res['forces'][a0:a1].cpu().numpy() - f).max(initial=0.0) <= 1e-5 * fs


def test_sevennet_model_replays_after_rattle(models):
    import torch
    from sevenn_b200.batch import SevenNetModel
    _, meta, arrays = models['B']
    model = SevenNetModel((meta, arrays), device='cuda')
    structs = _structs(meta)[:4]
    a = _flat(structs)
    state = types.SimpleNamespace(
        positions=torch.tensor(a['positions'], device='cuda'), row_vector_cell=torch.tensor(a['cells'], device='cuda'),
        pbc=True, atomic_numbers=torch.tensor(a['numbers'], device='cuda'),
        system_idx=torch.tensor(a['system_idx'], device='cuda'))
    model(state)
    c0, r0 = model.engine.graph_stats()
    g = torch.Generator(device='cuda').manual_seed(5)
    state.positions = state.positions + 0.02 * torch.randn(state.positions.shape, generator=g, device='cuda',
                                                         dtype=state.positions.dtype)
    out = model(state)
    torch.cuda.synchronize()
    assert model.engine.graph_stats() == (c0, r0 + 1)          # replayed, not re-captured
    pos = state.positions.cpu().numpy()
    o = _oracle(meta, arrays)
    from sevenn_b200.neighbors import build_graph
    for b in (0, 3):
        a0, a1 = a['atom_ptr'][b], a['atom_ptr'][b + 1]
        ei, ev = build_graph(pos[a0:a1], a['cells'][b], True, 5.0)
        sp = np.array([model.type_map[int(z)] for z in a['numbers'][a0:a1]])
        ref = o.forward(sp, ei, ev)
        assert abs(float(out['energy'][b]) - float(ref['energy'])) <= 1e-4
        fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
        assert np.allclose(out['forces'][a0:a1].cpu().numpy(), ref['forces'].numpy(), atol=5e-5 * fs, rtol=0)


def test_split_stages_match_compute(models, engines):
    import torch
    from sevenn_b200 import engine as E
    from sevenn_b200.neighbors import diamond_si
    _, meta, _ = models['D']
    eng = engines('D')
    pos, cell, z = diamond_si(3, 2, 2, sigma=0.05, seed=2)
    sp = np.full(len(pos), eng.spec.type_map[14], dtype=np.int32)
    eng.set_positions(sp, pos, cell, True)
    eng.compute()
    torch.cuda.synchronize()
    full = {k: v.cpu().numpy().copy() for k, v in eng.results().items() if hasattr(v, 'cpu')}
    eng.set_interior(len(pos) // 3)
    T = eng.spec.n_layers
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
    torch.cuda.synchronize()
    split = {k: v.cpu().numpy().copy() for k, v in eng.results().items() if hasattr(v, 'cpu')}
    eng.set_interior(len(pos))
    # the forward has no atomics: per-atom energies are bit-identical
    assert np.array_equal(split['atomic_energy'].view(np.uint32), full['atomic_energy'].view(np.uint32))
    # the (split) backward adds edge terms atomically: fp32 reordering only
    fs = max(1.0, float(np.abs(full['forces']).max()))
    assert np.abs(split['forces'] - full['forces']).max() <= 1e-5 * fs
    vs = max(1.0, float(np.abs(full['virial']).max()))
    assert np.abs(split['virial'] - full['virial']).max() <= 1e-5 * vs


class _Atoms:
    """the part of ase.Atoms the calculator reads"""

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


def test_calculator_from_checkpoint_path(models):
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import build_graph, rocksalt_nacl
    path, meta, arrays = models['C']
    calc = SevenNetCalculator(model=path)
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.1, seed=1)
    calc.calculate(_Atoms(z, pos, cell, (True, True, True)))
    ei, ev = build_graph(pos, cell, True, 5.0)
    sp = np.array([calc.type_map[int(a)] for a in z])
    ref = _oracle(meta, arrays).forward(sp, ei, ev, volume=abs(np.linalg.det(cell)))
    out = dict(energy=calc.results['energy'], atomic_energy=calc.results['energies'], forces=calc.results['forces'],
               virial=ref['virial'].numpy())
    _check(out, ref, len(z))
    vol = abs(np.linalg.det(cell))
    want = -(ref['virial'].numpy() / vol)[[0, 1, 2, 4, 5, 3]]
    fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
    assert np.allclose(calc.results['stress'], want, atol=5e-4 * fs / vol, rtol=1e-5)


def test_export_flat_and_cpp_host(models, tmp_path):
    from sevenn_b200.export import export_flat
    from sevenn_b200.neighbors import build_graph, diamond_si
    _, meta, arrays = models['B']
    exe = str(tmp_path / 'host_entry')
    lib_dir = os.path.join(ROOT, 'sevenn_b200', 'lib')
    subprocess.check_call(['g++', '-O1', '-std=c++17', os.path.join(ROOT, 'examples', 'host_entry.cpp'), '-o', exe,
                           f'-L{lib_dir}', '-lsevenn_b200', f'-Wl,-rpath,{lib_dir}'])
    model = str(tmp_path / 'synthetic_B.s7b')
    export_flat(model, meta, arrays)
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=9)
    ei, ev = build_graph(pos, cell, True, 5.0)
    z = z.astype(np.int32)
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
    ref = _oracle(meta, arrays).forward(np.array([tm[int(a)] for a in z]), ei, ev)
    fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
    assert abs(energy - float(ref['energy'])) < 1e-4
    assert np.allclose(forces, ref['forces'].numpy(), atol=5e-5 * fs)


# ---- refusals --------------------------------------------------------------------------------------------------
def test_width_48_refused_by_engine_and_plugin(models):
    from sevenn_b200.conv_op import B200Convolution
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.checkpoint import random_weights
    meta = dict(models['B'][1])
    meta['irreps_per_layer'] = ['64x0e', '48x0e+32x1e', '64x0e']
    with pytest.raises(RuntimeError, match='positive multiples of 32'):
        B200Engine(meta, random_weights(meta))
    from sevenn_b200.spec import build_layer
    L = build_layer(0, [48, 32], [32, 32, 32], 1)
    with pytest.raises(RuntimeError, match='positive multiples of 32'):
        B200Convolution('48x0e+32x1e', '1x0e+1x1e', '+'.join(f'{p.mul}x{p.l3}e' for p in L.paths),
                        [(p.l1, p.l2, p.slot, 'uvu', True) for p in L.paths], shared_weights=False,
                        internal_weights=False)


def test_parity_checkpoint_refused(tmp_path):
    from sevenn_b200.calculator import SevenNetCalculator
    path = write_checkpoint(tmp_path / 'parity.pth', 'A', parity=True)
    with pytest.raises(NotImplementedError, match='is_parity'):
        SevenNetCalculator(model=path)
