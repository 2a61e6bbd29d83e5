"""The radial path on the GPU at radial shapes other than the shipped models' (tests/radial_models.py: cutoffs 4.0,
5.0, 5.3, 6.0; XPLOR with r_on on and off the 2000-interval grid; poly_cut p = 3 and 9; n_basis 5, 6, 8; radial
hidden widths [48, 96] and [50, 70]), against fp64: the edge kernel's buffers, per-edge forces of isolated dimers
across the radial range, whole models, the device neighbour list at those cutoffs, the calculator and the flat-file
C++ host; and the FP32 SIMT GEMM at row lengths and widths that are not multiples of 4 (the radial MLP's GEMMs
with radial='mlp')."""
import ctypes
import functools
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import graphs
from helpers import ROOT, first_divergence, format_stage_errors, stage_errors
from radial_models import CONFIGS, convert_radial, write_radial_checkpoint

pytestmark = pytest.mark.gpu
CIDS = sorted(CONFIGS)


@functools.lru_cache(maxsize=None)
def _ckpt(cid):
    d = tempfile.mkdtemp(prefix='radial_ckpt_')
    path = write_radial_checkpoint(f'{d}/{cid}.pth', cid)
    return (path,) + convert_radial(path, cid)


@functools.lru_cache(maxsize=None)
def _engine(cid, radial, knots=None):
    from sevenn_b200.engine import B200Engine
    _, meta, arrays = _ckpt(cid)
    return B200Engine(meta, arrays, radial=radial, knots=knots)


@functools.lru_cache(maxsize=None)
def _oracle(cid):
    import torch
    from oracle.oracle import Oracle
    _, meta, arrays = _ckpt(cid)
    return Oracle(meta, arrays, dtype=torch.float64)


def _spec(cid):
    from sevenn_b200.spec import build_spec
    return build_spec(_ckpt(cid)[1])


def _run(e, species, ei, ev):
    import torch
    e.set_graph(species, ei, ev)
    e.compute()
    torch.cuda.synchronize()
    r = e.results()
    return dict(energy=float(r['energy'].cpu()[0]), atomic_energy=r['atomic_energy'].cpu().numpy(),
                forces=r['forces'].cpu().numpy(), edge_force=r['edge_force'].cpu().numpy(),
                virial=r['virial'].cpu().numpy())


def _local_scale(r, mag, width=0.1, floor=0.1):
    """per edge: max of mag over edges with |r' - r| <= width, floored at floor * max(mag)"""
    o = np.argsort(r)
    rs, ms = r[o], mag[o]
    lo, hi = np.searchsorted(rs, rs - width), np.searchsorted(rs, rs + width, side='right')
    loc = np.array([ms[a:b].max() for a, b in zip(lo, hi)])
    out = np.empty_like(loc)
    out[o] = np.maximum(loc, floor * ms.max())
    return out


# ---- the edge kernel -------------------------------------------------------------------------------------------
def _edge_buffers(e, vec):
    import torch
    from sevenn_b200 import engine as E
    n = len(vec)
    e.set_graph(np.zeros(2 * n, dtype=np.int64), np.stack([np.arange(n), np.arange(n) + n]), vec)
    e.run_stage(E.STAGE_FWD_BEGIN)
    torch.cuda.synchronize()
    y = e.buffer('edge_Y').cpu().numpy().reshape(n, -1)
    rec = e.buffer('edge_rec', dtype='i4', shape=(n, 4)).cpu().numpy()
    rlen = e.buffer('edge_len', shape=(n,)).cpu().numpy()
    emb = e.buffer('edge_emb').cpu().numpy().reshape(n, -1) if e.radial == 'mlp' else None
    return y, rec, rlen, emb


def _directions():
    """the axes, 1e-7 off the poles, random directions"""
    axes = np.concatenate([np.eye(3), -np.eye(3)])
    poles = np.array([[1e-7, 0, 1], [0, -1e-7, -1], [1e-7, 1e-7, 1], [-1e-7, 0, -1]])
    rnd = np.random.RandomState(3).normal(size=(40, 3))
    u = np.concatenate([axes, poles, rnd])
    return u / np.linalg.norm(u, axis=1, keepdims=True)


@pytest.mark.parametrize('cid', ['R1', 'R3', 'R4'])     # lmax_filter 1, 2, 2
def test_edge_kernel_against_fp64(cid):
    import torch
    from oracle.oracle import _sh_torch
    spec = _spec(cid)
    lf = spec.lmax_filter
    u = _directions()
    rng = np.random.RandomState(7)
    r = np.concatenate([[1e-3, 0.2, spec.cutoff - 1e-6, spec.cutoff, spec.cutoff + 0.5],
                        rng.uniform(0.3, spec.cutoff, len(u) - 5)])
    vec = (u * r[:, None]).astype(np.float32)
    v64 = vec.astype(np.float64)
    r64 = np.linalg.norm(v64, axis=1)
    want_y = _sh_torch(lf, torch.tensor(v64 / r64[:, None])).numpy()[:, 1:]
    for radial in ('table', 'mlp'):
        e = _engine(cid, radial)
        y, rec, rlen, emb = _edge_buffers(e, vec)
        ny = want_y.shape[1]
        assert np.abs(y[:, :ny] - want_y).max() < 2e-6, (radial, np.abs(y[:, :ny] - want_y).max())
        assert (y[:, ny:] == 0).all()                                    # padding of the Y rows
        assert np.allclose(rlen, r64, rtol=2e-7, atol=0)
        assert (rec[:, 0] == np.arange(len(r)) + len(r)).all()           # neighbour index
        if radial == 'table':
            knots = e.knots
            tk, tt = rec[:, 1], rec[:, 2].view(np.float32).astype(np.float64)
            assert ((tk >= 0) & (tk < knots) & (tt >= 0) & (tt <= 1)).all()
            s = r64 * knots / spec.cutoff
            inside = r64 < spec.cutoff * (1 - 1e-6)
            beyond = r64 > spec.cutoff * (1 + 1e-6)
            assert np.abs((tk + tt - s)[inside]).max() < 1e-3                # interval + fraction = r / h (fp32 s)
            assert (tk[~inside] == knots - 1).all() and (tt[~inside] > 1 - 1e-3).all()
            assert (tt[beyond] == 1.0).all()                                 # r > rc: the end of the table
        else:
            from sevenn_b200.engine import radial_embedding
            _, _, arrays = _ckpt(cid)
            want, _ = radial_embedding(spec, arrays['bessel_coeffs'], r64)
            assert emb.shape == (len(r), spec.n_basis)
            assert np.abs(emb - want).max() < 2e-6 * max(1.0, np.abs(want).max()), np.abs(emb - want).max()


def test_zero_length_edge_stays_finite():
    """an r = 0 edge (a caller's degenerate pair) has no direction: zero harmonics, no NaN anywhere downstream"""
    spec = _spec('R4')
    for radial in ('table', 'mlp'):
        e = _engine('R4', radial)
        y, rec, rlen, emb = _edge_buffers(e, np.zeros((1, 3), np.float32))
        assert np.isfinite(y).all() and rlen[0] == 0 and rec[0, 1] == 0
        tm = spec.type_map
        sp = np.array([tm[14], tm[8], tm[8]])
        ei = np.array([[0, 0, 1, 1, 2], [1, 2, 0, 2, 1]])
        ev = np.array([[0, 0, 0], [1.6, 0, 0], [0, 0, 0], [1.6, 0, 0], [-1.6, 0, 0]], dtype=np.float64)
        out = _run(e, sp, ei, ev)
        assert all(np.isfinite(v).all() for v in out.values()), radial


# ---- per-edge dE/dr of isolated dimers --------------------------------------------------------------------------
def _dimers(spec, knots):
    """~400 isolated dimers over the radial range: H-H below 1 A, Si-O above, plus knots, r_on +- {1e-6, h/3} and
    rc - 1e-6.  Returns species, edge_index, edge_vec (two directed edges per dimer) and the pair distances."""
    rc = spec.cutoff
    h = rc / knots
    r = [np.linspace(0.35, 0.99, 40), np.linspace(1.0, rc - 0.01, 340), [rc - 1e-6]]
    r.append(h * np.array([int(1.2 / h), int(2.5 / h), int(0.9 * knots), knots - 1]))
    if spec.cutoff_fn == 'XPLOR':
        r.append([spec.cutoff_on + d for d in (-h / 3, -1e-6, 0.0, 1e-6, h / 3)])
    r = np.concatenate(r)
    rng = np.random.RandomState(11)
    u = rng.normal(size=(len(r), 3))
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    v = u * r[:, None]
    tm = spec.type_map
    n = len(r)
    sp = np.empty(2 * n, dtype=np.int64)
    sp[0::2] = np.where(r < 1.0, tm[1], tm[14])
    sp[1::2] = np.where(r < 1.0, tm[1], tm[8])
    i = np.arange(n)
    ei = np.stack([np.stack([2 * i, 2 * i + 1], 1).ravel(), np.stack([2 * i + 1, 2 * i], 1).ravel()])
    ev = np.stack([v, -v], 1).reshape(-1, 3)
    return sp, ei, ev, np.repeat(r, 2)


def _dimer_errors(cid, radial, knots=None):
    """per-edge |f - f_ref| over the local scale of |f_ref|, and the edge lengths"""
    from sevenn_b200.engine import default_table_knots
    e = _engine(cid, radial, knots)
    spec = _spec(cid)
    sp, ei, ev, r = _dimers(spec, e.knots or default_table_knots(spec))
    out = _run(e, sp, ei, ev.astype(np.float32))
    ref = _oracle(cid).forward(sp, ei, ev.astype(np.float32).astype(np.float64))
    fr = ref['edge_force'].numpy()
    err = np.linalg.norm(out['edge_force'] - fr, axis=1)
    return err / _local_scale(r, np.linalg.norm(fr, axis=1)), r


# Per-edge force error over the local scale of |f| (max within 0.1 A, floored at 0.1 of the global max).  Measured on
# an H100 with r_on on a knot: table 1.4e-4 .. 2.8e-4 (median 7e-6 .. 2e-5), mlp <= 7e-6 (fp32 arithmetic only).
# With r_on inside an interval (2000 knots) the edges next to r_on reach 5.5e-4 (R1) and 2.4e-3 (R5).
DIMER_BOUND = {'table': 4e-4, 'mlp': 3e-5}


def _near_r_on(spec, r, knots):
    return np.abs(r - spec.cutoff_on) < spec.cutoff / knots


@pytest.mark.parametrize('radial', ['table', 'mlp'])
@pytest.mark.parametrize('cid', CIDS)
def test_dimer_edge_forces_against_oracle(cid, radial):
    rel, r = _dimer_errors(cid, radial)
    j = int(np.argmax(rel))
    print(f'\n{cid} {radial}: per-edge force error / local scale: max {rel[j]:.2e} at r = {r[j]:.5f}, '
          f'median {np.median(rel):.2e}')
    assert rel[j] < DIMER_BOUND[radial], (rel[j], r[j])


@pytest.mark.parametrize('cid', ['R1', 'R5'])
def test_dimer_check_fails_with_r_on_between_knots(cid):
    """negative control: the same model tabulated on 2000 intervals (r_on inside one) fails the bound, at r_on, and
    is several times worse there than on the knot rule's grid"""
    spec = _spec(cid)
    rel, r = _dimer_errors(cid, 'table', knots=2000)
    near = _near_r_on(spec, r, 2000)
    rel_ok, r_ok = _dimer_errors(cid, 'table')
    near_ok = _near_r_on(spec, r_ok, 2000)
    j = int(np.argmax(rel))
    print(f'\n{cid} table, 2000 knots: max {rel[j]:.2e} at r = {r[j]:.5f}; next to r_on {rel[near].max():.2e} '
          f'(on the knot rule\'s grid: {rel_ok[near_ok].max():.2e}), elsewhere {rel[~near].max():.2e}')
    assert rel[j] > DIMER_BOUND['table'] and near[j]
    assert rel[near].max() > 3 * rel_ok[near_ok].max()


# ---- whole models ----------------------------------------------------------------------------------------------
def _system(name, meta, cutoff):
    from sevenn_b200.neighbors import build_graph, diamond_si
    if name == 'si64':
        pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
        pbc = (True, True, True)
    else:
        g = graphs.build(name, meta)        # dense fcc / triclinic cell with heights below the cutoff / hub
        pos, cell, z, pbc = g.positions, g.cell, g.numbers, g.pbc
    ei, ev = build_graph(pos, cell, pbc, cutoff) if all(pbc) else build_graph(pos, cell, False, cutoff)
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    vol = abs(np.linalg.det(cell)) if all(pbc) else 0.0
    return np.array([tm[int(a)] for a in z]), ei, ev, vol


# The virial sums r (x) f over every edge, so a smooth error in dw/dr adds up instead of cancelling: its bound grows
# with sum_e |r_a f_b| (dense cells at 6 A: ~80 eV over 22 000 - 44 000 edges).  Measured on an H100: table 1.4e-5 ..
# 3.2e-5 of that sum (the tables' dw/dr error, ~1e-5 of its global scale), mlp below 2e-5.
VIRIAL_SUM_RTOL = {'table': 1e-4, 'mlp': 2e-5}


@pytest.mark.parametrize('system', ['si64', 'dense', 'tiny_cell', 'hub'])
@pytest.mark.parametrize('cid', CIDS)
def test_model_against_oracle(cid, system):
    _, meta, arrays = _ckpt(cid)
    sp, ei, ev, vol = _system(system, meta, meta['cutoff'])
    ref = _oracle(cid).forward(sp, ei, ev, volume=vol, keep=True)
    f_ref, v_ref = ref['forces'].numpy(), ref['virial'].numpy()
    fe = ref['edge_force'].numpy()
    v_sum = np.abs(ev[:, [0, 1, 2, 0, 1, 2]] * fe[:, [0, 1, 2, 1, 2, 0]]).sum(0)
    fs = max(1.0, float(np.abs(f_ref).max()) / 5.0)
    es = max(1.0, float(np.abs(ref['atomic_energy'].numpy()).max()) / 10.0)
    n = len(sp)
    failures = []
    for radial in ('table', 'mlp'):
        e = _engine(cid, radial)
        out = _run(e, sp, ei, ev)
        errs = dict(energy=abs(out['energy'] - float(ref['energy'])),
                    atomic=np.abs(out['atomic_energy'] - ref['atomic_energy'].numpy()).max(),
                    forces=np.abs(out['forces'] - f_ref).max(),
                    virial=np.abs(out['virial'] - v_ref).max())
        ok = (errs['energy'] <= 1e-4 * es * max(1.0, n / 64.0) and errs['atomic'] <= 2e-5 * es
              and errs['forces'] <= 5e-5 * fs
              and (np.abs(out['virial'] - v_ref) <= 5e-4 * fs + VIRIAL_SUM_RTOL[radial] * v_sum).all())
        if not ok:
            st = stage_errors(e, arrays, sp, ei, ev, ref=ref)
            failures.append(f'{cid} {system} {radial}: {errs} (E = {ei.shape[1]}, sum|r f| = {v_sum.max():.3g})\n'
                            f'first divergence: {first_divergence(st)}\n{format_stage_errors(st)}')
    assert not failures, '\n'.join(failures)


# ---- the device neighbour list at other cutoffs ----------------------------------------------------------------
def _planted(rc):
    """pairs at rc - 1e-6 (edges) and rc + 1e-6 (none), 40 A apart from each other and from everything else"""
    pos = []
    for k, d in enumerate((rc - 1e-6, rc + 1e-6)):
        u = np.array([np.cos(0.7 * k + 0.3), np.sin(0.7 * k + 0.3), 0.2 * k])
        u /= np.linalg.norm(u)
        base = np.array([60.0 + 40.0 * k, -50.0, 30.0])
        pos += [base, base + d * u]
    return np.array(pos)


@pytest.mark.parametrize('cid', ['R3', 'R4', 'R1'])        # cutoffs 4.0, 5.3 (not exact in fp32), 6.0
def test_device_neighbor_list_at_model_cutoff(cid):
    """the device list keeps pairs with |d| < the model's fp32 cutoff (S7bModelDesc.cutoff, widened to double):
    identical to the numpy builders at that cutoff, periodic and not"""
    from sevenn_b200.neighbors import neighbor_list_brute
    _, meta, _ = _ckpt(cid)
    rc = meta['cutoff']
    rc32 = float(np.float32(rc))
    e = _engine(cid, 'table')
    rng = np.random.RandomState(2)
    cluster = rng.uniform(0, 9.0, size=(40, 3))
    cases = []
    pos = np.concatenate([cluster, _planted(rc)])
    if rc32 != rc:          # a pair between the fp64 and the fp32 cutoff is an edge of the device list
        pos = np.concatenate([pos, [[0, 0, -80.0], [0, 0, -80.0 + 0.5 * (rc + rc32)]]])
    cases.append((pos, np.zeros((3, 3)), (False, False, False)))
    g = graphs.build('tiny_cell', meta)
    cases.append((g.positions, g.cell, (True, True, True)))
    g = graphs.build('dense', meta)
    cases.append((g.positions, g.cell, (True, True, True)))
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    for pos, cell, pbc in cases:
        sp = np.full(len(pos), tm[14], dtype=np.int32)
        e.set_positions(sp, pos, cell, pbc)
        rowptr, src, vec = (t.cpu().numpy() for t in e.graph_arrays())
        ei, ev, _ = neighbor_list_brute(pos, cell, np.asarray(pbc), rc32)
        dst = np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))
        got = sorted(zip(dst.tolist(), src.tolist(), np.rint(vec * 1e4).astype(int).tolist()))
        want = sorted(zip(ei[0].tolist(), ei[1].tolist(), np.rint(ev * 1e4).astype(int).tolist()))
        assert len(got) == len(want) and [g[:2] for g in got] == [w[:2] for w in want], (cid, pbc)
        if not any(pbc):
            n0 = len(cluster)
            have = set(zip(dst.tolist(), src.tolist()))
            assert (n0, n0 + 1) in have and (n0 + 2, n0 + 3) not in have
            if rc32 != rc:
                assert (n0 + 4, n0 + 5) in have


# ---- front ends ------------------------------------------------------------------------------------------------
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


def test_calculator_from_r1_checkpoint():
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import build_graph, rocksalt_nacl
    path, meta, arrays = _ckpt('R1')
    calc = SevenNetCalculator(model=path)
    assert calc.cutoff == 6.0 and calc.engine.knots == 2004
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.1, seed=1)
    calc.calculate(_Atoms(z, pos, cell, (True, True, True)))
    ei, ev = build_graph(pos, cell, True, 6.0)
    assert calc.results['num_edges'] == ei.shape[1]
    sp = np.array([calc.type_map[int(a)] for a in z])
    vol = abs(np.linalg.det(cell))
    ref = _oracle('R1').forward(sp, ei, ev, volume=vol)
    fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
    assert abs(calc.results['energy'] - float(ref['energy'])) < 1e-4 * max(1.0, len(z) / 64.0)
    assert np.allclose(calc.results['forces'], ref['forces'].numpy(), atol=5e-5 * fs, rtol=0)
    want = -(ref['virial'].numpy() / vol)[[0, 1, 2, 4, 5, 3]]
    assert np.allclose(calc.results['stress'], want, atol=5e-4 * fs / vol, rtol=1e-5)


def test_export_flat_and_cpp_host_r5(tmp_path):
    from sevenn_b200.export import export_flat
    from sevenn_b200.neighbors import build_graph, diamond_si
    _, meta, arrays = _ckpt('R5')
    exe = str(tmp_path / 'host_entry')
    lib_dir = os.path.join(ROOT, 'sevenn_b200', 'lib')
    subprocess.check_call(['g++', '-O1', '-std=c++17', os.path.join(ROOT, 'examples', 'host_entry.cpp'), '-o', exe,
                           f'-L{lib_dir}', '-lsevenn_b200', f'-Wl,-rpath,{lib_dir}'])
    model = str(tmp_path / 'r5.s7b')
    export_flat(model, meta, arrays)
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=9)
    ei, ev = build_graph(pos, cell, True, 5.3)
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
    ref = _oracle('R5').forward(np.array([tm[int(a)] for a in z]), ei, ev)
    fs = max(1.0, float(ref['forces'].abs().max()) / 5.0)
    assert abs(energy - float(ref['energy'])) < 1e-4
    assert np.allclose(forces, ref['forces'].numpy(), atol=5e-5 * fs)


# ---- the FP32 SIMT GEMM at unaligned shapes ----------------------------------------------------------------------
def _stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize('N', [1, 3, 6, 50, 70])
@pytest.mark.parametrize('K', [1, 2, 3, 5, 6, 7, 13, 50])
def test_simt_dense_linear_unaligned(K, N):
    """s7b_dense_linear(use_tc=0) with K or N not a multiple of 4 (rows of A and W off 16-byte boundaries), and with
    A, W and C one float past a 16-byte boundary; the floats around C stay as they were"""
    import torch
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    rng = np.random.RandomState(K * 100 + N)
    rows = 300
    A = rng.normal(size=(rows, K)).astype(np.float32)
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    ref = A.astype(np.float64) @ W.astype(np.float64)
    for shift in (0, 1):
        a = torch.tensor(np.concatenate([np.zeros(shift, np.float32), A.ravel()]), device='cuda')
        w = torch.tensor(np.concatenate([np.zeros(shift, np.float32), W.ravel()]), device='cuda')
        c = torch.full((rows * N + 2 * shift + 8,), -7.0, device='cuda')
        check(lib.s7b_dense_linear(a.data_ptr() + 4 * shift, w.data_ptr() + 4 * shift, c.data_ptr() + 4 * shift,
                                   rows, K, N, 0, _stream()))
        torch.cuda.synchronize()
        got = c.cpu().numpy()
        out = got[shift:shift + rows * N].reshape(rows, N)
        assert np.abs(out - ref).max() < 3e-6 * np.sqrt(K) * max(1.0, np.abs(ref).max()), (shift, np.abs(out - ref).max())
        assert (got[:shift] == -7.0).all() and (got[shift + rows * N:] == -7.0).all()


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('a_K,c_N,pad', [([5, 3, 7], [6, 1, 3], (1, 3)), ([8, 12], [4, 8], (3, 5)),
                                         ([50, 13], [70, 6], (0, 1))])
def test_simt_block_linear_odd_leading_dimensions(a_K, c_N, pad, accumulate):
    """s7b_block_linear(use_tc=0) with odd lda / ldc and block offsets: blocks vs fp64, pad columns untouched"""
    import torch
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    rng = np.random.RandomState(sum(a_K) + sum(c_N))
    n_nodes, n_l = 200, len(a_K)
    a_off, c_off, lda, ldc = [], [], pad[0], pad[1]
    for l in range(n_l):
        a_off.append(lda)
        lda += (2 * l + 1) * a_K[l]
        c_off.append(ldc)
        ldc += (2 * l + 1) * c_N[l]
    lda += 3
    ldc += 1
    A = rng.normal(size=(n_nodes, lda)).astype(np.float32)
    C0 = rng.normal(size=(n_nodes, ldc)).astype(np.float32)
    Ws = [(rng.normal(size=(a_K[l], c_N[l])) / np.sqrt(a_K[l])).astype(np.float32) for l in range(n_l)]
    W = np.ascontiguousarray(np.concatenate([w.ravel() for w in Ws]))
    ref = C0.astype(np.float64).copy()
    for l in range(n_l):
        d = 2 * l + 1
        a = A[:, a_off[l]:a_off[l] + d * a_K[l]].reshape(n_nodes, d, a_K[l]).astype(np.float64)
        blk = ref[:, c_off[l]:c_off[l] + d * c_N[l]].reshape(n_nodes, d, c_N[l])
        ref[:, c_off[l]:c_off[l] + d * c_N[l]] = ((blk if accumulate else 0.0) + a @ Ws[l].astype(np.float64)).reshape(n_nodes, -1)
    a_t, c_t = torch.tensor(A, device='cuda'), torch.tensor(C0, device='cuda')
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ao, ak, co, cn = i32(a_off), i32(a_K), i32(c_off), i32(c_N)
    check(lib.s7b_block_linear(a_t.data_ptr(), lda, n_nodes, n_l, ao.ctypes.data, ak.ctypes.data, W.ctypes.data,
                               c_t.data_ptr(), ldc, co.ctypes.data, cn.ctypes.data, int(accumulate), 0, _stream()))
    torch.cuda.synchronize()
    got = c_t.cpu().numpy()
    assert np.abs(got - ref).max() < 3e-6 * np.sqrt(max(a_K)) * max(1.0, np.abs(ref).max())
    pads = np.ones(ldc, bool)
    for l in range(n_l):
        pads[c_off[l]:c_off[l] + (2 * l + 1) * c_N[l]] = False
    assert np.array_equal(got[:, pads], C0[:, pads])


def test_species_linear_refuses_unaligned_blocks():
    import torch
    from sevenn_b200.engine import load_library
    lib = load_library()
    a = torch.zeros(10, 8, device='cuda')
    c = torch.zeros(10, 8, device='cuda')
    sp = torch.zeros(10, dtype=torch.int32, device='cuda')
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    zero, k, n = i32([0]), i32([5]), i32([8])
    W = np.zeros(40, np.float32)
    rc = lib.s7b_species_linear(a.data_ptr(), 8, 10, sp.data_ptr(), 1, 1, zero.ctypes.data, k.ctypes.data, W.ctypes.data,
                                c.data_ptr(), 8, zero.ctypes.data, n.ctypes.data, 0, _stream())
    torch.cuda.synchronize()
    assert rc != 0 and b'multiples of 4' in lib.s7b_last_error()
