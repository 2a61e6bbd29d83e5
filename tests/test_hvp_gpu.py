"""The engine's Hessian-vector product (s7b_engine_hvp, B200Engine.hvp, SevenNetCalculator.get_hessian) on the GPU.

Reference: H v = -dF/de of the fp64 oracle's forces along edge_vec + e (v[neighbour] - v[centre]) with the edge list
held fixed, by central differences at h = 1e-3 and 2e-3 combined by Richardson extrapolation (truncation ~h^4, below
1e-9 of max|Hv| here).

Bounds.  The pass is fp32 throughout: every H v element sums over the ~40 edges of an atom and, per edge, over the
W radial channels and the channels of each layer, so its rounding error is a few hundred fp32 ulps of the largest
terms, ~1e-5 of max|Hv|, and the tensor-core node linears are error-free in the bf16x3 split.  The 'mlp' radial mode
evaluates the same radial MLP as the oracle: bound 2e-4 of max|Hv|.  The 'table' mode runs its forward on the
tabulated weights (value table: ~1e-5 relative error of w, whose effect on Hv is of the same order) and its second
order on the MLP: bound 5e-4 of max|Hv|.  Both stay below 1e-3 of max|Hv|.  The observed errors are printed."""
import ctypes
import os

import numpy as np
import pytest

from helpers import ROOT, model_weights

pytestmark = pytest.mark.gpu

BOUND = {'mlp': 2e-4, 'table': 5e-4}


def _species(meta, z):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z], dtype=np.int32)


def _si(meta, n=2, periodic=True, seed=4, cutoff=None):
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, z = diamond_si(n, n, n, sigma=0.05, seed=seed)
    from sevenn_b200.spec import build_spec
    rc = cutoff or build_spec(meta).cutoff
    if periodic:
        ei, ev = build_graph(pos, cell, True, rc)
    else:
        ei, ev = build_graph(pos, np.zeros((3, 3)), False, rc)
    return _species(meta, z), ei, ev


def _irr(muls):
    return '+'.join(f'{m}x{l}e' for l, m in enumerate(muls))


def _synthetic(le, ln, tmp):
    from synthetic_models import convert, layered, write_checkpoint
    mid = _irr([32] * (ln + 1))
    arch = layered(f'hvp_{le}{ln}', le, ln, ['32x0e', mid, mid, '32x0e'])
    path = write_checkpoint(os.path.join(tmp, f'hvp_{le}{ln}.pth'), arch, seed=70 + 10 * le + ln)
    return convert(path, arch)


def _weights(case, tmp):
    if case.startswith('synth_'):
        return _synthetic(int(case[6]), int(case[7]), tmp)
    if case.startswith('radial_'):
        from radial_models import convert_radial, write_radial_checkpoint
        cid = case[7:]
        return convert_radial(write_radial_checkpoint(os.path.join(tmp, f'{cid}.pth'), cid), cid)
    if case == 'nequip_A':
        from synthetic_nequip import convert, write_nequip_checkpoint
        return convert(write_nequip_checkpoint(os.path.join(tmp, 'nq_A.pth'), 'A', seed=3), 'A')
    return model_weights(case)


def fd_hvp(meta, arrays, species, ei, ev, v):
    """-dF/de of the fp64 oracle along edge_vec + e (v[nb] - v[centre]), Richardson-extrapolated.  The XPLOR envelope
    is only C1 at r_on (w'' jumps; the third-neighbour shell of Si, 4.50 A, sits on SevenNet-0's r_on = 4.5), so the
    steps stay below a fifth of the distance of every edge from r_on and from the cutoff: no difference straddles
    a kink of the forces' derivative."""
    import torch
    from oracle.oracle import Oracle
    from nequip_oracle import nequip_oracle
    from sevenn_b200.spec import build_spec
    spec = build_spec(meta)
    dev = 'cuda' if torch.cuda.is_available() else 'cpu'
    make = nequip_oracle if spec.self_connection == 'nequip' else Oracle
    o = make(meta, arrays, dtype=torch.float64, device=dev)
    dvec = v[ei[1]] - v[ei[0]]
    r = np.linalg.norm(ev.astype(np.float64), axis=1)
    kinks = [spec.cutoff] + ([spec.cutoff_on] if spec.cutoff_fn == 'XPLOR' else [])
    margin = min(np.abs(r - k).min() for k in kinks)
    h = min(1e-3, margin / (5 * 2 * np.linalg.norm(dvec, axis=1).max()))
    F = lambda s: o.forward(species, ei, ev.astype(np.float64) + s * dvec)['forces'].cpu().numpy().astype(np.float64)
    D = lambda s: -(F(s) - F(-s)) / (2 * s)
    return (4 * D(h) - D(2 * h)) / 3


def engine_hvp(meta, arrays, radial, species, ei, ev, vs):
    import torch
    from sevenn_b200.engine import B200Engine
    e = B200Engine(meta, arrays, radial=radial)
    e.set_graph(species, ei, ev)
    e.compute()
    out = [e.hvp(v).double().cpu().numpy() for v in vs]
    torch.cuda.synchronize()
    return e, out


CASES = [('sevennet_0', 'table', 'si64'), ('sevennet_0', 'mlp', 'si64'), ('sevennet_0', 'table', 'cluster'),
         ('sevennet_l3i5', 'table', 'si64'), ('sevennet_l3i5', 'mlp', 'cluster'),
         ('radial_R1', 'table', 'si64'), ('radial_R3', 'mlp', 'si64'), ('radial_R5', 'mlp', 'cluster'),
         ('nequip_A', 'mlp', 'si64'), ('nequip_A', 'table', 'cluster')]
CASES += [(f'synth_{le}{ln}', 'mlp' if (le + ln) % 2 else 'table', 'si64' if le != ln else 'cluster')
          for le in (1, 2, 3) for ln in (1, 2, 3)]


@pytest.mark.parametrize('case,radial,system', CASES)
def test_hvp_against_fp64_differences(case, radial, system, tmp_path):
    meta, arrays = _weights(case, str(tmp_path))
    if system == 'si64':
        species, ei, ev = _si(meta)
    else:      # 8-atom non-periodic cluster
        species, ei, ev = _si(meta, n=1, periodic=False)
    r = np.linalg.norm(ev, axis=1)
    rng = np.random.RandomState(sum(map(ord, case + radial + system)))
    v = rng.normal(size=(len(species), 3))
    ref = fd_hvp(meta, arrays, species, ei, ev, v)
    _, (out,) = engine_hvp(meta, arrays, radial, species, ei, ev, [v])
    err = np.abs(out - ref).max() / np.abs(ref).max()
    print(f'HVP {case} {radial} {system}: E = {len(r)}, r in [{r.min():.2f}, {r.max():.2f}], max|Hv| = '
          f'{np.abs(ref).max():.3e}, max err / max|Hv| = {err:.2e} (bound {BOUND[radial]:.0e})')
    assert err < BOUND[radial]


def test_r_on_straddled():
    """the R1 cell of test_hvp_against_fp64_differences has edges on both sides of r_on = 5.5"""
    from radial_models import CONFIGS
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, _ = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    _, ev = build_graph(pos, cell, True, CONFIGS['R1']['cutoff'])
    r = np.linalg.norm(ev, axis=1)
    assert (r < 5.5).any() and ((r > 5.5) & (r < 6.0)).any()


@pytest.fixture(scope='module')
def si0():
    meta, arrays = model_weights('sevennet_0')
    return meta, arrays, _si(meta)


def test_symmetry_and_translation(si0):
    """u^T (H v) = v^T (H u), and H (uniform translation) = 0"""
    meta, arrays, (species, ei, ev) = si0
    rng = np.random.RandomState(1)
    n = len(species)
    u, v = rng.normal(size=(n, 3)), rng.normal(size=(n, 3))
    tr = [np.tile(np.eye(3)[a], (n, 1)) for a in range(3)]
    _, (hu, hv, *ht) = engine_hvp(meta, arrays, 'table', species, ei, ev, [u, v] + tr)
    a, b = float((u * hv).sum()), float((v * hu).sum())
    scale = np.abs(u).sum() * np.abs(hv).max()
    print(f'symmetry: u.Hv = {a:.6e}, v.Hu = {b:.6e}, |diff| / (sum|u| max|Hv|) = {abs(a - b) / scale:.2e}')
    assert abs(a - b) < 1e-5 * scale
    for h in ht:
        print(f'translation: max|H t| / max|Hv| = {np.abs(h).max() / np.abs(hv).max():.2e}')
        assert np.abs(h).max() < 1e-4 * np.abs(hv).max()


class _Atoms:
    def __init__(self, pos, cell, z):
        self.pos, self.cell, self.z = pos, cell, z

    def get_positions(self):
        return self.pos

    def get_cell(self):
        return self.cell

    def get_pbc(self):
        return np.array([True] * 3)

    def get_atomic_numbers(self):
        return self.z


def test_calculator_hessian_si64():
    """SevenNetCalculator.get_hessian of a 64-atom Si cell: [192, 192] float64, symmetric to 1e-4 of max|H| (twice
    the HVP's fp32 error: each triangle is a different product), and results untouched"""
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=4)
    atoms = _Atoms(pos, cell, z)
    calc = SevenNetCalculator('7net-0')
    calc.calculate(atoms)
    before = {k: np.copy(v) for k, v in calc.results.items()}
    H = calc.get_hessian(atoms)
    assert H.shape == (192, 192) and H.dtype == np.float64 and np.isfinite(H).all()
    asym = np.abs(H - H.T).max() / np.abs(H).max()
    print(f'get_hessian(Si64): max|H| = {np.abs(H).max():.3e} eV/A^2, max|H - H^T| / max|H| = {asym:.2e}, '
          f'max|sum_j H| / max|H| = {np.abs(H.reshape(64, 3, 64, 3).sum(axis=2)).max() / np.abs(H).max():.2e}')
    assert asym < 1e-4
    assert all(np.array_equal(before[k], calc.results[k]) for k in before)


def test_batch_has_no_cross_structure_coupling():
    """on a union graph of set_positions_batch, H v equals the per-structure HVPs"""
    import torch
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = model_weights('sevennet_0')
    structs = [diamond_si(1, 1, 2, sigma=0.05, seed=s) for s in (1, 2, 3)]
    rng = np.random.RandomState(5)
    vs = [rng.normal(size=(len(p), 3)) for p, _, _ in structs]
    e = B200Engine(meta, arrays)
    singles = []
    for (p, c, z), v in zip(structs, vs):
        e.set_positions(_species(meta, z), p, c, True)
        e.compute()
        singles.append(e.hvp(v).double().cpu().numpy())
    ap = np.cumsum([0] + [len(p) for p, _, _ in structs])
    e.set_positions_batch(np.concatenate([_species(meta, z) for _, _, z in structs]),
                          np.concatenate([p for p, _, _ in structs]), ap, np.stack([c for _, c, _ in structs]), True)
    e.compute()
    hb = e.hvp(np.concatenate(vs)).double().cpu().numpy()
    torch.cuda.synchronize()
    ref = np.concatenate(singles)
    err = np.abs(hb - ref).max() / np.abs(ref).max()
    print(f'batch: max|H_batch v - H_single v| / max|Hv| = {err:.2e}')
    assert err < 1e-5


def test_no_edges_and_zero_tangent(si0):
    import torch
    from sevenn_b200.engine import B200Engine
    meta, arrays, (species, ei, ev) = si0
    e = B200Engine(meta, arrays)
    e.set_graph(species[:3], np.zeros((2, 0), np.int64), np.zeros((0, 3), np.float32))
    e.compute()
    assert torch.equal(e.hvp(np.ones((3, 3))).cpu(), torch.zeros(3, 3))
    e.set_graph(species, ei, ev)
    e.compute()
    h = e.hvp(np.zeros((len(species), 3))).cpu()
    assert torch.isfinite(h).all() and bool((h == 0).all())


def test_refusals(si0):
    from sevenn_b200.engine import B200Engine, check
    meta, arrays, (species, ei, ev) = si0
    n = len(species)
    v = np.ones((n, 3))
    e = B200Engine(meta, arrays)
    e.set_graph(species, ei, ev)
    with pytest.raises(RuntimeError, match='needs an s7b_engine_compute'):
        e.hvp(v)
    e.compute()
    e.hvp(v)
    # setting a parameter the step reads invalidates the forward
    check(e.lib.s7b_engine_set_param(e._h, b'scale', -1, np.ones(meta_species(meta), np.float32).ctypes.data,
                                     meta_species(meta)))
    with pytest.raises(RuntimeError, match='needs an s7b_engine_compute'):
        e.hvp(v)
    # ghosts: the last 8 atoms have no edges of their own
    keep = ei[0] < n - 8
    e.set_graph(species, ei[:, keep], ev[keep], n_local=n - 8)
    e.compute()
    with pytest.raises(RuntimeError, match='ghost'):
        e.hvp(v)
    # a table-mode engine without its radial MLP (the C ABI directly, Python uploads it on the first hvp)
    t = B200Engine(meta, arrays)
    t.set_graph(species, ei, ev)
    t.compute()
    import torch
    vv = torch.ones(n, 3, device=t.device)
    out = torch.empty(n, 3, device=t.device)
    with pytest.raises(RuntimeError, match='mlp0 of layer 0 is missing'):
        check(t.lib.s7b_engine_hvp(t._h, vv.data_ptr(), out.data_ptr(), t._stream()))


def meta_species(meta):
    from sevenn_b200.spec import build_spec
    return build_spec(meta).num_species


def test_compute_unchanged_by_hvp(si0):
    """compute() after hvp() gives the results of compute() before it (to the step's own run-to-run rounding); an engine that never meets an HVP
    keeps one captured step graph (no allocation since: every one bumps the capture key) and the same launches per
    step; after the first HVP the step is recaptured at most once, with the same launch count"""
    import torch
    from sevenn_b200.engine import B200Engine
    meta, arrays, (species, ei, ev) = si0
    e = B200Engine(meta, arrays)
    e.set_graph(species, ei, ev)

    def step():
        e.launch_count(reset=True)
        e.compute()
        torch.cuda.synchronize()
        r = e.results()
        return e.launch_count(), {k: r[k].cpu().numpy() for k in ('energy', 'forces', 'virial')}

    step()
    n1, r1 = step()
    n2, r2 = step()
    cap, _ = e.graph_stats()
    assert n1 == n2 and cap == 1        # any (re)allocation would have forced a recapture
    e.hvp(np.ones((len(species), 3)))
    n3, r3 = step()
    n4, _ = step()
    cap2, _ = e.graph_stats()
    assert n3 == n1 and n4 == n1 and cap2 <= cap + 1
    # the force scatter adds with float atomics, so two steps on the same inputs may already differ in the last
    # bits (arrival order); after the HVP the step stays within that rounding
    for k in r1:
        print(f'{k}: max|step 2 - step 1| = {np.abs(r2[k] - r1[k]).max():.2e}, '
              f'max|after HVP - step 1| = {np.abs(r3[k] - r1[k]).max():.2e}')
        assert np.allclose(r3[k], r1[k], rtol=1e-6, atol=1e-6 * np.abs(r1[k]).max()), k
