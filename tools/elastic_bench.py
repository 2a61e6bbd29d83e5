"""Cost of the elastic-tensor path: one strain product (B200Engine.hvp_strain) against one plain Hessian-vector
product, SevenNetCalculator.get_elastic_tensor on 2-, 8- and 64-atom Si cells, and DeviceBatch.elastic_tensors for 64
cells of 2 and of 8 atoms in one batch (SevenNet-0, table mode).  Prints one JSON line per measurement and writes them
all to --out; the card, its power limit and its SM clocks are read in the same run.

    python tools/elastic_bench.py --out /tmp/elastic_bench.json
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from hvp_bench import _Atoms, card, species_of, timed  # noqa: E402


def si_cell(kind, seed=1):
    """(pos, cell, z): 'prim' the 2-atom primitive cell, else diamond_si(k, k, k) with k = kind"""
    from sevenn_b200.neighbors import diamond_si
    a = 5.431
    if kind == 'prim':
        cell = 0.5 * a * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]])
        return np.array([[0.0, 0.0, 0.0], [0.25 * a] * 3]), cell, np.array([14, 14])
    return diamond_si(kind, kind, kind, sigma=0.0, seed=seed)


def product_vs_hvp(reps):
    import torch
    from sevenn_b200.checkpoint import load_weights
    from sevenn_b200.elastic import voigt_strains
    from sevenn_b200.engine import B200Engine
    meta, arrays = load_weights(os.path.join(ROOT, 'weights', 'sevennet_0.npz'))
    rows = []
    for k in (2, 4):
        pos, cell, z = si_cell(k)
        e = B200Engine(meta, arrays)
        e.set_positions(species_of(meta, z), pos, cell, True)
        e.compute()
        v = torch.randn(len(z), 3, device=e.device)
        eps = torch.as_tensor(voigt_strains()[3][None], device=e.device)
        e.hvp(v)
        e.hvp_strain(None, eps)
        t_hvp = timed(lambda: e.hvp(v), reps)
        t_str = timed(lambda: e.hvp_strain(None, eps), reps)
        rows.append(dict(kind='strain_product_vs_hvp', model='sevennet_0', atoms=len(z), edges=e.n_edges,
                         hvp_ms=t_hvp, strain_product_ms=t_str, ratio=t_str / t_hvp))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def calculator(reps):
    import torch
    from sevenn_b200.calculator import SevenNetCalculator
    calc = SevenNetCalculator('7net-0')
    rows = []
    for kind in ('prim', 1, 2):
        atoms = _Atoms(*si_cell(kind))
        for relaxed in (False, True):
            calc.get_elastic_tensor(atoms, relaxed=relaxed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                C = calc.get_elastic_tensor(atoms, relaxed=relaxed)
            dt = (time.perf_counter() - t0) / reps
            rows.append(dict(kind='get_elastic_tensor', model='sevennet_0', atoms=len(atoms.z), relaxed=relaxed, s=dt,
                             C11_C12_C44_GPa=[round(float(C[0, 0]) / 0.006241509, 2),
                                              round(float(C[0, 1]) / 0.006241509, 2),
                                              round(float(C[3, 3]) / 0.006241509, 2)]))
            print(json.dumps(rows[-1]), flush=True)
    return rows


def batch(reps, B=64):
    import torch
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.calculator import SevenNetCalculator
    calc = SevenNetCalculator('7net-0')
    db = DeviceBatch(calc.engine)
    rows = []
    for kind in ('prim', 1):
        cells = [si_cell(kind) for _ in range(B)]
        scale = 1.0 + 0.01 * np.linspace(-1, 1, B)          # 64 different lattice constants
        pos = np.concatenate([p * s for (p, _, _), s in zip(cells, scale)])
        cell = np.stack([c * s for (_, c, _), s in zip(cells, scale)])
        z = np.concatenate([z for _, _, z in cells])
        idx = np.repeat(np.arange(B), len(cells[0][2]))
        for relaxed in (False, True):
            db.elastic_tensors(z, pos, cell, True, idx, relaxed=relaxed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(reps):
                db.elastic_tensors(z, pos, cell, True, idx, relaxed=relaxed)
            dt = (time.perf_counter() - t0) / reps
            one = _Atoms(cells[0][0] * scale[0], cells[0][1] * scale[0], cells[0][2])
            calc.get_elastic_tensor(one, relaxed=relaxed)
            t0 = time.perf_counter()
            for _ in range(reps):
                calc.get_elastic_tensor(one, relaxed=relaxed)
            t1 = (time.perf_counter() - t0) / reps
            rows.append(dict(kind='batch_elastic_tensors', model='sevennet_0', structures=B, atoms_each=len(cells[0][2]),
                             relaxed=relaxed, batch_s=dt, per_structure_ms=1e3 * dt / B, single_call_s=t1,
                             speedup_vs_B_single_calls=B * t1 / dt))
            print(json.dumps(rows[-1]), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('elastic_bench.py needs a CUDA device')
    rows = [dict(kind='card', **card())]
    print(json.dumps(rows[0]), flush=True)
    rows += product_vs_hvp(20 * a.reps)
    rows += calculator(a.reps)
    rows += batch(a.reps)
    rows.append(dict(kind='card_after', **card()))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
