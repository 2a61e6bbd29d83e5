"""Cost of the D3 second order: one D3 Hessian-vector product (D3Engine.hvp_strain, position and strain tangent)
against the three forward stages on rock-salt NaCl of 1 000 and 50 000 atoms for both dampings (default cutoffs),
SevenNetD3Calculator.get_hessian against SevenNetCalculator.get_hessian on a 64-atom NaCl cell, and
DeviceBatch.elastic_tensors with and without d3 for 16 rattled 8-atom NaCl cells.  Prints one JSON line per
measurement and writes them all to --out; the card, its power limit and its SM clocks are read in the same run.

    python tools/d3_hvp_bench.py --out /tmp/d3_hvp_bench.json
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

from hvp_bench import _Atoms, card, timed  # noqa: E402


def hvp_vs_forward(reps):
    import torch
    from sevenn_b200.d3 import D3Engine
    from sevenn_b200.neighbors import rocksalt_nacl
    rows = []
    for nc in ((5, 5, 5), (23, 23, 12)):                 # 1 000 and 50 784 atoms
        pos, cell, z = rocksalt_nacl(*nc, sigma=0.05, seed=1)
        for damping in ('damp_bj', 'damp_zero'):
            eng = D3Engine(damping, 'pbe')
            eng.set_system(z, pos, cell, (True, True, True))
            rng = np.random.RandomState(0)
            v = torch.as_tensor(rng.normal(size=pos.shape), device=eng.device)
            eps = torch.as_tensor(rng.normal(size=(1, 3, 3)), device=eng.device)

            def fwd():
                for s in (1, 2, 3):
                    eng.run_stage(s)
            fwd()
            eng.hvp_strain(v, eps)
            torch.cuda.synchronize()
            r = max(1, reps if len(z) < 10000 else reps // 5)
            t_f = timed(fwd, r)
            t_h = timed(lambda: eng.hvp_strain(v, eps), r)
            rows.append(dict(kind='d3_hvp_vs_forward', atoms=len(z), damping=damping, forward_ms=round(t_f, 3),
                             hvp_ms=round(t_h, 3), ratio=round(t_h / t_f, 2)))
    return rows


def hessians():
    import torch
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.d3 import SevenNetD3Calculator
    from sevenn_b200.neighbors import rocksalt_nacl
    pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.05, seed=1)
    atoms = _Atoms(pos, cell, z)
    rows = []
    for name, calc in (('SevenNetCalculator', SevenNetCalculator('7net-0')),
                       ('SevenNetD3Calculator', SevenNetD3Calculator('7net-0', device='cuda'))):
        calc.get_hessian(atoms)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        calc.get_hessian(atoms)
        torch.cuda.synchronize()
        rows.append(dict(kind='get_hessian', calculator=name, atoms=len(z), ms=round(1e3 * (time.perf_counter() - t0), 1)))
    return rows


def batch_elastic():
    import torch
    from sevenn_b200.batch import DeviceBatch, SevenNetD3Model
    from sevenn_b200.neighbors import rocksalt_nacl
    B = 16
    structs = [rocksalt_nacl(1, 1, 1, sigma=0.05, seed=s) for s in range(B)]
    pos = torch.as_tensor(np.concatenate([s[0] for s in structs]), device='cuda')
    cells = np.stack([s[1] for s in structs])
    z = torch.as_tensor(np.concatenate([s[2] for s in structs]), device='cuda')
    si = torch.repeat_interleave(torch.arange(B, device='cuda'), 8)
    model = SevenNetD3Model('7net-0', device='cuda')
    db = DeviceBatch(model.engine)
    rows = []
    for tag, d3 in (('without_d3', None), ('with_d3', model.d3)):
        db.elastic_tensors(z, pos, cells, True, si, d3=d3)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        db.elastic_tensors(z, pos, cells, True, si, d3=d3)
        torch.cuda.synchronize()
        rows.append(dict(kind='DeviceBatch.elastic_tensors', d3=tag, structures=B, atoms_each=8,
                         ms=round(1e3 * (time.perf_counter() - t0), 1)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('d3_hvp_bench needs a CUDA device')
    rows = [dict(kind='card', **card())]
    print(json.dumps(rows[0]), flush=True)
    for part in (lambda: hvp_vs_forward(args.reps), hessians, batch_elastic):
        for r in part():
            print(json.dumps(r), flush=True)
            rows.append(r)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
