"""Cost of the engine's Hessian-vector product (B200Engine.hvp) against its energy/force step, and of a full Hessian
(SevenNetCalculator.get_hessian, 3N HVPs) against 6N central-difference force evaluations batched through
DeviceBatch.  Prints one JSON line per measurement and writes them all to --out; the card, its power limit and its
SM clocks are read in the same run.

    python tools/hvp_bench.py --out /tmp/hvp_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader'], capture_output=True, text=True)
    return dict(zip(q.split(','), [s.strip() for s in out.stdout.strip().splitlines()[0].split(',')]))


def timed(fn, reps):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def species_of(meta, z):
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    return np.array([tm[int(a)] for a in z], dtype=np.int32)


def step_vs_hvp(name, reps):
    import torch
    from sevenn_b200.checkpoint import load_weights
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = load_weights(os.path.join(ROOT, 'weights', f'{name}.npz'))
    rows = []
    for nc in ((2, 2, 2), (4, 4, 4), (10, 10, 15)):
        pos, cell, z = diamond_si(*nc, sigma=0.05, seed=1)
        e = B200Engine(meta, arrays)
        e.set_positions(species_of(meta, z), pos, cell, True)
        v = torch.randn(len(z), 3, device=e.device)
        for _ in range(3):
            e.compute()
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        e.hvp(v)
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info()[0]
        e.compute()
        t_step = timed(e.compute, reps)
        e.hvp(v)
        t_hvp = timed(lambda: e.hvp(v), max(reps // 4, 3))
        rows.append(dict(kind='hvp_vs_step', model=name, atoms=len(z), edges=e.n_edges, step_ms=t_step, hvp_ms=t_hvp,
                         ratio=t_hvp / t_step, hvp_alloc_GB=(free0 - free1) / 1e9))
        print(json.dumps(rows[-1]), flush=True)
        del e
        torch.cuda.empty_cache()
    return rows


class _Atoms:
    def __init__(self, pos, cell, z):
        self.p, self.c, self.z = pos, cell, z

    def get_positions(self):
        return self.p

    def get_cell(self):
        return self.c

    def get_pbc(self):
        return np.array([True] * 3)

    def get_atomic_numbers(self):
        return self.z


def full_hessian(nc, h=1e-2):
    import torch
    from sevenn_b200.batch import DeviceBatch
    from sevenn_b200.calculator import SevenNetCalculator
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(*nc, sigma=0.05, seed=1)
    n = len(z)
    calc = SevenNetCalculator('7net-0')
    atoms = _Atoms(pos, cell, z)
    calc.get_hessian(atoms)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    H = calc.get_hessian(atoms)
    torch.cuda.synchronize()
    t_hvp = time.perf_counter() - t0
    # 6N displaced copies, force differences: H[3i + a, :] = -(F(+h e_ia) - F(-h e_ia)) / 2h
    db = DeviceBatch(calc.engine)
    disp = np.repeat(pos[None], 6 * n, axis=0)
    for k in range(3 * n):
        disp[2 * k].reshape(-1)[k] += h
        disp[2 * k + 1].reshape(-1)[k] -= h
    chunk = max(2, (2 * 40000 // n) // 2 * 2)      # structures per batch (even: +h and -h together)

    def fd():
        out = []
        for s in range(0, 6 * n, chunk):
            m = min(chunk, 6 * n - s)
            idx = np.repeat(np.arange(m), n)
            r = db.compute(np.tile(z, m), disp[s:s + m].reshape(-1, 3), np.repeat(cell[None], m, axis=0), True, idx)
            out.append(torch.as_tensor(r['forces']).reshape(m, n * 3).double().cpu().numpy())
        F = np.concatenate(out)
        return -(F[0::2] - F[1::2]) / (2 * h)
    fd()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    Hfd = fd()
    torch.cuda.synchronize()
    t_fd = time.perf_counter() - t0
    row = dict(kind='full_hessian', model='sevennet_0', atoms=n, hvp_s=t_hvp, fd_6N_s=t_fd,
               max_abs_H=float(np.abs(H).max()), max_diff_vs_fd_rel=float(np.abs(H - Hfd).max() / np.abs(H).max()),
               asym_rel=float(np.abs(H - H.T).max() / np.abs(H).max()))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('hvp_bench.py needs a CUDA device')
    rows = [dict(kind='card', **card())]
    print(json.dumps(rows[0]), flush=True)
    for name in ('sevennet_0', 'sevennet_l3i5'):
        rows += step_vs_hvp(name, a.reps)
    for nc in ((2, 2, 2), (3, 3, 3)):
        rows.append(full_hessian(nc))
    rows.append(dict(kind='card_after', **card()))
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
