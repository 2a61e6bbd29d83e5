"""Cost of the engine's heat flux (B200Engine.heat_flux, one tangent-forward pass of four channels) against one
energy/force step and one Hessian-vector product, on Si cells of 64 / 512 / 12 000 atoms, SevenNet-0 and
SevenNet-l3i5, both radial modes; the device memory the first flux call allocates; and, with --profile, a
torch.profiler kernel breakdown of one pass (SevenNet-0, 512 atoms).  Prints one JSON line per measurement and writes
them all to --out; the card, its power limit and its SM clocks are read in the same run.

    python tools/heat_flux_bench.py --out /tmp/heat_flux_bench.json --profile
"""
import argparse
import json
import os
import subprocess
import sys

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


def engine_on(name, radial, nc):
    import torch
    from sevenn_b200.checkpoint import load_weights
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import diamond_si
    meta, arrays = load_weights(os.path.join(ROOT, 'weights', f'{name}.npz'))
    pos, cell, z = diamond_si(*nc, sigma=0.05, seed=1)
    e = B200Engine(meta, arrays, radial=radial)
    e.set_positions(species_of(meta, z), pos, cell, True)
    v = torch.randn(len(z), 3, device=e.device)
    return e, v


def measure(name, radial, nc, reps):
    import torch
    e, v = engine_on(name, radial, nc)
    for _ in range(3):
        e.compute()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    e.heat_flux(v)
    torch.cuda.synchronize()
    flux_mem = free0 - torch.cuda.mem_get_info()[0]
    e.hvp(v)
    e.compute()
    torch.cuda.synchronize()
    step = timed(e.compute, reps)
    flux = timed(lambda: e.heat_flux(v), reps)
    hvp = timed(lambda: e.hvp(v), max(1, reps // 2))
    row = dict(model=name, radial=radial, atoms=int(e.n_nodes), edges=int(e.n_edges), step_ms=round(step, 3),
               flux_ms=round(flux, 3), hvp_ms=round(hvp, 3), flux_over_step=round(flux / step, 2),
               flux_over_hvp=round(flux / hvp, 2), first_flux_call_bytes=int(flux_mem))
    del e
    torch.cuda.empty_cache()
    return row


def profile(out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    e, v = engine_on('sevennet_0', 'table', (4, 4, 4))
    e.compute()
    e.heat_flux(v)
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        e.heat_flux(v)
        torch.cuda.synchronize()
    rows = {}
    for ev in p.key_averages():
        if ev.device_type.name == 'CUDA' and ev.device_time_total > 0:
            k = ev.key.split('<')[0].split('(')[0]
            rows[k] = rows.get(k, 0.0) + ev.device_time_total / 1000.0
    total = sum(rows.values())
    table = sorted(rows.items(), key=lambda kv: -kv[1])
    if out_dir:
        p.export_chrome_trace(os.path.join(out_dir, 'heat_flux_trace.json'))
    return dict(profile='sevennet_0 table Si512 one flux pass', total_kernel_ms=round(total, 3),
                kernels={k: round(t, 3) for k, t in table[:15]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--profile', action='store_true')
    ap.add_argument('--sizes', default='2,2,2;4,4,4;10,10,15')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('heat_flux_bench needs a CUDA device')
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for name in ('sevennet_0', 'sevennet_l3i5'):
        for radial in ('table', 'mlp'):
            for s in args.sizes.split(';'):
                nc = tuple(int(x) for x in s.split(','))
                row = measure(name, radial, nc, args.reps if nc[0] < 10 else max(3, args.reps // 4))
                rows.append(row)
                print(json.dumps(row), flush=True)
    if args.profile:
        row = profile(os.path.dirname(args.out) if args.out else None)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(rows, open(args.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
