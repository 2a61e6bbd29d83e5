#!/usr/bin/env python
"""Step time of the synthetic architectures A-D (tests/synthetic_models.py: other widths, lmax_edge != lmax_node,
lmax 1), which run the runtime-width convolution kernels, on a rattled 12 000-atom Si cell.

    python tools/arch_bench.py --out DIR [--steps 20] [--warmup 5] [--archs A B C D]

For each model: ms per device-resident step (energy + forces + virial, the captured CUDA graph of
``s7b_engine_compute``; median of --steps synchronised steps after --warmup), atom-updates per second, and the
per-kernel breakdown of one step from torch.profiler (CUDA time per kernel name, summed over launches).  Prints
one line per model plus the top kernels and writes DIR/arch_bench.json with the GPU name, power limit and SM
clocks read in the same run.  Random weights: the numbers say nothing about accuracy.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        row = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # noqa: BLE001
        return {'error': str(ex)}
    return dict(zip(q.split(','), [c.strip() for c in row.split(',')]))


def bench(arch, pos, cell, steps, warmup):
    import torch
    from synthetic_models import convert, write_checkpoint
    from sevenn_b200.engine import B200Engine
    with tempfile.TemporaryDirectory() as tmp:
        meta, arrays = convert(write_checkpoint(os.path.join(tmp, f'{arch}.pth'), arch), arch)
    eng = B200Engine(meta, arrays, radial='table')
    sp = np.full(len(pos), eng.spec.type_map[14], dtype=np.int32)
    eng.set_positions(sp, pos, cell, True)
    for _ in range(warmup):
        eng.compute()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(steps):
        t0.record()
        eng.compute()
        t1.record()
        t1.synchronize()
        times.append(t0.elapsed_time(t1))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.compute()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, 'device_time_total', None)
        if t is None:
            t = getattr(ev, 'cuda_time_total', 0.0)
        if t > 0:
            kernels[ev.key] = kernels.get(ev.key, 0.0) + t / 1000.0
    ms = statistics.median(times)
    return dict(arch=arch, atoms=len(pos), edges=int(eng.n_edges), ms_per_step=ms,
                ms_min=min(times), ms_max=max(times), atom_updates_per_s=len(pos) / (ms * 1e-3),
                kernels_ms=dict(sorted(kernels.items(), key=lambda kv: -kv[1])))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--archs', nargs='+', default=['A', 'B', 'C', 'D'])
    args = ap.parse_args()
    from sevenn_b200.neighbors import diamond_si
    pos, cell, _ = diamond_si(15, 10, 10, sigma=0.05, seed=0)       # 12 000 atoms
    info = gpu_info()
    print('gpu:', info)
    res = []
    for arch in args.archs:
        r = bench(arch, pos, cell, args.steps, args.warmup)
        res.append(r)
        print(f'{arch}: {r["atoms"]} atoms, {r["edges"]} edges, {r["ms_per_step"]:.3f} ms/step '
              f'({r["ms_min"]:.3f}-{r["ms_max"]:.3f}), {r["atom_updates_per_s"]:.3e} atom-updates/s')
        for k, v in list(r['kernels_ms'].items())[:12]:
            print(f'    {v:8.3f} ms  {k[:140]}')
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'arch_bench.json'), 'w') as f:
        json.dump(dict(gpu=info, results=res), f, indent=1)


if __name__ == '__main__':
    main()
