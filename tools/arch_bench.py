#!/usr/bin/env python
"""Step time of the synthetic architectures A-D (tests/synthetic_models.py: other widths, lmax_edge != lmax_node,
lmax 1), which run the runtime-width convolution kernels, on a rattled 12 000-atom Si cell.

    python tools/arch_bench.py --out DIR [--steps 20] [--warmup 5] [--archs A B C D]
                               [--self-connection linear nequip] [--parity]

For each model: ms per device-resident step (energy + forces + virial, the captured CUDA graph of
``s7b_engine_compute``; median of --steps synchronised steps after --warmup), atom-updates per second, and the
per-kernel breakdown of one step from torch.profiler (CUDA time per kernel name, summed over launches).  Prints
one line per model plus the top kernels and writes DIR/arch_bench.json with the GPU name, power limit and SM
clocks read in the same run.  Random weights: the numbers say nothing about accuracy.

``--self-connection``: the self-connection type(s) to time, 'linear' (the synthetic_models.py checkpoints) and / or
'nequip' (the species-wise self-connection of tests/synthetic_nequip.py); each run also reports the CUDA-event
times of the self-connection linears (``sc_gemm`` forward, ``si1T_scT_gemm`` backward) from the engine's profile.
``--parity``: compare the engine's energy and forces on the cell with the fp64 oracle (on the GPU, edge-chunked)
within the tolerance bench.py applies (|dE| <= 1e-4 eV * sqrt(N / 64), max |dF| <= 5e-5 eV/A).
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


def bench(arch, pos, cell, steps, warmup, sc='linear', parity=False):
    import torch
    from sevenn_b200.engine import B200Engine
    with tempfile.TemporaryDirectory() as tmp:
        if sc == 'nequip':
            from synthetic_nequip import convert, write_nequip_checkpoint
            meta, arrays = convert(write_nequip_checkpoint(os.path.join(tmp, f'{arch}.pth'), arch), arch)
        else:
            from synthetic_models import convert, write_checkpoint
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
    # CUDA-event times of the self-connection linears (profiled steps run without the CUDA graph)
    eng.set_profiling(True)
    for _ in range(3):
        eng.compute()
    torch.cuda.synchronize()
    sc_ms = {k: v[0] / v[1] for k, v in eng.profile().items()
             if k.startswith(('sc_gemm', 'si1T_scT_gemm', 'species_segment'))}
    eng.set_profiling(False)
    out = dict(arch=arch, self_connection=sc, atoms=len(pos), edges=int(eng.n_edges), ms_per_step=ms,
               ms_min=min(times), ms_max=max(times), atom_updates_per_s=len(pos) / (ms * 1e-3), sc_linears_ms=sc_ms,
               kernels_ms=dict(sorted(kernels.items(), key=lambda kv: -kv[1])))
    if parity:
        out['parity'] = oracle_parity(eng, meta, arrays, sp, pos, cell)
    return out


def oracle_parity(eng, meta, arrays, sp, pos, cell):
    import torch
    from nequip_oracle import nequip_oracle
    from sevenn_b200.neighbors import build_graph
    eng.compute()
    torch.cuda.synchronize()
    r = eng.results()
    energy, forces = float(r['energy'].cpu()[0]), r['forces'].cpu().numpy().astype(np.float64)
    ei, ev = build_graph(pos, cell, True, float(meta['cutoff']))
    ref = nequip_oracle(meta, arrays, dtype=torch.float64, device='cuda').forward(sp, ei, ev, edge_chunk=32768)
    dE = energy - float(ref['energy'])
    dF = float(np.abs(forces - ref['forces'].cpu().numpy()).max())
    tolE, tolF = 1e-4 * (max(len(sp), 64) / 64.0) ** 0.5, 5e-5
    del ref
    torch.cuda.empty_cache()
    return dict(dE_eV=dE, max_dF_eV_per_A=dF, tol_dE_eV=tolE, tol_dF_eV_per_A=tolF, ok=bool(abs(dE) <= tolE and dF <= tolF))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--archs', nargs='+', default=['A', 'B', 'C', 'D'])
    ap.add_argument('--self-connection', nargs='+', default=['linear'], choices=['linear', 'nequip'])
    ap.add_argument('--parity', action='store_true')
    args = ap.parse_args()
    from sevenn_b200.neighbors import diamond_si
    pos, cell, _ = diamond_si(15, 10, 10, sigma=0.05, seed=0)       # 12 000 atoms
    info = gpu_info()
    print('gpu:', info)
    res = []
    for arch, sc in [(a, c) for a in args.archs for c in args.self_connection]:
        r = bench(arch, pos, cell, args.steps, args.warmup, sc, args.parity)
        res.append(r)
        print(f'{arch} ({sc}): {r["atoms"]} atoms, {r["edges"]} edges, {r["ms_per_step"]:.3f} ms/step '
              f'({r["ms_min"]:.3f}-{r["ms_max"]:.3f}), {r["atom_updates_per_s"]:.3e} atom-updates/s')
        print('    self-connection linears (ms):', ', '.join(f'{k} {v:.4f}' for k, v in sorted(r['sc_linears_ms'].items())))
        if 'parity' in r:
            print('    parity vs fp64 oracle:', r['parity'])
        for k, v in list(r['kernels_ms'].items())[:12]:
            print(f'    {v:8.3f} ms  {k[:140]}')
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'arch_bench.json'), 'w') as f:
        json.dump(dict(gpu=info, results=res), f, indent=1)


if __name__ == '__main__':
    main()
