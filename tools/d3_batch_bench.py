#!/usr/bin/env python
"""Batched D3 on the GPU: one ``D3Engine.compute`` per structure (host wrap and upload, two synchronisations per
structure) against ``D3Batch`` (one pass from device-resident arrays), and ``SevenNetModel`` against
``SevenNetD3Model`` (network alone, network + D3 in one batch).

    python tools/d3_batch_bench.py --out DIR [--runs 20] [--warmup 5]

Workloads: B in {1, 16, 128, 512} rattled 64-atom NaCl cells (one seed per cell) and one mixed batch (the systems
of tests/d3_cells.py).  For each workload the legs are alternated in the same process; each time is the median of
--runs synchronised calls after --warmup calls.  Before timing, the per-structure loop and the batch are compared
(energies 1e-12 relative, forces bit for bit).  Prints one line per workload and writes DIR/d3_batch_bench.json with
the GPU name, power limit and SM clocks read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from batch_bench import gpu_info, state_of, timed  # noqa: E402


def nacl_batch(B, seed0=0):
    from sevenn_b200.neighbors import rocksalt_nacl
    out = []
    for b in range(B):
        pos, cell, z = rocksalt_nacl(2, 2, 2, sigma=0.05, seed=seed0 + b)
        out.append((z, pos, cell, (True, True, True)))
    return out


def mixed_batch():
    import d3_cells as C
    return [C.FIXTURES[k]() for k in ('sheared', 'rotated', 'slab', 'wire', 'compressed_cs', 'species16', 'molecule')]


def loop_d3(eng, structs, max_cutoff):
    """the per-structure path: D3Calculator's rule for a missing cell, then one D3Engine.compute each"""
    out = []
    for z, pos, cell, pbc in structs:
        if np.all(np.asarray(cell) == 0):
            cell, pbc = np.eye(3) * (pos.max(axis=0) - pos.min(axis=0) + max_cutoff + 1.0), (True, True, True)
        out.append(eng.compute(z, pos, cell, pbc))
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', required=True)
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--sizes', default='1,16,128,512')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('d3_batch_bench needs a CUDA device')
    from sevenn_b200.batch import SevenNetD3Model, SevenNetModel
    from sevenn_b200.d3 import D3Batch, D3Engine
    os.makedirs(args.out, exist_ok=True)
    info_before = gpu_info()
    print('gpu:', info_before, flush=True)
    eng, d3b = D3Engine(), D3Batch()
    net, netd3 = SevenNetModel('7net-0', device='cuda'), SevenNetD3Model('7net-0', device='cuda')
    workloads = [(f'nacl64_x{B}', nacl_batch(B, 1000 * k)) for k, B in enumerate(int(s) for s in args.sizes.split(','))]
    workloads.append(('mixed', mixed_batch()))
    results = []
    for name, structs in workloads:
        state = state_of(structs)
        n_atoms = int(state.positions.shape[0])
        cells = state.row_vector_cell.detach().cpu().numpy()
        counts = [len(s[0]) for s in structs]
        atom_ptr = np.concatenate([[0], np.cumsum(counts)])
        # agreement first
        old = loop_d3(eng, structs, d3b.max_cutoff)
        new = d3b.compute(state.atomic_numbers, state.positions, cells, state.pbc, atom_ptr=atom_ptr)
        e_new, f_new = new['energy'].cpu().numpy(), new['forces'].cpu().numpy()
        de = max(abs(e_new[b] / old[b][0] - 1.0) for b in range(len(structs)))
        f_same = all(np.array_equal(f_new[atom_ptr[b]:atom_ptr[b + 1]], old[b][1]) for b in range(len(structs)))
        agree = dict(max_rel_de=float(de), forces_bitwise=f_same, ok=bool(de <= 1e-12 and f_same))
        legs = {
            'd3_loop': lambda: loop_d3(eng, structs, d3b.max_cutoff),
            'd3_batch': lambda: d3b.compute(state.atomic_numbers, state.positions, cells, state.pbc, system_idx=state.system_idx),
            'forward_net': lambda: net(state),
            'forward_net_d3': lambda: netd3(state),
        }
        times = {k: [] for k in legs}
        for rep in range(args.warmup + args.runs):
            for k, fn in legs.items():
                t = timed(fn, torch)
                if rep >= args.warmup:
                    times[k].append(t)
        med = {k: statistics.median(v) for k, v in times.items()}
        row = dict(workload=name, structures=len(structs), atoms=n_atoms, median_ms=med,
                   min_ms={k: min(v) for k, v in times.items()}, speedup_d3=med['d3_loop'] / med['d3_batch'],
                   d3_share_of_forward=1.0 - med['forward_net'] / med['forward_net_d3'], agreement=agree)
        results.append(row)
        print(f"{name:>12s}  B={len(structs):4d} n={n_atoms:6d}  D3 {med['d3_loop']:8.2f} -> {med['d3_batch']:7.2f} ms"
              f"  forward net {med['forward_net']:7.2f} / net+D3 {med['forward_net_d3']:7.2f} ms  agree={agree}", flush=True)
    out = dict(gpu_before=info_before, gpu_after=gpu_info(), runs=args.runs, warmup=args.warmup, results=results)
    with open(os.path.join(args.out, 'd3_batch_bench.json'), 'w') as f:
        json.dump(out, f, indent=1)
    if not all(r['agreement']['ok'] for r in results):
        raise SystemExit('the two D3 paths disagree')


if __name__ == '__main__':
    main()
