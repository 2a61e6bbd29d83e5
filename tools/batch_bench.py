#!/usr/bin/env python
"""Batched evaluation on the GPU: the per-structure host path (``batch.BatchedEvaluator``, as the TorchSim
adapter used it before ``batch.DeviceBatch``) against the device path (``DeviceBatch``: one batched device
neighbour list and fp64 per-structure sums on the device).

    python tools/batch_bench.py --out DIR [--runs 20] [--warmup 5]

Workloads: B in {1, 16, 128, 512} rattled 64-atom Si cells (one seed per cell), the batch sizes of
high-throughput relaxation and screening, and one mixed batch of 2-1 000-atom structures (triclinic, slab,
molecule) that takes the bounding-box pass of the non-periodic directions.  For each workload the two paths are
alternated in the same process, each on its own engine (so that neither evicts the other's captured CUDA graph):
the graph build alone, and the whole ``SevenNetModel.forward`` (state on the device -> energy, forces, stress).
Each time is the median of --runs synchronised calls after --warmup calls.  Before timing, the two paths'
energies and forces are compared.  Prints one line per workload and writes DIR/batch_bench.json with the GPU
name, power limit and SM clocks read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

E_RTOL, F_ATOL = 2e-5, 2e-5     # the adapter test's bounds (tests/test_batch_device_gpu.py)


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        row = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # noqa: BLE001
        return {'error': str(ex)}
    return dict(zip(q.split(','), [c.strip() for c in row.split(',')]))


def si_batch(B, seed0=0):
    from sevenn_b200.neighbors import diamond_si
    out = []
    for b in range(B):
        pos, cell, z = diamond_si(2, 2, 2, sigma=0.08, seed=seed0 + b)
        out.append((z, pos, cell, (True, True, True)))
    return out


def mixed_batch():
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    rng = np.random.RandomState(3)
    out = []
    a = 5.431
    prim = 0.5 * a * np.array([[0.0, 1.0, 1.0], [1.0, 0.0, 1.0], [1.0, 1.0, 0.0]])       # 2-atom triclinic Si
    out.append((np.full(2, 14), np.array([[0, 0, 0], [0.25, 0.25, 0.25]]) @ prim + rng.normal(0, .05, (2, 3)),
                prim, (True, True, True)))
    pos, cell, z = diamond_si(3, 3, 3, sigma=0.05, seed=4)                            # sheared 216-atom Si
    shear = np.array([[1.0, 0.0, 0.0], [0.3, 1.0, 0.0], [-0.2, 0.1, 1.0]])
    out.append((z, pos @ shear, cell @ shear, (True, True, True)))
    pos, cell, z = rocksalt_nacl(3, 3, 2, sigma=0.05, seed=5)                          # 144-atom NaCl slab
    cell = cell.copy()
    cell[2, 2] = 30.0
    out.append((z, pos, cell, (True, True, False)))
    pos, cell, z = diamond_si(2, 2, 2, sigma=0.05, seed=6)                             # 35-atom Si cluster, no cell
    keep = np.argsort(np.linalg.norm(pos - pos.mean(0), axis=1))[:35]
    out.append((z[keep], pos[keep], np.zeros((3, 3)), (False, False, False)))
    pos, cell, z = diamond_si(5, 5, 5, sigma=0.05, seed=7)                             # 1 000-atom Si
    out.append((z, pos, cell, (True, True, True)))
    out += si_batch(12, 100)
    return out


def state_of(structs):
    import torch
    counts = [len(s[0]) for s in structs]
    return types.SimpleNamespace(
        positions=torch.tensor(np.concatenate([s[1] for s in structs]), dtype=torch.float64, device='cuda'),
        row_vector_cell=torch.tensor(np.stack([s[2] for s in structs]), dtype=torch.float64, device='cuda'),
        pbc=torch.tensor(np.array([s[3] for s in structs]), device='cuda'),
        atomic_numbers=torch.tensor(np.concatenate([s[0] for s in structs]), device='cuda'),
        system_idx=torch.tensor(np.repeat(np.arange(len(structs)), counts), device='cuda'))


def host_systems(state):
    """What the per-structure path did first: copy the state to the host and slice out every structure."""
    import torch
    pos = state.positions.detach().cpu().double().numpy()
    cells = state.row_vector_cell.detach().cpu().double().numpy().reshape(-1, 3, 3)
    numbers = state.atomic_numbers.cpu().numpy()
    sys_idx = state.system_idx.cpu().numpy()
    pbc = np.broadcast_to(torch.as_tensor(state.pbc).cpu().numpy().astype(bool), (len(cells), 3))
    return [dict(numbers=numbers[sys_idx == b], positions=pos[sys_idx == b], cell=cells[b], pbc=pbc[b])
            for b in range(len(cells))]


def stress_of(torch, virial, cells):
    vol = torch.as_tensor(np.abs(np.linalg.det(cells)), device=virial.device)
    v = -(virial / vol[:, None])[:, [0, 1, 2, 4, 5, 3]]
    return torch.stack([torch.stack([v[:, 0], v[:, 5], v[:, 4]], -1), torch.stack([v[:, 5], v[:, 1], v[:, 3]], -1),
                        torch.stack([v[:, 4], v[:, 3], v[:, 2]], -1)], -2)


def old_forward(torch, ev, state):
    """``SevenNetModel.forward`` on the per-structure path (host copy, one neighbour list per structure)."""
    systems = host_systems(state)
    out = ev.compute(systems)
    cells = np.stack([s['cell'] for s in systems])
    return {'energy': out['energy'].float(), 'forces': out['forces'],
            'stress': stress_of(torch, out['virial'], cells).float()}


def timed(fn, torch):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--out', required=True)
    ap.add_argument('--runs', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--sizes', default='1,16,128,512')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('batch_bench needs a CUDA device')
    from sevenn_b200.batch import BatchedEvaluator, SevenNetModel
    os.makedirs(args.out, exist_ok=True)
    info_before = gpu_info()
    print('gpu:', info_before, flush=True)
    new = SevenNetModel('7net-0', device='cuda')
    old_model = SevenNetModel('7net-0', device='cuda')
    ev = BatchedEvaluator(old_model.engine)
    workloads = [(f'si64_x{B}', si_batch(B, 1000 * k)) for k, B in enumerate(int(s) for s in args.sizes.split(','))]
    workloads.append(('mixed', mixed_batch()))
    results = []
    for name, structs in workloads:
        state = state_of(structs)
        n_atoms = int(state.positions.shape[0])
        # agreement first (positions in float64)
        o_new, o_old = new(state), old_forward(torch, ev, state)
        de = (o_new['energy'].double() - o_old['energy'].double()).abs()
        e_ok = bool((de <= E_RTOL * o_old['energy'].double().abs().clamp(min=1.0)).all())
        df = float((o_new['forces'] - o_old['forces']).abs().max()) if n_atoms else 0.0
        agree = dict(max_abs_de=float(de.max()), max_abs_df=df, ok=e_ok and df <= F_ATOL)
        legs = {
            'build_old': lambda: ev.set_batch(host_systems(state)),
            'build_new': lambda: new._batch.set_batch(state.atomic_numbers, state.positions,
                                                      state.row_vector_cell.detach().cpu(), state.pbc, state.system_idx),
            'forward_old': lambda: old_forward(torch, ev, state),
            'forward_new': lambda: new(state),
        }
        times = {k: [] for k in legs}
        for rep in range(args.warmup + args.runs):
            for k, fn in legs.items():          # alternated: old, new, old, new in every repetition
                t = timed(fn, torch)
                if rep >= args.warmup:
                    times[k].append(t)
        med = {k: statistics.median(v) for k, v in times.items()}
        row = dict(workload=name, structures=len(structs), atoms=n_atoms, n_edges=int(new.engine.n_edges),
                   median_ms=med, min_ms={k: min(v) for k, v in times.items()},
                   speedup_build=med['build_old'] / med['build_new'],
                   speedup_forward=med['forward_old'] / med['forward_new'], agreement=agree,
                   graph_stats_new=new.engine.graph_stats())
        results.append(row)
        print(f"{name:>10s}  B={len(structs):4d} n={n_atoms:6d}  build {med['build_old']:8.2f} -> {med['build_new']:7.2f} ms"
              f"  forward {med['forward_old']:8.2f} -> {med['forward_new']:7.2f} ms  agree={agree}", flush=True)
    out = dict(gpu_before=info_before, gpu_after=gpu_info(), runs=args.runs, warmup=args.warmup, results=results)
    with open(os.path.join(args.out, 'batch_bench.json'), 'w') as f:
        json.dump(out, f, indent=1)
    if not all(r['agreement']['ok'] for r in results):
        raise SystemExit('the two paths disagree')


if __name__ == '__main__':
    main()
