"""Cost of the distributed centroid virial (DESIGN.md §8.7), per rank, over NCCL:

    torchrun --nproc_per_node N tools/distributed_centroid_bench.py [--per-gpu 12500] [--reps 10] [--radial table]

Si (diamond) cells of about --per-gpu atoms per GPU, SevenNet-0, split into N bricks along x.  Each rank prints one
JSON line: step ms (DistributedRunner.compute), CV-sequence ms (DistributedRunner.centroid_virials: CV stages plus
their reverse exchanges), the single-GPU one-shot B200Engine.centroid_virial ms on a cell of the same per-GPU size,
bytes per reverse exchange computed from the shapes, and the GPU's name and power limit.  With fewer than two GPUs
it prints "not measured": a single-GPU host-staged timing is not a multi-GPU cost."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu_info(rank):
    try:
        out = subprocess.run(['nvidia-smi', f'--id={rank}', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def _timed(fn, sync, reps):
    fn()
    sync()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    sync()
    return (time.perf_counter() - t0) / reps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--per-gpu', type=int, default=12500)
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--radial', default='table')
    args = ap.parse_args()
    import torch
    world = int(os.environ.get('WORLD_SIZE', '1'))
    if world < 2 or torch.cuda.device_count() < 2:
        print(json.dumps({'distributed_centroid': 'not measured', 'reason': 'needs torchrun with two or more GPUs'}))
        return
    import torch.distributed as dist
    from sevenn_b200.checkpoint import load_weights
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import build_graph, diamond_si
    from sevenn_b200.parallel import DistributedRunner, brick_decompose
    rank = int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', device_id=torch.device('cuda', rank))
    meta, arrays = load_weights(os.path.join(ROOT, 'weights', 'sevennet_0.npz'))
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    ny = max(2, round((args.per_gpu / 8) ** (1 / 3)))          # per-GPU brick of ny^3 conventional cells ...
    pos, cell, z = diamond_si(ny * world, ny, ny, sigma=0.05, seed=1)      # ... stacked along x
    species = np.array([tm[int(a)] for a in z], dtype=np.int32)
    sync = torch.cuda.synchronize
    part = brick_decompose(pos, cell, species, (world, 1, 1), rank, 5.0)
    run = DistributedRunner(B200Engine(meta, arrays, radial=args.radial, device=rank), part)
    step_ms = _timed(run.compute, sync, args.reps)
    cv_ms = _timed(run.centroid_virials, sync, args.reps)
    # one-shot pass on one GPU at the same per-GPU size
    p1, c1, z1 = diamond_si(ny, ny, ny, sigma=0.05, seed=1)
    ei, ev = build_graph(p1, c1, True, 5.0)
    one = B200Engine(meta, arrays, radial=args.radial, device=rank)
    one.set_graph(np.array([tm[int(a)] for a in z1]), ei, ev)
    one.compute()
    one_ms = _timed(one.centroid_virial, sync, args.reps)
    n_ghost, n_send = part['n_nodes'] - part['n_local'], int(sum(run.exchange.send_counts))
    dims = [L.dim_x for L in run.engine.spec.layers]
    per_layer = {t: 4 * 4 * dims[t] * (n_ghost + n_send) for t in range(1, len(dims))}       # 4 fp32 planes, out + in
    print(json.dumps({'rank': rank, 'world': world, 'gpu': _gpu_info(rank), 'radial': args.radial,
                      'atoms_per_gpu': int(part['n_local']), 'ghosts': int(n_ghost), 'step_ms': round(step_ms, 3),
                      'cv_sequence_ms': round(cv_ms, 3), 'one_gpu_centroid_ms': round(one_ms, 3),
                      'one_gpu_atoms': len(p1), 'bytes_per_cv_exchange': per_layer,
                      'bytes_wc_exchange': 8 * 9 * (n_ghost + n_send)}), flush=True)
    run.close()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
