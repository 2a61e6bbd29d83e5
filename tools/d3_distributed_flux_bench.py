"""Cost of D3's heat flux and per-atom centroid virial on the distributed partial-range driver (DESIGN.md §8.8), per
rank, over NCCL:

    torchrun --nproc_per_node N tools/d3_distributed_flux_bench.py [--reps 10] [--out result.json]

World 1 is allowed.  The cells of §8.4 / §8.6: rattled rock-salt NaCl of 50 784 atoms and rattled diamond Si of 49 096
atoms, PBE, default cutoffs, both dampings.  Each rank prints one JSON line per cell and damping: the distributed
forward (``distributed_d3``), centroid (``distributed_d3_centroid_virials``) and flux (``distributed_d3_heat_flux``)
ms, the one-GPU one-shot ms of the same three at the same total size (three stages, ``D3Engine.centroid_virial``,
``D3Engine.heat_flux``), the bytes of each all-gather computed from the shapes, and the GPU's name and power limit
read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# bytes per atom of each all-gather: (name, width, item size)
GATHERS = dict(centroid=(('ct_nb', 4, 4), ('ct_out', 9, 8)), flux=(('fx_nb', 8, 4), ('fx_out', 6, 8)))


def _gpu_info(rank):
    try:
        return subprocess.run(['nvidia-smi', f'--id={rank}', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
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
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    from sevenn_b200.d3 import (D3Engine, distributed_d3, distributed_d3_centroid_virials,
                                distributed_d3_heat_flux)
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    if not torch.cuda.is_available():
        raise SystemExit('d3_distributed_flux_bench needs a CUDA device')
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', rank))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', local))
    rows = []
    try:
        def sync():
            torch.cuda.synchronize()
            dist.barrier()

        cells = [('nacl', rocksalt_nacl, (23, 23, 12)), ('si', diamond_si, (19, 19, 17))]   # 50 784 / 49 096 atoms
        for material, fn, nc in cells:
            pos, cell, z = fn(*nc, sigma=0.05, seed=1)
            n, pbc = len(z), (True, True, True)
            v = torch.as_tensor(np.random.RandomState(0).normal(size=pos.shape), device='cuda')
            chunk = (n + world - 1) // world
            for damping in ('damp_bj', 'damp_zero'):
                eng = D3Engine(damping, 'pbe')
                t_fwd = _timed(lambda: distributed_d3(eng, z, pos, cell, pbc), sync, args.reps)
                distributed_d3(eng, z, pos, cell, pbc)
                t_ct = _timed(lambda: distributed_d3_centroid_virials(eng), sync, args.reps)
                t_fx = _timed(lambda: distributed_d3_heat_flux(eng, v), sync, args.reps)
                one = D3Engine(damping, 'pbe')
                one.set_system(z, pos, cell, pbc)

                def stages():
                    for s in (1, 2, 3):
                        one.run_stage(s)
                t1_fwd = _timed(stages, torch.cuda.synchronize, args.reps)
                t1_ct = _timed(one.centroid_virial, torch.cuda.synchronize, args.reps)
                t1_fx = _timed(lambda: one.heat_flux(v), torch.cuda.synchronize, args.reps)
                row = dict(kind='d3_distributed_flux', rank=rank, world=world, material=material, atoms=n,
                           damping=damping, forward_ms=round(t_fwd, 3), centroid_ms=round(t_ct, 3),
                           flux_ms=round(t_fx, 3), one_gpu_forward_ms=round(t1_fwd, 3),
                           one_gpu_centroid_ms=round(t1_ct, 3), one_gpu_flux_ms=round(t1_fx, 3),
                           gather_bytes={k: {name: world * chunk * w * b for name, w, b in g}
                                         for k, g in GATHERS.items()},
                           gpu=_gpu_info(local))
                if world < 2:
                    row['multi_gpu'] = 'not measured: world 1 runs the range passes over all atoms'
                print(json.dumps(row), flush=True)
                rows.append(row)
                del eng, one
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(f'{args.out}.rank{rank}' if world > 1 else args.out, 'w') as f:
                json.dump(rows, f, indent=1)
    finally:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
