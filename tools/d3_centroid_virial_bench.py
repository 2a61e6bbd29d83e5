"""Cost of D3's per-atom centroid virial: one D3Engine.centroid_virial call against the three forward stages, one D3
heat-flux call and one D3 Hessian-vector product, at the default cutoffs, both dampings, on rattled rock-salt NaCl of
1 000 and 50 784 atoms and on rattled diamond Si of 1 000 and 49 096 atoms.  In rock salt every atom's C6 weights are
one-hot (CN far above the references of Na and Cl), so the moment pass skips the damping of every pair there; in Si
(CN ~4, between silicon's references) it evaluates it for every pair.  Also one SevenNet-0 + D3 step
(SevenNetD3Model.forward, 64 rattled NaCl cells of 64 atoms) with and without both centroid passes
(DeviceBatch.centroid_virials with d3).  Prints one JSON line per measurement and writes them all to --out; the card,
its power limit and its SM clocks are read in the same run.

    python tools/d3_centroid_virial_bench.py --out /tmp/d3_centroid_virial_bench.json
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from hvp_bench import card, timed  # noqa: E402


def centroid_vs_forward(reps):
    import torch
    from sevenn_b200.d3 import D3Engine
    from sevenn_b200.neighbors import diamond_si, rocksalt_nacl
    rows = []
    cases = [('nacl', rocksalt_nacl, (5, 5, 5)), ('nacl', rocksalt_nacl, (23, 23, 12)),     # 1 000, 50 784 atoms
             ('si', diamond_si, (5, 5, 5)), ('si', diamond_si, (19, 19, 17))]              # 1 000, 49 096 atoms
    for material, fn, nc in cases:
        pos, cell, z = fn(*nc, sigma=0.05, seed=1)
        for damping in ('damp_bj', 'damp_zero'):
            eng = D3Engine(damping, 'pbe')
            eng.set_system(z, pos, cell, (True, True, True))
            v = torch.as_tensor(np.random.RandomState(0).normal(size=pos.shape), device=eng.device)

            def fwd():
                for s in (1, 2, 3):
                    eng.run_stage(s)
            fwd()
            eng.centroid_virial()
            eng.heat_flux(v)
            eng.hvp(v)
            torch.cuda.synchronize()
            r = max(1, reps if len(z) < 10000 else reps // 5)
            t_f = timed(fwd, r)
            t_c = timed(eng.centroid_virial, r)
            t_x = timed(lambda: eng.heat_flux(v), r)
            t_h = timed(lambda: eng.hvp(v), r)
            rows.append(dict(kind='d3_centroid_vs_forward', material=material, atoms=len(z), damping=damping,
                             forward_ms=round(t_f, 3), centroid_ms=round(t_c, 3), flux_ms=round(t_x, 3),
                             hvp_ms=round(t_h, 3), centroid_over_forward=round(t_c / t_f, 2),
                             centroid_over_flux=round(t_c / t_x, 2), centroid_over_hvp=round(t_c / t_h, 2)))
    return rows


def md_step(reps):
    import torch
    from sevenn_b200.batch import SevenNetD3Model
    from sevenn_b200.neighbors import rocksalt_nacl

    class State:
        pass
    B = 64
    structs = [rocksalt_nacl(2, 2, 2, sigma=0.05, seed=s) for s in range(B)]
    st = State()
    st.positions = torch.as_tensor(np.concatenate([s[0] for s in structs]), device='cuda')
    st.row_vector_cell = torch.as_tensor(np.stack([s[1] for s in structs]))
    st.atomic_numbers = torch.as_tensor(np.concatenate([s[2] for s in structs]), device='cuda')
    st.pbc = True
    st.system_idx = torch.repeat_interleave(torch.arange(B, device='cuda'), 64)
    model = SevenNetD3Model('7net-0', device='cuda')

    def step():
        return model(st)

    def step_centroid():
        out = model(st)
        return out, model._batch.centroid_virials(d3=model.d3)
    step()
    step_centroid()
    torch.cuda.synchronize()
    t_s = timed(step, reps)
    t_c = timed(step_centroid, reps)
    return [dict(kind='sevennet_d3_step', structures=B, atoms_each=64, step_ms=round(t_s, 3),
                 step_with_centroid_ms=round(t_c, 3), ratio=round(t_c / t_s, 2))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=20)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('d3_centroid_virial_bench needs a CUDA device')
    rows = [dict(kind='card', **card())]
    print(json.dumps(rows[0]), flush=True)
    for part in (lambda: centroid_vs_forward(args.reps), lambda: md_step(args.reps)):
        for r in part():
            print(json.dumps(r), flush=True)
            rows.append(r)
    rows.append(dict(kind='card_after', **card()))
    print(json.dumps(rows[-1]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
