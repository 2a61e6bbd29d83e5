"""Cost of the engine's per-atom centroid virial (B200Engine.centroid_virial, one reverse pass of four channels) against
one energy/force step, one heat-flux pass and one Hessian-vector product, on rattled Si cells of 64 / 512 / 12 000
atoms, SevenNet-0 and SevenNet-l3i5, both radial modes; the device memory the first centroid call allocates; and, with
--profile, a torch.profiler kernel breakdown of one pass (SevenNet-0, 512 atoms).  Prints one JSON line per
measurement and writes them all to --out; the card, its power limit and its SM clocks are read in the same run.

    python tools/centroid_virial_bench.py --out /tmp/centroid_virial_bench.json --profile
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from heat_flux_bench import card, engine_on, timed  # noqa: E402


def measure(name, radial, nc, reps):
    import torch
    e, v = engine_on(name, radial, nc)
    for _ in range(3):
        e.compute()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    e.centroid_virial()
    torch.cuda.synchronize()
    mem = free0 - torch.cuda.mem_get_info()[0]
    e.heat_flux(v)
    e.hvp(v)
    e.compute()
    torch.cuda.synchronize()
    step = timed(e.compute, reps)
    wc = timed(e.centroid_virial, reps)
    flux = timed(lambda: e.heat_flux(v), reps)
    hvp = timed(lambda: e.hvp(v), max(1, reps // 2))
    row = dict(model=name, radial=radial, atoms=int(e.n_nodes), edges=int(e.n_edges), step_ms=round(step, 3),
               centroid_ms=round(wc, 3), flux_ms=round(flux, 3), hvp_ms=round(hvp, 3),
               centroid_over_step=round(wc / step, 2), centroid_over_flux=round(wc / flux, 2),
               centroid_over_hvp=round(wc / hvp, 2), first_centroid_call_bytes=int(mem))
    del e
    torch.cuda.empty_cache()
    return row


def profile(out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile as prof
    e, _ = engine_on('sevennet_0', 'table', (4, 4, 4))
    e.compute()
    e.centroid_virial()
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        e.centroid_virial()
        torch.cuda.synchronize()
    rows = {}
    for ev in p.key_averages():
        if ev.device_type.name == 'CUDA' and ev.device_time_total > 0:
            k = ev.key.split('<')[0].split('(')[0]
            rows[k] = rows.get(k, 0.0) + ev.device_time_total / 1000.0
    total = sum(rows.values())
    table = sorted(rows.items(), key=lambda kv: -kv[1])
    if out_dir:
        p.export_chrome_trace(os.path.join(out_dir, 'centroid_virial_trace.json'))
    return dict(profile='sevennet_0 table Si512 one centroid pass', total_kernel_ms=round(total, 3),
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
        sys.exit('centroid_virial_bench needs a CUDA device')
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
