#!/usr/bin/env python
"""Time the operator-level convolution's forward, backward and double backward (the C ABI ``s7b_conv_*``) on
SevenNet-0 layer 1 and SevenNet-l3i5 layer 2 over the edges of the rattled 12 000-atom Si cell (10 x 10 x 15,
336 000 edges at 5 A), and compare the fused second-order kernels (``s7b_conv_double_backward``: conv_jvp_kernel +
conv_bwd_tangent_kernel per l1 role) with the same result composed from the first-order kernels (three
``s7b_conv_forward`` + three ``s7b_conv_backward`` calls and the sums, the weights with the Y_0 paths zeroed built
beforehand).

    python tools/conv_double_backward_bench.py [--reps 20] [--warmup 3] [--out DIR]

All three tangents present.  Times: median of --reps CUDA-event intervals after --warmup calls.  Prints one JSON line
per layer and the GPU name and power limit read in the same run (and writes DIR/conv_double_backward_bench.json).
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LAYERS = [('sevennet_0', 1), ('sevennet_l3i5', 2)]


def gpu_info():
    q = 'name,power.limit,clocks.sm,clocks.max.sm'
    try:
        row = subprocess.run(['nvidia-smi', f'--query-gpu={q}', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:   # noqa: BLE001
        return {'error': str(ex)}
    return dict(zip(q.split(','), [c.strip() for c in row.split(',')]))


def timed(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def bench_layer(name, t, ei, ev, reps, warmup):
    import torch
    from sevenn_b200.checkpoint import load_weights
    from sevenn_b200.engine import check, load_library
    from sevenn_b200.sh import spherical_harmonics
    from sevenn_b200.spec import build_spec
    lib = load_library()
    meta, _ = load_weights(os.path.join(ROOT, 'weights', f'{name}.npz'))
    spec = build_spec(meta)
    L, lf = spec.layers[t], spec.lmax_filter
    plan = ctypes.c_void_p()
    muls = (ctypes.c_int32 * len(L.x_muls))(*L.x_muls)
    lmax_out = max(p.l3 for p in L.paths)
    check(lib.s7b_conv_plan_create(len(L.x_muls), muls, lf, lmax_out, ctypes.byref(plan)))
    dims = [ctypes.c_int32() for _ in range(4)]
    check(lib.s7b_conv_plan_dims(plan, *[ctypes.byref(d) for d in dims]))
    dim_x, dim_mid, W, n_sh = (d.value for d in dims)

    order = np.argsort(ei[0], kind='stable')
    dst, src = ei[0][order], ei[1][order]
    n, E = int(ei.max()) + 1, len(order)
    dev = torch.device('cuda')
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g)
    rowptr = torch.zeros(n + 1, dtype=torch.int64)
    rowptr[1:] = torch.cumsum(torch.bincount(torch.as_tensor(dst), minlength=n), 0)
    rowptr = rowptr.to(torch.int32).to(dev)
    src32 = torch.as_tensor(src, dtype=torch.int32, device=dev)
    sh = torch.as_tensor(spherical_harmonics(lf, ev[order]), dtype=torch.float32, device=dev).contiguous()
    x, w, gout = rnd(n, dim_x), rnd(E, W), rnd(n, dim_mid)
    tx, tw = rnd(n, dim_x), rnd(E, W)
    tsh = rnd(E, n_sh)
    tsh[:, 0] = 0.0
    l2_0 = torch.zeros(W, dtype=torch.bool, device=dev)     # weight columns of the l2 = 0 paths
    for p in L.paths:
        if p.l2 == 0:
            l2_0[p.w_off:p.w_off + p.mul] = True
    w0 = w.masked_fill(l2_0, 0.0)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    P = lambda a: a.data_ptr()

    def fwd(x_, sh_, w_, out):
        check(lib.s7b_conv_forward(plan, P(x_), P(sh_), P(w_), P(rowptr), P(src32), n, n, E, P(out), st))

    def bwd(x_, sh_, w_, g_, dx, dsh, dw):
        check(lib.s7b_conv_backward(plan, P(x_), P(sh_), P(w_), P(rowptr), P(src32), n, n, E, P(g_),
                                    P(dx), P(dsh), P(dw), st))

    out = torch.empty(n, dim_mid, device=dev)
    gx, gsh, gw = torch.empty_like(x), torch.empty_like(sh), torch.empty_like(w)
    fused = [torch.empty_like(gout), torch.empty_like(x), torch.empty_like(sh), torch.empty_like(w)]

    def double_fused():
        check(lib.s7b_conv_double_backward(plan, P(x), P(sh), P(w), P(rowptr), P(src32), n, n, E, P(gout),
                                           P(tx), P(tsh), P(tw), *[P(a) for a in fused], st))

    parts = [torch.empty_like(gout) for _ in range(3)]
    bA = [torch.empty_like(x), torch.empty_like(sh), torch.empty_like(w)]
    bB = [torch.empty_like(x), torch.empty_like(sh), torch.empty_like(w)]
    bC = [torch.empty_like(x), torch.empty_like(sh), torch.empty_like(w)]
    comp = [None] * 4

    def double_composed():
        fwd(tx, sh, w, parts[0])
        fwd(x, tsh, w0, parts[1])
        fwd(x, sh, tw, parts[2])
        bwd(tx, sh, w, gout, *bA)           # dsh, dw
        bwd(x, tsh, w0, gout, *bB)          # dx, dw (l2 > 0 columns)
        bwd(x, sh, tw, gout, *bC)           # dx, dsh
        comp[0] = parts[0] + parts[1] + parts[2]
        comp[1] = bB[0] + bC[0]
        comp[2] = bA[1] + bC[1]
        comp[3] = bA[2] + bB[2].masked_fill(l2_0, 0.0)

    res = dict(model=name, layer=t, atoms=n, edges=E, dim_x=dim_x, dim_mid=dim_mid, weight_numel=W,
               forward_ms=timed(lambda: fwd(x, sh, w, out), reps, warmup),
               backward_ms=timed(lambda: bwd(x, sh, w, gout, gx, gsh, gw), reps, warmup),
               double_backward_fused_ms=timed(double_fused, reps, warmup),
               double_backward_composed_ms=timed(double_composed, reps, warmup))
    torch.cuda.synchronize()
    res['fused_vs_composed_max_rel'] = max(float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
                                           for a, b in zip(fused, comp))
    res['speedup'] = res['double_backward_composed_ms'] / res['double_backward_fused_ms']
    lib.s7b_conv_plan_destroy(plan)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit('conv_double_backward_bench.py needs a CUDA device')
    from sevenn_b200.neighbors import build_graph, diamond_si
    pos, cell, _ = diamond_si(10, 10, 15)
    ei, ev = build_graph(pos, cell, True, 5.0)
    info = gpu_info()
    rows = [dict(bench_layer(name, t, ei, ev, args.reps, args.warmup), gpu=info) for name, t in LAYERS]
    for r in rows:
        print(json.dumps(r))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'conv_double_backward_bench.json'), 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
