"""Node linears against the HBM roofline on the benchmark cell (SevenNet-0, Si 10x10x15 = 12 000 atoms).

Runs the engine with its CUDA-event profile on, and prints for every linear label (si1, sc, si2 forward; si2T,
si1T_scT backward; per layer) the measured ms, the algorithmic bytes -- A read once plus C written once, fp32,
per node sum_l (2l+1) (K_l + N_l) over the blocks the call multiplies; the read of C by the accumulating calls,
the row-exponent pass and the zero fill of dh / g are not counted -- and the fraction of the HBM floor
(bytes / peak bandwidth) the kernel time reaches.  The peak is the data sheet's 3.35 TB/s unless given.

    python tools/linear_roofline.py [--steps 10] [--peak-gbs 3350]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)


def _block_bytes(Ks, Ns, n_nodes):
    return 4 * n_nodes * sum((2 * l + 1) * (K + N) for l, (K, N) in enumerate(zip(Ks, Ns)) if K and N)


def linear_bytes(spec, n_nodes):
    """{profile label: algorithmic bytes} of the node linears of one step (labels as the engine names them)."""
    out = {}
    for t, L in enumerate(spec.layers):
        x, g, mid = list(L.x_muls), list(L.gate_muls), list(L.mid_K)
        n_sc = min(len(x), len(g))
        if t > 0:       # layer 0's input is the species embedding: no si1 / sc of its own
            out[f'si1_gemm.t{t}'] = _block_bytes(x, x, n_nodes)
            out[f'sc_gemm.t{t}'] = _block_bytes(x[:n_sc], g[:n_sc], n_nodes)
            out[f'si1T_scT_gemm.t{t}'] = _block_bytes(g[:n_sc], x[:n_sc], n_nodes) + _block_bytes(x, x, n_nodes)
        out[f'si2_gemm.t{t}'] = _block_bytes(mid[:len(g)], g, n_nodes)
        out[f'si2T_gemm.t{t}'] = _block_bytes(g, mid[:len(g)], n_nodes)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--peak-gbs', type=float, default=3350.0)
    args = ap.parse_args()
    import torch
    from sevenn_b200.checkpoint import load_weights
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import build_graph, diamond_si

    meta, arrays = load_weights(os.path.join(ROOT, 'weights', 'sevennet_0.npz'))
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    pos, cell, z = diamond_si(10, 10, 15)
    ei, ev = build_graph(pos, cell, True, 5.0)
    eng = B200Engine(meta, arrays, radial='table')
    eng.set_graph(np.array([tm[int(a)] for a in z], dtype=np.int32), ei, ev)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')   # > 50 MB L2, evicted between steps
    for _ in range(args.warmup):
        eng.compute()
    torch.cuda.synchronize()
    eng.set_profiling(True)
    for _ in range(args.steps):
        flush.fill_(1)
        eng.compute()
    torch.cuda.synchronize()
    prof = eng.profile()
    eng.set_profiling(False)
    props = torch.cuda.get_device_properties(0)
    print(f'{props.name}, {len(z)} atoms, {args.steps} profiled steps, HBM peak {args.peak_gbs:.0f} GB/s')
    print(f'{"label":20s} {"ms":>8s} {"MB":>8s} {"floor ms":>9s} {"of floor":>9s}')
    tot_ms = tot_b = 0.0
    for label, nbytes in sorted(linear_bytes(eng.spec, len(z)).items(), key=lambda kv: (kv[0].split('.')[1], kv[0])):
        if label not in prof:
            continue
        ms = prof[label][0] / args.steps
        floor = nbytes / (args.peak_gbs * 1e9) * 1e3
        tot_ms += ms
        tot_b += nbytes
        print(f'{label:20s} {ms:8.4f} {nbytes / 1e6:8.1f} {floor:9.4f} {floor / ms:9.1%}')
    floor = tot_b / (args.peak_gbs * 1e9) * 1e3
    print(f'{"all linears":20s} {tot_ms:8.4f} {tot_b / 1e6:8.1f} {floor:9.4f} {floor / tot_ms:9.1%}')


if __name__ == '__main__':
    main()
