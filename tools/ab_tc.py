"""A/B of the node-linear kernels (tensor-core bf16x3 vs FP32 SIMT): accuracy vs the fp64 oracle on the
64-atom cell and step time on the 12 000-atom cell."""
import os, sys, time
import numpy as np, torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from oracle.oracle import Oracle
from sevenn_b200.checkpoint import load_weights
from sevenn_b200.engine import B200Engine, set_option
from sevenn_b200.neighbors import build_graph, diamond_si
meta, arrays = load_weights(os.path.join(ROOT, 'weights', 'sevennet_0.npz'))
tm = {int(k): int(v) for k, v in meta['type_map'].items()}
e = B200Engine(meta, arrays)
pos, cell, z = diamond_si(2, 2, 2)
ei, ev = build_graph(pos, cell, True, 5.0)
sp = np.array([tm[int(a)] for a in z])
ref = Oracle(meta, arrays, dtype=torch.float64).forward(sp, ei, ev)
e.set_graph(sp, ei, ev)
for tc in (0, 1):
    set_option('tc_gemm', tc)
    e.compute(); torch.cuda.synchronize()
    r = e.results()
    dE = float(r['energy'].cpu()[0]) - float(ref['energy'])
    dF = np.abs(r['forces'].cpu().numpy() - ref['forces'].numpy()).max()
    dA = np.abs(r['atomic_energy'].cpu().numpy() - ref['atomic_energy'].numpy()).max()
    print(f'tc_gemm={tc}: dE {dE:+.2e} eV, max|dE_atom| {dA:.2e}, max|dF| {dF:.2e} eV/A')
pos, cell, z = diamond_si(10, 10, 15)
ei, ev = build_graph(pos, cell, True, 5.0)
e.set_graph(np.array([tm[int(a)] for a in z]), ei, ev)
for tc in (0, 1):
    set_option('tc_gemm', tc)
    for _ in range(3): e.compute()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(10): e.compute()
    b.record(); torch.cuda.synchronize()
    print(f'tc_gemm={tc}: {a.elapsed_time(b)/10:.3f} ms/step (12000 atoms, L2 warm)')
