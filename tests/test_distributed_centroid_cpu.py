"""CPU tests of DistributedRunner.centroid_virials / heat_flux (gloo, world 2 and 4): the CV stage protocol with its
per-layer reverse exchange of four adjoint channels and the final fp64 reverse-add of the per-atom centroid virial,
driven with a stand-in engine (test_parallel_gloo.FakeEngine plus CV stages that run DESIGN.md §8.7's recursion for
its toy model in fp64).  The serial stand-in is the oracle; it is itself checked against the sum rule
sum_i Wc_i = -sum_e vec_e (x) f_e."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from sevenn_b200.engine import (STAGE_BWD_END, STAGE_BWD_LAYER_A, STAGE_BWD_LAYER_B, STAGE_CV_BEGIN, STAGE_CV_END,
                                STAGE_CV_LAYER_A, STAGE_CV_LAYER_B, STAGE_FWD_BEGIN, STAGE_FWD_END, STAGE_FWD_LAYER)
from sevenn_b200.neighbors import build_graph
from sevenn_b200.parallel import DistributedRunner, brick_decompose
from test_parallel_gloo import FakeEngine, _free_port, _system


class CentroidFakeEngine(FakeEngine):
    """FakeEngine with the CV stages.  Toy model: a_t[j] = sum_{e: centre j} w_e x_t[k_e], w_e = |vec_e|,
    h_t = tanh(a_t), x_{t+1} = c_t h_t, U_j = sum_d h_{T-1}[j, d].  Channels per feature: A = dE/df and
    B_a = sum_m (r_m - r_j)_a dU_m/df.  The neighbour of edge e receives w_e (B_a - vec_a A) and w_e A; the per-edge
    sums G_c = (channel c of the centre . x_t[k]) vec / w accumulate over the layers; CV_END adds G'_a (x) e_b to the
    neighbour's row and -(G'_a + vec_a f) to the centre's (f = G_0).  Smaller x_0 and c_t than FakeEngine's keep
    tanh out of saturation, so every derivative is far from zero."""

    def __init__(self):
        super().__init__()
        self.coef = [0.02, 0.03, 0.02]

    def buffer(self, name, t=0, dtype='f4', shape=None):
        if name.startswith('cv_dx'):
            return self.cv_dx[int(name[5:])]
        if name == 'centroid_virial':
            return self.wc
        if name == 'atomic_energy_f64':
            return self.h.sum(1)
        return super().buffer(name, t, dtype, shape)

    def run_stage(self, stage, t=0):
        if stage not in (STAGE_CV_BEGIN, STAGE_CV_LAYER_A, STAGE_CV_LAYER_B, STAGE_CV_END):
            super().run_stage(stage, t)
            if stage == STAGE_FWD_BEGIN:
                self.x[0] *= 0.01
            return
        nl, n, D = self.n_local, self.n_nodes, self.D
        j, k, vec, w = self.dst, self.src, self.vec, self.w
        if stage == STAGE_CV_BEGIN:
            self.ch = [torch.ones(nl, D, dtype=torch.float64)] + [torch.zeros(nl, D, dtype=torch.float64) for _ in range(3)]
            self.G = torch.zeros(len(w), 4, 3, dtype=torch.float64)
        elif stage == STAGE_CV_LAYER_A:
            s = 1 - torch.tanh(self.a[t]) ** 2                         # owned rows only
            cen = [s * c for c in self.ch]
            ce = [cen[0][j]] + [cen[1 + a][j] - vec[:, a, None] * cen[0][j] for a in range(3)]   # what k receives / w
            u = vec / w[:, None]
            for c in range(4):
                self.G[:, c] += (ce[c] * self.x[t][k]).sum(1)[:, None] * u
            self.cv_dx = [torch.zeros(n, D, dtype=torch.float64) for _ in range(4)]
            if t > 0:
                for c in range(4):
                    self.cv_dx[c].index_add_(0, k, w[:, None] * ce[c])
        elif stage == STAGE_CV_LAYER_B:
            self.ch = [self.coef[t - 1] * d[:nl] for d in self.cv_dx]
        else:
            f, Gp = self.G[:, 0], self.G[:, 1:]                        # Gp [E, a, b]
            self.wc = torch.zeros(n, 9, dtype=torch.float64)
            self.wc.index_add_(0, k, Gp.reshape(-1, 9))
            self.wc.index_add_(0, j, -(Gp + vec[:, :, None] * f[:, None, :]).reshape(-1, 9))


def _serial(kind):
    pos, cell, species = _system(kind)
    ei, ev = build_graph(pos, cell, True, 5.0)
    ser = CentroidFakeEngine()
    ser.set_graph(species, ei, ev)
    ser.run_stage(STAGE_FWD_BEGIN)
    for t in range(ser.T):
        ser.run_stage(STAGE_FWD_LAYER, t)
    ser.run_stage(STAGE_FWD_END)
    for t in range(ser.T - 1, -1, -1):
        ser.run_stage(STAGE_BWD_LAYER_A, t)
        if t > 0:
            ser.run_stage(STAGE_BWD_LAYER_B, t)
    ser.run_stage(STAGE_BWD_END)
    ser.run_stage(STAGE_CV_BEGIN)
    for t in range(ser.T - 1, -1, -1):
        ser.run_stage(STAGE_CV_LAYER_A, t)
        if t > 0:
            ser.run_stage(STAGE_CV_LAYER_B, t)
    ser.run_stage(STAGE_CV_END)
    return ser


def _inputs(n):
    rs = np.random.RandomState(31)
    return rs.normal(size=(n, 3)), rs.uniform(1.0, 30.0, size=n)


def _worker(rank, world, port, grid, kind, q):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        pos, cell, species = _system(kind)
        part = brick_decompose(pos, cell, species, grid, rank, 5.0)
        run = DistributedRunner(CentroidFakeEngine(), part)
        run.compute()
        wc = run.centroid_virials().numpy()
        v, m = _inputs(len(pos))
        j_all = run.heat_flux(v, m).numpy()
        j_pot = run.heat_flux(torch.as_tensor(v), convective=False).numpy()
        with pytest.raises(ValueError, match='masses'):
            run.heat_flux(v)
        nl = part['n_local']
        # a remote atom that is a neighbour through several images (one shared ghost row)
        ei, ev = part['edge_index'], part['edge_vec']
        ghost = ei[1] >= nl
        lattice_free = np.round(pos[part['global_ids'][ei[0][ghost]]] + ev[ghost], 3)
        images = {}
        for g, r in zip(ei[1][ghost], map(tuple, lattice_free)):
            images.setdefault(int(g), set()).add(r)
        multi = max((len(s) for s in images.values()), default=0)
        q.put((rank, part['global_ids'][:nl].copy(), wc, j_all, j_pot, multi))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world,grid,kind', [(2, (2, 1, 1), 'si'), (2, (1, 1, 2), 'nacl'), (4, (2, 2, 1), 'si'),
                                             (2, (2, 1, 1), 'si_long')])
def test_distributed_centroid_virial_and_heat_flux_match_serial(world, grid, kind):
    ser = _serial(kind)
    pos = _system(kind)[0]
    n = len(pos)
    wc_ser = ser.wc.numpy().reshape(n, 3, 3)
    # the stand-in's recursion meets the sum rule: sum_i Wc_i = -sum_e vec_e (x) f_e
    vir = -(ser.vec[:, :, None] * ser.fedge[:, None, :]).sum(0).numpy()
    assert np.abs(wc_ser.sum(0) - vir).max() < 1e-12 * np.abs(wc_ser).sum()
    assert np.abs(wc_ser - wc_ser.transpose(0, 2, 1)).max() > 1e-3 * np.abs(wc_ser).max()    # not the pairwise split
    v, m = _inputs(n)
    u = ser.h.sum(1).numpy()
    jpot_ser = np.einsum('iab,ib->a', wc_ser, v)
    j_ser = jpot_ser + ((u + 0.5 * m * (v * v).sum(1))[:, None] * v).sum(0)

    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, grid, kind, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    wc = np.zeros((n, 3, 3))
    seen = np.zeros(n, dtype=int)
    for rank, gids, w, j_all, j_pot, multi in res:
        wc[gids] = w
        seen[gids] += 1
        assert np.abs(j_all - j_ser).max() < 1e-10 * np.abs(j_ser).max()
        assert np.abs(j_pot - jpot_ser).max() < 1e-10 * np.abs(jpot_ser).max()
    assert (seen == 1).all()
    assert np.array_equal(res[0][3], res[-1][3])                    # the same flux on every rank, bit for bit
    assert np.abs(wc - wc_ser).max() < 1e-12 * np.abs(wc_ser).sum()
    if kind == 'si':
        assert max(r[5] for r in res) >= 2                          # a ghost row stands for several images
