"""CPU tests of DistributedRunner.centroid_virials(d3=) / heat_flux(..., d3=) (gloo, world 2 and 4): the network's part
comes from the stand-in engine of test_distributed_centroid_cpu.py, D3's from a stand-in of the distributed D3 functions
whose rows and flux are known.  Checks that D3's rows reach the owned atoms of their global ids, that its flux is added
once to the rank sum (not once per rank), that its sum U v is added only with the convective part, and that a D3
forward of another system is refused."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from sevenn_b200.parallel import DistributedRunner, brick_decompose
from test_distributed_centroid_cpu import CentroidFakeEngine, _inputs
from test_parallel_gloo import _free_port, _system


class StandInD3:
    """what the runner reads of a D3Engine (its atom count), plus the values the stand-in functions return"""

    def __init__(self, n):
        rs = np.random.RandomState(7)
        self.n = n
        self.rows = rs.normal(size=(n, 3, 3))
        self.jpot, self.ju = rs.normal(size=3), rs.normal(size=3)
        self.calls = []


def _stand_in_rows(d3, group=None):
    d3.calls.append('centroid')
    return torch.as_tensor(d3.rows)


def _stand_in_flux(d3, v, group=None):
    d3.calls.append('flux')
    d3.v = np.array(v)
    return torch.as_tensor(d3.jpot), torch.as_tensor(d3.ju)


def _worker(rank, world, port, grid, kind, q):
    import sevenn_b200.d3 as d3mod
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        d3mod.distributed_d3_centroid_virials = _stand_in_rows
        d3mod.distributed_d3_heat_flux = _stand_in_flux
        pos, cell, species = _system(kind)
        n = len(pos)
        part = brick_decompose(pos, cell, species, grid, rank, 5.0)
        run = DistributedRunner(CentroidFakeEngine(), part)
        run.compute()
        v, m = _inputs(n)
        d3 = StandInD3(n)
        out = dict(gids=part['global_ids'][:part['n_local']].copy(),
                   wc=run.centroid_virials().numpy(), wc_d3=run.centroid_virials(d3=d3).numpy(),
                   j=run.heat_flux(v, m).numpy(), j_d3=run.heat_flux(v, m, d3=d3).numpy(),
                   jpot=run.heat_flux(v, convective=False).numpy(),
                   jpot_d3=run.heat_flux(v, convective=False, d3=d3).numpy(), calls=list(d3.calls),
                   v_seen=d3.v, rows=d3.rows, d3_jpot=d3.jpot, d3_ju=d3.ju)
        with pytest.raises(ValueError, match='distributed_d3 of the whole system'):
            run.centroid_virials(d3=StandInD3(n + 1))
        with pytest.raises(ValueError, match='distributed_d3 of the whole system'):
            run.heat_flux(v, m, d3=StandInD3(n - 1))
        q.put((rank, out))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('world,grid,kind', [(2, (2, 1, 1), 'si'), (4, (2, 2, 1), 'si'), (2, (1, 1, 2), 'nacl')])
def test_runner_adds_d3_rows_and_flux_once(world, grid, kind):
    n = len(_system(kind)[0])
    v = _inputs(n)[0]
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
    seen = np.zeros(n, dtype=int)
    for rank, o in res:
        gids = o['gids']
        seen[gids] += 1
        # D3's rows land on the owned atoms of their global ids; the network's part is that of the call without d3
        assert np.allclose(o['wc_d3'] - o['wc'], o['rows'][gids], rtol=0, atol=1e-12 * np.abs(o['wc']).max())
        # D3's flux once, after the rank sum; its sum U v only with the convective part
        assert np.allclose(o['j_d3'], o['j'] + o['d3_jpot'] + o['d3_ju'], rtol=1e-14, atol=0)
        assert np.allclose(o['jpot_d3'], o['jpot'] + o['d3_jpot'], rtol=1e-14, atol=0)
        assert o['calls'] == ['centroid', 'flux', 'flux']                 # heat_flux takes no D3 rows
        assert np.array_equal(o['v_seen'], v)                             # every atom's velocity, global-id order
    assert (seen == 1).all()
    assert all(np.array_equal(res[0][1]['j_d3'], o['j_d3']) for _, o in res)
