"""The per-atom centroid virial on graphs with ghost atoms (stages CV_BEGIN .. CV_END, DESIGN.md §8.7) on the GPU.

Most tests drive the host-staged protocol a parallel LAMMPS pair style would use, with 2 or 3 engines on one GPU:
s7b_engine_set_graph_host, ghost rows through s7b_engine_read_rows_host / write_rows_host between the stages, and the
Wc rows through s7b_engine_read_rows_f64_host, reverse-added into their owners in fp64.  Two ghost conventions:
'brick' (parallel.brick_decompose: one ghost row per remote atom, images of owned atoms point at owned rows) and
'lammps' (every periodic image its own ghost row, images of owned atoms included, on cells short along the split axis).
The owned rows must equal the single engine's s7b_engine_centroid_virial of the whole cell; the bound 1e-5 of max |Wc|
is that of batch-vs-alone (fp32 atomics in the convolution's scatter).  The observed errors are printed."""
import os

import numpy as np
import pytest

from helpers import model_weights, species_of

pytestmark = pytest.mark.gpu

BOUND = 1e-5
ORACLE_BOUND = {'mlp': 2e-4, 'table': 5e-4}


def _weights(case, tmp):
    if case == 'synth_A_nequip':
        from synthetic_nequip import convert, write_nequip_checkpoint
        return convert(write_nequip_checkpoint(os.path.join(tmp, 'cv_A_nequip.pth'), 'A', seed=21), 'A')
    return model_weights(case)


def _system(case, meta, reps, seed=3):
    from sevenn_b200.neighbors import diamond_si
    pos, cell, z = diamond_si(*reps, sigma=0.05, seed=seed)
    if case.startswith('synth'):
        from synthetic_models import NUMBERS
        z = np.array([NUMBERS[i % 3] for i in range(len(pos))])
    return pos, cell, species_of(meta, z).astype(np.int32)


def partition(pos, cell, species, n_ranks, style, cutoff):
    """Per rank: n_local, species, edges (centre, neighbour, vec) sorted by centre, global ids of the owned rows and,
    per ghost row, the (rank, row) of the owned row it stands for.  Split along x into n_ranks bricks."""
    from sevenn_b200.neighbors import build_graph
    from sevenn_b200.parallel import brick_decompose, owner_of
    grid = (n_ranks, 1, 1)
    if style == 'brick':
        parts = [brick_decompose(pos, cell, species, grid, r, cutoff) for r in range(n_ranks)]
        owner_row = {int(g): (r, i) for r, p in enumerate(parts) for i, g in enumerate(p['global_ids'][:p['n_local']])}
        out = []
        for p in parts:
            o = np.argsort(p['edge_index'][0], kind='stable')
            out.append(dict(n_local=p['n_local'], n_nodes=p['n_nodes'], species=p['species'], gids=p['global_ids'][:p['n_local']],
                            centre=p['edge_index'][0][o], neighbour=p['edge_index'][1][o], vec=p['edge_vec'][o],
                            src=[owner_row[int(g)] for g in p['global_ids'][p['n_local']:]]))
        return out
    ei, ev = build_graph(pos, cell, True, cutoff)
    inv = np.linalg.inv(cell)
    shift = np.rint((ev - (pos[ei[1]] - pos[ei[0]])) @ inv).astype(np.int64)        # image of the neighbour
    frac = pos @ inv
    owner = owner_of(frac - np.floor(frac), grid)
    owned = [np.nonzero(owner == r)[0] for r in range(n_ranks)]
    row_of = {int(g): (r, i) for r in range(n_ranks) for i, g in enumerate(owned[r])}
    out = []
    for r in range(n_ranks):
        keep = owner[ei[0]] == r
        c, k, s, v = ei[0][keep], ei[1][keep], shift[keep], ev[keep]
        local = (owner[k] == r) & (s == 0).all(1)
        keys = sorted({(int(a),) + tuple(int(x) for x in b) for a, b in zip(k[~local], s[~local])})
        ghost_row = {key: len(owned[r]) + i for i, key in enumerate(keys)}
        nb = np.array([row_of[int(a)][1] if l else ghost_row[(int(a),) + tuple(int(x) for x in b)]
                       for a, b, l in zip(k, s, local)], dtype=np.int64)
        cen = np.array([row_of[int(a)][1] for a in c], dtype=np.int64)
        o = np.argsort(cen, kind='stable')
        gids = np.concatenate([owned[r], np.array([key[0] for key in keys], dtype=np.int64)])
        out.append(dict(n_local=len(owned[r]), n_nodes=len(gids), species=species[gids], gids=owned[r],
                        centre=cen[o], neighbour=nb[o], vec=v[o], src=[row_of[key[0]] for key in keys],
                        own_images=sum(row_of[key[0]][0] == r for key in keys),
                        multi_images=max(np.unique([key[0] for key in keys], return_counts=True)[1], default=0)))
    return out


class Staged:
    """One engine per rank on this GPU, ghost rows exchanged through host arrays between the stages"""

    def __init__(self, meta, arrays, radial, parts):
        from sevenn_b200.engine import B200Engine
        self.parts = parts
        self.engs = [B200Engine(meta, arrays, radial=radial) for _ in parts]
        for e, p in zip(self.engs, parts):
            e.set_graph_host(p['species'], p['centre'], p['neighbour'], p['vec'], p['n_local'])
        self.T = self.engs[0].spec.n_layers
        self.dims = [L.dim_x for L in self.engs[0].spec.layers]

    def forward_exchange(self, name, layer, width):
        owned = [e.read_rows(name, layer, 0, p['n_local'], width) for e, p in zip(self.engs, self.parts)]
        for e, p in zip(self.engs, self.parts):
            if p['src']:
                e.write_rows(name, layer, p['n_local'], np.stack([owned[q][row] for q, row in p['src']]))

    def reverse_exchange(self, name, layer, width, f64=False):
        read = (lambda e, n: e.read_rows_f64(name, layer, 0, n, width)) if f64 else (lambda e, n: e.read_rows(name, layer, 0, n, width))
        full = [read(e, p['n_nodes']) for e, p in zip(self.engs, self.parts)]
        acc = [f[:p['n_local']].astype(np.float64) for f, p in zip(full, self.parts)]
        for f, p in zip(full, self.parts):
            for i, (q, row) in enumerate(p['src']):
                acc[q][row] += f[p['n_local'] + i]
        if not f64:
            for e, a in zip(self.engs, acc):
                e.write_rows(name, layer, 0, a.astype(np.float32))
        return acc

    def run(self, stage, layer=0):
        for e in self.engs:
            e.run_stage(stage, layer)

    def step(self, backward=True):
        from sevenn_b200 import engine as E
        self.run(E.STAGE_FWD_BEGIN)
        for t in range(self.T):
            self.run(E.STAGE_FWD_LAYER, t)
            if t + 1 < self.T:
                self.forward_exchange('x', t + 1, self.dims[t + 1])
        self.run(E.STAGE_FWD_END)
        if not backward:
            return None
        for t in range(self.T - 1, -1, -1):
            self.run(E.STAGE_BWD_LAYER_A, t)
            if t > 0:
                self.reverse_exchange('dx', t, self.dims[t])
                self.run(E.STAGE_BWD_LAYER_B, t)
        self.run(E.STAGE_BWD_END)
        forces = self.reverse_exchange('forces', 0, 3)
        return (sum(e.read_scalars()[0] for e in self.engs), sum(e.read_scalars()[1] for e in self.engs), forces)

    def centroid(self):
        """[n_global, 3, 3]: every rank's owned rows after the reverse-add of the ghost rows"""
        from sevenn_b200 import engine as E
        for e in self.engs:
            e._upload_hvp_mlp()
        self.run(E.STAGE_CV_BEGIN)
        for t in range(self.T - 1, -1, -1):
            self.run(E.STAGE_CV_LAYER_A, t)
            if t > 0:
                for c in range(4):
                    self.reverse_exchange(f'cv_dx{c}', t, self.dims[t])
                self.run(E.STAGE_CV_LAYER_B, t)
        self.run(E.STAGE_CV_END)
        acc = self.reverse_exchange('centroid_virial', 0, 9, f64=True)
        n = sum(p['n_local'] for p in self.parts)
        wc = np.zeros((n, 3, 3))
        for a, p in zip(acc, self.parts):
            wc[p['gids']] = a.reshape(-1, 3, 3)
        return wc


def _whole(meta, arrays, radial, species, pos, cell, cutoff):
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.neighbors import build_graph
    ei, ev = build_graph(pos, cell, True, cutoff)
    w = B200Engine(meta, arrays, radial=radial)
    w.set_graph(species, ei, ev)
    w.compute()
    return w, w.centroid_virial().cpu().numpy()


CASES = [('sevennet_0', 'table', 'brick', 2), ('sevennet_0', 'mlp', 'lammps', 3), ('sevennet_0', 'table', 'lammps', 2),
         ('sevennet_l3i5', 'table', 'lammps', 2), ('sevennet_l3i5', 'mlp', 'brick', 3),
         ('synth_A_nequip', 'mlp', 'lammps', 2), ('synth_A_nequip', 'table', 'brick', 2)]


@pytest.mark.parametrize('case,radial,style,n_ranks', CASES)
def test_host_staged_ranks_equal_the_whole_cell(case, radial, style, n_ranks, tmp_path):
    from sevenn_b200.spec import build_spec
    meta, arrays = _weights(case, str(tmp_path))
    cutoff = build_spec(meta).cutoff
    # 'lammps': bricks of one conventional cell (5.43 A) along x, shorter than the cutoff; 'brick': two cells each
    reps = (n_ranks, 2, 2) if style == 'lammps' else (2 * n_ranks, 2, 2)
    pos, cell, species = _system(case, meta, reps)
    parts = partition(pos, cell, species, n_ranks, style, cutoff)
    if style == 'lammps':
        assert all(p['own_images'] > 0 and p['multi_images'] >= 2 for p in parts)
    st = Staged(meta, arrays, radial, parts)
    st.step(backward=False)
    wc = st.centroid()
    _, ref = _whole(meta, arrays, radial, species, pos, cell, cutoff)
    err = np.abs(wc - ref).max() / np.abs(ref).max()
    print(f'{case} {radial} {style} x{n_ranks}: {len(pos)} atoms, ghosts {[p["n_nodes"] - p["n_local"] for p in parts]}: '
          f'max |staged - whole| / max |Wc| = {err:.1e}')
    assert err < BOUND


@pytest.mark.parametrize('radial', ['table', 'mlp'])
def test_against_the_fp64_oracle(radial):
    """8-atom Si cell cut into two 2.7 A bricks: nearly every neighbour is a per-image ghost row"""
    import torch
    from centroid_reference import reference_centroid_cell
    from flux_reference import make_oracle
    from sevenn_b200.spec import build_spec
    meta, arrays = model_weights('sevennet_0')
    spec = build_spec(meta)
    pos, cell, species = _system('sevennet_0', meta, (1, 1, 1), seed=7)
    st = Staged(meta, arrays, radial, partition(pos, cell, species, 2, 'lammps', spec.cutoff))
    st.step(backward=False)
    wc = st.centroid()
    ref = reference_centroid_cell(make_oracle(meta, arrays, 'cuda'), spec, species, pos, cell)
    torch.cuda.synchronize()
    err = np.abs(wc - ref).max() / np.abs(ref).sum()
    print(f'staged x2 vs fp64 oracle ({radial}): err / sum|Wc| = {err:.1e} (bound {ORACLE_BOUND[radial]:.0e})')
    assert err < ORACLE_BOUND[radial]


def test_identities():
    """summed over ranks, sum_i Wc_i = the whole cell's virial, and sum_i Wc_i v_i = its heat flux J_pot"""
    meta, arrays = model_weights('sevennet_0')
    pos, cell, species = _system('sevennet_0', meta, (2, 2, 2), seed=5)
    st = Staged(meta, arrays, 'table', partition(pos, cell, species, 2, 'lammps', 5.0))
    energy, virial, _ = st.step()
    wc = st.centroid()
    whole, _ = _whole(meta, arrays, 'table', species, pos, cell, 5.0)
    w = whole.buffer('virial', dtype='f8', shape=(6,)).cpu().numpy()
    W = np.array([[w[0], w[3], w[5]], [w[3], w[1], w[4]], [w[5], w[4], w[2]]])
    scale = np.abs(wc).sum()
    err_w = np.abs(wc.sum(0) - W).max() / scale
    err_staged = np.abs(virial - w).max() / scale
    print(f'sum_i Wc_i vs whole-cell virial: {err_w:.1e} of sum|Wc| (staged virial vs whole: {err_staged:.1e})')
    assert err_w < 1e-5 and err_staged < 1e-5
    for seed in range(2):
        v = np.random.RandomState(40 + seed).normal(size=pos.shape)
        J = whole.heat_flux(v)[0][0].cpu().numpy()
        Jc = np.einsum('iab,ib->a', wc, v.astype(np.float32).astype(np.float64))
        err = np.abs(J - Jc).max() / np.abs(wc * np.abs(v)[:, None, :]).sum()
        print(f'sum Wc v vs whole-cell J_pot: {err:.1e} of sum|terms|')
        assert err < 1e-5


def test_refusals_change_nothing():
    import torch
    from sevenn_b200 import engine as E
    from sevenn_b200.engine import B200Engine, check, prepare_params
    meta, arrays = model_weights('sevennet_0')
    pos, cell, species = _system('sevennet_0', meta, (2, 2, 2))
    p = partition(pos, cell, species, 2, 'lammps', 5.0)[0]
    T = 5
    e = B200Engine(meta, arrays, radial='mlp')
    e.set_graph_host(p['species'], p['centre'], p['neighbour'], p['vec'], p['n_local'])
    with pytest.raises(RuntimeError, match='needs FWD_END'):
        e.run_stage(E.STAGE_CV_BEGIN)
    e.run_stage(E.STAGE_FWD_BEGIN)
    for t in range(T):
        e.run_stage(E.STAGE_FWD_LAYER, t)
    with pytest.raises(RuntimeError, match='needs FWD_END'):
        e.run_stage(E.STAGE_CV_BEGIN)
    e.run_stage(E.STAGE_FWD_END)
    with pytest.raises(RuntimeError, match='needs CV_BEGIN'):
        e.run_stage(E.STAGE_CV_LAYER_A, T - 1)
    e.run_stage(E.STAGE_CV_BEGIN)
    with pytest.raises(RuntimeError, match='1 <= layer'):
        e.run_stage(E.STAGE_CV_LAYER_B, 0)
    for t in range(T - 1, -1, -1):
        e.run_stage(E.STAGE_CV_LAYER_A, t)
        if t > 0:
            e.run_stage(E.STAGE_CV_LAYER_B, t)
    e.run_stage(E.STAGE_CV_END)
    n, d1 = p['n_nodes'], e.spec.layers[1].dim_x

    def snapshot():
        torch.cuda.synchronize()
        return e.read_rows_f64('centroid_virial', 0, 0, n, 9), [e.read_rows(f'cv_dx{c}', 1, 0, n, d1) for c in range(4)]

    before = snapshot()
    assert np.abs(before[0]).max() > 0
    prm = prepare_params(e.spec, arrays, 'mlp', 0)[('si2', 0)]
    n0 = e.launch_count()
    check(e.lib.s7b_engine_set_param(e._h, b'si2', 0, prm.ctypes.data, prm.size))     # same values: still a new parameter
    for stage, t in [(E.STAGE_CV_BEGIN, 0), (E.STAGE_CV_LAYER_A, 1), (E.STAGE_CV_END, 0)]:
        with pytest.raises(RuntimeError, match='needs FWD_END'):
            e.run_stage(stage, t)
    assert e.launch_count() == n0
    e.set_graph_host(p['species'], p['centre'], p['neighbour'], p['vec'], p['n_local'])
    n0 = e.launch_count()
    with pytest.raises(RuntimeError, match='needs FWD_END'):
        e.run_stage(E.STAGE_CV_BEGIN)
    assert e.launch_count() == n0
    after = snapshot()
    assert np.array_equal(before[0], after[0]) and all(np.array_equal(a, b) for a, b in zip(before[1], after[1]))
    with pytest.raises(RuntimeError, match='f64'):
        e.read_rows('centroid_virial', 0, 0, n, 9)
    # a table-mode engine without its radial MLP (Python's run_stage does not upload it)
    tb = B200Engine(meta, arrays)
    tb.set_graph_host(p['species'], p['centre'], p['neighbour'], p['vec'], p['n_local'])
    tb.run_stage(E.STAGE_FWD_BEGIN)
    for t in range(T):
        tb.run_stage(E.STAGE_FWD_LAYER, t)
    tb.run_stage(E.STAGE_FWD_END)
    n0 = tb.launch_count()
    with pytest.raises(RuntimeError, match='mlp0 of layer 0 is missing'):
        tb.run_stage(E.STAGE_CV_BEGIN)
    assert tb.launch_count() == n0


@pytest.mark.parametrize('stage_graphs', [0, 1])
def test_step_after_a_centroid_sequence_is_unchanged(stage_graphs):
    """energy, forces and virial of the stage sequence before and after a CV sequence, within the run-to-run difference
    of two sequences (float atomics) or 1e-6 of the largest value; with option stage_graphs the step's stages replay
    their graphs and the CV stages launch directly, with the same rows"""
    import torch
    from sevenn_b200.engine import set_option
    meta, arrays = model_weights('sevennet_0')
    pos, cell, species = _system('sevennet_0', meta, (4, 2, 2))
    parts = partition(pos, cell, species, 2, 'brick', 5.0)
    try:
        set_option('stage_graphs', stage_graphs)
        st = Staged(meta, arrays, 'table', parts)
        a, b = st.step(), st.step()
        wc1 = st.centroid()
        c = st.step()
        wc2 = st.centroid()
        torch.cuda.synchronize()
        captures = st.engs[0].stage_graph_stats()[0]
    finally:
        set_option('stage_graphs', 0)
    for i, name in enumerate(('energy', 'virial', 'forces')):
        x, y, z = (np.concatenate([np.ravel(f) for f in r[i]]) if name == 'forces' else np.ravel(r[i]) for r in (a, b, c))
        run_to_run = np.abs(x - y).max()
        bound = max(run_to_run, 1e-6 * np.abs(x).max())
        print(f'stage_graphs={stage_graphs} {name}: after a CV sequence {np.abs(x - z).max():.2e}, run to run {run_to_run:.2e}')
        assert np.abs(x - z).max() <= bound
    err = np.abs(wc1 - wc2).max() / np.abs(wc1).max()
    print(f'stage_graphs={stage_graphs}: two CV sequences differ by {err:.1e} of max |Wc|; stage graphs captured: {captures}')
    assert err < BOUND
    assert (captures > 0) == bool(stage_graphs)


def _runner_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    from sevenn_b200.engine import B200Engine
    from sevenn_b200.parallel import DistributedRunner, brick_decompose
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        meta, arrays = model_weights('sevennet_0')
        pos, cell, species = _system('sevennet_0', meta, (4, 3, 3), seed=2)
        part = brick_decompose(pos, cell, species, (world, 1, 1), rank, 5.0)
        run = DistributedRunner(B200Engine(meta, arrays, device=rank), part)
        run.compute()
        wc = run.centroid_virials().cpu().numpy()
        v = np.random.RandomState(9).normal(size=pos.shape)
        m = np.full(len(pos), 28.0855)
        j = run.heat_flux(v, m).cpu().numpy()
        jp = run.heat_flux(v, convective=False).cpu().numpy()
        run.close()
        q.put((rank, part['global_ids'][:part['n_local']], wc, j, jp))
    finally:
        dist.destroy_process_group()


def test_distributed_runner_over_nccl():
    import socket
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    meta, arrays = model_weights('sevennet_0')
    pos, cell, species = _system('sevennet_0', meta, (4, 3, 3), seed=2)
    whole, ref = _whole(meta, arrays, 'table', species, pos, cell, 5.0)
    v = np.random.RandomState(9).normal(size=pos.shape)
    jpot, ju = (x[0].cpu().numpy() for x in whole.heat_flux(v))
    j_ref = jpot + ju + (0.5 * 28.0855 * (v * v).sum(1)[:, None] * v).sum(0)
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_runner_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        res = [q.get(timeout=300) for _ in range(2)]
        for p in procs:
            p.join(timeout=120)
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
    wc = np.zeros_like(ref)
    for _, gids, w, j, jp in res:
        wc[gids] = w
        scale = np.abs(ref).sum()
        print(f'runner: J {j} vs {j_ref}, J_pot {jp} vs {jpot}')
        assert np.abs(jp - jpot).max() < 1e-5 * scale
        assert np.abs(j - j_ref).max() < 1e-5 * scale
    assert np.array_equal(res[0][3], res[1][3])
    err = np.abs(wc - ref).max() / np.abs(ref).max()
    print(f'runner over NCCL: max |Wc - whole| / max |Wc| = {err:.1e}')
    assert err < BOUND
