"""Timeline of CTA 0 of one tensor-core linear launch (debug aid; see TC_TRACE in csrc/tc_gemm.cuh).
Prints, per role, the gaps between consecutive events -- where a tile's time goes."""
import ctypes, os, sys
import numpy as np, torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from sevenn_b200.engine import check, load_library
lib = load_library()
ROLE = {0: 'prodA', 1: 'xform', 2: 'mma0', 3: 'epi0', 4: 'prodW', 5: 'mma1', 6: 'epi1'}
EV = {(0, 0): 'issue', (1, 0): 'raw_landed', (1, 1): 'ops_free', (1, 2): 'written', (2, 0): 'w_landed', (2, 1): 'ops_ready',
      (2, 2): 'wait1_ret', (3, 0): 'acc_full', (3, 1): 'tile_done', (3, 2): 'stage_free', (3, 3): 'staged', (4, 0): 'issue'}
EV.update({(5, e): EV[(2, e)] for e in range(3)})
EV.update({(6, e): EV[(3, e)] for e in range(4)})
MMA_WG = [(2, 3), (5, 6)]           # (MMA role, epilogue role) of each MMA warpgroup
N_ROLES = 7


def run(n_nodes, a_K, c_N, acc, label, warm=True):
    rng = np.random.RandomState(0)
    n_l = len(a_K)
    a_off, c_off, lda, ldc = [], [], 0, 0
    for l in range(n_l):
        a_off.append(lda); lda += (2 * l + 1) * a_K[l]
        c_off.append(ldc); ldc += (2 * l + 1) * c_N[l]
    A = torch.tensor(rng.normal(size=(n_nodes, lda)).astype(np.float32), device='cuda')
    C = torch.zeros(n_nodes, ldc, device='cuda')
    W = np.ascontiguousarray(np.concatenate([(rng.normal(size=(a_K[l], c_N[l])) / np.sqrt(a_K[l])).astype(np.float32).ravel() for l in range(n_l)]))
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ao, ak, co, cn = i32(a_off), i32(a_K), i32(c_off), i32(c_N)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    call = lambda: check(lib.s7b_block_linear(A.data_ptr(), lda, n_nodes, n_l, ao.ctypes.data, ak.ctypes.data, W.ctypes.data,
                                              C.data_ptr(), ldc, co.ctypes.data, cn.ctypes.data, int(acc), 1, st))
    if warm:
        call()
    cap = 20000
    buf = ctypes.c_void_p()
    check(lib.s7b_tc_trace_enable(cap, ctypes.byref(buf)))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    call()
    torch.cuda.synchronize()
    from sevenn_b200.engine import _DevView
    view = torch.as_tensor(_DevView(buf.value, (8 + 3 * cap,), '<i8'), device='cuda')
    host = view.cpu().numpy().copy()
    check(lib.s7b_tc_trace_enable(0, ctypes.byref(buf)))
    per = cap // N_ROLES
    recs = []
    for role in range(N_ROLES):
        n_r = int(min(host[1 + role], per))
        blk = host[8 + 3 * role * per: 8 + 3 * (role * per + n_r)].reshape(n_r, 3)
        recs.append(np.concatenate([np.full((n_r, 1), role, dtype=np.int64), blk], axis=1))
    rec = np.concatenate(recs)
    n = len(rec)
    rec = rec[np.argsort(rec[:, 3], kind='stable')]
    t0 = rec[:, 3].min()
    print(f'== {label}: nodes {n_nodes} K {a_K} N {c_N} acc {acc}: {n} records, CTA 0 span {rec[:, 3].max() - t0} clk')
    for role in sorted(set(rec[:, 0])):
        r = rec[rec[:, 0] == role]
        for ev in sorted(set(r[:, 1])):
            e = r[r[:, 1] == ev]
            ts = e[:, 3] - t0
            gaps = np.diff(ts)
            print(f'   {ROLE[role]:6s} {EV[(role, ev)]:11s} n={len(e):4d} first {ts[0]:7d} last {ts[-1]:7d}  gap mean {gaps.mean() if len(gaps) else 0:8.0f} max {gaps.max() if len(gaps) else 0:7d}'
                  f'  first 12: {ts[:12].tolist()}')
    # per-chunk latencies: issue -> landed -> written -> mma ready
    def ev(role, e_):
        m = rec[(rec[:, 0] == role) & (rec[:, 1] == e_)]
        return dict(zip(m[:, 2].tolist(), (m[:, 3] - t0).tolist()))
    issue, landed, free, written, ready = ev(0, 0), ev(1, 0), ev(1, 1), ev(1, 2), {**ev(2, 1), **ev(5, 1)}
    lat = [(k, landed[k] - issue[k], free[k] - landed[k], written[k] - free[k], ready[k] - written[k]) for k in sorted(issue) if k in landed and k in written and k in ready and k in free]
    arr = np.array(lat)
    if len(arr):
        print('   per chunk (mean clk): TMA issue->landed %.0f | landed->ops slot free %.0f | convert %.0f | written->MMA sees it %.0f' % tuple(arr[:, 1:].mean(0)))
        print('   first 10 chunks:', arr[:10].tolist())
    # MMA warpgroup, per chunk: waiting in w_landed / ops_ready (from the warpgroup's previous event: the last
    # chunk's wait_group 1 return, or the end of its previous epilogue), then ops_ready -> wait_group 1 returned
    # (issuing this chunk and retiring the previous one); chunk interval = ops_ready to ops_ready inside a tile
    for mma_role, epi_role in MMA_WG:
        wl, rd, wt = ev(mma_role, 0), ev(mma_role, 1), ev(mma_role, 2)
        marks = np.sort(np.array(list(wt.values()) + list(ev(epi_role, 1).values()), dtype=np.int64))
        tile_ends = np.sort(np.array(list(ev(epi_role, 1).values()), dtype=np.int64))
        rows = []
        for k in sorted(rd):
            if k not in wl or k not in wt:
                continue
            i = np.searchsorted(marks, wl[k]) - 1
            if i < 0:
                continue
            prev_rd = rd.get(k - 1)
            same_tile = prev_rd is not None and not np.any((tile_ends > prev_rd) & (tile_ends < rd[k]))
            rows.append((wl[k] - marks[i], rd[k] - wl[k], wt[k] - rd[k], rd[k] - prev_rd if same_tile else -1))
        if rows:
            r = np.array(rows, dtype=np.float64)
            iv = r[r[:, 3] >= 0, 3]
            print(f'   {ROLE[mma_role]} per chunk (mean clk, {len(r)} chunks): wait w_landed {r[:, 0].mean():.0f} | wait ops_ready '
                  f'{r[:, 1].mean():.0f} | ops_ready->wait_group 1 returned {r[:, 2].mean():.0f} | chunk interval in a tile '
                  f'{iv.mean() if len(iv) else 0:.0f} (median {np.median(iv) if len(iv) else 0:.0f})')


run(12000, [128, 64, 32], [128, 64, 32], False, 'self_interaction_1')
run(12000, [224, 384, 352], [224, 64, 32], True, 'self_interaction_2')
run(12000, [224, 64, 32], [224, 384, 352], False, 'self_interaction_2^T')
