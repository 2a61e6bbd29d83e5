"""Timeline of CTA 0 of one tensor-core linear launch (debug aid; see TC_TRACE in csrc/tc_gemm.cuh).
Prints, per role, the gaps between consecutive events -- where a tile's time goes."""
import ctypes, os, sys
import numpy as np, torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
from sevenn_b200.engine import check, load_library
lib = load_library()
ROLE = {0: 'prodA', 1: 'xform', 2: 'mma', 3: 'epi', 4: 'prodW'}
EV = {(0, 0): 'issue', (1, 0): 'raw_landed', (1, 1): 'ops_free', (1, 2): 'written', (2, 0): 'w_landed', (2, 1): 'ops_ready',
      (2, 2): 'acc_free', (3, 0): 'acc_full', (3, 1): 'tile_done', (3, 2): 'stage_free', (3, 3): 'staged', (4, 0): 'issue'}


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
    per = cap // 5
    recs = []
    for role in range(5):
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
    issue, landed, free, written, ready = ev(0, 0), ev(1, 0), ev(1, 1), ev(1, 2), ev(2, 1)
    lat = [(k, landed[k] - issue[k], free[k] - landed[k], written[k] - free[k], ready[k] - written[k]) for k in sorted(issue) if k in landed and k in written and k in ready and k in free]
    arr = np.array(lat)
    if len(arr):
        print('   per chunk (mean clk): TMA issue->landed %.0f | landed->ops slot free %.0f | convert %.0f | written->MMA sees it %.0f' % tuple(arr[:, 1:].mean(0)))
        print('   first 10 chunks:', arr[:10].tolist())


run(12000, [128, 64, 32], [128, 64, 32], False, 'self_interaction_1')
run(12000, [224, 384, 352], [224, 64, 32], True, 'self_interaction_2')
run(12000, [224, 64, 32], [224, 384, 352], False, 'self_interaction_2^T')
