import os, sys, ctypes, numpy as np, torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from sevenn_b200.engine import check, load_library
lib = load_library()
def run(rows, K, N, use_tc, scale=1.0, seed=0):
    rng = np.random.RandomState(seed)
    A = (rng.normal(size=(rows, K)) * scale).astype(np.float32)
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    a, w = torch.tensor(A, device='cuda'), torch.tensor(W, device='cuda')
    c = torch.zeros((rows, N), device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.s7b_dense_linear(a.data_ptr(), w.data_ptr(), c.data_ptr(), rows, K, N, use_tc, st))
    torch.cuda.synchronize()
    ref = A.astype(np.float64) @ W.astype(np.float64)
    got = c.cpu().numpy().astype(np.float64)
    t32 = (torch.tensor(A) @ torch.tensor(W)).numpy().astype(np.float64)
    return np.abs(got-ref).max(), np.sqrt(((got-ref)**2).mean()), (got-ref).mean(), np.abs(t32-ref).max(), np.abs(ref).max()
for (rows,K,N) in [(1024,224,224),(1024,384,64),(1024,128,128),(1024,32,32)]:
    for tc in (0,1):
        print(rows,K,N,'tc' if tc else 'simt', 'max|err| %.2e rms %.2e bias %.2e | torch-cpu-fp32 max %.2e | ref max %.2f' % run(rows,K,N,tc))
