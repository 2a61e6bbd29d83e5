"""Tensor-core (wgmma) linear kernel (TMA-fed, error-free bf16x3 slices; csrc/tc_gemm.cuh) vs fp64 numpy, and vs the FP32
SIMT kernel inside the engine."""
import ctypes

import numpy as np
import pytest

from helpers import model_weights, species_of

pytestmark = pytest.mark.gpu


def _dense(rows, K, N, use_tc, seed=0):
    import torch
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    rng = np.random.RandomState(seed)
    A = rng.normal(size=(rows, K)).astype(np.float32)
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    a, w = torch.tensor(A, device='cuda'), torch.tensor(W, device='cuda')
    c = torch.full((rows, N), float('nan'), device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.s7b_dense_linear(a.data_ptr(), w.data_ptr(), c.data_ptr(), rows, K, N, use_tc, st))
    torch.cuda.synchronize()
    return c.cpu().numpy(), A.astype(np.float64) @ W.astype(np.float64)


@pytest.mark.parametrize('rows,K,N', [(128, 32, 32), (300, 64, 64), (1000, 224, 224), (257, 416, 64),
                                      (640, 352, 32), (513, 128, 384), (128, 32, 16), (4096, 384, 256)])
def test_tc_linear_matches_fp64(rows, K, N):
    got, ref = _dense(rows, K, N, 1, seed=rows + K)
    assert np.isfinite(got).all()
    err = np.abs(got - ref).max()
    # fp32-level: a plain fp32 dot product of length K has ~1e-7 * sqrt(K) relative error
    assert err < 4e-7 * np.sqrt(K) * max(1.0, np.abs(ref).max()), err
    simt, _ = _dense(rows, K, N, 0, seed=rows + K) if K % 4 == 0 else (got, None)
    assert np.abs(got - simt).max() < 6e-7 * np.sqrt(K) * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize('rows,K,N', [(300, 64, 64), (1000, 224, 224), (77, 8, 64)])
def test_simt_linear_matches_fp64(rows, K, N):
    got, ref = _dense(rows, K, N, 0, seed=1)
    assert np.abs(got - ref).max() < 3e-6 * np.sqrt(K) * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize('rows,K,N', [(1000, 224, 224), (5000, 384, 64)])
def test_tc_linear_has_no_accumulation_bias(rows, K, N):
    """The tensor core's truncating accumulation biased the round-1 3xTF32 kernel (~ -3e-7 relative); the
    fixed-point slices make the first-order accumulator exact, so the signed error averages to zero."""
    got, ref = _dense(rows, K, N, 1, seed=11)
    scale = np.abs(ref).mean()
    signed = (got - ref) * np.sign(ref) / scale
    assert abs(signed.mean()) < 4.0 * signed.std() / np.sqrt(signed.size) + 1e-10
    assert np.sqrt(((got - ref) ** 2).mean()) / scale < 3e-6


def test_tc_linear_swizzled_and_plain_tma_tiles_agree():
    from sevenn_b200.engine import set_option
    try:
        set_option('tc_swizzle', 0)
        plain, ref = _dense(777, 224, 112, 1, seed=3)
        set_option('tc_swizzle', 1)
        swz, _ = _dense(777, 224, 112, 1, seed=3)
    finally:
        set_option('tc_swizzle', 1)
    assert np.array_equal(plain, swz)
    assert np.abs(swz - ref).max() < 4e-7 * np.sqrt(224) * max(1.0, np.abs(ref).max())


def test_engine_tc_and_simt_linears_agree():
    import torch
    from sevenn_b200.engine import B200Engine, set_option
    from sevenn_b200.neighbors import build_graph, diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos, cell, z = diamond_si(3, 3, 3)
    ei, ev = build_graph(pos, cell, True, 5.0)
    e = B200Engine(meta, arrays)
    e.set_graph(species_of(meta, z), ei, ev)
    out = {}
    try:
        for tc in (0, 1):
            set_option('tc_gemm', tc)
            e.compute()
            torch.cuda.synchronize()
            r = e.results()
            out[tc] = (float(r['energy'].cpu()[0]), r['forces'].cpu().numpy())
    finally:
        set_option('tc_gemm', 1)
    # 216 atoms: no systematic per-atom energy shift between the two GEMM paths (round 1: -8.7e-6 eV/atom)
    assert abs(out[0][0] - out[1][0]) < 216 * 3e-7, (out[0][0], out[1][0])
    assert np.allclose(out[0][1], out[1][1], atol=2e-5)


def _block_linear(n_nodes, a_K, c_N, accumulate, use_tc, seed=0, pad=(32, 64)):
    """C_l (+)= A_l W_l for irrep blocks l = 0.. through the engine's kernels; returns (got, fp64 reference)."""
    import torch
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    rng = np.random.RandomState(seed)
    n_l = len(a_K)
    a_off, c_off, lda, ldc = [], [], pad[0], pad[1]        # leading pads: blocks do not start at column 0
    for l in range(n_l):
        a_off.append(lda)
        lda += (2 * l + 1) * a_K[l]
        c_off.append(ldc)
        ldc += (2 * l + 1) * c_N[l]
    lda += 32
    ldc += 32
    A = (rng.normal(size=(n_nodes, lda)) * np.exp(rng.normal(size=(n_nodes, 1)))).astype(np.float32)
    C0 = rng.normal(size=(n_nodes, ldc)).astype(np.float32)
    Ws = [(rng.normal(size=(a_K[l], c_N[l])) / np.sqrt(a_K[l])).astype(np.float32) for l in range(n_l)]
    W = np.ascontiguousarray(np.concatenate([w.ravel() for w in Ws]))
    ref = C0.astype(np.float64).copy()
    for l in range(n_l):
        d = 2 * l + 1
        a = A[:, a_off[l]:a_off[l] + d * a_K[l]].reshape(n_nodes, d, a_K[l]).astype(np.float64)
        out = a @ Ws[l].astype(np.float64)
        blk = ref[:, c_off[l]:c_off[l] + d * c_N[l]].reshape(n_nodes, d, c_N[l])
        blk[...] = (blk if accumulate else 0.0) + out
        ref[:, c_off[l]:c_off[l] + d * c_N[l]] = blk.reshape(n_nodes, -1)
    a_t, c_t = torch.tensor(A, device='cuda'), torch.tensor(C0, device='cuda')
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ao, ak, co, cn = i32(a_off), i32(a_K), i32(c_off), i32(c_N)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.s7b_block_linear(a_t.data_ptr(), lda, n_nodes, n_l, ao.ctypes.data, ak.ctypes.data, W.ctypes.data,
                               c_t.data_ptr(), ldc, co.ctypes.data, cn.ctypes.data, int(accumulate), int(use_tc), st))
    torch.cuda.synchronize()
    return c_t.cpu().numpy(), ref


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('n_nodes,a_K,c_N', [
    (1000, [224, 384, 352], [224, 64, 32]),          # 7net-0 mid layer, self_interaction_2
    (1000, [224, 64, 32], [224, 384, 352]),          # ... its transpose (backward)
    (333, [128, 64, 32], [128, 64, 32]),             # self_interaction_1
    (4100, [128, 64, 32], [224, 64, 32]),            # self connection; 33 node tiles: several tiles per CTA
    (515, [256, 480, 416, 352], [256, 64, 32, 32]),  # lmax 3 shapes (SevenNet-l3i5 self_interaction_2)
    (515, [256, 64, 32, 32], [256, 480, 416, 352]),  # ... its transpose: column tiles of 128 / 96 / 32 / 32
    (300, [128, 64, 32, 32], [256, 64, 32, 32]),     # lmax 3 self connection
    (20000, [224, 384, 352], [224, 64, 32]),         # many tiles per CTA: the operand rings wrap many times
    (333, [64, 32, 96], [48, 96, 40]),               # tile widths 48 / 96 / 48 (padded)
    (129, [96, 64, 32], [180, 72, 100]),             # 2 x 96 (padded), 80 (padded), 112 (padded)
])
def test_block_linear_tc_matches_fp64(n_nodes, a_K, c_N, accumulate):
    got, ref = _block_linear(n_nodes, a_K, c_N, accumulate, 1, seed=n_nodes)
    assert np.isfinite(got).all()
    scale = np.abs(ref).max(axis=1, keepdims=True) + 1e-30
    assert (np.abs(got - ref) / scale).max() < 2e-5, (np.abs(got - ref) / scale).max()
    simt, _ = _block_linear(n_nodes, a_K, c_N, accumulate, 0, seed=n_nodes)
    assert (np.abs(simt - ref) / scale).max() < 2e-5
    # untouched columns (pads between / around the blocks) stay as they were
    pad_cols = np.ones(ref.shape[1], dtype=bool)
    off = 64
    for l in range(len(c_N)):
        pad_cols[off:off + (2 * l + 1) * c_N[l]] = False
        off += (2 * l + 1) * c_N[l]
    assert np.array_equal(got[:, pad_cols], ref[:, pad_cols].astype(np.float32))


# ---- every tile width of tc_pick_nt (16 .. 128 in steps of 16) and the padded last tile -------------------
# N -> NT: 40 -> 48, 48 -> 48, 72 -> 80, 80 -> 80, 96 -> 96, 100 -> 112, 136 -> 2 x 80, 160 -> 2 x 80,
# 180 -> 2 x 96, 260 -> 3 x 96 (asserted on the CPU in test_tc_pack_cpu.py)
TILE_WIDTH_N = [40, 48, 72, 80, 96, 100, 136, 160, 180, 260]


@pytest.mark.parametrize('N', TILE_WIDTH_N)
def test_tc_dense_linear_every_tile_width(N):
    got, ref = _dense(300, 96, N, 1, seed=N)
    assert np.isfinite(got).all()
    assert np.abs(got - ref).max() < 4e-7 * np.sqrt(96) * max(1.0, np.abs(ref).max())
    simt, _ = _dense(300, 96, N, 0, seed=N)
    assert np.abs(got - simt).max() < 6e-7 * np.sqrt(96) * max(1.0, np.abs(ref).max())


def _linear_rows(A, W, C0, n_nodes, accumulate, use_tc):
    """C[:n_nodes] (+)= A[:n_nodes] W through s7b_block_linear with one l = 0 block; A, C0 may hold more rows
    (and C0 more columns) than the product touches.  Returns the whole C."""
    import torch
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    K, N = W.shape
    a_t, c_t = torch.tensor(A, device='cuda'), torch.tensor(C0, device='cuda')
    i32 = lambda v: np.ascontiguousarray(v, dtype=np.int32)
    ao, ak, co, cn = i32([0]), i32([K]), i32([0]), i32([N])
    Wc = np.ascontiguousarray(W, dtype=np.float32)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(lib.s7b_block_linear(a_t.data_ptr(), A.shape[1], n_nodes, 1, ao.ctypes.data, ak.ctypes.data, Wc.ctypes.data,
                               c_t.data_ptr(), C0.shape[1], co.ctypes.data, cn.ctypes.data, int(accumulate), int(use_tc), st))
    torch.cuda.synchronize()
    return c_t.cpu().numpy()


@pytest.mark.parametrize('accumulate', [False, True])
@pytest.mark.parametrize('rows', [1, 63, 65, 129])
@pytest.mark.parametrize('N', TILE_WIDTH_N)
def test_tc_row_counts_leave_pads_and_extra_rows_alone(N, rows, accumulate):
    rng = np.random.RandomState(N + rows)
    K, extra, pad = 64, 70, 12
    A = rng.normal(size=(rows + extra, K)).astype(np.float32)
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    C0 = rng.normal(size=(rows + extra, N + pad)).astype(np.float32)
    ref = (C0[:rows, :N].astype(np.float64) if accumulate else 0.0) + A[:rows].astype(np.float64) @ W.astype(np.float64)
    for use_tc in (1, 0):
        got = _linear_rows(A, W, C0, rows, accumulate, use_tc)
        assert np.abs(got[:rows, :N] - ref).max() < 1e-6 * np.sqrt(K) * max(1.0, np.abs(ref).max()), use_tc
        assert np.array_equal(got[:, N:], C0[:, N:])            # pad columns
        assert np.array_equal(got[rows:], C0[rows:])            # rows beyond n_nodes


def _wide_range_operands(K=64, N=80, seed=0):
    """A: rows at scales 2^-100 .. 2^100, all-zero rows, rows of subnormals, rows with one dominant element;
    W: an all-zero column and columns at scales 2^-20 .. 2^20"""
    rng = np.random.RandomState(seed)
    scales = [2.0 ** e for e in range(-100, 101, 5)]
    A = [rng.normal(size=K) * s for s in scales]
    A += [np.zeros(K), np.zeros(K)]
    A += [rng.normal(size=K) * 2.0 ** -140, np.full(K, 2.0 ** -149)]         # subnormal rows
    for e in (-60, 0, 60):
        r = rng.normal(size=K) * 2.0 ** (e - 30)
        r[rng.randint(K)] = 2.0 ** e                                          # one dominant element
        A.append(r)
    A = np.array(A, dtype=np.float32)
    A = A[rng.permutation(len(A))]
    W = rng.normal(size=(K, N)) / np.sqrt(K) * 2.0 ** rng.randint(-20, 21, size=N)[None, :]
    W[:, 3] = 0.0
    W[:, 7] *= 2.0 ** rng.randint(-30, 31, size=K)                            # one column with a wide spread
    return A, W.astype(np.float32)


@pytest.mark.parametrize('use_tc', [1, 0])
def test_tc_linear_error_contract_over_the_exponent_range(use_tc):
    """|C - A W| <= c 2^-24 max_k|A_ik| max_k|W_kj| sqrt(K) for every element; all-zero rows and rows of
    subnormals give exactly 0 on the tensor-core path (the SIMT path multiplies them out within the same bound)."""
    A, W = _wide_range_operands()
    K, N = W.shape
    rows = len(A)
    got = _linear_rows(A, W, np.zeros((rows, N), np.float32), rows, False, use_tc).astype(np.float64)
    ref = A.astype(np.float64) @ W.astype(np.float64)
    amax = np.abs(A.astype(np.float64)).max(1)
    bound = 8 * 2.0 ** -24 * np.outer(amax, np.abs(W.astype(np.float64)).max(0)) * np.sqrt(K)
    assert np.isfinite(got).all()
    tiny = amax < 2.0 ** -126
    assert (amax[tiny] > 0).any() and (amax == 0).sum() == 2
    if use_tc:
        assert (got[tiny] == 0.0).all()
    else:
        assert (np.abs(got - ref)[tiny] <= bound[tiny] + K * 2.0 ** -149).all()     # K subnormal roundings
    err = np.abs(got - ref)[~tiny]
    assert (err <= bound[~tiny]).all(), (err / np.maximum(bound[~tiny], 1e-300)).max()
    assert (got[:, 3] == 0.0).all()


@pytest.mark.parametrize('use_tc', [1, 0])
def test_tc_linear_non_finite_rows_stay_non_finite(use_tc):
    """A row holding NaN or Inf gives a row of non-finite outputs on both paths (never finite numbers); the
    other rows are unaffected."""
    rng = np.random.RandomState(5)
    rows, K, N = 130, 64, 96
    A = rng.normal(size=(rows, K)).astype(np.float32)
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    W[:, 5] = 0.0
    bad = {3: np.nan, 64: np.inf, 65: -np.inf, 129: np.nan}
    for i, v in bad.items():
        A[i, rng.randint(K)] = v
    got = _linear_rows(A, W, np.zeros((rows, N), np.float32), rows, False, use_tc)
    for i in bad:
        assert not np.isfinite(got[i]).any(), (i, got[i][np.isfinite(got[i])][:4])
    good = np.setdiff1d(np.arange(rows), list(bad))
    ref = A[good].astype(np.float64) @ W.astype(np.float64)
    assert np.abs(got[good] - ref).max() < 1e-6 * np.sqrt(K) * np.abs(ref).max()
