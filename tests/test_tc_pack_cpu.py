"""Host-side logic of the tensor-core linear (sevenn_b200/csrc/tc_gemm.cuh), no GPU needed:
the C++ weight packing exported as ``s7b_tc_pack_weights`` and a bit-faithful numpy emulation of the
kernel's fixed-point slicing.  Claims checked: (1) the three bf16 slices reproduce W to 2^-24 of the
column bound; (2) the first-order accumulator ACC0 holds integers below 2^24, so the tensor core's
truncating fp32 accumulation has nothing to truncate; (3) the result is as accurate as an fp32 FMA chain
and has no systematic bias."""
import ctypes

import numpy as np
import pytest


def _pack(W):
    from sevenn_b200.engine import check, load_library
    lib = load_library()
    K, N = W.shape
    W = np.ascontiguousarray(W, dtype=np.float32)
    q = np.zeros(3 * K * (N + 127), dtype=np.uint16)
    fb = np.zeros(N, dtype=np.float32)
    nt = ctypes.c_int32()
    check(lib.s7b_tc_pack_weights(W.ctypes.data, K, N, q.ctypes.data, fb.ctypes.data, ctypes.byref(nt)))
    NT = nt.value
    # undo the [n tile][K/32][slice][canonical NT x 32] arrangement -> slices [3, N, K] as float64
    vals = (q.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    n_kc = K // 32
    out = np.zeros((3, N, K))
    r = np.arange(NT)[:, None]
    kk = np.arange(32)[None, :]
    elem = ((r & 7) * 16 + (r >> 3) * 512 + (kk >> 3) * 128 + (kk & 7) * 2) // 2
    tiles = (N + NT - 1) // NT
    padded = np.zeros((3, tiles * NT, K))
    for t in range(tiles):
        for kc in range(n_kc):
            for s in range(3):
                base = ((t * n_kc + kc) * 3 + s) * NT * 32
                padded[s, t * NT:(t + 1) * NT, kc * 32:(kc + 1) * 32] = vals[base + elem]
    assert not padded[:, N:].any()                      # pad columns of the last tile carry zero weights
    out[:] = padded[:, :N]
    return out, fb.astype(np.float64), NT


def _slice_rows(A):
    """numpy float32 replica of the transform warps (magic-number rounding, exact residuals)."""
    A = A.astype(np.float32)
    bits = (np.abs(A).max(axis=1).view(np.uint32) >> 23).astype(np.int64)
    Ea = bits - 126
    sc = np.ldexp(np.float32(1.0), (23 - Ea).astype(np.int32)).astype(np.float32)[:, None]
    M = np.float32(12582912.0)
    t = A * sc
    q0 = (t * np.float32(2.0 ** -16) + M) - M
    r1 = (t.astype(np.float64) - q0.astype(np.float64) * 65536.0).astype(np.float32)
    assert np.array_equal(r1.astype(np.float64), t.astype(np.float64) - q0.astype(np.float64) * 65536.0)   # exact
    q1 = (r1 * np.float32(2.0 ** -8) + M) - M
    r2 = (r1.astype(np.float64) - q1.astype(np.float64) * 256.0).astype(np.float32)
    assert np.array_equal(r2.astype(np.float64), r1.astype(np.float64) - q1.astype(np.float64) * 256.0)    # exact
    q2 = (r2 + M) - M
    for q in (q0, q1, q2):
        assert np.abs(q).max() <= 128 and np.array_equal(q, np.rint(q))
    fa = np.ldexp(1.0, (Ea - 7).astype(np.int32))
    return q0.astype(np.float64), q1.astype(np.float64) / 256.0, q2.astype(np.float64) / 65536.0, fa


# tile width tc_pick_nt chooses for N (fewest tiles of <= 128 columns, width a multiple of 16): the GPU tests of
# tests/test_tc_gemm_gpu.py use these N to reach the wgmma widths 48 / 80 / 96 / 112 and a padded last tile
TILE_WIDTHS = {40: 48, 48: 48, 72: 80, 80: 80, 96: 96, 100: 112, 136: 80, 160: 80, 180: 96, 260: 96,
               16: 16, 32: 32, 64: 64, 128: 128, 224: 112, 384: 128}


@pytest.mark.parametrize('N,NT', sorted(TILE_WIDTHS.items()))
def test_pack_picks_the_tile_width(N, NT):
    W = np.random.RandomState(N).normal(size=(64, N)).astype(np.float32)
    sl, fb, nt = _pack(W)
    assert nt == NT
    rec = (sl.sum(0) * fb[:, None]).T
    assert np.all(np.abs(rec - W) <= np.abs(W).max(axis=0) * 2.0 ** -23)


@pytest.mark.parametrize('K,N', [(32, 32), (224, 224), (384, 64), (352, 32), (64, 384), (256, 256), (32, 352), (64, 480), (32, 416), (32, 24)])
def test_pack_reproduces_weights(K, N):
    rng = np.random.RandomState(K + N)
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    W[:, 0] = 0.0                                      # an all-zero column
    sl, fb, NT = _pack(W)
    assert NT <= 128 and NT % 16 == 0 and (N + NT - 1) // NT == (N + 127) // 128     # fewest tiles of <= 128 columns
    rec = (sl.sum(0) * fb[:, None]).T                  # [K, N]
    bound = np.abs(W).max(axis=0)
    assert np.all(np.abs(rec - W) <= np.maximum(bound, 1e-30) * 2.0 ** -23 + 1e-30)
    q0 = sl[0]
    assert np.array_equal(q0, np.rint(q0)) and np.abs(q0).max() <= 128
    assert np.array_equal(sl[1] * 256, np.rint(sl[1] * 256)) and np.abs(sl[1]).max() <= 0.5 + 1e-12
    assert np.array_equal(sl[2] * 65536, np.rint(sl[2] * 65536))


@pytest.mark.parametrize('K,N', [(224, 224), (384, 64), (352, 32)])
def test_emulated_kernel_is_exact_and_unbiased(K, N):
    rng = np.random.RandomState(7)
    rows = 4096
    A = (rng.normal(size=(rows, K)) * np.exp(rng.normal(size=(rows, 1)))).astype(np.float32)   # rows of varied scale
    W = (rng.normal(size=(K, N)) / np.sqrt(K)).astype(np.float32)
    B, fb, _ = _pack(W)
    A0, A1, A2, fa = _slice_rows(A)
    acc0 = A0 @ B[0].T
    assert np.abs(acc0).max() < 2 ** 23 and np.array_equal(acc0, np.rint(acc0))      # exact in an fp32 accumulator
    acc1 = A0 @ B[1].T + A1 @ B[0].T + A0 @ B[2].T + A1 @ B[1].T + A2 @ B[0].T
    got = ((acc0.astype(np.float32) + acc1.astype(np.float32)).astype(np.float64) * fa[:, None] * fb[None, :])
    ref = A.astype(np.float64) @ W.astype(np.float64)
    simt = A @ W                                                                      # numpy fp32 (pairwise/blocked)
    scale = np.abs(ref).mean()
    err, err32 = got - ref, simt.astype(np.float64) - ref
    assert np.sqrt((err ** 2).mean()) < 3.0 * np.sqrt((err32 ** 2).mean()) + 1e-9 * scale
    # no systematic component: the mean signed error (relative to sign(ref)) is consistent with zero
    signed = err * np.sign(ref) / scale
    bias, sem = signed.mean(), signed.std() / np.sqrt(signed.size)
    assert abs(bias) < 4.0 * sem + 1e-10, (bias, sem)        # (a truncating 3xTF32 accumulation shows ~ -3e-7 here)
