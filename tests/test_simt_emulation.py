"""The warp-collective node kernels run on the CPU: their SOURCE is cut out of the .cuh files and compiled with g++
against tests/cpu_harness/simt_emu.h (one std::thread per CUDA thread, warp collectives on a barrier), then compared
with numpy.  Covers the kernels that produce the row exponents of the tensor-core linears' inputs
(gate_fwd_rows_kernel -- default path; gate_bwd_rows_kernel -- option gate_bwd_rows; row_exponent_kernel) and the
plain gate kernels they must agree with bit for bit."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'sevenn_b200', 'csrc')
KMAXL = 4
SILU = 1.6791767923989418


def _cut(src, start_pat):
    """text from the line matching start_pat up to and including the closing brace of the first '{' block after it"""
    m = re.search(start_pat, src, re.M)
    assert m, start_pat
    i = src.index('{', m.start())
    depth, j = 0, i
    while True:
        depth += {'{': 1, '}': -1}.get(src[j], 0)
        j += 1
        if depth == 0:
            break
    tail = ';' if src[j:j + 1] == ';' else ''
    return src[m.start():j] + tail + '\n'


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
    node = open(os.path.join(CSRC, 'node_kernels.cuh')).read()
    tc = open(os.path.join(CSRC, 'tc_gemm.cuh')).read()
    common = open(os.path.join(CSRC, 'common.cuh')).read()
    parts = ['#include "simt_emu.h"\nnamespace s7b {\n',
             'constexpr float kSiluNorm = 1.6791767923989418f;\nconstexpr int kMaxL = 4;\nconstexpr int kTcZeroRow = -1000;\n',
             _cut(common, r'^S7B_HD float silu_n\('), _cut(common, r'^S7B_HD float dsilu_n\('),
             _cut(node, r'^struct GateDesc '),
             _cut(node, r'^__global__ void gate_fwd_kernel\('), _cut(node, r'^__global__ void gate_bwd_kernel\('),
             _cut(node, r'^__device__ __forceinline__ void row_max_update\('),
             _cut(node, r'^__device__ __forceinline__ void row_exponents_store\('),
             _cut(node, r'^__global__ void gate_fwd_rows_kernel\('), _cut(node, r'^__global__ void gate_bwd_rows_kernel\('),
             _cut(tc, r'^struct RowExpArgs '), _cut(tc, r'^__global__ void row_exponent_kernel\('),
             '}  // namespace s7b\nusing namespace s7b;\nextern "C" {\n',
             'void emu_gate_fwd(const GateDesc* d, const float* g, float* h, int n) {'
             ' emu_launch(3, 256, [&] { gate_fwd_kernel(*d, g, h, n); }); }\n',
             'void emu_gate_bwd(const GateDesc* d, const float* g, const float* dh, float* dg, int n) {'
             ' emu_launch(3, 256, [&] { gate_bwd_kernel(*d, g, dh, dg, n); }); }\n',
             'void emu_gate_fwd_rows(const GateDesc* d, const float* g, float* h, int n, int* E, int rows) {'
             ' emu_launch((n + 7) / 8, 256, [&] { gate_fwd_rows_kernel(*d, g, h, n, E, rows, kTcZeroRow); }); }\n',
             'void emu_gate_bwd_rows(const GateDesc* d, const float* g, const float* dh, float* dg, int n, unsigned* bits, int rows, int grid) {'
             ' emu_launch(grid, 256, [&] { gate_bwd_rows_kernel(*d, g, dh, dg, n, bits, rows); }); }\n',
             'void emu_row_exponent(const RowExpArgs* a) {'
             ' emu_launch((a->n_nodes + 7) / 8, 256, [&] { row_exponent_kernel(*a); }); }\n',
             '}\n']
    d = tmp_path_factory.mktemp('simt')
    src = d / 'emu_kernels.cpp'
    src.write_text(''.join(parts))
    lib = str(d / 'libemu.so')
    subprocess.check_call(['g++', '-std=c++17', '-O1', '-shared', '-fPIC', '-pthread', '-I', os.path.join(ROOT, 'tests', 'cpu_harness'),
                           str(src), '-o', lib])
    return ctypes.CDLL(lib)


class GateDesc(ctypes.Structure):
    _fields_ = [('n_scalars', ctypes.c_int), ('lmax', ctypes.c_int), ('mul', ctypes.c_int * KMAXL), ('dim_g', ctypes.c_int),
                ('dim_h', ctypes.c_int), ('g_off', ctypes.c_int * KMAXL), ('h_off', ctypes.c_int * KMAXL), ('gate_off', ctypes.c_int * KMAXL)]


class RowExpArgs(ctypes.Structure):
    _fields_ = [('A', ctypes.c_void_p), ('E', ctypes.c_void_p), ('lda', ctypes.c_int), ('n_nodes', ctypes.c_int),
                ('rows_per_node', ctypes.c_int), ('nblocks', ctypes.c_int), ('d', ctypes.c_int * KMAXL), ('K', ctypes.c_int * KMAXL),
                ('a_off', ctypes.c_int * KMAXL), ('row_base', ctypes.c_int * KMAXL)]


def gate_desc(muls):
    """the descriptor engine.cu:build_layer_cfg fills: g row = [scalars | gate scalars | l = 1 block | ...], h row = blocks"""
    n_lo = len(muls)
    gates = sum(muls[1:])
    g_muls0 = muls[0] + gates
    g_off = [0] + list(np.cumsum([g_muls0] + [(2 * l + 1) * muls[l] for l in range(1, n_lo)]))[:-1][:n_lo - 1]
    g_off = [0]
    acc = g_muls0
    for l in range(1, n_lo):
        g_off.append(acc)
        acc += (2 * l + 1) * muls[l]
    dim_g = acc
    h_off, acc = [], 0
    for l in range(n_lo):
        h_off.append(acc)
        acc += (2 * l + 1) * muls[l]
    dim_h = acc
    d = GateDesc()
    d.n_scalars, d.lmax, d.dim_g, d.dim_h = muls[0], n_lo - 1, dim_g, dim_h
    goff = muls[0]
    for l in range(KMAXL):
        d.mul[l] = muls[l] if l < n_lo else 0
        d.g_off[l] = g_off[l] if l < n_lo else dim_g
        d.h_off[l] = h_off[l] if l < n_lo else dim_h
        d.gate_off[l] = g_muls0
    for l in range(1, n_lo):
        d.gate_off[l] = goff
        goff += muls[l]
    return d


def silu(z):
    return SILU * z / (1.0 + np.exp(-z))


def dsilu(z):
    s = 1.0 / (1.0 + np.exp(-z))
    return SILU * s * (1.0 + z * (1.0 - s))


def gate_numpy(d, g, dh=None):
    """h (and dg for a given dh) in float64"""
    n = len(g)
    g = g.astype(np.float64)
    h = np.zeros((n, d.dim_h))
    h[:, :d.n_scalars] = silu(g[:, :d.n_scalars])
    dg = None if dh is None else np.zeros((n, d.dim_g))
    if dh is not None:
        dg[:, :d.n_scalars] = dh[:, :d.n_scalars] * dsilu(g[:, :d.n_scalars])
    for l in range(1, d.lmax + 1):
        m = d.mul[l]
        gate = g[:, d.gate_off[l]:d.gate_off[l] + m]
        blk = g[:, d.g_off[l]:d.g_off[l] + (2 * l + 1) * m].reshape(n, 2 * l + 1, m)
        h[:, d.h_off[l]:d.h_off[l] + (2 * l + 1) * m] = (blk * silu(gate)[:, None, :]).reshape(n, -1)
        if dh is not None:
            dhb = dh[:, d.h_off[l]:d.h_off[l] + (2 * l + 1) * m].astype(np.float64).reshape(n, 2 * l + 1, m)
            dg[:, d.g_off[l]:d.g_off[l] + (2 * l + 1) * m] = (dhb * silu(gate)[:, None, :]).reshape(n, -1)
            dg[:, d.gate_off[l]:d.gate_off[l] + m] = (dhb * blk).sum(1) * dsilu(gate)
    return h, dg


def exponents_of_bits(bits, zero_row=-1000):
    """the row exponent the kernels derive from the bits of max |row| (node_kernels.cuh row_exponents_store):
    zero_row for zero / subnormal / Inf / NaN maxima, otherwise max |row| < 2^E with E clamped at -104"""
    ex = (np.asarray(bits, dtype=np.uint32) >> 23).astype(np.int64)
    return np.where((ex == 0) | (ex == 255), zero_row, np.maximum(ex - 126, -104))


def row_exponents(a, blocks, zero_row=-1000):
    """E[n, row_base + i] with max |row| < 2^E from the fp32 bit pattern, as tc_gemm.cuh defines it"""
    out = []
    for dcomp, K, off in blocks:
        rows = np.abs(a[:, off:off + dcomp * K]).reshape(len(a), dcomp, K).max(2).astype(np.float32)
        out.append(exponents_of_bits(rows.view(np.uint32), zero_row))
    return np.concatenate(out, 1)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize('muls', [(128, 64, 32), (128, 64, 32, 32), (128,)])
def test_gate_kernels_and_row_exponents_on_the_emulator(emu, muls):
    rng = np.random.RandomState(len(muls))
    d = gate_desc(list(muls))
    n = 21
    g = (rng.normal(size=(n, d.dim_g)) * np.exp(rng.uniform(-6, 3, size=(n, 1)))).astype(np.float32)
    g[3] = 0.0                                   # an all-zero node: zero rows must be flagged, not given an exponent
    g[5, d.g_off[1] if d.lmax else 0:] = 0.0
    dh = rng.normal(size=(n, d.dim_h)).astype(np.float32)
    rows = (d.lmax + 1) ** 2
    blocks_h = [(2 * l + 1, d.mul[l], d.h_off[l]) for l in range(d.lmax + 1)]
    g_muls0 = d.gate_off[KMAXL - 1] if d.lmax < KMAXL - 1 else d.g_off[1]
    blocks_g = [(1, g_muls0 if d.lmax else d.n_scalars, 0)] + [(2 * l + 1, d.mul[l], d.g_off[l]) for l in range(1, d.lmax + 1)]

    h0, h1 = np.zeros((n, d.dim_h), np.float32), np.zeros((n, d.dim_h), np.float32)
    E1 = np.full((n, rows), 7777, np.int32)
    emu.emu_gate_fwd(ctypes.byref(d), _ptr(g), _ptr(h0), n)
    emu.emu_gate_fwd_rows(ctypes.byref(d), _ptr(g), _ptr(h1), n, _ptr(E1), rows)
    ref_h, ref_dg = gate_numpy(d, g, dh)
    assert np.allclose(h0, ref_h, rtol=2e-6, atol=1e-30)
    assert np.array_equal(h0, h1)                                   # same arithmetic, bit for bit
    assert np.array_equal(E1, row_exponents(h1, blocks_h))
    assert (E1[3] == -1000).all()

    # the stand-alone row pass over h must give the same exponents
    a = RowExpArgs()
    E2 = np.full((n, rows), 7777, np.int32)
    a.A, a.E, a.lda, a.n_nodes, a.rows_per_node, a.nblocks = h1.ctypes.data, E2.ctypes.data, d.dim_h, n, rows, d.lmax + 1
    for l, (dc, K, off) in enumerate(blocks_h):
        a.d[l], a.K[l], a.a_off[l], a.row_base[l] = dc, K, off, l * l
    emu.emu_row_exponent(ctypes.byref(a))
    assert np.array_equal(E2, E1)

    dg0, dg1 = np.zeros((n, d.dim_g), np.float32), np.zeros((n, d.dim_g), np.float32)
    bits = np.zeros((n, rows), np.uint32)
    emu.emu_gate_bwd(ctypes.byref(d), _ptr(g), _ptr(dh), _ptr(dg0), n)
    grid = (n * d.dim_g + 255) // 256
    emu.emu_gate_bwd_rows(ctypes.byref(d), _ptr(g), _ptr(dh), _ptr(dg1), n, _ptr(bits), rows, min(grid, 7))   # 7 blocks: grid-stride loop
    assert np.allclose(dg0, ref_dg, rtol=2e-5, atol=1e-6)
    assert np.array_equal(dg0, dg1)
    E_bits = exponents_of_bits(bits)                                 # what tc_gemm.cuh's row_exp() makes of the bits
    assert np.array_equal(E_bits, row_exponents(dg1, blocks_g))


def test_row_exponents_across_the_float_range(emu):
    """row_exponent_kernel on rows whose maxima span the whole fp32 range: zero and subnormal rows (and Inf / NaN)
    are flagged, rows down to 2^-104 get their exact exponent, smaller normal rows the clamped -104 (never the
    zero flag: the tensor-core linear must not drop them)."""
    K = 8
    exps = list(range(-125, 128, 3)) + [-104, -105, -97, -96, 127]       # 0.75 * 2^e is normal for e >= -125
    A = [np.full(K, 0.75 * 2.0 ** e) for e in exps]
    A += [np.zeros(K), np.full(K, 2.0 ** -140), np.full(K, 2.0 ** -149)]
    inf_row, nan_row = np.ones(K), np.ones(K)
    inf_row[3], nan_row[5] = np.inf, np.nan
    A += [inf_row, nan_row]
    A = np.ascontiguousarray(np.array(A, dtype=np.float32))
    n = len(A)
    a = RowExpArgs()
    E = np.full((n, 1), 7777, np.int32)
    a.A, a.E, a.lda, a.n_nodes, a.rows_per_node, a.nblocks = A.ctypes.data, E.ctypes.data, K, n, 1, 1
    a.d[0], a.K[0], a.a_off[0], a.row_base[0] = 1, K, 0, 0
    emu.emu_row_exponent(ctypes.byref(a))
    E = E[:, 0]
    m = len(exps)
    want = np.array([max(e, -104) for e in exps])                  # 0.75 * 2^e < 2^e
    assert np.array_equal(E[:m], want)
    assert (E[m:] == -1000).all()
    assert np.array_equal(E, exponents_of_bits(np.abs(A).max(1).view(np.uint32)))
