"""CPU checks of the radial path at radial shapes other than the shipped models' (tests/radial_models.py): the
packed radial table read back exactly as the convolution kernels read it, against the fp64 radial MLP; the knot
rule that keeps XPLOR's switching radius on a knot; the converter's radial fields; the refusal of radial MLPs
without exactly two hidden layers."""
import ctypes
import functools
import tempfile

import numpy as np
import pytest

from helpers import model_weights
from radial_models import CONFIGS, convert_radial, write_radial_checkpoint

# Errors relative to the local scale: the max over channels within 0.1 A, floored at 0.1 of the global max (near
# rc the envelope takes w and dw/dr to zero).  Measured with every XPLOR r_on on a knot: dw/dr <= 3.0e-4 (R5 next
# to rc), w <= 1.3e-6; the synthetic models' weights are O(1), so their a2 / a3 coefficients sit near fp16's
# subnormal range and dw/dr carries an absolute error of ~1e-5 of its global max everywhere.  With r_on inside an
# interval (R1, R5 on 2000 knots) every layer reaches 1.2e-3 .. 2.1e-3 at r_on.  The shipped models stay below
# 4.5e-5 (SevenNet-l3i5 layer 3 at 0.27 A; 1e-5 elsewhere).
DW_BOUND = 6e-4
DW_BOUND_SHIPPED = 1e-4
W_BOUND = 5e-6


@functools.lru_cache(maxsize=None)
def _radial_model(cid, hidden=None):
    d = tempfile.mkdtemp(prefix='radial_ckpt_')
    path = write_radial_checkpoint(f'{d}/{cid}.pth', cid, None if hidden is None else list(hidden))
    return convert_radial(path, cid)


def _model(name):
    return _radial_model(name) if name in CONFIGS else model_weights(name)


def device_table_read(t01, t23, knots, cutoff, r):
    """w, dw/dr [len(r), W] as the kernels read the packed table (engine.py pack_table_pairs) at fp32 radii r:
    s = f32(r) * f32(knots / cutoff) in fp32, interval tk = (int)s clamped to [0, knots - 1], tt = s - tk clamped
    to [0, 1] (edge_fwd_kernel), a0 + tt(a1 + tt(a2 + tt a3)) and (a1 + tt(2 a2 + 3 tt a3)) * inv_h
    (conv_kernels.cuh)."""
    K = knots
    a01 = t01.astype(np.float64).reshape(K, -1, 2, 2)                     # [k, pair, coef, parity]
    a23 = t23.view(np.float16).astype(np.float64).reshape(K, -1, 2, 2)
    tab = np.concatenate([a01, a23], axis=2).transpose(0, 1, 3, 2).reshape(K, -1, 4)
    inv_h = np.float32(np.float32(K) / np.float32(cutoff))
    s = np.asarray(r, dtype=np.float32) * inv_h
    tk = np.clip(s.astype(np.int64), 0, K - 1)
    tt = np.clip(s - tk.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float64)[:, None]
    a = tab[tk]
    w = a[..., 0] + tt * (a[..., 1] + tt * (a[..., 2] + tt * a[..., 3]))
    dw = (a[..., 1] + tt * (2.0 * a[..., 2] + 3.0 * tt * a[..., 3])) * float(inv_h)
    return w, dw


def sample_radii(spec, knots):
    """fp32 radii in [0.2, rc): every interval at several fractions, the knots, r_on +- {1e-6, h/3}, rc - 1e-6"""
    h = spec.cutoff / knots
    frac = np.array([0.0, 0.1, 0.3, 0.5, 0.7, 0.9, 0.999])
    r = ((np.arange(knots)[:, None] + frac) * h).ravel()
    extra = [spec.cutoff - 1e-6]
    if spec.cutoff_fn == 'XPLOR':
        extra += [spec.cutoff_on + d for d in (-h / 3, -1e-6, 1e-6, h / 3)]
    r = np.concatenate([r, extra])
    r = r[(r >= 0.2) & (r <= spec.cutoff - 1e-6)]
    return np.unique(r.astype(np.float32))


def table_errors(spec, arrays, t, knots):
    """(max w error / local max |w|, max dw/dr error / local max |dw/dr|, r of the worst dw/dr) of layer t's packed
    table; the local scale is the max over channels and over radii within 0.1 A, floored at 0.1 of the global max"""
    from scipy.ndimage import maximum_filter1d
    from sevenn_b200.engine import pack_table_pairs, radial_table, radial_weights
    t01, t23 = pack_table_pairs(radial_table(spec, arrays, t, knots))
    step = 0.002
    rg = np.arange(0.0, spec.cutoff + step / 2, step)
    fg, dfg = radial_weights(spec, arrays, t, np.maximum(rg, 1e-9))
    win = int(round(0.1 / step))
    sw = maximum_filter1d(np.abs(fg).max(1), 2 * win + 1)
    sdw = maximum_filter1d(np.abs(dfg).max(1), 2 * win + 1)
    sw, sdw = np.maximum(sw, 0.1 * sw.max()), np.maximum(sdw, 0.1 * sdw.max())
    r32 = sample_radii(spec, knots)
    ew, edw = np.zeros(len(r32)), np.zeros(len(r32))
    for i in range(0, len(r32), 2048):
        r = r32[i:i + 2048]
        w, dw = device_table_read(t01, t23, knots, spec.cutoff, r)
        f, df = radial_weights(spec, arrays, t, r.astype(np.float64))
        g = np.rint(r.astype(np.float64) / step).astype(int)
        ew[i:i + 2048] = np.abs(w - f).max(1) / sw[g]
        edw[i:i + 2048] = np.abs(dw - df).max(1) / sdw[g]
    j = int(np.argmax(edw))
    return float(ew.max()), float(edw[j]), float(r32[j])


MODELS = sorted(CONFIGS) + ['sevennet_0', 'sevennet_l3i5']


@pytest.mark.parametrize('name', MODELS)
def test_table_matches_radial_mlp(name):
    from sevenn_b200.engine import default_table_knots
    from sevenn_b200.spec import build_spec
    meta, arrays = _model(name)
    spec = build_spec(meta)
    knots = default_table_knots(spec)
    bound = DW_BOUND if name in CONFIGS else DW_BOUND_SHIPPED
    for t in range(spec.n_layers):
        ew, edw, r = table_errors(spec, arrays, t, knots)
        assert ew < W_BOUND and edw < bound, (name, knots, t, ew, edw, r)


@pytest.mark.parametrize('name', MODELS)
def test_table_is_exactly_zero_at_the_cutoff(name):
    """Edges at or beyond the cutoff read the end of the last interval (t = 1): the kernels' fp32 sums there,
    w = fma(1, fma(1, fma(1, a3, a2), a1), a0) and dw/dr h = fma(1, fma(3, a3, 2 a2), a1), must be exactly 0 with the
    fp16 a2, a3 the device holds (regression: 1e-11 of w and 1e-8 of dw/dr were left), and closing the interval
    moves a0 and a1 by no more than that rounding"""
    from sevenn_b200.engine import default_table_knots, pack_table_pairs, prepare_params, radial_table
    from sevenn_b200.spec import build_spec
    meta, arrays = _model(name)
    spec = build_spec(meta)
    knots = default_table_knots(spec)
    p = prepare_params(spec, arrays, 'table', knots)
    for t in range(spec.n_layers):
        t01, t23 = p[('table', t)][-1], p[('table23', t)].view(np.float16)[-1].astype(np.float32)
        a0, a1, a2, a3 = t01[:, 0:2], t01[:, 2:4], t23[:, 0:2], t23[:, 2:4]
        f32 = lambda v: np.asarray(v, dtype=np.float64).astype(np.float32)
        w = (((a3 + a2) + a1) + a0)                          # fp32 adds: fma(1, x, y) rounds x + y once
        dw = f32(3.0 * a3.astype(np.float64) + 2.0 * a2.astype(np.float64)) + a1
        assert np.all(w == 0) and np.all(dw == 0), (name, t, np.abs(w).max(), np.abs(dw).max())
        # fp16 rounds a2 and a3 by at most 2^-11 of their size, or half the subnormal spacing 2^-25
        raw, _ = pack_table_pairs(radial_table(spec, arrays, t, knots))
        e16 = 2.0 ** -25 + 2.0 ** -11 * (np.abs(a2) + np.abs(a3))
        d = np.abs(raw[-1] - p[('table', t)][-1])
        assert np.all(d <= 8 * np.concatenate([e16, e16], 1) + 2.0 ** -22 * np.abs(raw[-1])), (name, t, d.max())
        assert np.array_equal(raw[:-1], p[('table', t)][:-1])


@pytest.mark.parametrize('cid', ['R1', 'R5'])
def test_table_check_fails_with_r_on_between_knots(cid):
    """negative control: on the 2000-interval grid r_on of R1 (6.0 / 5.5) and R5 (5.3 / 4.8) is not a knot, and the
    interval that spans it breaks the dw/dr bound next to r_on"""
    from sevenn_b200.spec import build_spec
    meta, arrays = _model(cid)
    spec = build_spec(meta)
    h = spec.cutoff / 2000
    assert abs(spec.cutoff_on / h - round(spec.cutoff_on / h)) > 0.2
    for t in range(spec.n_layers):
        ew, edw, r = table_errors(spec, arrays, t, 2000)
        assert edw > DW_BOUND and abs(r - spec.cutoff_on) < h, (t, edw, r)


def test_knot_rule_puts_r_on_on_a_knot():
    from sevenn_b200.engine import default_table_knots
    from sevenn_b200.spec import build_spec
    want = {'R1': 2004, 'R2': 2000, 'R3': 2048, 'R4': 2048, 'R5': 2014, 'sevennet_0': 2000, 'sevennet_l3i5': 2048}
    for name, n in want.items():
        spec = build_spec(_model(name)[0])
        assert default_table_knots(spec) == n, name
        if spec.cutoff_fn == 'XPLOR':
            s = spec.cutoff_on * n / spec.cutoff
            assert abs(s - round(s)) < 1e-9, name
    # no count in [2000, 4096] puts r_on = 4.123456789 on a knot of [0, 5]: the closest one, the smallest on a tie
    spec = build_spec(dict(_model('R2')[0], cutoff_on=4.123456789))
    dist = [abs(0.8246913578 * n - round(0.8246913578 * n)) for n in range(2000, 4097)]
    assert min(dist) > 1e-9
    assert default_table_knots(spec) == 2000 + int(np.argmin(dist))


@pytest.mark.parametrize('cid', sorted(CONFIGS))
def test_converter_reads_every_radial_field(cid):
    from radial_models import radial_checkpoint
    c = CONFIGS[cid]
    meta, arrays = _model(cid)
    assert meta['cutoff'] == c['cutoff'] and meta['cutoff_fn'] == c['cutoff_fn']
    if c['cutoff_fn'] == 'XPLOR':
        assert meta['cutoff_on'] == c['cutoff_on']
    else:
        assert meta['poly_p'] == c['poly_p']
    assert meta['n_basis'] == c['n_basis'] and meta['radial_hidden'] == c['hidden']
    sd = radial_checkpoint(cid)['model_state_dict']
    assert np.array_equal(arrays['bessel_coeffs'], sd['edge_embedding.basis_function.coeffs'].numpy())
    nominal = np.arange(1, c['n_basis'] + 1) * np.pi / c['cutoff']
    assert 0 < np.abs(arrays['bessel_coeffs'] / nominal - 1).max() <= 0.05
    for j, (k, n) in enumerate(zip([c['n_basis']] + c['hidden'], c['hidden'])):
        assert arrays[f'0.mlp{j}'].shape == (k, n)


def test_export_flat_carries_the_knot_count(tmp_path):
    from sevenn_b200.engine import S7bModelDesc
    from sevenn_b200.export import export_flat
    meta, arrays = _model('R5')
    path = str(tmp_path / 'r5.s7b')
    export_flat(path, meta, arrays)
    with open(path, 'rb') as f:
        f.read(12)
        d = S7bModelDesc.from_buffer_copy(f.read(ctypes.sizeof(S7bModelDesc)))
    assert d.table_knots == 2014 and d.cutoff_fn == 0 and d.n_basis == 5
    assert d.cutoff == np.float32(5.3) and d.cutoff_on == np.float32(4.8)
    assert list(d.radial_hidden) == [50, 70]


@pytest.mark.parametrize('hidden', [(64,), (32, 32, 32)])
def test_radial_mlp_depth_other_than_two_refused(hidden, tmp_path):
    from sevenn_b200.engine import model_desc
    from sevenn_b200.export import export_flat
    from sevenn_b200.spec import build_spec
    meta, arrays = _radial_model('R3', hidden)
    assert meta['radial_hidden'] == list(hidden) and f'0.mlp{len(hidden)}' in arrays
    with pytest.raises(NotImplementedError, match='radial MLP must have two hidden layers'):
        model_desc(build_spec(meta), 2048)
    for radial in ('table', 'mlp'):
        with pytest.raises(NotImplementedError, match='radial MLP must have two hidden layers'):
            export_flat(str(tmp_path / 'm.s7b'), meta, arrays, radial=radial)
