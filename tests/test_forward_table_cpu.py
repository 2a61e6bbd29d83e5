"""CPU checks of the forward convolution's radial value table (engine.py ``radial_value_table``): knot values on a
grid three times finer than the backward's cubic table, read the way ``conv_fwd`` reads it (linear interpolation,
``value_table_read``), against the fp64 radial MLP for every layer of both shipped models and of the radial shapes
of tests/radial_models.py, including that the error averages to zero over r; the knot rule (XPLOR's r_on on a knot,
size no larger than the cubic table but one row); the parameter ``prepare_params`` hands to the engine."""
import functools
import tempfile

import numpy as np
import pytest

from helpers import model_weights
from radial_models import CONFIGS, convert_radial, write_radial_checkpoint

# Measured (tools/forward_table_error.py): see the numbers there and in DESIGN.md section 3.  The cubic table's w
# error is 4.3e-8 of max |w|: linear interpolation on three times the knots trades ~20x that for a third fewer
# bytes per weight; the forces still come from the cubic table.
W_BOUND_GLOBAL = 2.5e-6
W_BOUND_LOCAL = 2e-5
R_ON_OFF_GRID = 4.123456789     # on no knot of any count the knot rule can pick for R2's [0, 5] (test_radial_cpu)


@functools.lru_cache(maxsize=None)
def _model(name):
    if name not in CONFIGS:
        return model_weights(name)
    d = tempfile.mkdtemp(prefix='fwd_table_ckpt_')
    return convert_radial(write_radial_checkpoint(f'{d}/{name}.pth', name), name)


def dense_radii(spec, fknots):
    """fp32 radii in [0.2, rc): every interval of the value grid at several fractions, r_on +- {1e-6, h/3}, rc - 1e-6"""
    h = spec.cutoff / fknots
    frac = np.array([0.0, 0.1, 0.3, 0.5, 0.7, 0.9, 0.999])
    r = ((np.arange(fknots)[:, None] + frac) * h).ravel()
    extra = [spec.cutoff - 1e-6]
    if spec.cutoff_fn == 'XPLOR':
        extra += [spec.cutoff_on + d for d in (-h / 3, -1e-6, 1e-6, h / 3)]
    r = np.concatenate([r, extra])
    r = r[(r >= 0.2) & (r <= spec.cutoff - 1e-6)]
    return np.unique(r.astype(np.float32))


def forward_table_errors(spec, arrays, t, tab, seed=0):
    """(max, rms) of |w - w_fp64| / max |w| at 3000 random fp32 radii in [1.5, rc), and (max, r of the max) of
    |w - w_fp64| over the local scale (max over channels within 0.1 A, floored at 0.1 of the global max) at
    ``dense_radii``, of layer t's value table ``tab`` read as conv_fwd reads it"""
    from scipy.ndimage import maximum_filter1d
    from sevenn_b200.engine import radial_weights, value_table_read
    r = np.random.default_rng(seed).uniform(1.5, spec.cutoff, 3000).astype(np.float32)
    f, _ = radial_weights(spec, arrays, t, r.astype(np.float64))
    err = value_table_read(tab, spec.cutoff, r) - f
    scale = np.abs(f).max()
    step = 0.002
    rg = np.arange(0.0, spec.cutoff + step / 2, step)
    fg, _ = radial_weights(spec, arrays, t, np.maximum(rg, 1e-9))
    sw = maximum_filter1d(np.abs(fg).max(1), 2 * int(round(0.1 / step)) + 1)
    sw = np.maximum(sw, 0.1 * sw.max())
    r32 = dense_radii(spec, tab.shape[0] - 1)
    worst, at = 0.0, 0.0
    for i in range(0, len(r32), 4096):
        rc = r32[i:i + 4096]
        fc, _ = radial_weights(spec, arrays, t, rc.astype(np.float64))
        e = np.abs(value_table_read(tab, spec.cutoff, rc) - fc).max(1) / sw[np.rint(rc.astype(np.float64) / step).astype(int)]
        j = int(np.argmax(e))
        if e[j] > worst:
            worst, at = float(e[j]), float(rc[j])
    return float(np.abs(err).max() / scale), float(np.sqrt(np.mean(err ** 2)) / scale), worst, at


MODELS = sorted(CONFIGS) + ['sevennet_0', 'sevennet_l3i5']


@pytest.mark.parametrize('name', MODELS + ['R2@r_on_off_grid'])
def test_forward_table_matches_radial_mlp(name):
    from sevenn_b200.engine import default_table_knots, forward_table_knots, radial_value_table
    from sevenn_b200.spec import build_spec
    base, _, variant = name.partition('@')
    meta, arrays = _model(base)
    if variant:
        meta = dict(meta, cutoff_on=R_ON_OFF_GRID)
    spec = build_spec(meta)
    fknots = forward_table_knots(default_table_knots(spec))
    for t in range(spec.n_layers):
        tab = radial_value_table(spec, arrays, t, fknots)
        e_max, e_rms, e_loc, r = forward_table_errors(spec, arrays, t, tab)
        assert e_max < W_BOUND_GLOBAL and e_rms < e_max and e_loc < W_BOUND_LOCAL, (name, fknots, t, e_max, e_loc, r)


def test_forward_table_read_is_exact_at_the_knots_and_clamps_at_the_cutoff():
    from sevenn_b200.engine import value_table_read
    tab = np.random.default_rng(1).standard_normal((301, 8)).astype(np.float32)
    rc = 5.0
    k = np.array([0, 1, 150, 299, 300])
    r = (k * rc / 300).astype(np.float32)
    # exact at the knots (fp32 r lands within one rounding of the knot: the interpolation weight is ~1e-5 or less)
    assert np.allclose(value_table_read(tab, rc, r), tab[k], rtol=0, atol=2e-5 * np.abs(tab).max())
    # at and beyond the cutoff, and at r = 0: the end knots, no extrapolation
    far = value_table_read(tab, rc, np.array([rc, rc + 0.3, 100.0], np.float32))
    assert np.array_equal(far, np.repeat(tab[300:301].astype(np.float64), 3, 0))
    assert np.array_equal(value_table_read(tab, rc, np.zeros(1, np.float32)), tab[:1].astype(np.float64))


@pytest.mark.parametrize('name', MODELS + ['R2@r_on_off_grid'])
def test_forward_knot_rule(name):
    """three value intervals per cubic interval: r_on stays on a knot when the cubic grid has it there (and comes
    three times closer in units of an interval when it does not); the value table is at most one 4-byte row per
    weight larger than the cubic table (12 B per weight and interval)"""
    from sevenn_b200.engine import default_table_knots, forward_table_knots
    from sevenn_b200.spec import build_spec
    base, _, variant = name.partition('@')
    meta = dict(_model(base)[0], **({'cutoff_on': R_ON_OFF_GRID} if variant else {}))
    spec = build_spec(meta)
    K = default_table_knots(spec)
    Kf = forward_table_knots(K)
    assert Kf == 3 * K
    for L in spec.layers:
        W = L.weight_numel
        assert (Kf + 1) * W * 4 <= K * W * 12 + W * 4
    if spec.cutoff_fn == 'XPLOR':
        s, sf = spec.cutoff_on * K / spec.cutoff, spec.cutoff_on * Kf / spec.cutoff
        assert abs(sf - round(sf)) <= 3 * abs(s - round(s)) + 1e-9
        if not variant:
            assert abs(sf - round(sf)) < 1e-8, name


@pytest.mark.parametrize('name', ['sevennet_0', 'R5'])
def test_prepare_params_carries_the_value_table(name):
    from sevenn_b200.engine import default_table_knots, prepare_params, radial_weights
    from sevenn_b200.spec import build_spec
    meta, arrays = _model(name)
    spec = build_spec(meta)
    K = default_table_knots(spec)
    P = prepare_params(spec, arrays, 'table', K)
    assert not any(n == 'table_fwd' for n, _ in prepare_params(spec, arrays, 'mlp', 0))
    for t in range(spec.n_layers):
        W = P[('table', t)].shape[1] * 2
        tab = P[('table_fwd', t)]
        assert tab.dtype == np.float32 and tab.shape == (3 * K + 1, W)
        # knot values w_k - (w_k+1 - 2 w_k + w_k-1) / 12, the last one w(cutoff) = 0
        k = np.array([1, K, 3 * K - 1])
        h = spec.cutoff / (3 * K)
        f, _ = radial_weights(spec, arrays, t, np.concatenate([k - 1, k, k + 1]) * h)
        fm, f0, fp = np.split(f, 3)
        assert np.array_equal(tab[k], (f0 - (fp - 2 * f0 + fm) / 12).astype(np.float32))
        assert (tab[3 * K] == 0).all()        # exactly: conv_fwd sends the edges it leaves to the cubic table here


@pytest.mark.parametrize('name', ['sevennet_0', 'R1'])
def test_forward_table_error_averages_to_zero(name):
    """the knot values cancel linear interpolation's one-signed error: the mean error over r of every channel (what
    a sum over many edges sees) is below 1e-8 of max |w|, where plain interpolation of w leaves up to ~5e-8"""
    from sevenn_b200.engine import default_table_knots, forward_table_knots, radial_value_table, radial_weights, value_table_read
    from sevenn_b200.spec import build_spec
    meta, arrays = _model(name)
    spec = build_spec(meta)
    fknots = forward_table_knots(default_table_knots(spec))
    r = np.random.default_rng(2).uniform(1.5, spec.cutoff, 100000).astype(np.float32)
    for t in range(spec.n_layers):
        f, _ = radial_weights(spec, arrays, t, r.astype(np.float64))
        bias = (value_table_read(radial_value_table(spec, arrays, t, fknots), spec.cutoff, r) - f).mean(0)
        assert np.abs(bias).max() < 1e-8 * np.abs(f).max(), (name, t, np.abs(bias).max() / np.abs(f).max())
