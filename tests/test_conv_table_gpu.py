"""The table-mode convolution kernels (``TABLE = true``, what every production run uses), one layer at a time, against
an fp64 evaluation of the same operation on the engine's own inputs.

Per layer t the forward runs ``FWD_CONV_INTERIOR`` on random x[t] and is compared with
    mid[n] = sum over the edges e of row n of TP(x[src_e], Y_e, w_e)          (Oracle.tensor_product, fp64)
where Y is the engine's ``edge_Y``, and w_e is read from the host tables that were uploaded, as the kernel reads
them: the value table (``engine.value_table_read``) at r >= 0.6 A, the cubic table at the edge record's interval and
fraction below (``test_radial_cpu.device_table_read``; the record is checked against it).  The backward runs
``BWD_LAYER_A`` on random x[t], gate_in[t] and dh, reads the gout it used from ``mid``, and is compared with the
autograd of sum gout . conv with w from the cubic table: dx, and per l1 role dY (``dY_acc``) and
dE/dr = sum_p (dE/dw_p) dw_p/dr (``dEdr_acc``).  The reference has the kernels' tables and fp32 knot placement, so
what is left is fp32 rounding; a wrong table image, address or edge selection shows at full size.

Bound, per element: C_BOUND * 2^-24 * (n_sum + n_paths) * the same reference on |x|, |Y|, |w|, |gout| and |CG|
(|w| = the interpolation of |knot values|, sum |a_i| t^i for the cubic, and its dw/dr of |a_i|: near a zero of
dw/dr, and at the cutoff, its terms cancel).  n_sum is the length of the sum the element
is: the row length (mid), the in-degree (dx), the role's channels (dY, dE/dr); n_paths the paths of the layer (mid,
dx) or of the role.  u * n is the first-order bound of a sum of n rounded terms; C_BOUND = 8 covers the roundings
inside one term (two or three FMAs of the table read, the product w x Y CG and the short CG contraction) with a
factor of two to spare.  It was fixed before any comparison ran.

Models: for every (lmax_edge, lmax_node) in {1, 2, 3}^2 a synthetic model whose layers run group (lf, ln) (three
with every l1 role, two with l1 = 0 only) and group (lf, 0) (two), at widths chosen so that every l1 role of every
group meets a half-warp node (32 channels), a warp with one channel pair per lane (64), two pairs per lane (l1 = 0,
128 | mul) and a role split over several CTAs (96, 256), whose backward adds atomically; SevenNet-0 and
SevenNet-l3i5 add the width-specialised kernels of (2, 2), (2, 0), (3, 3) and (3, 0).  ``test_coverage`` states
and checks the map.
"""
import ctypes

import numpy as np
import pytest

import graphs
from helpers import model_weights
from synthetic_models import convert, layered, write_checkpoint
from test_radial_cpu import device_table_read

pytestmark = pytest.mark.gpu

C_BOUND = 8.0
U32 = 2.0 ** -24
R_MIN_VALUE = np.float32(0.6)          # conv_kernels.cuh kValueTableMinR
SHORT_R = (0.05, 0.2, 0.5, float(np.nextafter(np.float32(0.6), np.float32(0))))
RAGGED = (0, 1, 15, 16, 17, 31, 32, 33, 65)
SHORT_AT = (0, 15, 16, 31, 32, 33)      # short-edge positions in long rows (and the last edge)
N_GHOST = 16


# ---- models -----------------------------------------------------------------------------------------------------
def y_stride(ny):
    return (ny - 1 + 3) // 4 * 4          # common.cuh y_stride: Y_1 .. Y_{NY-1} padded to float4


def _irr(muls):
    return '+'.join(f'{m}x{l}e' for l, m in enumerate(muls))


W3 = (32, 64, 96)
# x widths of the two (lf, 0) layers per lmax_node, l = 0 .. ln (l = 3 at 32 comes from SevenNet-l3i5)
TAIL = {1: ([32, 32], [128, 64]), 2: ([64, 96, 32], [96, 32, 64]), 3: ([256, 64, 96, 64], [32, 96, 64, 96])}


def model_irreps(le, ln):
    """[x of layer 0, ..., out of layer 6]: layers 0 and 4 run (le, ln) with l1 = 0 only (x = scalars), 1, 2 and 5 with
    every l1 role, 3 and 6 run (le, 0)"""
    full = lambda k, w0: _irr([w0] + [W3[(l + k) % 3] for l in range(1, ln + 1)])
    c, e = TAIL[ln]
    return ['128x0e', full(0, 32), full(1, 64), _irr(c), '96x0e', full(2, 256), _irr(e), '32x0e']


SYNTH = [(le, ln) for le in (1, 2, 3) for ln in (1, 2, 3)]
CASES = [f'synth_{le}{ln}' for le, ln in SYNTH] + ['sevennet_0', 'sevennet_l3i5']


def lane_map(l1, mul, spec_group):
    """(LPN, NV, split, specialised) of a role's kernels (conv_dispatch.cuh)"""
    nv = 2 if (l1 == 0 and mul % 128 == 0) else 1
    lpn = 32 if mul % 64 == 0 else 16
    grid_y = mul // (2 * lpn * nv)
    kconv = (128, 64, 32, 32)
    return lpn, nv, grid_y > 1, spec_group and mul == kconv[l1]


SPEC_GROUPS = {(2, 2), (2, 0), (3, 3), (3, 0)}


def roles_of(spec):
    """[(t, lf, lo, l1, mul)] of every role with paths"""
    out = []
    for L in spec.layers:
        lo = len(L.out_muls) - 1
        for l1, mul in enumerate(L.x_muls):
            if any(p.l1 == l1 for p in L.paths):
                out.append((L.t, spec.lmax_filter, lo, l1, mul))
    return out


def _synthetic(le, ln, tmpdir):
    arch = layered(f'conv_table_{le}{ln}', le, ln, model_irreps(le, ln))
    path = write_checkpoint(f'{tmpdir}/conv_table_{le}{ln}.pth', arch, seed=10 * le + ln)
    return convert(path, arch)


def _weights(case, tmpdir):
    if case.startswith('synth_'):
        return _synthetic(int(case[6]), int(case[7]), tmpdir)
    return model_weights(case)


# ---- graphs ----------------------------------------------------------------------------------------------------
def _unit(rng):
    u = rng.normal(size=3)
    return u / np.linalg.norm(u)


def _axis(rng):
    u = np.zeros(3)
    u[rng.randint(3)] = rng.choice([-1.0, 1.0])
    return u


def table_graph(spec, knots, seed=0):
    """Rows (one per local node, edges in row order) with every length of RAGGED, short edges at SHORT_AT and last,
    rows of short edges only, adjacent node pairs with a short edge in one node only, edges at 0.6 A, on value and
    cubic knots, at r_on, at the fp32 cutoff and one ulp above, rows of only those beyond-the-cutoff edges, and the
    ragged / hub degree patterns of tests/graphs.py.  Radii that must arrive exactly lie on a coordinate axis
    (sqrt(r^2) = r in fp32).  Returns the arrays for set_graph and the row kinds."""
    from sevenn_b200.engine import forward_table_knots
    rng = np.random.RandomState(seed)
    cut = np.float32(spec.cutoff)
    kf = forward_table_knots(knots)
    long_r = lambda: min(float(rng.uniform(0.6, spec.cutoff)), float(np.nextafter(cut, np.float32(0))))
    rows, kinds = [], []

    def add(radii, kind, exact=()):
        # 0.05, 0.2 and 0.5 A need not arrive exactly: they keep random directions (all harmonics nonzero)
        rows.append([(float(r), i in exact and r not in SHORT_R[:3]) for i, r in enumerate(radii)])
        kinds.append(kind)

    def pad_even():
        if len(rows) % 2:
            add([long_r() for _ in range(3)], 'long')

    for n in RAGGED:
        add([long_r() for _ in range(n)], 'long')
    for j, n in enumerate(RAGGED[1:]):
        r = [long_r() for _ in range(n)]
        at = sorted({p for p in SHORT_AT if p < n} | {n - 1})
        for i, p in enumerate(at):
            r[p] = SHORT_R[(i + j) % len(SHORT_R)]
        add(r, 'mixed', exact=at)
    for j, n in enumerate((1, 4, 17, 33)):
        add([SHORT_R[(i + j) % len(SHORT_R)] for i in range(n)], 'short', exact=range(n))
    # LPN = 16 puts nodes 2k and 2k + 1 in one warp: exactly one of them has a short edge
    for n, p, first in ((9, 4, False), (20, 0, True), (33, 32, False), (17, 16, True)):
        pad_even()
        r = [long_r() for _ in range(n)]
        r[p] = SHORT_R[p % len(SHORT_R)]
        plain = [long_r() for _ in range(n)]
        if first:
            add(r, 'mixed', exact=[p])
            add(plain, 'long')
        else:
            add(plain, 'long')
            add(r, 'mixed', exact=[p])
    special = [0.6, float(np.float32(1000 * spec.cutoff / kf)), float(np.float32(1001 * spec.cutoff / kf)),
               float(np.float32((kf - 1) * spec.cutoff / kf)), float(np.float32(300 * spec.cutoff / knots)),
               float(np.float32((knots - 1) * spec.cutoff / knots))]
    if spec.cutoff_fn == 'XPLOR':
        special.append(spec.cutoff_on)
    beyond = [float(cut), float(np.nextafter(cut, np.float32(np.inf)))]
    mix = [long_r() for _ in range(12)] + special + beyond
    order = rng.permutation(len(mix))
    add([mix[i] for i in order], 'mixed', exact=[k for k, i in enumerate(order) if i >= 12])
    for r in special:
        add([r], 'long', exact=[0])
    add(beyond + beyond[::-1], 'beyond', exact=range(4))
    add(beyond[:1], 'beyond', exact=[0])
    for name, keep in (('ragged', 44), ('hub', 24)):      # one cycle of the ragged lengths; the hub next to empty rows
        for n in graphs.degrees(graphs.fixture(name, 'sevennet_0'))[:keep]:
            add([long_r() for _ in range(int(n))], 'long')

    n_local = len(rows)
    n_nodes = n_local + N_GHOST
    dst, src, vec, exact = [], [], [], []
    for i, row in enumerate(rows):
        for r, ex in row:
            dst.append(i)
            src.append(rng.randint(n_nodes))
            d = _axis(rng) if ex else _unit(rng)
            vec.append(d * np.float32(r) if ex else d * r)
            exact.append(np.float32(r) if ex else np.nan)
    return dict(species=rng.randint(spec.num_species, size=n_nodes), n_local=n_local, kinds=kinds,
                edge_index=np.array([dst, src], dtype=np.int64), edge_vec=np.array(vec, dtype=np.float32),
                exact=np.array(exact, dtype=np.float32))


# ---- the engine side -------------------------------------------------------------------------------------------
def _raw(e, name, layer, numel):
    """torch view of `numel` floats of an engine buffer (its capacity may exceed what s7b_engine_buffer reports)"""
    import torch
    from sevenn_b200.engine import _DevView
    n = ctypes.c_size_t()
    ptr = e.lib.s7b_engine_buffer(e._h, name.encode(), int(layer), ctypes.byref(n))
    assert ptr, (name, layer)
    return torch.as_tensor(_DevView(ptr, (numel,), '<f4'), device=e.device)


class Case:
    """An engine in table mode on table_graph, the host tables it was given, and the fp64 reference pieces"""

    def __init__(self, meta, arrays, seed=0):
        import torch
        from oracle.oracle import Oracle
        from sevenn_b200 import engine as eng
        self.torch, self.eng = torch, eng
        spec = eng.build_spec(meta)
        self.knots = eng.default_table_knots(spec)
        self.params = eng.prepare_params(spec, arrays, 'table', self.knots)
        prepare, eng.prepare_params = eng.prepare_params, lambda *a: self.params     # the engine uploads these
        try:
            self.e = eng.B200Engine(meta, arrays, radial='table')
        finally:
            eng.prepare_params = prepare
        self.spec = self.e.spec
        assert self.e.knots == self.knots
        self._cubic = {}
        self.dev = torch.device('cuda')
        self.o = Oracle(meta, arrays, dtype=torch.float64, device='cuda')
        self.oa = Oracle.__new__(Oracle)
        self.oa.__dict__.update(self.o.__dict__)
        self.oa.cg = {k: v.abs() for k, v in self.o.cg.items()}
        g = table_graph(self.spec, self.knots, seed)
        self.g = g
        self.n_local, self.n_nodes = g['n_local'], len(g['species'])
        self.e.set_graph(g['species'], g['edge_index'], g['edge_vec'], n_local=self.n_local)
        self.E = g['edge_index'].shape[1]
        self.dst, self.src = g['edge_index']
        self.deg = np.bincount(self.dst, minlength=self.n_local)
        self.indeg = np.bincount(self.src, minlength=self.n_nodes)
        self.e.run_stage(eng.STAGE_FWD_BEGIN)
        torch.cuda.synchronize()
        ny = self.spec.n_sh
        Y = self.e.buffer('edge_Y').view(self.E, y_stride(ny))[:, :ny - 1].double()
        self.Y = torch.cat([torch.ones(self.E, 1, dtype=torch.float64, device=self.dev), Y], 1)
        self.r = self.e.buffer('edge_len').cpu().numpy()
        self.rec = self.e.buffer('edge_rec', dtype='i4').view(self.E, 4).cpu().numpy()
        self.short = self.r < R_MIN_VALUE

    def check_inputs(self):
        """the engine's edge lengths and records are the ones the reference assumes"""
        g = self.g
        ex = ~np.isnan(g['exact'])
        assert np.array_equal(self.r[ex], g['exact'][ex])
        assert np.array_equal(self.rec[:, 0], self.src) and np.array_equal(self.rec[:, 3].view(np.float32), self.r)
        inv_h = np.float32(np.float32(self.knots) / np.float32(self.spec.cutoff))
        s = self.r * inv_h
        tk = np.clip(s.astype(np.int64), 0, self.knots - 1)
        tt = np.clip(s - tk.astype(np.float32), np.float32(0), np.float32(1))
        assert np.array_equal(self.rec[:, 1], tk) and np.array_equal(self.rec[:, 2].view(np.float32), tt)

    # -- weights as the kernels read them (float64 [E, W]) and their absolute-value counterparts
    def cubic(self, t):
        """w, dw/dr and the same reads of |coefficients| (w and dw/dr as sums of absolute terms)"""
        if t not in self._cubic:
            t01, t23 = self.params[('table', t)], self.params[('table23', t)]
            w, dw = device_table_read(t01, t23, self.knots, self.spec.cutoff, self.r)
            wa, dwa = device_table_read(np.abs(t01), np.abs(t23.view(np.float16)).view(np.float32), self.knots,
                                        self.spec.cutoff, self.r)
            self._cubic[t] = w, dw, wa, dwa
        return self._cubic[t]

    def forward_weights(self, t, short_from_value=False):
        from sevenn_b200.engine import value_table_read
        tab = self.params[('table_fwd', t)]
        wv = value_table_read(tab, self.spec.cutoff, self.r)
        wva = value_table_read(np.abs(tab), self.spec.cutoff, self.r)
        wc, _, wca, _ = self.cubic(t)
        s = self.short[:, None] & (not short_from_value)
        return np.where(s, wc, wv), np.where(s, wca, wva)

    def t64(self, a):
        return self.torch.as_tensor(np.asarray(a, dtype=np.float64), device=self.dev)

    def conv(self, o, L, x, w, Y=None):
        """fp64 [n_local, dim_mid] e3nn layout: sum over each row of TP(x[src], Y, w)"""
        torch = self.torch
        msg = o.tensor_product(L, x[torch.as_tensor(self.src, device=self.dev)], self.Y if Y is None else Y, w)
        out = torch.zeros(self.n_local, L.dim_mid, dtype=torch.float64, device=self.dev)
        return out.index_add_(0, torch.as_tensor(self.dst, device=self.dev), msg)


def _mulir(cm, perm):
    out = np.empty_like(cm)
    out[:, perm] = cm
    return out


def ratio(got, want, scale, n):
    """max of |got - want| / bound, bound = C_BOUND u n scale; elements with bound 0 must match exactly"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    bound = C_BOUND * U32 * np.asarray(n, np.float64) * np.asarray(scale, np.float64)
    err = np.abs(got - want)
    zero = bound == 0
    assert not np.any(err[zero] != 0), 'nonzero where the reference is exactly 0'
    return float((err[~zero] / bound[~zero]).max()) if np.any(~zero) else 0.0


def forward_layer(c, t, rng, short_from_value=False, table_fwd=None):
    """run FWD_CONV_INTERIOR on random x[t]; returns (engine mid cm, reference cm, abs reference cm, n)"""
    from sevenn_b200.spec import perm_cm_from_mulir
    torch, eng, e = c.torch, c.eng, c.e
    L = c.spec.layers[t]
    e.run_stage(eng.STAGE_FWD_BEGIN)
    x = rng.normal(size=(c.n_nodes, L.dim_x)).astype(np.float32)
    e.buffer('x', t).copy_(torch.from_numpy(x.ravel()))
    e.buffer('mid', t).fill_(float('nan'))                 # a row the kernels leave unwritten fails the comparison
    e.set_interior(c.n_local)
    e.run_stage(eng.STAGE_FWD_CONV_INTERIOR, t)
    torch.cuda.synchronize()
    mid = e.buffer('mid', t).view(c.n_local, L.dim_mid).cpu().numpy()
    w, wa = c.forward_weights(t, short_from_value)
    xm = _mulir(x, perm_cm_from_mulir(list(L.x_muls)))
    pm = L.mid_perm_cm_from_mulir()
    ref = c.conv(c.o, L, c.t64(xm), c.t64(w)).cpu().numpy()[:, pm]
    ref_a = c.conv(c.oa, L, c.t64(np.abs(xm)), c.t64(wa), c.Y.abs()).cpu().numpy()[:, pm]
    n = (c.deg + len(L.paths))[:, None]
    return mid, ref, ref_a, n


def backward_layer(c, t, rng, stages=None, interior=None):
    """BWD_LAYER_A (or the given split stages) on random x[t], gate_in[t], dh; returns engine and reference values:
    {'dx': (got, ref, abs, n) or None, 'dY': [per l1], 'dEdr': [per l1]} and the dx sentinel check for t = 0"""
    import torch
    from sevenn_b200.spec import irreps_dim, perm_cm_from_mulir
    eng, e = c.eng, c.e
    L = c.spec.layers[t]
    e.run_stage(eng.STAGE_FWD_BEGIN)
    x = rng.normal(size=(c.n_nodes, L.dim_x)).astype(np.float32)
    e.buffer('x', t).copy_(torch.from_numpy(x.ravel()))
    e.buffer('gate_in', t).copy_(torch.from_numpy(rng.normal(size=c.n_local * L.dim_gate).astype(np.float32)))
    dim_h = irreps_dim(list(L.out_muls))
    _raw(e, 'dh', t, c.n_local * dim_h).copy_(torch.from_numpy(rng.normal(size=c.n_local * dim_h).astype(np.float32)))
    dx_view = _raw(e, 'dx', t, c.n_nodes * L.dim_x)
    if t == 0:
        dx_view.fill_(7.0)
    e.set_interior(c.n_local if interior is None else interior)
    for st in stages or (eng.STAGE_BWD_LAYER_A,):
        e.run_stage(st, t)
    torch.cuda.synchronize()
    gout = e.buffer('mid', t).view(c.n_local, L.dim_mid).cpu().numpy()
    dx = dx_view.view(c.n_nodes, L.dim_x).cpu().numpy()
    ny = c.spec.n_sh
    dY = [e.buffer('dY_acc', l1).view(c.E, y_stride(ny))[:, :ny - 1].cpu().numpy() for l1 in range(len(L.x_muls))]
    dEdr = [e.buffer('dEdr_acc', l1).cpu().numpy() for l1 in range(len(L.x_muls))]
    # the parts of the l1 roles this layer does not have (up to the widest layer) stay as FWD_BEGIN left them
    for l1 in range(len(L.x_muls), max(len(M.x_muls) for M in c.spec.layers)):
        assert not e.buffer('dY_acc', l1).any() and not e.buffer('dEdr_acc', l1).any(), (t, l1)

    px = perm_cm_from_mulir(list(L.x_muls))
    xm, gm = _mulir(x, px), _mulir(gout, L.mid_perm_cm_from_mulir())
    w, dw, wa, dwa = c.cubic(t)
    out = dict(dY=[], dEdr=[], dx=None, dx_untouched=None, terms=[], raw=(dY, dEdr))
    gx, gxa = np.zeros_like(xm, dtype=np.float64), np.zeros_like(xm, dtype=np.float64)
    for l1 in range(len(L.x_muls)):
        cols = np.zeros(L.weight_numel)
        paths = [p for p in L.paths if p.l1 == l1]
        for p in paths:
            cols[p.w_off:p.w_off + p.mul] = 1.0
        if not paths:
            out['dY'].append((dY[l1], np.zeros_like(dY[l1]), np.zeros_like(dY[l1]), 1))
            out['dEdr'].append((dEdr[l1], np.zeros_like(dEdr[l1]), np.zeros_like(dEdr[l1]), 1))
            out['terms'].append(None)
            continue
        res = []
        for o, xs, ws, Ys, gs in ((c.o, xm, w, c.Y, gm), (c.oa, np.abs(xm), wa, c.Y.abs(), np.abs(gm))):
            xt = c.t64(xs).requires_grad_(True)
            wt = c.t64(ws * cols).requires_grad_(True)
            Yt = Ys.clone().requires_grad_(True)
            (c.conv(o, L, xt, wt, Yt) * c.t64(gs)).sum().backward()
            res.append((xt.grad.cpu().numpy(), Yt.grad[:, 1:].cpu().numpy(), wt.grad.cpu().numpy()))
        (gx1, gY, gw), (gxa1, gYa, gwa) = res
        gx += gx1
        gxa += gxa1
        n_role = L.x_muls[l1] + len(paths)
        out['dY'].append((dY[l1], gY, gYa, n_role))
        # dE/dw of the other roles' columns is not zero (only their w is): keep this role's
        terms = gw * cols * dw
        out['dEdr'].append((dEdr[l1], terms.sum(1), (np.abs(gwa) * cols * dwa).sum(1), n_role))
        out['terms'].append(terms)
    if t > 0:
        out['dx'] = (dx, gx[:, px], gxa[:, px], (c.indeg + len(L.paths))[:, None])
    else:
        out['dx_untouched'] = bool(np.all(dx == 7.0))
    return out


def backward_ratios(res):
    r = {}
    if res['dx'] is not None:
        r['dx'] = ratio(*res['dx'])
    for l1, (got, ref, ra, n) in enumerate(res['dY']):
        r[f'dY{l1}'] = ratio(got, ref, ra, n)
    for l1, (got, ref, ra, n) in enumerate(res['dEdr']):
        r[f'dEdr{l1}'] = ratio(got, ref, ra, n)
    return r


@pytest.fixture(scope='module')
def cases(tmp_path_factory):
    """case name -> Case, built once per module and released (engines, tables, fp64 oracles) at its end"""
    import torch
    d = str(tmp_path_factory.mktemp('conv_table_ckpt'))
    made = {}

    def get(case):
        if case not in made:
            made[case] = Case(*_weights(case, d))
        return made[case]
    yield get
    made.clear()
    torch.cuda.empty_cache()


# ---- the comparisons ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('case', CASES)
def test_conv_table_layers(case, cases):
    c = cases(case)
    c.check_inputs()
    # dY_acc / dEdr_acc: part l1 for 0 <= l1 < the widest x, part 0 for -1, nothing else
    n_part = max(len(L.x_muls) for L in c.spec.layers)
    for name in ('dY_acc', 'dEdr_acc'):
        ptr = lambda layer: c.e.lib.s7b_engine_buffer(c.e._h, name.encode(), layer, None)
        assert ptr(-1) == ptr(0) and ptr(n_part - 1) and not ptr(n_part) and not ptr(-2), name
    rng = np.random.RandomState(sum(map(ord, case)))
    worst = {}
    for L in c.spec.layers:
        t = L.t
        mid, ref, ref_a, n = forward_layer(c, t, rng)
        worst[f'{t} mid'] = ratio(mid, ref, ref_a, n)
        # rows whose edges all sit at or beyond the cutoff add exactly 0
        beyond = [i for i, k in enumerate(c.g['kinds']) if k == 'beyond']
        assert np.all(mid[beyond] == 0.0)
        res = backward_layer(c, t, rng)
        if t == 0:
            assert res['dx_untouched'], 'the first layer runs without dx and must leave it untouched'
        # ... and edges at or beyond the cutoff add exactly 0 to dE/dY and dE/dr (engine.close_table_at_cutoff)
        far = c.r >= np.float32(c.spec.cutoff)
        assert far.sum() >= 4
        for dY, dEdr in zip(*res['raw']):
            assert not dY[far].any() and not dEdr[far].any(), t
        for k, v in backward_ratios(res).items():
            worst[f'{t} {k}'] = v
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    print(f'\n{case}: largest error / bound {max(worst.values()):.3g} ({max(worst, key=worst.get)})')
    assert not bad, (case, bad)


SPLIT_CASE = 'synth_32'


def test_conv_table_split_stages(cases):
    """FWD_CONV_INTERIOR + FWD_LAYER_A2 give mid bit for bit as one pass (every row written: mid is filled with NaN
    first); BWD_LAYER_A1 + A2 stay within the bound"""
    c = cases(SPLIT_CASE)
    eng, torch, e = c.eng, c.torch, c.e
    t = 2
    L = c.spec.layers[t]
    rng = np.random.RandomState(3)
    x = rng.normal(size=(c.n_nodes, L.dim_x)).astype(np.float32)

    def fwd(k):
        e.run_stage(eng.STAGE_FWD_BEGIN)
        e.buffer('x', t).copy_(torch.from_numpy(x.ravel()))
        e.buffer('mid', t).fill_(float('nan'))
        e.set_interior(k)
        e.run_stage(eng.STAGE_FWD_CONV_INTERIOR, t)
        if k < c.n_local:
            e.run_stage(eng.STAGE_FWD_LAYER_A2, t)
        torch.cuda.synchronize()
        return e.buffer('mid', t).view(c.n_local, L.dim_mid).cpu().numpy().copy()

    one = fwd(c.n_local)
    for k in (0, 1, c.n_local // 2 | 1):
        assert np.array_equal(fwd(k), one), k
    for k in (0, 1, c.n_local // 2 | 1, c.n_local):
        res = backward_layer(c, t, np.random.RandomState(k), stages=(eng.STAGE_BWD_LAYER_A1, eng.STAGE_BWD_LAYER_A2),
                             interior=k)
        r = backward_ratios(res)
        assert max(r.values()) <= 1.0, (k, r)


# ---- negative controls: each perturbation must break the comparison it targets -------------------------------
NEG_CASE = 'synth_21'


def _single_edge(c):
    """an edge alone in its row, long (the forward reads the value table) and inside 0.9 cutoff"""
    single = [i for i, k in enumerate(c.g['kinds']) if k == 'long' and c.deg[i] == 1]
    e_idx = np.searchsorted(c.dst, single)
    e_idx = e_idx[c.r[e_idx] < np.float32(c.spec.cutoff) * 0.9]
    return int(e_idx[0])


def test_negative_control_value_knot(cases):
    """one interior knot of one channel of one path of one role of table_fwd scaled by 1 + 1e-4"""
    c = cases(NEG_CASE)
    t = 1
    L = c.spec.layers[t]
    ei = _single_edge(c)
    kf = c.params[('table_fwd', t)].shape[0] - 1
    inv_h = np.float32(np.float32(kf) / np.float32(c.spec.cutoff))
    s = c.r[ei] * inv_h
    k = int(s)
    k = k if s - k < 0.5 else k + 1                     # the knot with the larger interpolation weight
    # path (1, 0, 1): its message is w x CG with Y_0 = 1, no cancelling sum; the channel whose weight at this edge
    # is most nearly its knot value at k (not a near-zero mix of two knots of opposite sign)
    p = next(q for q in L.paths if q.l1 == 1 and q.l2 == 0)
    tab = c.params[('table_fwd', t)].copy()
    frac = 1.0 - abs(float(s) - k)
    cols = np.arange(p.w_off, p.w_off + p.mul)
    wa = np.abs(tab[int(s), cols]) * (1 - (s - int(s))) + np.abs(tab[int(s) + 1, cols]) * (s - int(s))
    col = int(cols[np.argmax(frac * np.abs(tab[k, cols]) / np.maximum(wa, 1e-30))])
    tab[k, col] *= np.float32(1 + 1e-4)
    _upload(c, 'table_fwd', t, tab)
    try:
        mid, ref, ref_a, n = forward_layer(c, t, np.random.RandomState(1))
    finally:
        _upload(c, 'table_fwd', t, c.params[('table_fwd', t)])
    assert ratio(mid, ref, ref_a, n) > 1.0


def test_negative_control_cubic_slope(cases):
    """the slope a1 of one cubic knot of one channel scaled by 1 + 1e-4: the dE/dr comparison must fail"""
    c = cases(NEG_CASE)
    t = 3                                              # group (2, 0), x = 32x0e+32x1e: role l1 = 0 has one path
    L = c.spec.layers[t]
    rng = np.random.RandomState(5)
    state = rng.get_state()
    res = backward_layer(c, t, rng)
    assert max(backward_ratios(res).values()) <= 1.0
    # the (edge, channel) whose term is the largest share of the bound on its edge's dE/dr in role 0
    p = [q for q in L.paths if q.l1 == 0][0]
    _, _, scale, _ = res['dEdr'][0]
    share = np.abs(res['terms'][0][:, p.w_off:p.w_off + p.mul]) / np.maximum(scale, 1e-300)[:, None]
    ei, u = np.unravel_index(np.argmax(share), share.shape)
    tk = int(c.rec[ei, 1])
    col = p.w_off + u
    t01 = c.params[('table', t)].copy()                 # [K, W/2, 4] {a0e, a0o, a1e, a1o}
    t01[tk, col // 2, 2 + col % 2] *= np.float32(1 + 1e-4)
    _upload(c, 'table', t, t01)
    try:
        rng.set_state(state)
        res2 = backward_layer(c, t, rng)
    finally:
        _upload(c, 'table', t, c.params[('table', t)])
    got, ref, ra, n = res2['dEdr'][0]
    assert ratio(got, ref, ra, n) > 1.0


def test_negative_control_short_edges_from_value_table(cases):
    """a reference that reads the short edges from the value table does not match: they went through the cubic pass"""
    c = cases(NEG_CASE)
    worst = 0.0
    for t in range(c.spec.n_layers):
        mid, ref, ref_a, n = forward_layer(c, t, np.random.RandomState(t))
        assert ratio(mid, ref, ref_a, n) <= 1.0
        _, ref_v, ref_va, _ = forward_layer(c, t, np.random.RandomState(t), short_from_value=True)
        worst = max(worst, ratio(mid, ref_v, ref_a, n))
    assert worst > 1.0


def _upload(c, name, t, arr):
    arr = np.ascontiguousarray(arr, dtype=np.float32)
    c.eng.check(c.e.lib.s7b_engine_set_param(c.e._h, name.encode(), t, arr.ctypes.data, arr.size))

# ---- what ran --------------------------------------------------------------------------------------------------
def _meta(case):
    """the meta of a case (for a synthetic model, enough of it to build its spec)"""
    from sevenn_b200.spec import parse_even_irreps
    if case.startswith('synth_'):
        le, ln = int(case[6]), int(case[7])
        irreps = model_irreps(le, ln)
        return dict(name=case, cutoff=5.0, cutoff_fn='poly_cut', n_basis=8, lmax_filter=le, num_species=1,
                    type_map={'1': 0}, radial_hidden=[64, 64], irreps_per_layer=irreps,
                    readout_hidden=parse_even_irreps(irreps[-1])[0] // 2)
    return model_weights(case)[0]


def n_layers():
    from sevenn_b200.spec import build_spec
    return sum(build_spec(_meta(case)).n_layers for case in CASES)


def coverage():
    """{(lf, lo): {l1: {(mul, LPN, NV, split, specialised)}}} of every case, from the models' irreps and the
    dispatch rule of conv_dispatch.cuh"""
    from sevenn_b200.spec import build_spec
    cov = {}
    for case in CASES:
        for t, lf, lo, l1, mul in roles_of(build_spec(_meta(case))):
            m = lane_map(l1, mul, (lf, lo) in SPEC_GROUPS)
            cov.setdefault((lf, lo), {}).setdefault(l1, set()).add((mul,) + m)
    return cov


def test_coverage():
    cov = coverage()
    assert sorted(cov) == [(lf, lo) for lf in (1, 2, 3) for lo in range(4)]
    n_roles = n_maps = 0
    lines = []
    for g in sorted(cov):
        for l1, maps in sorted(cov[g].items()):
            cats = {(lpn, nv, split) for _, lpn, nv, split, _ in maps}
            need = [lambda c: (16, 1, False) in c, lambda c: (32, 1, False) in c, lambda c: any(s for _, _, s in c)]
            if l1 == 0:
                need.append(lambda c: any(nv == 2 for _, nv, _ in c))
            assert all(f(cats) for f in need), (g, l1, sorted(maps))
            n_roles += 1
            n_maps += len(maps)
            lines.append(f'  group {g} l1 = {l1}: ' + ', '.join(
                f'{mul} (LPN {lpn}, NV {nv}{", split" if s else ""}{", specialised" if sp else ""})'
                for mul, lpn, nv, s, sp in sorted(maps)))
    print(f'\n{n_layers()} layers in {len(CASES)} models, {len(cov)} groups, {n_roles} l1 roles, '
          f'{n_maps} (role, width, LPN, NV) mappings, table = true:\n' + '\n'.join(lines))
