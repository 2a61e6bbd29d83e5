"""Second order of the operator-level drop-in: B200Convolution differentiated twice (forces inside a loss,
Hessian-vector products) against the oracle's fp64 tensor product + index_add under torch autograd.

Per layer: first-order gradients (gx, gsh, gw) are taken with create_graph=True, contracted with random
(a_x, a_sh, a_w), and the contraction is differentiated to x, sh, w and grad_out.  The tangent cases are each of
a_x, a_sh, a_w alone (the other two incoming gradients are then None) and all three.  Layers: SevenNet-0 t = 0, 1,
4, SevenNet-l3i5 t = 2, 4, and for every (lmax_filter, lmax_node) in {1, 2, 3}^2 a synthetic model whose layers 0
and 1 run group (lf, ln) (l1 = 0 only at 128 channels, then every role at 64 / 96 / 32 / 64 channels: two pairs per
lane, one pair, half warps, a role split over three CTAs) and layer 2 group (lf, 0) (256 / 32 / 64 / 96): all twelve
groups of the runtime-width kernels.
"""
import numpy as np
import pytest

from helpers import model_weights, oracle
from synthetic_models import convert, layered, write_checkpoint

pytestmark = pytest.mark.gpu

TANGENTS = {'x': (1, 0, 0), 'sh': (0, 1, 0), 'w': (0, 0, 1), 'all': (1, 1, 1)}


def _irr(muls):
    return '+'.join(f'{m}x{l}e' for l, m in enumerate(muls))


_SYNTH = {}


def _synthetic_oracle(le, ln, tmpdir):
    import torch
    from oracle.oracle import Oracle
    key = (le, ln)
    if key not in _SYNTH:
        irreps = ['128x0e', _irr([64, 96, 32, 64][:ln + 1]), _irr([256, 32, 64, 96][:ln + 1]), '64x0e']
        arch = layered(f'conv_dbwd_{le}{ln}', le, ln, irreps)
        meta, arrays = convert(write_checkpoint(f'{tmpdir}/conv_dbwd_{le}{ln}.pth', arch, seed=7 * le + ln), arch)
        _SYNTH[key] = Oracle(meta, arrays, dtype=torch.float64)
    return _SYNTH[key]


def _conv_of(o, L):
    from sevenn_b200.conv_op import B200Convolution
    mid = '+'.join(f'{p.mul}x{p.l3}e' for p in L.paths)
    inst = [(p.l1, p.l2, p.slot, 'uvu', True) for p in L.paths]
    return B200Convolution(_irr(L.x_muls), _irr([1] * (o.spec.lmax_filter + 1)), mid, inst).cuda()


def _second_order(conv_fn, tensors, a, tan):
    """d/d(x, sh, w, gout) of sum_i a_i . (first-order gradient i), the gradients taken with create_graph=True;
    `tan` selects which of the three first-order gradients enter the contraction"""
    import torch
    x, sh, w, gout = tensors
    out = conv_fn(x, sh, w)
    g1 = torch.autograd.grad(out, (x, sh, w), grad_outputs=gout, create_graph=True)
    s = sum((ai * gi).sum() for ai, gi, on in zip(a, g1, tan) if on)
    return torch.autograd.grad(s, (x, sh, w, gout), allow_unused=True)


def _check_layer(o, t, n=37, E=400):
    import torch
    from sevenn_b200.sh import spherical_harmonics
    L = o.spec.layers[t]
    rng = np.random.RandomState(100 + t)
    x = rng.normal(size=(n, L.dim_x))
    sh = spherical_harmonics(o.spec.lmax_filter, rng.normal(size=(E, 3)))
    w = rng.normal(size=(E, L.weight_numel))
    src = rng.randint(0, n, size=E)
    dst = rng.randint(0, n - 3, size=E)            # unsorted, some nodes without edges
    gout = rng.normal(size=(n, L.dim_mid))
    a = [rng.normal(size=x.shape), rng.normal(size=sh.shape), rng.normal(size=w.shape)]
    a[1][:, 0] = 0.0     # Y_0 is the constant 1: its first-order gradient is 0 here, a function of sh in the oracle
    conv = _conv_of(o, L)
    src_c = torch.as_tensor(src, device='cuda', dtype=torch.int32)
    dst_c = torch.as_tensor(dst, device='cuda', dtype=torch.int32)
    src_t, dst_t = torch.as_tensor(src), torch.as_tensor(dst)

    def ref_fn(x_, sh_, w_):
        msg = o.tensor_product(L, x_[src_t], sh_, w_)
        return torch.zeros(n, L.dim_mid, dtype=torch.float64).index_add_(0, dst_t, msg)

    for name, tan in TANGENTS.items():
        ref = _second_order(ref_fn, [torch.tensor(v, dtype=torch.float64, requires_grad=True)
                                     for v in (x, sh, w, gout)],
                            [torch.as_tensor(v) for v in a], tan)
        got = _second_order(lambda x_, sh_, w_: conv(x_, sh_, w_, src_c, dst_c),
                            [torch.tensor(v, dtype=torch.float32, device='cuda', requires_grad=True)
                             for v in (x, sh, w, gout)],
                            [torch.as_tensor(v, dtype=torch.float32, device='cuda') for v in a], tan)
        for what, shape, r, g in zip(('x', 'sh', 'w', 'grad_out'), (x.shape, sh.shape, w.shape, gout.shape),
                                     ref, got):
            # a derivative that autograd reports as unused (None) is zero
            r = np.zeros(shape) if r is None else r.numpy().copy()
            g = np.zeros(shape) if g is None else g.detach().cpu().numpy()
            if what == 'sh':
                assert np.all(g[:, 0] == 0.0), (name, 'd/d sh[:, 0] must be exactly 0')
                r[:, 0] = 0.0
            # the first-order bounds of tests/test_conv_op_gpu.py (fp32 sums over a row, an in-degree or a role)
            assert np.allclose(g, r, atol=2e-3, rtol=1e-4), \
                (name, what, float(np.abs(g - r).max()), float(np.abs(r).max()))


@pytest.mark.parametrize('name,t', [('sevennet_0', 0), ('sevennet_0', 1), ('sevennet_0', 4),
                                    ('sevennet_l3i5', 2), ('sevennet_l3i5', 4)])
def test_double_backward_pretrained(name, t):
    _check_layer(oracle(name), t)


@pytest.mark.parametrize('t', [0, 1, 2])
@pytest.mark.parametrize('le,ln', [(le, ln) for le in (1, 2, 3) for ln in (1, 2, 3)])
def test_double_backward_groups(le, ln, t, tmp_path_factory):
    o = _synthetic_oracle(le, ln, tmp_path_factory.mktemp('ckpt'))
    group = (o.spec.lmax_filter, max(p.l3 for p in o.spec.layers[t].paths))
    if t > 0:
        assert group == ((le, ln) if t == 1 else (le, 0))
    _check_layer(o, t)


def test_double_backward_empty_and_third_order():
    """E == 0 gives zeros; differentiating a third time raises instead of returning a silent zero."""
    import torch
    L = oracle('sevennet_0').spec.layers[1]
    conv = _conv_of(oracle('sevennet_0'), L)
    x = torch.randn(5, L.dim_x, device='cuda', requires_grad=True)
    sh = torch.zeros(0, 9, device='cuda', requires_grad=True)
    w = torch.zeros(0, L.weight_numel, device='cuda', requires_grad=True)
    gout = torch.randn(5, L.dim_mid, device='cuda', requires_grad=True)
    e = torch.zeros(0, dtype=torch.int32, device='cuda')
    (gx,) = torch.autograd.grad(conv(x, sh, w, e, e), x, grad_outputs=gout, create_graph=True)
    gg = torch.autograd.grad((torch.randn_like(gx) * gx).sum(), (x, gout), allow_unused=True)
    for g in gg:
        assert g is None or float(g.abs().max()) == 0.0

    n, E = 12, 60
    rng = np.random.RandomState(0)
    from sevenn_b200.sh import spherical_harmonics
    sh = torch.tensor(spherical_harmonics(2, rng.normal(size=(E, 3))), dtype=torch.float32, device='cuda',
                      requires_grad=True)
    w = torch.randn(E, L.weight_numel, device='cuda', requires_grad=True)
    src = torch.as_tensor(rng.randint(0, n, size=E), dtype=torch.int32, device='cuda')
    dst = torch.as_tensor(rng.randint(0, n, size=E), dtype=torch.int32, device='cuda')
    x = torch.randn(n, L.dim_x, device='cuda', requires_grad=True)
    gout = torch.randn(n, L.dim_mid, device='cuda')
    (gw,) = torch.autograd.grad(conv(x, sh, w, src, dst), w, grad_outputs=gout, create_graph=True)
    (hx,) = torch.autograd.grad((gw * gw).sum(), x, create_graph=True)
    with pytest.raises(RuntimeError):      # autograd.grad: x is not reachable through the third derivative
        torch.autograd.grad(hx.sum(), x)
    with pytest.raises(RuntimeError, match='once_differentiable'):
        hx.sum().backward()


def test_double_backward_launches():
    """Two convolution kernels per l1 role (jvp and bwd_tangent), besides the packing of Y, of the tangent of Y and
    the unpacking of dY; the composition from first-order kernels would take six."""
    import torch
    from sevenn_b200.engine import load_library
    lib = load_library()
    o = oracle('sevennet_0')
    L = o.spec.layers[1]
    conv = _conv_of(o, L)
    n, E = 40, 500
    rng = np.random.RandomState(1)
    from sevenn_b200.sh import spherical_harmonics
    t32 = lambda v: torch.tensor(v, dtype=torch.float32, device='cuda', requires_grad=True)
    x, sh, w = t32(rng.normal(size=(n, L.dim_x))), t32(spherical_harmonics(2, rng.normal(size=(E, 3)))), \
        t32(rng.normal(size=(E, L.weight_numel)))
    src = torch.as_tensor(rng.randint(0, n, size=E), dtype=torch.int32, device='cuda')
    dst = torch.as_tensor(np.sort(rng.randint(0, n, size=E)), dtype=torch.int32, device='cuda')
    gout = t32(rng.normal(size=(n, L.dim_mid)))
    g1 = torch.autograd.grad(conv(x, sh, w, src, dst), (x, sh, w), grad_outputs=gout, create_graph=True)
    s = sum((torch.randn_like(g) * g).sum() for g in g1)
    torch.cuda.synchronize()
    lib.s7b_launch_count(1)
    torch.autograd.grad(s, (x, sh, w, gout))
    torch.cuda.synchronize()
    roles = len({p.l1 for p in L.paths})
    assert lib.s7b_launch_count(1) == 2 * roles + 3


# ---- end to end: a force loss and a Hessian-vector product through a SevenNet-0 energy ----------------------------
def _energy(o, species, src, dst, ev, conv=None):
    """The oracle's energy (Oracle.forward's module order) as a differentiable function of the edge vectors and of
    o.w; `conv(L, x, sh, weight)` replaces the convolution's tensor product + index_add when given"""
    import math
    import torch
    s, n = o.spec, species.shape[0]
    r, emb, sh = o.edge_embedding(ev)
    x = o.w['embed'].reshape(s.num_species, -1)[species] / math.sqrt(s.num_species)
    for L in s.layers:
        t = L.t
        xb = o._blocks(L.x_muls)
        sc = o.linear(x, o.w[f'{t}.sc'], xb, list(L.gate_muls))
        x = o.linear(x, o.w[f'{t}.si1'], xb, list(L.x_muls))
        weight = o.radial_mlp(t, emb)
        if conv is None:
            agg = torch.zeros(n, L.dim_mid, dtype=x.dtype, device=x.device).index_add_(
                0, dst, o.tensor_product(L, x[src], sh, weight))
        else:
            agg = conv(L, x, sh, weight)
        agg = agg / o.w[f'{t}.den']
        mid_blocks, off = [], 0
        for p in L.paths:
            mid_blocks.append((p.l3, p.mul, off))
            off += p.mul * (2 * p.l3 + 1)
        g = o.linear(agg, o.w[f'{t}.si2'], mid_blocks, list(L.gate_muls)) + sc
        x = o.gate(L, g)
    Lz = s.layers[-1]
    h = o.linear(x, o.w['readout1'], o._blocks(Lz.out_muls), [s.readout_hidden])
    e = o.linear(h, o.w['readout2'], [(0, s.readout_hidden, 0)], [1])
    return (e[:, 0] * o.w['scale'][species] + o.w['shift'][species]).sum()


def test_force_loss_gradients_and_hvp():
    """Energy of a rattled 16-atom periodic Si cell with SevenNet-0 weights, forces by autograd with
    create_graph=True, loss = sum (F - F0)^2: its gradients with respect to the radial-MLP and the linear weights,
    and one Hessian-vector product d(F . v)/d pos, with B200Convolution (fp32) against the all-fp64 oracle.  Bound:
    relative 2-norm error 2e-3 per tensor (fp32 convolutions in an fp64 model give about 1e-5 .. 1e-4; without the
    convolution's second order the MLP gradients are off by O(1))."""
    import torch
    from oracle.oracle import Oracle
    from sevenn_b200.neighbors import build_graph, diamond_si
    meta, arrays = model_weights('sevennet_0')
    pos0, cell, z = diamond_si(2, 1, 1)
    rng = np.random.RandomState(5)
    pos0 = pos0 + rng.normal(scale=0.1, size=pos0.shape)
    ei, ev0 = build_graph(pos0, cell, True, float(meta['cutoff']))
    tm = {int(k): int(v) for k, v in meta['type_map'].items()}
    species = torch.as_tensor([tm[int(a)] for a in z], device='cuda')
    dst_t = torch.as_tensor(ei[0], device='cuda')
    src_t = torch.as_tensor(ei[1], device='cuda')
    shift = torch.as_tensor(ev0 - (pos0[ei[1]] - pos0[ei[0]]), device='cuda')
    F0 = torch.as_tensor(rng.normal(scale=0.3, size=pos0.shape), device='cuda')
    v = torch.as_tensor(rng.normal(size=pos0.shape), device='cuda')
    keys = [k for k in arrays if any(k.endswith(s) for s in ('.mlp0', '.mlp1', '.mlp2', '.si1', '.si2'))]
    keys += ['readout1']
    convs = {}

    def b200(L, x, sh, weight):
        if L.t not in convs:
            convs[L.t] = _conv_of(oracle('sevennet_0'), L)
        out = convs[L.t](x.float(), sh.float(), weight.float(), src_t.to(torch.int32), dst_t.to(torch.int32))
        return out.double()

    res = {}
    for impl, conv in (('fp64', None), ('b200', b200)):
        o = Oracle(meta, arrays, dtype=torch.float64, device='cuda')
        params = [o.w[k].requires_grad_(True) for k in keys]
        pos = torch.as_tensor(pos0, device='cuda').requires_grad_(True)
        ev = pos[src_t] - pos[dst_t] + shift
        E = _energy(o, species, src_t, dst_t, ev, conv)
        (dE,) = torch.autograd.grad(E, pos, create_graph=True)
        F = -dE
        loss = ((F - F0) ** 2).sum()
        grads = torch.autograd.grad(loss, params, retain_graph=True)
        (hvp,) = torch.autograd.grad((F * v).sum(), pos)
        res[impl] = [g.detach().cpu().numpy() for g in grads] + [hvp.detach().cpu().numpy()]
    for k, a, b in zip(keys + ['hvp'], res['b200'], res['fp64']):
        rel = np.linalg.norm(a - b) / np.linalg.norm(b)
        assert rel < 2e-3, (k, rel)
