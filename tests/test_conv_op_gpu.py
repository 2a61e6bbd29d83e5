"""Operator-level drop-in (`convolution_cls` contract, reference convolution.py:243-247,270-276):
B200Convolution vs the oracle's e3nn-semantics tensor product + index_add + torch autograd."""
import numpy as np
import pytest

from helpers import model_weights, oracle

pytestmark = pytest.mark.gpu


def _irreps_str(muls):
    return '+'.join(f'{m}x{l}e' for l, m in enumerate(muls))


def _compare_with_oracle(name, t, x, sh, w, src, dst, gout, g=1.0):
    """B200Convolution of layer t vs the oracle's fp64 tensor product + index_add, forward and the three
    gradients; `g` widens the absolute bounds of sums over many edges"""
    import torch
    from sevenn_b200.conv_op import B200Convolution
    o = oracle(name)
    L = o.spec.layers[t]
    lf = o.spec.lmax_filter
    mid = '+'.join(f'{p.mul}x{p.l3}e' for p in L.paths)
    inst = [(p.l1, p.l2, p.slot, 'uvu', True) for p in L.paths]
    conv = B200Convolution(_irreps_str(L.x_muls), _irreps_str([1] * (lf + 1)), mid, inst,
                           shared_weights=False, internal_weights=False).cuda()
    n = x.shape[0]

    xt, sht, wt = (torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (x, sh, w))
    msg = o.tensor_product(L, xt[torch.as_tensor(src)], sht, wt)
    ref = torch.zeros(n, L.dim_mid, dtype=torch.float64).index_add_(0, torch.as_tensor(dst), msg)
    (ref * torch.as_tensor(gout)).sum().backward()

    xc, shc, wc = (torch.tensor(a, dtype=torch.float32, device='cuda', requires_grad=True) for a in (x, sh, w))
    out = conv(xc, shc, wc, torch.as_tensor(src, device='cuda', dtype=torch.int32),
               torch.as_tensor(dst, device='cuda', dtype=torch.int32))
    assert out.shape == (n, L.dim_mid)
    assert np.allclose(out.detach().cpu().numpy(), ref.detach().numpy(), atol=2e-4 * g, rtol=1e-5)
    (out * torch.as_tensor(gout, device='cuda', dtype=torch.float32)).sum().backward()
    assert np.allclose(xc.grad.cpu().numpy(), xt.grad.numpy(), atol=5e-4 * g, rtol=1e-4)
    assert np.allclose(wc.grad.cpu().numpy(), wt.grad.numpy(), atol=5e-4, rtol=1e-4)
    gsh_ref = sht.grad.numpy().copy()
    gsh_ref[:, 0] = 0.0          # Y_0 is the constant 1: no gradient is produced for it
    assert np.allclose(shc.grad.cpu().numpy(), gsh_ref, atol=2e-3, rtol=1e-4)
    return out


@pytest.mark.parametrize('name,t', [('sevennet_0', 0), ('sevennet_0', 1), ('sevennet_0', 4),
                                    ('sevennet_l3i5', 2), ('sevennet_l3i5', 4)])
def test_conv_op_forward_backward(name, t):
    L = oracle(name).spec.layers[t]
    rng = np.random.RandomState(t)
    n, E = 37, 400
    x = rng.normal(size=(n, L.dim_x))
    from sevenn_b200.sh import spherical_harmonics
    sh = spherical_harmonics(oracle(name).spec.lmax_filter, rng.normal(size=(E, 3)))
    w = rng.normal(size=(E, L.weight_numel))
    src = rng.randint(0, n, size=E)
    dst = rng.randint(0, n - 3, size=E)            # unsorted, some nodes without edges
    gout = rng.normal(size=(n, L.dim_mid))
    _compare_with_oracle(name, t, x, sh, w, src, dst, gout)


def _row_lengths(pattern, rng):
    """per-node edge counts: the ragged / hub fixtures of tests/graphs.py, or odd n with an empty last node"""
    if pattern == 'odd_last_empty':
        deg = rng.randint(1, 40, size=45)
        deg[-1] = 0
        return deg
    import graphs
    return graphs.degrees(graphs.fixture(pattern, 'sevennet_0'))


# sevennet_0 layer 1 and sevennet_l3i5 layer 2 hold 128-, 64- and 32-channel roles: both lane mappings (32 lanes per
# node, 16 for 32 channels); l3i5's lmax-3 roles take the atomic (split) backward.  ragged: rows of 0 .. 65 edges
# (every edge-record refill boundary, also side by side); hub: a 166-edge row next to empty ones
@pytest.mark.parametrize('pattern', ['ragged', 'hub', 'odd_last_empty'])
@pytest.mark.parametrize('name,t', [('sevennet_0', 1), ('sevennet_l3i5', 2)])
def test_conv_op_row_lengths(name, t, pattern):
    L = oracle(name).spec.layers[t]
    rng = np.random.RandomState(t)
    deg = _row_lengths(pattern, rng)
    n, E = len(deg), int(deg.sum())
    dst = np.repeat(np.arange(n), deg)[rng.permutation(E)]          # unsorted
    x = rng.normal(size=(n, L.dim_x))
    from sevenn_b200.sh import spherical_harmonics
    sh = spherical_harmonics(oracle(name).spec.lmax_filter, rng.normal(size=(E, 3)))
    w = rng.normal(size=(E, L.weight_numel))
    src = rng.randint(0, n, size=E)
    gout = rng.normal(size=(n, L.dim_mid))
    # fp32 sums of up to `fan` unit-scale terms: the absolute bounds grow as sqrt(fan) (about 12 in the test above)
    fan = max(np.bincount(dst).max(), np.bincount(src).max())
    out = _compare_with_oracle(name, t, x, sh, w, src, dst, gout, g=max(1.0, np.sqrt(fan / 12.0)))
    if pattern == 'odd_last_empty':
        assert float(out[-1].abs().max()) == 0.0


def test_conv_op_empty_edges():
    """reference convolution.py:265-268: E == 0 must work and give zeros."""
    import torch
    from sevenn_b200.conv_op import B200Convolution
    conv = B200Convolution('128x0e', '1x0e+1x1e+1x2e', '128x0e+128x1e+128x2e').cuda()
    x = torch.randn(5, 128, device='cuda', requires_grad=True)
    sh = torch.zeros(0, 9, device='cuda', requires_grad=True)
    w = torch.zeros(0, 384, device='cuda', requires_grad=True)
    e = torch.zeros(0, dtype=torch.int32, device='cuda')
    out = conv(x, sh, w, e, e)
    assert out.shape == (5, 1152) and float(out.abs().max()) == 0.0
    out.sum().backward()
    assert float(x.grad.abs().max()) == 0.0


def test_conv_op_rejects_unsupported():
    from sevenn_b200.conv_op import B200Convolution
    with pytest.raises(NotImplementedError):
        B200Convolution('128x0e+64x1o', '1x0e+1x1e', '128x0e')
    with pytest.raises(NotImplementedError):
        B200Convolution('128x0e', '1x0e+1x1e+1x2e', '128x0e+128x1e+128x2e',
                        [(0, 0, 0, 'uvw', True), (0, 1, 1, 'uvu', True), (0, 2, 2, 'uvu', True)])
