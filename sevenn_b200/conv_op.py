"""Drop-in for the reference's tensor-product accelerator plug-in point.

The reference swaps ``IrrepsScatterGatterFusedConvolution.convolution_cls`` for an accelerator
class (``sevenn/nn/convolution.py:145-284``; adapters ``sevenn/nn/flash_helper.py:33-48``,
``sevenn/nn/oeq_helper.py:30-70``).  The contract restated here:

  construct: ``cls(irreps_in1, irreps_in2, irreps_out, instructions, shared_weights=False,
             internal_weights=False)`` with 'uvu' instructions sorted by ``i_out``
             (``convolution.py:61-91``);
  call:      ``out = f(x, edge_filter, weight, edge_src.int32, edge_dst.int32)`` with
             ``x [n_nodes, dim_in]``, ``edge_filter [E, (lmax+1)^2]``, ``weight [E, W]`` and
             ``out [n_nodes, dim_mid]`` in e3nn ``mul_ir`` layout, differentiable in x,
             edge_filter and weight (``convolution.py:270-276``).

``B200Convolution`` keeps that interface and runs the fused gather -> tensor product -> scatter
kernels of ``libsevenn_b200.so`` (C ABI ``s7b_conv_forward`` / ``s7b_conv_backward``), with a
hand-written backward instead of autograd through e3nn.  The operator is twice differentiable: under
``create_graph=True`` (forces inside a training loss, Hessian-vector products) the backward is itself
differentiated by ``s7b_conv_double_backward``; a third derivative raises.  Layout conversion (mul_ir <-> the
engine's component-major layout) and the sort of edges by destination are torch index ops.
``edge_filter[:, 0]`` must be the constant Y_0 = 1 that ``SphericalEncoding`` produces
(component normalisation); its gradient is returned as zero.
"""
from __future__ import annotations

import ctypes
import re
from typing import List, Sequence

import numpy as np

from .engine import check, load_library
from .spec import build_layer, parse_even_irreps, perm_cm_from_mulir


def _parse_unsimplified(s: str):
    out = []
    for tok in str(s).replace(' ', '').split('+'):
        m = re.fullmatch(r'(\d+)x(\d+)([eo])', tok)
        if m is None:
            raise ValueError(f'cannot parse irreps token {tok!r}')
        if m.group(3) != 'e':
            raise NotImplementedError('odd-parity irreps are not supported by sevenn_b200')
        out.append((int(m.group(1)), int(m.group(2))))
    return out


def is_b200_available() -> bool:
    try:
        import torch
        load_library()
        return torch.cuda.is_available()
    except Exception:
        return False


def _make_module_class():
    import torch
    from torch.autograd.function import once_differentiable

    class _ConvFn(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, edge_filter, weight, edge_src, edge_dst, mod):
            lib = load_library()
            dev = x.device
            E, n_nodes = int(edge_src.shape[0]), int(x.shape[0])
            dst, src = edge_dst.long(), edge_src.long()
            perm = None
            inputs = (x, edge_filter, weight)
            if E > 1 and bool((dst[1:] < dst[:-1]).any()):
                perm = torch.argsort(dst, stable=True)
                dst, src = dst[perm], src[perm]
                edge_filter, weight = edge_filter[perm], weight[perm]
            rowptr = torch.zeros(n_nodes + 1, dtype=torch.int64, device=dev)
            if E > 0:
                rowptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n_nodes), 0)
            rowptr = rowptr.to(torch.int32)
            src32 = src.to(torch.int32).contiguous()
            x_cm = x.float().index_select(1, mod._perm_x).contiguous()
            sh = edge_filter.float().contiguous()
            w = weight.float().contiguous()
            out_cm = torch.empty(n_nodes, mod.dim_mid, dtype=torch.float32, device=dev)
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            with torch.cuda.device(dev):
                check(lib.s7b_conv_forward(mod._plan, x_cm.data_ptr(), sh.data_ptr(), w.data_ptr(),
                                           rowptr.data_ptr(), src32.data_ptr(), n_nodes, n_nodes, E,
                                           out_cm.data_ptr(), st))
            # the inputs as well: the backward is differentiated as a function of them (second order)
            ctx.save_for_backward(x_cm, sh, w, rowptr, src32, *inputs)
            ctx.perm, ctx.mod = perm, mod
            return out_cm.index_select(1, mod._perm_mid_inv)

        @staticmethod
        def backward(ctx, grad_out):
            x_cm, sh, w, rowptr, src32, x, edge_filter, weight = ctx.saved_tensors
            gx, gsh, gw = _ConvBwdFn.apply(grad_out, x, edge_filter, weight, x_cm, sh, w, rowptr, src32,
                                           ctx.perm, ctx.mod)
            return gx, gsh, gw, None, None, None

    class _ConvBwdFn(torch.autograd.Function):
        """The backward of _ConvFn as a function of (grad_out, x, edge_filter, weight), so that a graph built
        with create_graph=True differentiates it once more (s7b_conv_double_backward).  x, edge_filter and
        weight only tie the result to the graph; the kernels read their converted copies x_cm, sh and w."""

        @staticmethod
        def forward(ctx, grad_out, x, edge_filter, weight, x_cm, sh, w, rowptr, src32, perm, mod):
            lib = load_library()
            dev = x_cm.device
            n_nodes, E = int(x_cm.shape[0]), int(src32.shape[0])
            g_cm = grad_out.float().index_select(1, mod._perm_mid).contiguous()
            gx = torch.empty_like(x_cm)
            gsh = torch.zeros_like(sh)
            gw = torch.zeros_like(w)
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            with torch.cuda.device(dev):
                check(lib.s7b_conv_backward(mod._plan, x_cm.data_ptr(), sh.data_ptr(), w.data_ptr(),
                                            rowptr.data_ptr(), src32.data_ptr(), n_nodes, n_nodes, E,
                                            g_cm.data_ptr(), gx.data_ptr(), gsh.data_ptr(), gw.data_ptr(), st))
            if perm is not None:
                inv = torch.empty_like(perm)
                inv[perm] = torch.arange(E, device=dev)
                gsh, gw = gsh[inv], gw[inv]
            ctx.save_for_backward(x_cm, sh, w, rowptr, src32, g_cm)
            ctx.perm, ctx.mod = perm, mod
            ctx.set_materialize_grads(False)      # an absent incoming gradient skips its terms
            return gx.index_select(1, mod._perm_x_inv), gsh, gw

        @staticmethod
        @once_differentiable
        def backward(ctx, tan_x, tan_sh, tan_w):
            lib = load_library()
            x_cm, sh, w, rowptr, src32, g_cm = ctx.saved_tensors
            mod, perm = ctx.mod, ctx.perm
            dev = x_cm.device
            n_nodes, E = int(x_cm.shape[0]), int(src32.shape[0])

            def edges_sorted(t):      # per-edge tangent -> the kernels' dst-sorted edge order, fp32
                if t is None:
                    return None
                return (t if perm is None else t[perm]).float().contiguous()

            tx = None if tan_x is None else tan_x.float().index_select(1, mod._perm_x).contiguous()
            tsh, tw = edges_sorted(tan_sh), edges_sorted(tan_w)
            ggo = torch.empty_like(g_cm)
            gx = torch.empty_like(x_cm)
            gsh = torch.empty_like(sh)
            gw = torch.empty_like(w)
            ptr = lambda t: None if t is None else t.data_ptr()
            st = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            with torch.cuda.device(dev):
                check(lib.s7b_conv_double_backward(
                    mod._plan, x_cm.data_ptr(), sh.data_ptr(), w.data_ptr(), rowptr.data_ptr(), src32.data_ptr(),
                    n_nodes, n_nodes, E, g_cm.data_ptr(), ptr(tx), ptr(tsh), ptr(tw),
                    ggo.data_ptr(), gx.data_ptr(), gsh.data_ptr(), gw.data_ptr(), st))
            if perm is not None:
                inv = torch.empty_like(perm)
                inv[perm] = torch.arange(E, device=dev)
                gsh, gw = gsh[inv], gw[inv]
            return (ggo.index_select(1, mod._perm_mid_inv), gx.index_select(1, mod._perm_x_inv), gsh, gw,
                    None, None, None, None, None, None, None)

    class B200Convolution(torch.nn.Module):
        """``convolution_cls``-compatible fused 'uvu' tensor product (see module docstring)."""

        def __init__(self, irreps_in1, irreps_in2, irreps_out, instructions: Sequence = (),
                     shared_weights: bool = False, internal_weights: bool = False):
            super().__init__()
            if shared_weights or internal_weights:
                raise NotImplementedError('only per-edge external weights are supported')
            x_muls = parse_even_irreps(str(irreps_in1))
            filt = parse_even_irreps(str(irreps_in2))
            if any(m != 1 for m in filt):
                raise NotImplementedError('irreps_in2 must be spherical harmonics 1x0e+1x1e+...')
            mid = _parse_unsimplified(str(irreps_out))
            lmax_out = max(l for _, l in mid)
            layer = build_layer(0, x_muls, [32] * (lmax_out + 1), len(filt) - 1)
            expect = [(p.l1, p.l2, p.slot) for p in layer.paths]
            if instructions:
                got = [(int(i[0]), int(i[1]), int(i[2])) for i in instructions]
                if got != expect or any(str(i[3]) != 'uvu' for i in instructions):
                    raise NotImplementedError(
                        'instructions are not the complete, i_out-sorted uvu set of '
                        'sevenn/nn/convolution.py:61-82')
            if [(p.mul, p.l3) for p in layer.paths] != mid:
                raise NotImplementedError('irreps_out does not match the instruction set')
            self.layer = layer
            self.dim_x, self.dim_mid, self.weight_numel = layer.dim_x, layer.dim_mid, layer.weight_numel
            lib = load_library()
            self._plan = ctypes.c_void_p()
            muls = (ctypes.c_int32 * len(x_muls))(*x_muls)
            check(lib.s7b_conv_plan_create(len(x_muls), muls, len(filt) - 1, lmax_out, ctypes.byref(self._plan)))
            dims = [ctypes.c_int32() for _ in range(4)]
            check(lib.s7b_conv_plan_dims(self._plan, *[ctypes.byref(d) for d in dims]))
            assert [d.value for d in dims[:3]] == [self.dim_x, self.dim_mid, self.weight_numel]
            px = perm_cm_from_mulir(x_muls)
            pm = layer.mid_perm_cm_from_mulir()
            self.register_buffer('_perm_x', torch.as_tensor(px), persistent=False)
            self.register_buffer('_perm_x_inv', torch.as_tensor(np.argsort(px)), persistent=False)
            self.register_buffer('_perm_mid', torch.as_tensor(pm), persistent=False)
            self.register_buffer('_perm_mid_inv', torch.as_tensor(np.argsort(pm)), persistent=False)

        def __del__(self):
            try:
                if getattr(self, '_plan', None) is not None and self._plan.value:
                    load_library().s7b_conv_plan_destroy(self._plan)
                    self._plan = None
            except Exception:
                pass

        def forward(self, x, edge_filter, weight, edge_src, edge_dst):
            if not x.is_cuda:
                raise RuntimeError('B200Convolution needs CUDA tensors; there is no CPU path')
            return _ConvFn.apply(x, edge_filter, weight, edge_src, edge_dst, self)

    return B200Convolution


_cls = None


def __getattr__(name):
    global _cls
    if name == 'B200Convolution':
        if _cls is None:
            _cls = _make_module_class()
        return _cls
    raise AttributeError(name)


def patch_convolution(conv_module):
    """Mirror of ``flash_helper.patch_convolution`` (flash_helper.py:33-48): given an
    ``IrrepsScatterGatterFusedConvolution``-like object that has not been instantiated yet,
    point its ``convolution_cls`` at ``B200Convolution``."""
    if not is_b200_available():
        raise ImportError('sevenn_b200 CUDA library or device is not available')
    conv_module.convolution_cls = __getattr__('B200Convolution')
    return conv_module
