"""Code generator for the per-lane arithmetic of the fused gather -> tensor-product -> scatter
kernels and for the spherical harmonics.  Run as a script to (re)write ``generated/*.cuh``.

Nothing here is copied from the reference: e3nn generates its tensor-product code at run time
with torch.fx (``o3.TensorProduct``, used at reference ``sevenn/nn/convolution.py:84-100``);
this generator emits straight-line CUDA with the coupling coefficients baked in as FFMA
immediates, specialised per *kind* = (l1, lmax_filter, lmax_out): all triangle-allowed paths
(l1, l2, l3) with l2 <= lmax_filter, l3 <= lmax_out, in slot order (l3-major, then l2), which is
the path set of every even-parity SevenNet interaction layer (``convolution.py:61-82``).

Per-lane forward for one edge and one channel u (w_p = per-edge radial weight of path p):
    s_p[k]  = sum_ij C'_p[i,j,k] x[i] Y_l2[j]         C' = sqrt(2 l3 + 1) * w3j
    acc_p[k] += w_p * s_p[k]
Per-lane backward, given ga_p[k] = dE/d(acc_p[k]):
    dw_p      = sum_k ga_p[k] s_p[k]
    R_l2[i,j] = sum_{p with that l2} sum_k C'_p[i,j,k] w_p ga_p[k]
    dx[i]     = sum_{l2,j} R_l2[i,j] Y_l2[j]
    dY_l2[j] += sum_i x[i] R_l2[i,j]                   (partial: still to be summed over channels)
"""
from __future__ import annotations

import os
import sys
from typing import List, Tuple

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))

from sevenn_b200.cg import tp_path_coefficients  # noqa: E402
from sevenn_b200.sh import sh_polynomials, X, Y, Z  # noqa: E402

def kind_paths(l1: int, lf: int, lo: int) -> List[Tuple[int, int]]:
    """(l2, l3) in slot order restricted to this l1: sorted by l3, then by creation (l2)."""
    ps = [(l2, l3) for l2 in range(lf + 1) for l3 in range(abs(l1 - l2), l1 + l2 + 1) if l3 <= lo]
    return sorted(ps, key=lambda p: (p[1], p[0]))


# (lmax_filter, lmax_out) groups: each is one translation unit, conv_group_<LF><LO>.cu
GROUPS: List[Tuple[int, int]] = [(lf, lo) for lf in (1, 2, 3) for lo in range(4)]
# the groups of SevenNet-0 and SevenNet-l3i5, which also have kernels specialised for their widths (kConvMul)
SPECIALISED_GROUPS: List[Tuple[int, int]] = [(2, 2), (2, 0), (3, 3), (3, 0)]

KINDS: List[Tuple[int, int, int]] = (
    [(l1, 2, 2) for l1 in range(3)] + [(l1, 2, 0) for l1 in range(3)]       # SevenNet-0
    + [(l1, 3, 3) for l1 in range(4)] + [(l1, 3, 0) for l1 in range(4)]     # SevenNet-l3i5
)
# every other kind with at least one path: x of l1 <= 3, every group (a role without paths launches nothing)
KINDS += [(l1, lf, lo) for (lf, lo) in GROUPS for l1 in range(4)
          if (l1, lf, lo) not in KINDS and kind_paths(l1, lf, lo)]


def _f(v: float) -> str:
    return f'{float(v):.9g}f' if 'e' in f'{float(v):.9g}' or '.' in f'{float(v):.9g}' else f'{float(v):.9g}.0f'


def _y(l2: int, j: int) -> str:
    return '1.0f' if l2 == 0 else f'Y[{l2 * l2 + j}]'


def gen_kind(l1: int, lf: int, lo: int) -> str:
    paths = kind_paths(l1, lf, lo)
    d1 = 2 * l1 + 1
    ny = (lf + 1) ** 2
    acc_off, off = [], 0
    for (_, l3) in paths:
        acc_off.append(off)
        off += 2 * l3 + 1
    nacc = off
    npath = len(paths)
    name = f'TPKind<{l1}, {lf}, {lo}>'
    out = [f'// ---- kind (l1={l1}, lmax_filter={lf}, lmax_out={lo}): paths (l2,l3) = {paths}',
           f'template <> struct {name} {{',
           f'  static constexpr int L1 = {l1}, D1 = {d1}, NY = {ny}, NPATH = {npath}, NACC = {nacc};',
           f'  S7B_HD static constexpr int path_l2(int p) {{ constexpr int t[{npath}] = {{{", ".join(str(p[0]) for p in paths)}}}; return t[p]; }}',
           f'  S7B_HD static constexpr int path_l3(int p) {{ constexpr int t[{npath}] = {{{", ".join(str(p[1]) for p in paths)}}}; return t[p]; }}',
           f'  S7B_HD static constexpr int acc_off(int p) {{ constexpr int t[{npath}] = {{{", ".join(str(o) for o in acc_off)}}}; return t[p]; }}']

    l2_used = sorted({p[0] for p in paths})

    def products(lines: List[str]):
        """t_{l2}_{i}_{j} = x[i] * Y_l2[j] for every (i,j) that any path of this l2 touches."""
        for l2 in l2_used:
            if l2 == 0:
                continue
            need = set()
            for (q2, l3) in paths:
                if q2 != l2:
                    continue
                c = tp_path_coefficients(l1, l2, l3)
                for i, j, k in zip(*np.nonzero(c)):
                    need.add((int(i), int(j)))
            for (i, j) in sorted(need):
                lines.append(f'    const V t{l2}_{i}_{j} = mul_(x[{i}], {_y(l2, j)});')

    def s_expr(l2: int, l3: int, k: int) -> str:
        c = tp_path_coefficients(l1, l2, l3)
        terms = []
        for i in range(d1):
            for j in range(2 * l2 + 1):
                v = c[i, j, k]
                if v != 0.0:
                    t = f'x[{i}]' if l2 == 0 else f't{l2}_{i}_{j}'
                    terms.append((v, t))
        assert terms
        e = terms[0][1] if abs(terms[0][0] - 1.0) < 1e-12 else f'mul_({terms[0][1]}, {_f(terms[0][0])})'
        for v, t in terms[1:]:
            e = f'fma_({_f(v)}, {t}, {e})'
        return e

    # ---- forward
    out.append('  // acc[ACC_OFF[p] + k] += w[p] * sum_ij C\'[i,j,k] x[i] Y[j]')
    out.append('  template <class V>')
    out.append('  S7B_HD static void fwd(const V* __restrict__ x, const float* __restrict__ Y,')
    out.append('                         const V* __restrict__ w, V* __restrict__ acc) {')
    body: List[str] = []
    products(body)
    for p, (l2, l3) in enumerate(paths):
        for k in range(2 * l3 + 1):
            body.append(f'    acc[{acc_off[p] + k}] = fma_(w[{p}], {s_expr(l2, l3, k)}, acc[{acc_off[p] + k}]);')
    out += body
    out.append('  }')

    # ---- backward
    out.append('  // dw[p] = ...; dx[i] = ...; dY[j] += ... (see header comment of gen_kernels.py)')
    out.append('  template <class V>')
    out.append('  S7B_HD static void bwd(const V* __restrict__ x, const float* __restrict__ Y,')
    out.append('                         const V* __restrict__ w, const V* __restrict__ ga,')
    out.append('                         V* __restrict__ dw, V* __restrict__ dx, V* __restrict__ dY) {')
    body = []
    products(body)
    for p, (l2, l3) in enumerate(paths):
        e = f'mul_(ga[{acc_off[p]}], {s_expr(l2, l3, 0)})'
        for k in range(1, 2 * l3 + 1):
            e = f'fma_(ga[{acc_off[p] + k}], {s_expr(l2, l3, k)}, {e})'
        body.append(f'    dw[{p}] = {e};')
    for p, (l2, l3) in enumerate(paths):
        for k in range(2 * l3 + 1):
            body.append(f'    const V g{p}_{k} = mul_(w[{p}], ga[{acc_off[p] + k}]);')
    for i in range(d1):
        dx_terms = []
        for l2 in l2_used:
            for j in range(2 * l2 + 1):
                terms = []
                for p, (q2, l3) in enumerate(paths):
                    if q2 != l2:
                        continue
                    c = tp_path_coefficients(l1, l2, l3)
                    for k in range(2 * l3 + 1):
                        if c[i, j, k] != 0.0:
                            terms.append((c[i, j, k], f'g{p}_{k}'))
                if not terms:
                    continue
                e = terms[0][1] if abs(terms[0][0] - 1.0) < 1e-12 else f'mul_({terms[0][1]}, {_f(terms[0][0])})'
                for v, t in terms[1:]:
                    e = f'fma_({_f(v)}, {t}, {e})'
                body.append(f'    const V r{l2}_{i}_{j} = {e};')
                dx_terms.append((l2, j, f'r{l2}_{i}_{j}'))
                if l2 > 0:
                    body.append(f'    dY[{l2 * l2 + j}] = fma_(x[{i}], r{l2}_{i}_{j}, dY[{l2 * l2 + j}]);')
        assert dx_terms
        l2_, j_, r_ = dx_terms[0]
        e = r_ if l2_ == 0 else f'mul_({r_}, {_y(l2_, j_)})'
        for (l2_, j_, r_) in dx_terms[1:]:
            e = f'add_({r_}, {e})' if l2_ == 0 else f'fma_({_y(l2_, j_)}, {r_}, {e})'
        body.append(f'    dx[{i}] = {e};')
    out += body
    out.append('  }')
    out.append('};')
    return '\n'.join(out)


def op_counts(l1: int, lf: int, lo: int):
    """FP32 flops per (edge, channel) of the generated forward / backward bodies (fma = 2, mul/add = 1),
    used by bench.py for the FP32-pipe fraction of the convolution kernels."""
    import re
    text = gen_kind(l1, lf, lo)
    fwd = text[text.index('static void fwd('):text.index('static void bwd(')]
    bwd = text[text.index('static void bwd('):]
    count = lambda t: 2 * len(re.findall(r'fma_\(', t)) + len(re.findall(r'mul_\(', t)) + len(re.findall(r'add_\(', t))
    return count(fwd), count(bwd), len(kind_paths(l1, lf, lo))


def gen_sh(lmax: int) -> str:
    """sh_eval<L>: unit vector -> Y[1..];  sh_vjp<L>: g_c = sum_j gY[j] dY_j/du_c (c = x,y,z)."""
    import sympy as sp
    polys = sh_polynomials(lmax)
    n = len(polys)
    lines = [f'template <> struct SH<{lmax}> {{', f'  static constexpr int NY = {n};',
             '  // Y[0] = 1 is implicit; writes Y[1..NY-1]',
             '  S7B_HD static void eval(float x, float y, float z, float* __restrict__ Y) {',
             '    Y[0] = 1.0f;']
    exprs = [sp.nsimplify(p) for p in polys[1:]]
    repl, red = sp.cse([sp.N(sp.horner(e, wrt=Y) if e.has(Y) else e, 12) for e in exprs], optimizations='basic')
    for s, e in repl:
        lines.append(f'    const float {s} = {_cc(e)};')
    for j, e in enumerate(red):
        lines.append(f'    Y[{j + 1}] = {_cc(e)};')
    lines.append('  }')
    lines.append('  // vector-Jacobian product w.r.t. the (unconstrained) unit-vector components')
    lines.append('  S7B_HD static void vjp(float x, float y, float z, const float* __restrict__ gY,')
    lines.append('                                float& gx, float& gy, float& gz) {')
    gsym = sp.symbols(f'g1:{n}', real=True)
    tot = sum(g * p for g, p in zip(gsym, polys[1:]))
    grads = [sp.N(sp.expand(sp.diff(tot, v)), 12) for v in (X, Y, Z)]
    repl, red = sp.cse(grads, optimizations='basic')
    sub = {str(g): f'gY[{j + 1}]' for j, g in enumerate(gsym)}
    for s, e in repl:
        lines.append(f'    const float {s} = {_cc(e, sub)};')
    for nme, e in zip(('gx', 'gy', 'gz'), red):
        lines.append(f'    {nme} = {_cc(e, sub)};')
    lines.append('  }')
    lines.append('};')
    return '\n'.join(lines)


def gen_sh2(lmax: int) -> str:
    """SH2<L>::jvp: dY[j] = sum_c dY_j/du_c t_c (j = 1..);  SH2<L>::hvp: h_c = sum_d d2(gY . Y)/du_c du_d t_d,
    both w.r.t. the unconstrained unit-vector components like SH<L>::vjp (the Hessian-vector product's edge terms)."""
    import sympy as sp
    polys = sh_polynomials(lmax)
    n = len(polys)
    tsym = sp.symbols('tx ty tz', real=True)
    lines = [f'template <> struct SH2<{lmax}> {{',
             '  // Jacobian-vector product: writes dY[1..NY-1] (dY[0] = 0)',
             '  S7B_HD static void jvp(float x, float y, float z, float tx, float ty, float tz, float* __restrict__ dY) {',
             '    dY[0] = 0.0f;']
    jv = [sp.N(sp.expand(sum(sp.diff(p, v) * t for v, t in zip((X, Y, Z), tsym))), 12) for p in polys[1:]]
    repl, red = sp.cse(jv, optimizations='basic')
    for s, e in repl:
        lines.append(f'    const float {s} = {_cc(e)};')
    for j, e in enumerate(red):
        lines.append(f'    dY[{j + 1}] = {_cc(e)};')
    lines.append('  }')
    lines.append('  // Hessian of gY . Y(u) times t')
    lines.append('  S7B_HD static void hvp(float x, float y, float z, const float* __restrict__ gY, float tx, float ty,')
    lines.append('                         float tz, float& hx, float& hy, float& hz) {')
    gsym = sp.symbols(f'g1:{n}', real=True)
    tot = sum(g * p for g, p in zip(gsym, polys[1:]))
    hv = [sp.N(sp.expand(sum(sp.diff(tot, a, b) * t for b, t in zip((X, Y, Z), tsym))), 12) for a in (X, Y, Z)]
    repl, red = sp.cse(hv, optimizations='basic')
    sub = {str(g): f'gY[{j + 1}]' for j, g in enumerate(gsym)}
    for s, e in repl:
        lines.append(f'    const float {s} = {_cc(e, sub)};')
    for nme, e in zip(('hx', 'hy', 'hz'), red):
        lines.append(f'    {nme} = {_cc(e, sub)};')
    lines.append('  }')
    lines.append('};')
    return '\n'.join(lines)


def _cc(expr, sub=None) -> str:
    import sympy as sp
    from sympy.printing.c import C99CodePrinter

    class P(C99CodePrinter):
        def _print_Float(self, e):
            return _f(float(e))

        def _print_Integer(self, e):
            return f'{int(e)}.0f'

        def _print_Rational(self, e):
            return _f(float(e))

        def _print_Pow(self, e):
            b, ex = e.as_base_exp()
            if ex.is_Integer and 1 < int(ex) <= 4:
                return '(' + '*'.join([self._print(b)] * int(ex)) + ')'
            return super()._print_Pow(e)

        def _print_Symbol(self, e):
            if sub and str(e) in sub:
                return sub[str(e)]
            return str(e)

    return P().doprint(expr)


HEADER = '''// GENERATED by sevenn_b200/csrc/gen_kernels.py -- do not edit by hand.
#pragma once
#include "../vec_ops.cuh"
'''


def main():
    gen_dir = os.path.join(HERE, 'generated')
    os.makedirs(gen_dir, exist_ok=True)
    tp = HEADER + 'namespace s7b {\ntemplate <int L1, int LF, int LO> struct TPKind;\n\n'
    tp += ''.join(gen_kind(*k) + '\n\n' for k in KINDS) + '}  // namespace s7b\n'
    sh = HEADER + 'namespace s7b {\ntemplate <int LMAX> struct SH;\n\n'
    sh += ''.join(gen_sh(lmax) + '\n\n' for lmax in (1, 2, 3)) + '}  // namespace s7b\n'
    # second order (Hessian-vector products), appended so that the first-order text above stays as it is
    sh += '\n// second order: SH2<L>::jvp / SH2<L>::hvp\nnamespace s7b {\ntemplate <int LMAX> struct SH2;\n\n'
    sh += ''.join(gen_sh2(lmax) + '\n\n' for lmax in (1, 2, 3)) + '}  // namespace s7b\n'
    for fname, text in (('tp_kinds.cuh', tp), ('sh.cuh', sh)):
        path = os.path.join(gen_dir, fname)
        if not os.path.exists(path) or open(path).read() != text:   # keep mtimes for make
            with open(path, 'w') as f:
                f.write(text)
    print('generated', [os.path.join(gen_dir, n) for n in ('tp_kinds.cuh', 'sh.cuh')])


if __name__ == '__main__':
    main()
