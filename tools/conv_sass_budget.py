"""Static instruction budget of the convolution kernels' edge loops, on the CPU (no GPU needed).

Compiles the convolution groups (sevenn_b200/csrc/conv_group_*.cu) for sm_90a with nvcc, finds each
conv_fwd_kernel / conv_bwd_kernel instantiation in `cuobjdump -sass`, takes its edge loop (the longest
conditional backward branch: the loop body runs from the branch target to the branch) and prints per loop
iteration the SASS instructions in total, the FP32 arithmetic among them (FFMA / FMUL / FADD) and the rest
("other": address arithmetic, loads, shuffles, conversions, predicates, branches), plus registers and spill
bytes from `-Xptxas -v`.  One iteration handles one edge of a row, or two with 16 lanes per node (one per
half warp).  The counts are static: every instruction of the loop body once, including the edge-record refill
that runs once per 16 or 32 edges.

    python tools/conv_sass_budget.py [--groups 22 20 33 30 ...] [--all]

By default only the kernels the engine launches in table mode are listed (table radial weights; backward
with dx, and without dx for l1 = 0 as the first layer uses it); --all lists every instantiation.  The groups
default to all twelve (lmax_filter 1..3, lmax_out 0..3).  The first template argument after the kind is the
channel width: 128 / 64 / 32 for the kernels specialised to SevenNet-0 / SevenNet-l3i5, 0 for the runtime-width
kernels (any multiple of 32, read from ConvRole::mul), so the groups 22 / 20 / 33 / 30 list the same kind at its
compiled and at the runtime width side by side.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
CSRC = os.path.join(ROOT, 'sevenn_b200', 'csrc')
FP32 = ('FFMA', 'FMUL', 'FADD')


def _cuda_bin(name):
    home = os.environ.get('CUDA_HOME', '/usr/local/cuda')
    path = os.path.join(home, 'bin', name)
    return path if os.path.exists(path) else name


def compile_group(group, tmp):
    """-> (sass text, ptxas -v text) of conv_group_<group>.cu"""
    cubin = os.path.join(tmp, f'conv_group_{group}.cubin')
    cmd = [_cuda_bin('nvcc'), '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
           '--expt-relaxed-constexpr', '-Xptxas', '-v', '-cubin', '-o', cubin,
           os.path.join(CSRC, f'conv_group_{group}.cu')]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode:
        sys.exit(f'nvcc failed for conv_group_{group}.cu:\n{r.stderr}')
    sass = subprocess.run([_cuda_bin('cuobjdump'), '-sass', cubin], capture_output=True, text=True, check=True).stdout
    return sass, r.stderr


def demangle(names):
    r = subprocess.run(['c++filt'], input='\n'.join(names), capture_output=True, text=True, check=True)
    return r.stdout.split('\n')[:len(names)]


def ptxas_usage(text):
    """{mangled name: (registers, spill store bytes, spill load bytes)}"""
    out, cur, spill = {}, None, (0, 0)
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m:
            spill = (int(m.group(1)), int(m.group(2)))
            continue
        m = re.search(r'Used (\d+) registers', line)
        if m and cur:
            out[cur] = (int(m.group(1)),) + spill
            cur, spill = None, (0, 0)
    return out


def edge_loop(body):
    """(total, fp32) instructions of the longest conditional backward branch's range"""
    ins = [(int(a, 16), t.strip()) for a, t in re.findall(r'/\*([0-9a-f]{4,})\*/\s+([^;]*);', body)]
    best = None
    for addr, text in ins:
        m = re.match(r'@!?U?P\w+\s+BRA\s+(?:`\()?(?:\S+\s+)?0x([0-9a-f]+)', text)
        if m:
            target = int(m.group(1), 16)
            if target < addr and (best is None or addr - target > best[1] - best[0]):
                best = (target, addr)
    if best is None:
        return None
    loop = [t for a, t in ins if best[0] <= a <= best[1] and not t.startswith('NOP')]
    opcode = lambda t: re.sub(r'^@!?U?P\w+\s+', '', t).split()[0].split('.')[0]
    fp32 = sum(1 for t in loop if opcode(t) in FP32)
    return len(loop), fp32


def describe(demangled):
    """('fwd'|'bwd', l1, lmax_filter, lmax_out, rest of the template arguments)"""
    m = re.match(r'void s7b::conv_(fwd|bwd)_kernel<s7b::TPKind<(\d+), (\d+), (\d+)>, (.*)>\(', demangled)
    if not m:
        return None
    return m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4)), m.group(5).replace('float2', 'V2')


def launched_in_table_mode(kind, l1, args):
    """table radial weights; the backward with dx (and for l1 = 0 also without: first layer)"""
    flags = [a.strip() for a in args.split(',') if a.strip() in ('true', 'false')]
    if not flags or flags[0] != 'true':
        return False
    if kind == 'bwd' and len(flags) > 1 and flags[1] != 'true' and l1 != 0:
        return False
    return True


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--groups', nargs='+', default=[f'{lf}{lo}' for lf in (1, 2, 3) for lo in range(4)],
                    help='(lmax_filter, lmax_out) groups, as in conv_group_<LFLO>.cu')
    ap.add_argument('--all', action='store_true', help='every instantiation, not only those table mode launches')
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp, ThreadPoolExecutor(len(args.groups)) as pool:
        results = list(pool.map(lambda g: (g,) + compile_group(g, tmp), args.groups))
    print(f'{"group":>5} {"dir":>3} {"l1":>2}  {"template args":<34} {"SASS/it":>7} {"FP32":>5} {"other":>5} '
          f'{"other%":>6} {"regs":>4} {"spill":>5}')
    for group, sass, ptxas in results:
        usage = ptxas_usage(ptxas)
        funcs = re.split(r'\n\s+Function : ', sass)[1:]
        names = [f.split('\n', 1)[0].strip() for f in funcs]
        rows = []
        for name, dem, body in zip(names, demangle(names), funcs):
            d = describe(dem)
            if d is None:
                continue
            kind, l1, lf, lo, targs = d
            if not args.all and not launched_in_table_mode(kind, l1, targs):
                continue
            loop = edge_loop(body)
            regs, st, ld = usage.get(name, (-1, 0, 0))
            rows.append((kind, l1, targs, loop, regs, st + ld))
        for kind, l1, targs, loop, regs, spill in sorted(rows, key=lambda r: (r[0] != 'fwd', r[1], r[2])):
            tot, fp = loop if loop else (0, 0)
            other = tot - fp
            print(f'{group:>5} {kind:>3} {l1:>2}  {targs:<34} {tot:>7} {fp:>5} {other:>5} '
                  f'{100.0 * other / max(tot, 1):>5.0f}% {regs:>4} {spill:>5}')


if __name__ == '__main__':
    main()
