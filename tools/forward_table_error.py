"""Error of the forward's radial value table against the fp64 radial MLP, on the CPU.

The forward convolution interpolates w(r) linearly in a table of values on a grid three times finer than the
backward's cubic table (engine.py ``forward_table_knots`` / ``radial_value_table``).  For every layer of the two
pretrained models and of the radial shapes of tests/radial_models.py (cutoffs 4.0 / 5.0 / 5.3 / 6.0, XPLOR and
polynomial envelopes), plus R2 with XPLOR r_on = 4.123456789 (on no knot of any grid the knot rule can pick), this
reads the table as the kernel does (``value_table_read``) and prints:
  * max and rms of |w - w_fp64| over max |w|, at 3000 random fp32 radii in [1.5, cutoff) (seed 0);
  * max |w - w_fp64| over the local scale at every interval of the value grid (r >= 0.2 A) and where it is worst
    (``forward_table_errors`` of tests/test_forward_table_cpu.py, which bounds both);
  * the sizes of the value table and of the cubic table it sits beside.

    python tools/forward_table_error.py [--models sevennet_0 R1 ...]
"""
import argparse
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from sevenn_b200.engine import default_table_knots, forward_table_knots, radial_value_table  # noqa: E402
from sevenn_b200.spec import build_spec  # noqa: E402
from test_forward_table_cpu import forward_table_errors  # noqa: E402


def load_model(name):
    if name.startswith('sevennet'):
        from sevenn_b200.checkpoint import load_weights
        return load_weights(os.path.join(ROOT, 'weights', f'{name}.npz'))
    import tempfile
    from radial_models import convert_radial, write_radial_checkpoint
    cid, _, r_on = name.partition('@')
    meta, arrays = convert_radial(write_radial_checkpoint(os.path.join(tempfile.mkdtemp(), f'{cid}.pth'), cid), cid)
    if r_on:
        meta = dict(meta, cutoff_on=float(r_on))
    return meta, arrays


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--models', nargs='+',
                    default=['sevennet_0', 'sevennet_l3i5', 'R1', 'R2', 'R3', 'R4', 'R5', 'R2@4.123456789'])
    args = ap.parse_args()
    print(f'{"model":16s} {"t":>2s} {"W":>5s} {"K":>5s} {"Kf":>6s} {"MiB":>6s} {"cubic":>6s} '
          f'{"max/max|w|":>10s} {"rms/max|w|":>10s} {"max/local":>10s} {"at r":>8s}')
    for name in args.models:
        meta, arrays = load_model(name)
        spec = build_spec(meta)
        K = default_table_knots(spec)
        Kf = forward_table_knots(K)
        for t in range(spec.n_layers):
            tab = radial_value_table(spec, arrays, t, Kf)
            W = tab.shape[1]
            e_max, e_rms, e_loc, at = forward_table_errors(spec, arrays, t, tab)
            print(f'{name:16s} {t:2d} {W:5d} {K:5d} {Kf:6d} {tab.nbytes / 2**20:6.1f} {K * W * 12 / 2**20:6.1f} '
                  f'{e_max:10.2e} {e_rms:10.2e} {e_loc:10.2e} {at:8.4f}')

if __name__ == '__main__':
    main()
