"""The serial LAMMPS pair style's per-atom centroid virial (examples/lammps/pair_e3gnn_b200.cpp) inside
tests/mock_lammps_centroid/harness_centroid.cpp, against the CPU double of the library (tests/mock_lammps/stub_s7b.cpp)
and the harness's toy centroid rows: with the Pair declarations that carry the centroid members the style advertises
CENTROID_AVAIL and, when the centroid flag is set, fills cvatom with the library's rows in LAMMPS's order
(xx yy zz xy xz yz yx zx zy, xy = Wc[x][y]).  Against tests/mock_lammps (a Pair without those members) it still builds,
which tests/test_host_logic.py checks."""
import os
import subprocess

from helpers import ROOT


def test_serial_pair_style_fills_cvatom_in_lammps_order(tmp_path):
    mock = os.path.join(ROOT, 'tests', 'mock_lammps_centroid')
    ex = os.path.join(ROOT, 'examples', 'lammps')
    exe = str(tmp_path / 'harness_centroid')
    subprocess.run(['g++', '-std=c++17', '-O1', '-Wall', '-Werror', '-I', mock, '-I', ex,
                    os.path.join(mock, 'harness_centroid.cpp'), os.path.join(ex, 'pair_e3gnn_b200.cpp'),
                    os.path.join(ROOT, 'tests', 'mock_lammps', 'stub_s7b.cpp'), '-o', exe], check=True)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(p.stdout)
    assert p.returncode == 0 and p.stdout.strip().endswith('OK'), p.stdout + p.stderr


def test_only_the_serial_style_advertises_centroid_support():
    serial = open(os.path.join(ROOT, 'examples', 'lammps', 'pair_e3gnn_b200.cpp')).read()
    parallel = open(os.path.join(ROOT, 'examples', 'lammps', 'pair_e3gnn_b200_parallel.cpp')).read()
    mliap = open(os.path.join(ROOT, 'sevenn_b200', 'mliap.py')).read()
    assert 'self->centroidstressflag = 1' in serial
    assert 'CENTROID_AVAIL' not in parallel and 'centroid' not in mliap.lower()


def test_export_flat_radial_mlp_adds_the_mlp_to_a_table_file(tmp_path):
    import ctypes
    import struct
    from sevenn_b200.engine import S7bModelDesc, default_table_knots, prepare_params
    from sevenn_b200.export import export_flat
    from sevenn_b200.spec import build_spec
    from helpers import model_weights
    meta, arrays = model_weights('sevennet_0')
    spec = build_spec(meta)
    path = str(tmp_path / 'm.s7b')
    export_flat(path, meta, arrays, radial_mlp=True)
    want = dict(prepare_params(spec, arrays, 'table', default_table_knots(spec)))
    want.update({k: v for k, v in prepare_params(spec, arrays, 'mlp', 0).items() if k[0] in ('mlp0', 'mlp1', 'mlp2')})
    with open(path, 'rb') as f:
        f.read(12 + ctypes.sizeof(S7bModelDesc))
        n_arrays, n_types = struct.unpack('<ii', f.read(8))
        f.read(8 * n_types)
        seen = set()
        for _ in range(n_arrays):
            name = f.read(32).rstrip(b'\0').decode()
            layer, numel = struct.unpack('<iq', f.read(12))
            assert numel == want[(name, layer)].size
            f.read(4 * numel)
            seen.add((name, layer))
    assert seen == set(want) and ('mlp0', 0) in seen and ('table', 0) in seen
