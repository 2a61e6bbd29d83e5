"""The engine against the fp64 oracle on the adversarial graphs of tests/graphs.py (GPU, `pytest -m gpu`):
rows of 0 - 166 edges next to each other, every edge-record refill boundary, 1 - 256 atoms across the
64-row tensor-core, 128-row SIMT and 8-node conv tiles, every species, edges at both ends of the radial table
and a cell smaller than the cutoff; both models, both radial modes, and a subset with the FP32 SIMT linears.

Tolerances follow the fp32 error model: an absolute floor (the suite's usual one) plus a relative term on the
reference's own scale, taken per connected component of the graph (the radial_edges dimers are independent
systems whose forces span 1 - 1e3 eV/A):
    forces, edge forces   |dF| <= 1e-4 + 2e-5 max|F_ref|                 eV/A
    atomic energies       |dE_i| <= 3e-5 + 1.5e-5 max|E_ref_i|           eV
    total energy          |dE| <= (3e-5 + 3e-6 max|E_ref_i|) sqrt(n)     (independent roundings per atom)
    virial                |dW| <= 2e-4 + 5e-5 max|W_ref|                  eV
Force bounds of a component holding an edge shorter than 0.5 A use 3x the relative term (short_pair_factor).
The relative terms are ~100 - 300 fp32 ulps: a force is a sum of up to 2 x 166 edge forces, each the end of
five layers of fp32 sums over 128 - 480 channels, and where edge forces cancel (ragged: 1.6 A contacts, edge
forces far above the net forces) the error follows the edge forces, not max|F|.  The force bounds stay inside the
project tolerance (1e-3 eV/A) except on the 0.2 A H-H dimer of radial_edges (910 eV/A with SevenNet-0), where
fp32 resolution alone exceeds it; the total-energy bound exceeds 1e-4 eV from ~16 atoms on, as does the 12 000-atom
parity bound of bench.py (1.25e-5 eV sqrt(n)).
A failing comparison names the first intermediate that diverges (helpers.stage_errors).  The negative control
shows that these bounds catch a 2 % change of the radial weights of one path of one middle layer.

Measured on one H100 80GB HBM3 (SXM, 700 W): worst case per fixture over both models, both radial modes,
tensor-core and SIMT linears (the test prints one `ADV ...` line per run):
    fixture     longest row  |dE|/atom  max|dE_i|  max|dF| eV/A  rel |dW|
    dense              86     7.6e-07    1.2e-05    7.8e-05      2.1e-06
    hub               166     2.7e-07    6.2e-06    2.0e-05      2.7e-06
    ragged             65     3.8e-07    5.8e-05    4.7e-04      4.0e-06
    isolated           19     6.6e-07    3.5e-06    3.1e-05      3.8e-06
    many_species       30     4.1e-07    6.4e-06    1.2e-04      2.5e-06
    radial_edges        1     1.4e-05    1.1e-04    5.1e-03      1.4e-05   (0.2 A H-H: |F| up to 910 eV/A)
    tiny_cell          60     3.9e-07    2.6e-06    9.6e-06      5.9e-06
    sizes_1 .. 9     0 - 8    2.2e-06    2.4e-05    2.1e-05      9.5e-06
    sizes_63 .. 129 26 - 46   5.4e-07    2.0e-05    9.7e-05      2.8e-05
"""
import functools

import numpy as np
import pytest

import graphs
from helpers import first_divergence, format_stage_errors, model_weights, oracle, stage_errors

pytestmark = pytest.mark.gpu

MODELS = ['sevennet_0', 'sevennet_l3i5']
F_ABS, F_REL = 1e-4, 2e-5
E_ABS, E_REL = 3e-5, 1.5e-5
ET_REL = 3e-6
W_ABS, W_REL = 2e-4, 5e-5
SIMT_SUBSET = ['dense', 'hub', 'ragged', 'isolated', 'sizes_65', 'sizes_129']


@functools.lru_cache(maxsize=None)
def reference(model, fixture):
    g = graphs.fixture(fixture, model)
    r = oracle(model).forward(g.species, g.edge_index, g.edge_vec, volume=g.volume)
    return {k: (v.numpy() if hasattr(v, 'numpy') else v) for k, v in r.items()}


@functools.lru_cache(maxsize=None)
def components(model, fixture):
    """connected-component label of every atom (edges taken as undirected)"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    g = graphs.fixture(fixture, model)
    n = len(g.species)
    a = coo_matrix((np.ones(g.edge_index.shape[1]), (g.edge_index[0], g.edge_index[1])), shape=(n, n))
    return connected_components(a, directed=False)[1]


@functools.lru_cache(maxsize=None)
def short_pair_factor(model, fixture):
    """per atom: 3 in a component holding an edge shorter than 0.5 A, else 1.  There dE/dr of the Bessel basis,
    (2/rc)(c cos(cr)/r - sin(cr)/r^2), is a difference of terms several times its size: fp32 loses more digits."""
    g = graphs.fixture(fixture, model)
    comp = components(model, fixture)
    short = np.zeros(comp.max() + 1, dtype=bool)
    r = np.linalg.norm(g.edge_vec, axis=1)
    short[comp[g.edge_index[0][r < 0.5]]] = True
    return np.where(short[comp], 3.0, 1.0)


def _scale(values, comp):
    """per atom (or edge): max |value| over its connected component"""
    v = np.abs(values).reshape(len(comp), -1).max(1)
    m = np.zeros(comp.max() + 1)
    np.maximum.at(m, comp, v)
    return m[comp]


@pytest.fixture(scope='module')
def engines():
    from sevenn_b200.engine import B200Engine
    cache = {}

    def get(name, radial, atomic_virial=False, arrays=None):
        key = (name, radial, atomic_virial)
        if arrays is not None:
            meta, _ = model_weights(name)
            return B200Engine(meta, arrays, radial=radial, atomic_virial=atomic_virial)
        if key not in cache:
            meta, arr = model_weights(name)
            cache[key] = B200Engine(meta, arr, radial=radial, atomic_virial=atomic_virial)
        return cache[key]
    return get


def run(e, g):
    import torch
    e.set_graph(g.species, g.edge_index, g.edge_vec)
    e.compute()
    torch.cuda.synchronize()
    r = e.results()
    out = dict(energy=float(r['energy'].cpu()[0]), atomic_energy=r['atomic_energy'].cpu().numpy().astype(np.float64),
               forces=r['forces'].cpu().numpy().astype(np.float64), virial=r['virial'].cpu().numpy(),
               edge_force=r['edge_force'].cpu().numpy().astype(np.float64))
    if e.atomic_virial:
        out['atomic_virial'] = e.buffer('atomic_virial', shape=(len(g.species), 6)).cpu().numpy().astype(np.float64)
    perm = e._graph['perm']
    out['perm'] = None if perm is None else perm.cpu().numpy()
    return out


def errors(model, fixture, out, ref):
    """{quantity: (max error, max allowed)} with the bounds of the module docstring"""
    g = graphs.fixture(fixture, model)
    comp = components(model, fixture)
    n = len(g.species)
    res = {}
    ae = ref['atomic_energy']
    res['energy'] = (abs(out['energy'] - float(ref['energy'])),
                     (E_ABS + ET_REL * np.abs(ae).max()) * np.sqrt(n))
    res['atomic_energy'] = (np.abs(out['atomic_energy'] - ae), E_ABS + E_REL * _scale(ae, comp))
    cond = short_pair_factor(model, fixture)
    res['forces'] = (np.abs(out['forces'] - ref['forces']).max(1), F_ABS + F_REL * cond * _scale(ref['forces'], comp))
    if g.edge_index.shape[1]:
        centre = g.edge_index[0] if out['perm'] is None else g.edge_index[0][out['perm']]
        fe = ref['edge_force'] if out['perm'] is None else ref['edge_force'][out['perm']]
        res['edge_force'] = (np.abs(out['edge_force'] - fe).max(1),
                             F_ABS + F_REL * cond[centre] * _scale(fe, comp[centre]))
    res['virial'] = (np.abs(out['virial'] - ref['virial']).max(), W_ABS + W_REL * np.abs(ref['virial']).max())
    if 'atomic_virial' in out:
        av = ref['atomic_virial']
        res['atomic_virial'] = (np.abs(out['atomic_virial'] - av).max(1), W_ABS + W_REL * _scale(av, comp))
    return res


def failures(res):
    return [k for k, (err, tol) in res.items() if not np.all(np.asarray(err) <= tol)]


def check(e, model, fixture, tag, out=None):
    g = graphs.fixture(fixture, model)
    ref = reference(model, fixture)
    out = run(e, g) if out is None else out
    res = errors(model, fixture, out, ref)
    n = len(g.species)
    rel_w = res['virial'][0] / max(np.abs(ref['virial']).max(), 1e-30)
    print(f'ADV {model} {tag} {fixture}: rows<={graphs.degrees(g).max()} |dE|/atom {res["energy"][0] / n:.2e} '
          f'|dE_i| {res["atomic_energy"][0].max():.2e} |dF| {res["forces"][0].max():.2e} rel |dW| {rel_w:.2e}')
    bad = failures(res)
    if bad:
        meta, arrays = model_weights(model)
        full = oracle(model).forward(g.species, g.edge_index, g.edge_vec, keep=True)
        st = stage_errors(e, arrays, g.species, g.edge_index, g.edge_vec, full)
        worst = {k: float(np.max(np.asarray(res[k][0]) - res[k][1])) for k in bad}
        pytest.fail(f'{model} {tag} {fixture}: {bad} out of bounds (worst excess {worst}); first divergence: '
                    f'{first_divergence(st)}\n{format_stage_errors(st)}')


@pytest.mark.parametrize('fixture', graphs.FIXTURES)
@pytest.mark.parametrize('radial', ['table', 'mlp'])
@pytest.mark.parametrize('model', MODELS)
def test_engine_matches_oracle(engines, model, radial, fixture):
    check(engines(model, radial), model, fixture, f'{radial} tc')


@pytest.mark.parametrize('fixture', SIMT_SUBSET)
@pytest.mark.parametrize('model', MODELS)
def test_engine_with_simt_linears_matches_oracle(engines, model, fixture):
    from sevenn_b200.engine import set_option
    e = engines(model, 'table')
    g = graphs.fixture(fixture, model)
    try:
        set_option('tc_gemm', 0)
        out = run(e, g)
    finally:
        set_option('tc_gemm', 1)
    check(e, model, fixture, 'table simt', out)


@pytest.mark.parametrize('fixture', ['dense', 'hub'])
@pytest.mark.parametrize('model', MODELS)
def test_atomic_virial_matches_oracle(engines, model, fixture):
    e = engines(model, 'table', atomic_virial=True)
    check(e, model, fixture, 'table atomic-virial')
    out = run(e, graphs.fixture(fixture, model))
    assert np.allclose(out['atomic_virial'].sum(0), out['virial'], rtol=1e-5, atol=W_ABS)


def test_negative_control_one_path_of_one_layer(engines):
    """2 % on the radial weights of path (l1, l2, l3) = (2, 2, 0) of layer 2: the oracle's own forces move by
    more than 5x the force bound, and the engine run with these weights fails the comparison with the
    unperturbed oracle (and passes the one with the perturbed oracle)."""
    from oracle.oracle import Oracle
    from sevenn_b200.spec import build_spec
    model, fixture, eps = 'sevennet_0', 'sizes_65', 2e-2
    meta, arrays = model_weights(model)
    p = next(p for p in build_spec(meta).layers[2].paths if (p.l1, p.l2, p.l3) == (2, 2, 0))
    orig = np.array(arrays['2.mlp2'], copy=True)
    bumped = dict(arrays)
    w = np.array(arrays['2.mlp2'], copy=True)
    w[:, p.w_off:p.w_off + p.mul] *= 1.0 + eps
    bumped['2.mlp2'] = w
    g = graphs.fixture(fixture, model)
    ref = reference(model, fixture)
    ref_b = Oracle(meta, bumped).forward(g.species, g.edge_index, g.edge_vec, volume=g.volume)
    ref_b = {k: (v.numpy() if hasattr(v, 'numpy') else v) for k, v in ref_b.items()}
    f_tol = F_ABS + F_REL * np.abs(ref['forces']).max()
    assert np.abs(ref_b['forces'] - ref['forces']).max() >= 5 * f_tol
    out = run(engines(model, 'table', arrays=bumped), g)
    assert 'forces' in failures(errors(model, fixture, out, ref))
    assert not failures(errors(model, fixture, out, ref_b))
    assert np.array_equal(model_weights(model)[1]['2.mlp2'], orig)          # the cached weights are untouched
