"""fp64 reference heat flux on the oracle alone (DESIGN.md §8.3), for tests/test_heat_flux_*.py.

For atomic energies U_j and velocities v_i of a cluster (no periodic images):

  J_pot = sum_j sum_i (r_j - r_i) (dU_j/dr_i . v_i) = sum_j [ r_j dU_j(v) - dU_j(w^a) ],   w^a_i = r_i,a v_i

where dU_j(u) is the directional derivative of U_j along the displacement field u, taken here by central differences
at h and 2h combined by Richardson extrapolation, with the edge list held fixed.  A periodic cell is evaluated on its
unfolded cluster: every image within T * cutoff (+ a margin) of a cell atom, each moving with its atom's velocity;
j then runs over the cell's own atoms only."""
import numpy as np


def make_oracle(meta, arrays, device):
    import torch
    from oracle.oracle import Oracle
    from nequip_oracle import nequip_oracle
    from sevenn_b200.spec import build_spec
    make = nequip_oracle if build_spec(meta).self_connection == 'nequip' else Oracle
    return make(meta, arrays, dtype=torch.float64, device=device)


def cluster_graph(pos, cutoff):
    """edges of every pair closer than the cutoff, sorted by centre: (edge_index [2, E] = (centre, neighbour),
    edge_vec = pos[neighbour] - pos[centre])"""
    from scipy.spatial import cKDTree
    pairs = cKDTree(pos).query_pairs(cutoff, output_type='ndarray')
    if len(pairs) == 0:
        return np.zeros((2, 0), np.int64), np.zeros((0, 3))
    c = np.concatenate([pairs[:, 0], pairs[:, 1]])
    nb = np.concatenate([pairs[:, 1], pairs[:, 0]])
    order = np.lexsort((nb, c))
    ei = np.stack([c[order], nb[order]]).astype(np.int64)
    return ei, pos[ei[1]] - pos[ei[0]]


def unfold(pos, cell, radius):
    """(cluster positions, parent atom of each): the cell's atoms first, then every image within `radius` of one"""
    from scipy.spatial import cKDTree
    pos, cell = np.asarray(pos, np.float64), np.asarray(cell, np.float64)
    spacing = 1.0 / np.linalg.norm(np.linalg.inv(cell), axis=0)      # distances between lattice planes
    K = np.ceil(radius / spacing).astype(int) + 1
    n = np.stack(np.meshgrid(*[np.arange(-k, k + 1) for k in K], indexing='ij'), -1).reshape(-1, 3)
    n = n[np.argsort(np.abs(n).sum(1), kind='stable')]                # shift 0 first
    img = (pos[None, :, :] + (n @ cell)[:, None, :]).reshape(-1, 3)
    parent = np.tile(np.arange(len(pos)), len(n))
    d, _ = cKDTree(pos).query(img, k=1)
    keep = d < radius
    return img[keep], parent[keep]


def atomic_energies(o, species, ei, ev):
    return o.forward(species, ei, ev)['atomic_energy'].detach().cpu().numpy().astype(np.float64)


def directional(o, species, ei, ev, u, h):
    """dU/ds of U(edge_vec + s (u[neighbour] - u[centre])), Richardson-extrapolated central differences"""
    du = u[ei[1]] - u[ei[0]]
    U = lambda s: atomic_energies(o, species, ei, ev + s * du)
    D = lambda s: (U(s) - U(-s)) / (2 * s)
    return (4 * D(h) - D(2 * h)) / 3


def step(spec, ev, ei, fields):
    """a step that moves no edge across a kink of the radial functions (cutoff, and r_on of XPLOR) nor by more than a
    fifth of its distance from one"""
    r = np.linalg.norm(ev, axis=1)
    kinks = [spec.cutoff] + ([spec.cutoff_on] if spec.cutoff_fn == 'XPLOR' else [])
    margin = min(np.abs(r - k).min() for k in kinks)
    move = max(np.linalg.norm(u[ei[1]] - u[ei[0]], axis=1).max() for u in fields)
    return min(1e-3, margin / (5 * 2 * max(move, 1e-12)))


def reference_flux(o, spec, species, pos, v, n_cell=None):
    """(J_pot [3], per-atom contributions [n_cell, 3]) of a cluster with the fp64 oracle; j < n_cell (all atoms by
    default).  Positions are made relative to the cell atoms' centroid (J_pot is translation invariant)."""
    pos = np.asarray(pos, np.float64)
    n_cell = len(pos) if n_cell is None else n_cell
    pos = pos - pos[:n_cell].mean(0)
    ei, ev = cluster_graph(pos, spec.cutoff)
    fields = [v] + [pos[:, a:a + 1] * v for a in range(3)]
    h = step(spec, ev, ei, fields)
    dv = directional(o, species, ei, ev, v, h)[:n_cell]
    per = pos[:n_cell] * dv[:, None]
    for a in range(3):
        per[:, a] -= directional(o, species, ei, ev, fields[1 + a], h)[:n_cell]
    return per.sum(0), per


def n_layers(meta):
    from sevenn_b200.spec import build_spec
    return len(build_spec(meta).layers)
