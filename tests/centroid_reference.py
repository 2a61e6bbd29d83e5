"""fp64 reference per-atom centroid virial on the oracle alone (DESIGN.md §8.5), for tests/test_centroid_virial_*.py.

For atomic energies U_j of a cluster (no periodic images), with E = sum_j U_j and Phi_a = sum_j r_j,a U_j:

  Wc_i[a, b] = sum_j (r_j - r_i)_a dU_j/dr_i,b = dPhi_a/dr_i,b - r_i,a dE/dr_i,b

from four reverse passes of the oracle, each with the atomic energies weighted per atom (by 1, then by r_j,a): the
oracle's edge forces of sum_j c_j U_j, scattered onto the atoms.  A periodic cell is evaluated on its unfolded cluster
(flux_reference.unfold): j runs over the cell's own atoms, i over every atom of the cluster, and each image's row is
added onto its parent's."""
import numpy as np

from flux_reference import cluster_graph, unfold


def weighted_gradients(o, species, ei, ev, weights):
    """For each per-atom weight vector c: d(sum_j c_j U_j)/dr_i, [n, 3], with the oracle `o` (the weights multiply
    the readout's output rows, so the per-species scale is inside and the shift drops out of the gradient)"""
    import torch
    readout2 = o.w['readout2']
    base = o.linear
    n = len(species)
    out = []
    for c in weights:
        ct = torch.as_tensor(np.asarray(c, np.float64), dtype=o.dtype, device=o.device)

        def lin(x, W, *args, **kw):
            y = base(x, W, *args, **kw)
            return y * ct[:, None] if W is readout2 else y

        o.linear = lin
        try:
            f = o.forward(species, ei, ev)['edge_force'].detach().cpu().numpy().astype(np.float64)
        finally:
            del o.linear
        g = np.zeros((n, 3))
        np.add.at(g, ei[1], f)
        np.add.at(g, ei[0], -f)
        out.append(g)
    return out


def reference_centroid(o, spec, species, pos, n_cell=None):
    """(Wc [n, 3, 3] of every atom i of a cluster, the positions used) with the fp64 oracle, j < n_cell (all atoms by
    default).  Positions are made relative to the cell atoms' centroid."""
    pos = np.asarray(pos, np.float64)
    n = len(pos)
    n_cell = n if n_cell is None else n_cell
    pos = pos - pos[:n_cell].mean(0)
    ei, ev = cluster_graph(pos, spec.cutoff)
    mask = (np.arange(n) < n_cell).astype(np.float64)
    gE, *gP = weighted_gradients(o, species, ei, ev, [mask] + [mask * pos[:, a] for a in range(3)])
    Wc = np.stack(gP, axis=1) - pos[:, :, None] * gE[:, None, :]
    return Wc, pos


def reference_centroid_cell(o, spec, species, pos, cell=None):
    """Wc [n, 3, 3] of a structure: a cluster when `cell` is None, else the periodic cell through its unfolded
    cluster (radius T x cutoff + 1 A), images folded onto their parents"""
    species = np.asarray(species)
    if cell is None:
        return reference_centroid(o, spec, species, pos)[0]
    cpos, parent = unfold(pos, cell, len(spec.layers) * spec.cutoff + 1.0)
    Wc_c, _ = reference_centroid(o, spec, species[parent], cpos, n_cell=len(pos))
    Wc = np.zeros((len(pos), 3, 3))
    np.add.at(Wc, parent, Wc_c)
    return Wc
