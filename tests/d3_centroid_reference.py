"""fp64 reference for D3's per-atom centroid virial (DESIGN.md §8.6), for tests/test_d3_centroid_virial_*.py.

With D3's atomic energies U_j = -1/2 sum_{k,tau} C6_jk(CN_j, CN_k) g(r_jk) (self images included, as
``d3_flux_reference``), Wc_i[a, b] = sum_j sum_i' (r_j - r_i')_a dU_j/dr_i',b over atom i and its periodic images i'.
A numpy restatement of the three parts the kernels sum, on the periodic cell with all its images, with
vec_ik = r_k + tau - r_i and u = vec / r:

* direct part (explicit r at fixed CN): sum_k 1/2 C6 g'/r vec (x) vec, the forward pair pass's per-atom ``spair``;
* beta_i = sum_{j, images} dU_j/dCN_i (r_j' - r_i) = -1/2 sum_k g dC6_ik/dCN_i vec_ik (vdW radius);
* CN part: -sum_m f'(r_im) (beta_m + beta_i + alpha_m vec_im) (x) u_im over the CN radius (strict bound, as the
  forward's chain pass), alpha_m = dE/dCN_m and f' the derivative of the counting function.

The pair enumeration and damping are ``d3_flux_reference``'s; C6_ik, CN and alpha = -dc6i come from the fp64 oracle.
Only dC6_ik/dCN_i, which neither exposes per pair, is formed here from the oracle's coordination numbers.  Summed over
i, Wc is the virial; contracted with velocities, sum_i Wc_i v_i is ``recursion_flux``'s J_pot.
"""
import numpy as np

from d3_flux_reference import AU_TO_EV, K1, K3, _damping, _pairs, _wrapped


def _dc6_dcn_i(z, cn):
    """[n, n] dC6_ik/dCN_i of the normalised Gaussian weights at the coordination numbers cn (zero where the weight
    product underflows, den <= 1e-99, as the oracle and the kernels)"""
    from oracle.d3_oracle import d3_params
    P = d3_params()
    cnr, mxc = P['cnref'][z], P['mxc'][z]
    valid = np.arange(5)[None, :] < mxc[:, None]
    w = np.where(valid, np.exp(K3 * (cnr - cn[:, None]) ** 2), 0.0)
    dw = w * 2.0 * K3 * (cn[:, None] - cnr)
    c6r = P['c6ref'][z[:, None], z[None, :]]
    den = np.einsum('ia,jb->ij', w, w)
    ok = den > 1e-99
    sden = np.where(ok, den, 1.0)
    c6 = np.einsum('ijab,ia,jb->ij', c6r, w, w) / sden
    return np.where(ok, (np.einsum('ijab,ia,jb->ij', c6r, dw, w) - c6 * np.einsum('ia,jb->ij', dw, w)) / sden, 0.0)


def _cn_pairs(z, x, lat, pbc, cn_cutoff):
    """CN pairs inside the strict bound: (I, J, vec, r, f' = dCN/dr of the counting function)"""
    from oracle.d3_oracle import d3_params
    I, J, d, r = _pairs(x, lat, pbc, cn_cutoff)
    keep = r * r < cn_cutoff
    I, J, d, r = I[keep], J[keep], d[keep], r[keep]
    rcov = d3_params()['rcov'][z]
    rc = rcov[I] + rcov[J]
    ex = np.exp(-K1 * (rc / r - 1.0))
    return I, J, d, r, -K1 * rc * ex / (r * r * (1.0 + ex) ** 2)


def centroid_virials(numbers, positions, cell, pbc, damping, vdw_cutoff, cn_cutoff, parts=False):
    """Wc [n, 3, 3] in eV, row a the flux (moment) direction, column b the velocity direction; with ``parts``
    (Wc, direct part, CN part), each [n, 3, 3] in eV"""
    from oracle.d3_oracle import d3_reference
    z = np.asarray(numbers, dtype=np.int64) - 1
    n = len(z)
    ora = d3_reference(numbers, positions, cell, pbc, damping=damping, functional='pbe', vdw_cutoff=vdw_cutoff,
                       cn_cutoff=cn_cutoff)
    x, lat = _wrapped(positions, cell)
    dc6 = _dc6_dcn_i(z, ora['cn'])
    I, J, d, r = _pairs(x, lat, pbc, vdw_cutoff)
    g, dg = _damping(z, I, J, r, damping)
    direct = np.zeros((n, 3, 3))
    np.add.at(direct, I, (0.5 * ora['c6'][I, J] * dg / r)[:, None, None] * d[:, :, None] * d[:, None, :])
    beta = np.stack([np.bincount(I, weights=-0.5 * g * dc6[I, J] * d[:, a], minlength=n) for a in range(3)], 1)
    alpha = -ora['dc6i']
    I, J, d, r, f1 = _cn_pairs(z, x, lat, pbc, cn_cutoff)
    mom = beta[J] + beta[I] + alpha[J][:, None] * d
    cnp = np.zeros((n, 3, 3))
    np.add.at(cnp, I, -(f1 / r)[:, None, None] * mom[:, :, None] * d[:, None, :])
    direct, cnp = direct * AU_TO_EV, cnp * AU_TO_EV
    return (direct + cnp, direct, cnp) if parts else direct + cnp


def pairwise_split(numbers, positions, cell, pbc, damping, vdw_cutoff, cn_cutoff):
    """the forward's per-atom virial rows spair_i + schain_i as [n, 3, 3] in eV (symmetric): a split that sums to the
    virial but is not the centroid virial of D3's many-body atomic energies"""
    from oracle.d3_oracle import d3_reference
    z = np.asarray(numbers, dtype=np.int64) - 1
    n = len(z)
    dc6i = d3_reference(numbers, positions, cell, pbc, damping=damping, functional='pbe', vdw_cutoff=vdw_cutoff,
                        cn_cutoff=cn_cutoff)['dc6i']
    _, direct, _ = centroid_virials(numbers, positions, cell, pbc, damping, vdw_cutoff, cn_cutoff, parts=True)
    x, lat = _wrapped(positions, cell)
    I, J, d, r, f1 = _cn_pairs(z, x, lat, pbc, cn_cutoff)
    chain = np.zeros((n, 3, 3))
    np.add.at(chain, I, (0.5 * f1 * (dc6i[I] + dc6i[J]) / r)[:, None, None] * d[:, :, None] * d[:, None, :])
    return direct + chain * AU_TO_EV
