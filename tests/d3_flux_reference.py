"""fp64 references for the D3 heat flux (DESIGN.md §8.4), for tests/test_d3_heat_flux_*.py.

D3's atomic energy is the half-pair split of the pair pass, U_j = -1/2 sum_{k,tau} C6_jk(CN_j, CN_k) g(r_jk), self
images included.  Two independent routes to J_pot = sum_j sum_i (r_j - r_i) (dU_j/dr_i . v_i):

* ``recursion_flux``: a numpy fp64 restatement of the two passes the kernels run, on the periodic cell with all its
  images (pair enumeration as oracle/d3_oracle.py, weights and dC6/dCN restated here);
* ``difference_flux``: J_pot = sum_j [r_j dU_j(v) - dU_j(w^a)], w^a_i = r_i,a v_i (as tests/flux_reference.py),
  dU_j(u) by Richardson-extrapolated central differences of ``atomic_energies``.  Those take C6_ij(CN_i, CN_j) from the
  fp64 oracle and sum -1/2 C6 g per centre; a periodic cell is evaluated on its unfolded cluster (every image within
  the vdW + CN radius of a cell atom, each moving with its atom's velocity) and j runs over the cell's atoms only.
"""
import numpy as np

AU = 0.52917726
AU_TO_EV = 27.21138505
K1, K3 = 16.0, -4.0


def _wrapped(positions, cell):
    """positions (bohr) wrapped into the cell in every direction, as the oracle and the kernels do; lattice (bohr)"""
    lat = np.asarray(cell, dtype=np.float64) / AU
    frac = (np.asarray(positions, dtype=np.float64) / AU) @ np.linalg.inv(lat)
    return (frac - np.floor(frac)) @ lat, lat


def _pairs(x, lat, pbc, cut2):
    """every ordered pair (centre i, neighbour j, translation) with r^2 <= cut2, the atom itself at tau = 0 excepted:
    (i, j, vec = x_j + tau - x_i, r)"""
    from oracle.d3_oracle import _translations
    tau, g = _translations(lat, np.sqrt(cut2), pbc)
    zero = np.abs(g).sum(1) == 0
    I, J, V = [], [], []
    n = len(x)
    for i in range(n):
        d = x[None, :, :] - x[i][None, None, :] + tau[:, None, :]          # [t, n, 3]
        m = (d ** 2).sum(-1) <= cut2
        m[zero, i] = False
        t, j = np.nonzero(m)
        I.append(np.full(len(j), i))
        J.append(j)
        V.append(d[t, j])
    I, J, V = np.concatenate(I), np.concatenate(J), np.concatenate(V).reshape(-1, 3)
    return I, J, V, np.linalg.norm(V, axis=1)


def _damping(z, I, J, r, damping):
    """g and dg/dr of E_pair = -C6 g (the oracle's formulas)"""
    from oracle.d3_oracle import d3_params, damping_parameters
    P, dp = d3_params(), damping_parameters(damping, 'pbe')
    r2r4 = P['r2r4'][z]
    if damping == 'damp_bj':
        r42x3 = 3.0 * r2r4[I] * r2r4[J]
        R0 = dp['a1'] * np.sqrt(r42x3) + dp['a2']
        t6, t8 = 1.0 / (r ** 6 + R0 ** 6), 1.0 / (r ** 8 + R0 ** 8)
        g = dp['s6'] * t6 + dp['s8'] * r42x3 * t8
        dg = -(6.0 * dp['s6'] * r ** 5 * t6 ** 2 + 8.0 * dp['s8'] * r42x3 * r ** 7 * t8 ** 2)
    else:
        r0 = P['r0ab'][z[I], z[J]] / AU
        r42 = r2r4[I] * r2r4[J]
        t6, t8 = (dp['a1'] * r0 / r) ** dp['alp6'], (dp['a2'] * r0 / r) ** dp['alp8']
        d6, d8 = 1.0 / (1.0 + 6.0 * t6), 1.0 / (1.0 + 6.0 * t8)
        g = dp['s6'] * d6 / r ** 6 + 3.0 * dp['s8'] * r42 * d8 / r ** 8
        dg = (dp['s6'] * (-6.0 * d6 / r ** 7 + 6.0 * dp['alp6'] * t6 * d6 ** 2 / r ** 7)
              + 3.0 * dp['s8'] * r42 * (-8.0 * d8 / r ** 9 + 6.0 * dp['alp8'] * t8 * d8 ** 2 / r ** 9))
    return g, dg


def atomic_energies(numbers, positions, cell, pbc, damping, vdw_cutoff, cn_cutoff):
    """U_j (eV) from the fp64 oracle's C6_ij: -1/2 sum over j's pairs inside the vdW cutoff of C6 g"""
    from oracle.d3_oracle import d3_reference
    z = np.asarray(numbers, dtype=np.int64) - 1
    c6 = d3_reference(numbers, positions, cell, pbc, damping=damping, functional='pbe', vdw_cutoff=vdw_cutoff,
                      cn_cutoff=cn_cutoff)['c6']
    x, lat = _wrapped(positions, cell)
    I, J, _, r = _pairs(x, lat, pbc, vdw_cutoff)
    g, _ = _damping(z, I, J, r, damping)
    return np.bincount(I, weights=-0.5 * c6[I, J] * g, minlength=len(z)) * AU_TO_EV


def recursion_flux(numbers, positions, cell, pbc, v, damping, vdw_cutoff, cn_cutoff):
    """(J_pot [3], R [n, 3], U [n]) by the recursion of the kernels in fp64: J_pot in eV A x (the unit of v), R_j the
    per-atom terms, U_j the atomic energies (eV).  v [n, 3] in A x (a time unit)."""
    from oracle.d3_oracle import d3_params
    P = d3_params()
    z = np.asarray(numbers, dtype=np.int64) - 1
    n = len(z)
    vb = np.asarray(v, dtype=np.float64).reshape(n, 3) / AU
    x, lat = _wrapped(positions, cell)
    # CN pass: CN, dCN and P
    I, J, d, r = _pairs(x, lat, pbc, cn_cutoff)
    rc = P['rcov'][z][I] + P['rcov'][z][J]
    ex = np.exp(-K1 * (rc / r - 1.0))
    cn = np.bincount(I, weights=1.0 / (1.0 + ex), minlength=n)
    f1 = -K1 * rc * ex / (r * r * (1.0 + ex) ** 2)
    u = d / r[:, None]
    q, qi = (u * vb[J]).sum(1), (u * vb[I]).sum(1)
    dcn = np.bincount(I, weights=f1 * (q - qi), minlength=n)
    Pm = np.stack([np.bincount(I, weights=-d[:, a] * f1 * q, minlength=n) for a in range(3)], 1)
    # weights and C6_jk, dC6/dCN_j, dC6/dCN_k of every atom pair (the oracle's den > 1e-99 rule)
    cnr, mxc = P['cnref'][z], P['mxc'][z]
    valid = np.arange(5)[None, :] < mxc[:, None]
    w = np.where(valid, np.exp(K3 * (cnr - cn[:, None]) ** 2), 0.0)
    dw = w * 2.0 * K3 * (cn[:, None] - cnr)
    c6r = P['c6ref'][z[:, None], z[None, :]]
    num = np.einsum('ijab,ia,jb->ij', c6r, w, w)
    den = np.einsum('ia,jb->ij', w, w)
    ok = den > 1e-99
    sden = np.where(ok, den, 1.0)
    near = np.argmin(np.where(valid, (cnr - cn[:, None]) ** 2, np.inf), axis=1)
    c6 = np.where(ok, num / sden, c6r[np.arange(n)[:, None], np.arange(n)[None, :], near[:, None], near[None, :]])
    dc6_i = np.where(ok, (np.einsum('ijab,ia,jb->ij', c6r, dw, w) - c6 * np.einsum('ia,jb->ij', dw, w)) / sden, 0.0)
    dc6_j = np.where(ok, (np.einsum('ijab,ia,jb->ij', c6r, w, dw) - c6 * np.einsum('ia,jb->ij', w, dw)) / sden, 0.0)
    # pair pass
    I, J, d, r = _pairs(x, lat, pbc, vdw_cutoff)
    g, dg = _damping(z, I, J, r, damping)
    C6, D = c6[I, J], dc6_j[I, J]
    dc6i = np.bincount(I, weights=g * dc6_i[I, J], minlength=n)
    qk = ((d / r[:, None]) * vb[J]).sum(1)
    term = (D * g)[:, None] * (Pm[J] - d * dcn[J][:, None]) - (C6 * dg * qk)[:, None] * d
    R = -0.5 * (dc6i[:, None] * Pm + np.stack([np.bincount(I, weights=term[:, a], minlength=n) for a in range(3)], 1))
    R *= AU_TO_EV * AU
    U = np.bincount(I, weights=-0.5 * C6 * g, minlength=n) * AU_TO_EV
    return R.sum(0), R, U


def unfold(positions, cell, pbc, radius):
    """(cluster positions, parent atom of each): the cell's atoms first, then every image along the periodic
    directions within `radius` of one"""
    from scipy.spatial import cKDTree
    pos, cell = np.asarray(positions, np.float64), np.asarray(cell, np.float64)
    spacing = 1.0 / np.linalg.norm(np.linalg.inv(cell), axis=0)
    K = np.where(np.asarray(pbc, dtype=bool), np.ceil(radius / spacing).astype(int) + 1, 0)
    s = np.stack(np.meshgrid(*[np.arange(-k, k + 1) for k in K], indexing='ij'), -1).reshape(-1, 3)
    s = s[np.argsort(np.abs(s).sum(1), kind='stable')]
    img = (pos[None, :, :] + (s @ cell)[:, None, :]).reshape(-1, 3)
    parent = np.tile(np.arange(len(pos)), len(s))
    dist, _ = cKDTree(pos).query(img, k=1)
    keep = dist < radius
    return img[keep], parent[keep]


def _margin(pos, cut2s):
    """min over all pairs of a cluster of | r - rc | for the cutoffs (A)"""
    from scipy.spatial import cKDTree
    rcs = [np.sqrt(c) * AU for c in cut2s]
    pairs = cKDTree(pos).query_pairs(max(rcs) + 1.0, output_type='ndarray')
    r = np.linalg.norm(pos[pairs[:, 1]] - pos[pairs[:, 0]], axis=1)
    return min(float(np.abs(r - rc).min()) for rc in rcs)


def difference_flux(numbers, positions, cell, pbc, v, damping, vdw_cutoff, cn_cutoff):
    """(J_pot [3], per-atom terms [n, 3]) by Richardson differences of ``atomic_energies`` on the cluster: the
    structure itself without a periodic direction, else its unfolded cluster (radius vdW + CN cutoff + 1 A)"""
    numbers, pos, v = np.asarray(numbers), np.asarray(positions, np.float64), np.asarray(v, np.float64)
    n = len(pos)
    if np.any(pbc):
        radius = (np.sqrt(vdw_cutoff) + np.sqrt(cn_cutoff)) * AU + 1.0
        pos, parent = unfold(pos, cell, pbc, radius)
        numbers, v = numbers[parent], v[parent]
    pos = pos - pos[:n].mean(0)
    lo, hi = pos.min(0), pos.max(0)
    box = np.diag(hi - lo + 10.0)                            # holds the cluster: the oracle's wrap moves nothing
    base = pos - lo + 5.0
    fields = [v] + [pos[:, a:a + 1] * v for a in range(3)]
    move = max(2 * np.linalg.norm(f, axis=1).max() for f in fields)
    h = min(1e-3, _margin(pos, (vdw_cutoff, cn_cutoff)) / (4 * max(move, 1e-12)))
    U = lambda p: atomic_energies(numbers, p, box, (False,) * 3, damping, vdw_cutoff, cn_cutoff)[:n]

    def dU(f):
        D = lambda s: (U(base + s * f) - U(base - s * f)) / (2 * s)
        return (4 * D(h / 2) - D(h)) / 3
    per = pos[:n] * dU(v)[:, None]
    for a in range(3):
        per[:, a] -= dU(fields[1 + a])
    return per.sum(0), per
