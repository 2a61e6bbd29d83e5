"""Elastic tensors from the engine's second derivatives (numpy only: no torch, no engine).

Definitions (DESIGN.md §8):

- Deformation: r -> (I + eps) r for atoms and cell, with the edge list held fixed.
- The virial W = -sum_e vec_e (x) f_e, f_e = dE/dvec_e, so dE/deps = -W; ASE stress is -W / V in Voigt order.
- Voigt order is ASE's, (xx, yy, zz, yz, xz, xy), with engineering strains: the shear strain e_yz is the tensor with
  1/2 in both (y, z) and (z, y) (``voigt_strains``).
- Clamped-ion (Born) tensor C0 = (1/V) d2E/de de, V the volume before the strain.
- Internal-strain tensor Lambda = d2E/dr de, [3N, 6] in eV/A (row 3i + a: atom i, direction a).
- Relaxed-ion tensor C = C0 - (1/V) Lambda^T H+ Lambda, with H+ the pseudo-inverse of the Hessian on the complement
  of the three uniform translations (sum_i Lambda_i = 0 by translation invariance).
- Units: eV/A^3, the unit of ASE stress; divide by ``ase.units.GPa`` for GPa.

This is the second derivative of the energy.  At a stress-free, force-free structure it is the elastic tensor; no
pre-stress correction is made, and none is checked for.

The engine gives, per strain tangent eps_k (``B200Engine.hvp_strain(None, eps_k)``), the force-path product
Lambda eps_k [N, 3] and the virial tangent dW [6] in the virial's order (xx, yy, zz, xy, yz, zx); and the Hessian
(``SevenNetCalculator.get_hessian``).  The functions here assemble the tensors from those raw products.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

# Voigt component j -> tensor index pair; the virial's order (xx,yy,zz,xy,yz,zx) -> Voigt (xx,yy,zz,yz,xz,xy)
VOIGT_PAIRS = ((0, 0), (1, 1), (2, 2), (1, 2), (0, 2), (0, 1))
VIRIAL_TO_VOIGT = [0, 1, 2, 4, 5, 3]


def voigt_strains() -> np.ndarray:
    """The six engineering-strain tangents [6, 3, 3]: 1 on the diagonal for j < 3, 1/2 in both off-diagonal
    entries for the shears."""
    eps = np.zeros((6, 3, 3))
    for j, (a, b) in enumerate(VOIGT_PAIRS):
        eps[j, a, b] = eps[j, b, a] = 1.0 if a == b else 0.5
    return eps


def virial_to_voigt(w6) -> np.ndarray:
    """[..., 6] in the virial's order (xx,yy,zz,xy,yz,zx) -> ASE Voigt order (xx,yy,zz,yz,xz,xy)"""
    return np.asarray(w6, dtype=np.float64)[..., VIRIAL_TO_VOIGT]


def clamped_ion(dvirial, volume: float) -> np.ndarray:
    """C0 [6, 6] in eV/A^3 from the virial tangents dvirial [6, 6] (row k: dW along Voigt strain k, in the virial's
    order): dE/de_j = -W_j (Voigt), so C0[j, k] = -(dW along k)_j / V.  Not symmetrised."""
    dv = np.asarray(dvirial, dtype=np.float64).reshape(6, 6)
    return -virial_to_voigt(dv).T / float(volume)


def internal_strain(outs) -> np.ndarray:
    """Lambda [3N, 6] in eV/A from the six products out_k = Lambda eps_k, outs [6, N, 3]"""
    o = np.asarray(outs, dtype=np.float64)
    return o.reshape(6, -1).T


def translation_complement(n_atoms: int) -> np.ndarray:
    """Orthonormal basis [3N, 3N - 3] of the complement of the three uniform translations"""
    t = np.zeros((3 * n_atoms, 3))
    for a in range(3):
        t[a::3, a] = 1.0 / np.sqrt(n_atoms)
    q, _ = np.linalg.qr(np.concatenate([t, np.eye(3 * n_atoms)], axis=1))
    return q[:, 3:3 * n_atoms]


def pinv_hessian(hessian) -> np.ndarray:
    """H+ [3N, 3N]: the pseudo-inverse of the symmetrised Hessian on the complement of the uniform translations
    (which it maps to zero)."""
    h = np.asarray(hessian, dtype=np.float64)
    h = 0.5 * (h + h.T)
    q = translation_complement(h.shape[0] // 3)
    return q @ np.linalg.pinv(q.T @ h @ q, hermitian=True) @ q.T


def relaxed_ion(c0, lam, hessian, volume: float) -> np.ndarray:
    """C = C0 - (1/V) Lambda^T H+ Lambda [6, 6] in eV/A^3"""
    lam = np.asarray(lam, dtype=np.float64)
    return np.asarray(c0, dtype=np.float64) - lam.T @ pinv_hessian(hessian) @ lam / float(volume)


def elastic_tensor(dvirial, outs, volume: float, hessian: Optional[np.ndarray] = None) -> np.ndarray:
    """[6, 6] in eV/A^3 from the six strain products (dvirial [6, 6], outs [6, N, 3]): clamped-ion without a
    Hessian, relaxed-ion with one ([3N, 3N] in eV/A^2)."""
    c0 = clamped_ion(dvirial, volume)
    if hessian is None:
        return c0
    return relaxed_ion(c0, internal_strain(outs), hessian, volume)
