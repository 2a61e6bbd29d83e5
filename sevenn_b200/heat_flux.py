"""Green-Kubo heat flux of SevenNet models (DESIGN.md §8.3).

For the atomic energies U_j (the engine's ``atomic_energy``, scale and shift included) and velocities v_i:

  J = J_pot + J_conv
  J_pot  = sum_j sum_i (r_j - r_i) (dU_j/dr_i . v_i)
  J_conv = sum_j (U_j + m_j |v_j|^2 / 2) v_j

j runs over the cell's atoms; i over every atom and periodic image U_j depends on, an image moving with its atom's
velocity, and r_j - r_i is the actual vector from that image to j.  The definition follows from energy continuity,
de_j/dt = sum_k (dU_j/dr_k . v_k - dU_k/dr_j . v_j).  Units: eV A times the velocity unit; with ASE's units (A, amu,
eV, ASE time) m v^2 / 2 is in eV and ``J * ase.units.fs`` is in eV A^2/fs.

The engine computes J_pot and sum_j U_j v_j in one tangent-forward CUDA pass of four channels
(``B200Engine.heat_flux``, C ABI ``s7b_engine_heat_flux``): T_j = sum_i dh_j/dr_i . v_i and
R_j,a = sum_i (r_j - r_i)_a (dh_j/dr_i . v_i) for every node feature h_j, carried through the layers with edge vectors
only, so a periodic cell needs no unfolding; J_pot,a = sum_j scale_s readout(R_j,a).  D3 dispersion's atomic energies
have their own two-pass flux (``d3.D3Engine.heat_flux``, DESIGN.md §8.4), which adds to this one.  This module adds the
kinetic part, which needs the masses.
"""
import numpy as np


def kinetic_flux(velocities, masses, atom_ptr=None) -> np.ndarray:
    """sum_j m_j |v_j|^2 / 2 v_j per structure, [B, 3] float64 (B = len(atom_ptr) - 1, or 1 without atom_ptr), in
    a fixed order"""
    v = np.asarray(velocities, dtype=np.float64).reshape(-1, 3)
    m = np.asarray(masses, dtype=np.float64).reshape(-1)
    if m.shape[0] != v.shape[0]:
        raise ValueError(f'masses has {m.shape[0]} entries for {v.shape[0]} atoms')
    ptr = np.array([0, len(v)]) if atom_ptr is None else np.asarray(atom_ptr, dtype=np.int64)
    t = (0.5 * m * (v * v).sum(axis=1))[:, None] * v
    return np.stack([t[a:b].sum(axis=0) for a, b in zip(ptr[:-1], ptr[1:])]).reshape(-1, 3)
