"""ASE-style calculator with the reference's ``SevenNetCalculator`` surface
(``sevenn/calculator.py:20-233``): same constructor keywords, same ``results`` keys
(``free_energy, energy, energies, forces, stress, num_edges``), same stress convention
(ASE Voigt order ``-inferred_stress[[0,1,2,4,5,3]]``, ``calculator.py:198-203``).

ASE itself is optional: when importable the class derives from ``ase.calculators.calculator.
Calculator``; otherwise it is a duck-typed object with ``calculate(atoms, properties,
system_changes)`` and ``get_*`` helpers, where ``atoms`` needs ``get_positions()``,
``get_cell()``, ``get_pbc()`` and ``get_atomic_numbers()``.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np

from .checkpoint import convert_reference_checkpoint, load_weights
from .engine import B200Engine

_WEIGHTS_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'weights')
# names the reference resolves in sevenn/util.py:264-312
_ALIASES = {
    '7net-0': 'sevennet_0', '7net-0_11july2024': 'sevennet_0', 'sevennet-0': 'sevennet_0',
    'sevennet_0': 'sevennet_0', '7net-l3i5': 'sevennet_l3i5', 'sevennet-l3i5': 'sevennet_l3i5',
    'sevennet_l3i5': 'sevennet_l3i5',
}

try:  # pragma: no cover - ASE is not installed in the build container
    from ase.calculators.calculator import Calculator as _Base, all_changes as _all_changes
except Exception:  # noqa: BLE001
    _all_changes = ['positions', 'numbers', 'cell', 'pbc', 'initial_charges', 'initial_magmoms']

    class _Base:  # minimal stand-in for ase.calculators.calculator.Calculator
        def __init__(self, **kwargs):
            self.results = {}
            self.atoms = None

        def calculate(self, atoms=None, properties=None, system_changes=None):
            self.atoms = atoms

        def get_potential_energy(self, atoms=None, force_consistent=False):
            self.calculate(atoms)
            return self.results['free_energy' if force_consistent else 'energy']

        def get_forces(self, atoms=None):
            self.calculate(atoms)
            return self.results['forces']

        def get_stress(self, atoms=None):
            self.calculate(atoms)
            return self.results['stress']

        def get_potential_energies(self, atoms=None):
            self.calculate(atoms)
            return self.results['energies']


def resolve_model(model: str):
    """name | path to ``.npz`` (this repo's format) | path to a reference ``.pth`` checkpoint."""
    key = str(model).lower()
    if key in _ALIASES:
        return load_weights(os.path.join(_WEIGHTS_DIR, _ALIASES[key] + '.npz'))
    if os.path.isfile(model):
        if str(model).endswith('.npz'):
            return load_weights(model)
        return convert_reference_checkpoint(model, os.path.splitext(os.path.basename(model))[0])
    raise ValueError(f'unknown model {model!r}: expected one of {sorted(_ALIASES)} or a file path')


class SevenNetCalculator(_Base):
    implemented_properties = ['free_energy', 'energy', 'forces', 'stress', 'energies']

    def __init__(self, model: str = '7net-0', file_type: str = 'checkpoint', device='cuda',
                 modal: Optional[str] = None, enable_cueq: bool = False, enable_flash: bool = False,
                 enable_oeq: bool = False, compute_atomic_virial: bool = False,
                 sevennet_config: Optional[dict] = None, radial: str = 'table', **kwargs):
        super().__init__(**kwargs)
        if file_type != 'checkpoint':
            raise NotImplementedError("sevenn_b200 loads checkpoints only (file_type='checkpoint')")
        if modal is not None:
            raise NotImplementedError('multi-fidelity models are out of scope')
        if enable_cueq or enable_flash or enable_oeq:
            raise ValueError('enable_cueq/flash/oeq select other accelerators; this calculator '
                             'always runs the sevenn_b200 CUDA engine')
        import torch
        dev = torch.device(device)
        if dev.type != 'cuda':
            raise RuntimeError('sevenn_b200 has no CPU path; pass a CUDA device')
        self.meta, self.arrays = resolve_model(model) if isinstance(model, str) else model
        self.engine = B200Engine(self.meta, self.arrays, radial=radial,
                                 device=dev.index if dev.index is not None else None,
                                 atomic_virial=compute_atomic_virial)
        self.cutoff = self.engine.spec.cutoff
        self.type_map = self.engine.spec.type_map
        self.compute_atomic_virial = compute_atomic_virial
        self.sevennet_config = sevennet_config or dict(self.meta)
        self._engine_inputs = None     # (positions, cell, pbc, numbers) of the engine's current graph and forward

    def _remember(self, pos, cell, pbc, numbers):
        self._engine_inputs = tuple(np.array(a, copy=True) for a in (pos, cell, pbc, numbers))

    def _inputs(self, atoms):
        """(species, positions, cell, pbc, atomic numbers) of ``atoms`` for the engine"""
        pos = np.asarray(atoms.get_positions(), dtype=np.float64)
        cell = np.asarray(atoms.get_cell(), dtype=np.float64).reshape(3, 3)
        pbc = np.asarray(atoms.get_pbc(), dtype=bool)
        numbers = np.asarray(atoms.get_atomic_numbers())
        try:
            species = np.array([self.type_map[int(z)] for z in numbers], dtype=np.int32)
        except KeyError as e:  # same failure mode as sequential.py:131-137 for unknown elements
            raise ValueError(f'atomic number {e} is not known to this model') from None
        return species, pos, cell, pbc, numbers

    def calculate(self, atoms=None, properties=None, system_changes=_all_changes):
        super().calculate(atoms, properties, system_changes)
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        species, pos, cell, pbc, numbers = self._inputs(atoms)
        # neighbour list, graph build, model and force path all run on the GPU (one C-ABI call);
        # the reference builds the graph on the CPU every step (calculator.py:224-226)
        energy, energies, forces, virial, n_edges = self.engine.compute_positions(species, pos, cell, pbc)
        self._remember(pos, cell, pbc, numbers)
        # the reference divides by atoms.cell.volume whatever the pbc flags are (dataload.py:121,
        # force_output.py:227-228); a missing cell (volume 0) has no stress
        vol = abs(np.linalg.det(cell))
        self.results = {
            'free_energy': energy, 'energy': energy,
            'energies': energies.astype(np.float64),
            'forces': forces.astype(np.float64),
            'num_edges': n_edges,
        }
        if vol > 0:
            inferred_stress = virial / vol
            self.results['stress'] = -inferred_stress[[0, 1, 2, 4, 5, 3]]
        if self.compute_atomic_virial:   # calculator.py:211-216: 'stresses' = the per-atom virial as the model gives it
            self.results['stresses'] = self.engine.buffer('atomic_virial', shape=(len(numbers), 6)).cpu().numpy().astype(np.float64)
        return self.results

    def get_hessian(self, atoms=None) -> np.ndarray:
        """Hessian d2E/dr dr of ``atoms`` (default: the calculator's atoms), [3N, 3N] float64 in eV/A^2, row 3i + a
        = H e_(i,a).  Built from 3N Hessian-vector products (``B200Engine.hvp``) on the calculator's own graph of the
        atoms, with that edge list held fixed, so a periodic cell gives the Gamma-point (supercell) Hessian that
        phonon codes take force constants from.  Not symmetrised (the two triangles agree to the fp32 error of the
        products); ``.reshape(N, 3, N, 3)`` gives the force constants Phi[i, a, j, b].  ``results`` and the other
        ``get_*`` methods are not touched.  ``SevenNetD3Calculator.get_hessian`` adds D3 dispersion's."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        torch = self.engine.torch
        species, pos, cell, pbc, numbers = self._inputs(atoms)
        n = len(species)
        self.engine.set_positions(species, pos, cell, pbc)
        self.engine.compute()
        self._remember(pos, cell, pbc, numbers)
        eye = torch.eye(3 * n, dtype=torch.float32, device=self.engine.device)
        rows = [self.engine.hvp(eye[k].reshape(n, 3)).reshape(-1) for k in range(3 * n)]
        if not rows:
            return np.zeros((0, 0))
        return torch.stack(rows).double().cpu().numpy()

    def get_elastic_tensor(self, atoms=None, relaxed: bool = True) -> np.ndarray:
        """Elastic tensor d2E/de de / V of ``atoms`` (default: the calculator's atoms), [6, 6] float64 in eV/A^3 (the
        unit of ASE stress; ``/ ase.units.GPa`` gives GPa), ASE Voigt order (xx, yy, zz, yz, xz, xy), engineering
        strains, V the volume of the unstrained cell.  From six strain products (``B200Engine.hvp_strain``) on the
        calculator's own graph of the atoms, with that edge list held fixed.  ``relaxed=True`` gives the relaxed-ion
        tensor C0 - Lambda^T H+ Lambda / V, which also takes the Hessian (``get_hessian``, 3N more products);
        ``relaxed=False`` the clamped-ion tensor C0 (``sevenn_b200.elastic`` defines both).  This is the second
        derivative of the energy: at a stress-free, force-free structure it is the elastic tensor; no pre-stress
        correction is made and none is checked for.  All three directions must be periodic.  ``results`` and the other
        ``get_*`` methods are not touched.  ``SevenNetD3Calculator.get_elastic_tensor`` adds D3 dispersion's."""
        from . import elastic
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        return elastic.elastic_tensor(*self._strain_pieces(atoms, relaxed))

    def get_heat_flux(self, atoms=None, convective: bool = True) -> np.ndarray:
        """Energy-barycentre heat flux of ``atoms`` (default: the calculator's atoms), [3] float64, for Green-Kubo
        thermal conductivity (``sevenn_b200.heat_flux``, DESIGN.md §8.3):

          J = J_pot + J_conv,  J_pot = sum_j sum_i (r_j - r_i) (dU_j/dr_i . v_i),  J_conv = sum_j (U_j + m_j |v_j|^2 / 2) v_j

        with U_j the atomic energies ('energies'), j over the atoms, i over every atom and periodic image U_j depends
        on (T layers x cutoff away), an image moving with its atom.  This is exact for the message-passing model; the
        pairwise split of the per-atom virial (``compute_atomic_virial``, J = sum_k W_k v_k) is not.  Velocities and
        masses come from ``atoms.get_velocities()`` and ``get_masses()``.  Units: eV A^2 / (ASE time); multiply by
        ``ase.units.fs`` for eV A^2/fs.  ``convective=False`` gives J_pot alone.  One tangent-forward pass of four
        channels; the energy/force step runs only when positions, numbers, cell or pbc differ from those of the last
        calculation, so an MD observer that asked for forces this step adds only the flux pass.  ``results`` are not
        touched.  ``SevenNetD3Calculator.get_heat_flux`` adds D3 dispersion's."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        J, ju, v = self._flux_parts(atoms)
        if convective:
            from .heat_flux import kinetic_flux
            J = J + ju + kinetic_flux(v, atoms.get_masses())[0]
        return J

    def get_centroid_virials(self, atoms=None) -> np.ndarray:
        """Per-atom centroid virial of ``atoms`` (default: the calculator's atoms), [N, 3, 3] float64 in eV
        (``B200Engine.centroid_virial``, DESIGN.md §8.5):

          Wc_i[a, b] = sum_j sum_i' (r_j - r_i')_a dU_j/dr_i',b

        with U_j the atomic energies ('energies'), i' atom i and its periodic images.  Row a is the flux direction,
        column b the velocity direction: sum_i Wc_i v_i is ``get_heat_flux(convective=False)`` for any velocities, and
        sum_i Wc_i is the virial.  This is the quantity of LAMMPS's ``compute centroid/stress/atom`` (times -1 / V for
        a stress); the symmetric pairwise split of ``compute_atomic_virial`` ('stresses') is not, for a model of more
        than one layer.  One reverse pass of four channels; the energy/force step runs only when positions, numbers,
        cell or pbc differ from those of the last calculation.  ``results`` are not touched."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        self._step_if_changed(atoms)
        return self.engine.centroid_virial().cpu().numpy()

    def _step_if_changed(self, atoms):
        """Leave the engine on the graph and forward of ``atoms``: the energy/force step runs only when positions,
        numbers, cell or pbc differ from those of the last calculation"""
        species, pos, cell, pbc, numbers = self._inputs(atoms)
        last = self._engine_inputs
        if last is None or not all(np.array_equal(a, b) for a, b in zip(last, (pos, cell, pbc, numbers))):
            self.engine.set_positions(species, pos, cell, pbc)
            self.engine.compute()
            self._remember(pos, cell, pbc, numbers)

    def _flux_parts(self, atoms):
        """(J_pot [3], sum_j U_j v_j [3], velocities [n, 3]) of ``atoms``; the energy/force step runs only when
        positions, numbers, cell or pbc differ from those of the last calculation"""
        self._step_if_changed(atoms)
        v = np.asarray(atoms.get_velocities(), dtype=np.float64).reshape(-1, 3)
        jpot, ju = self.engine.heat_flux(v.astype(np.float32))
        return jpot[0].cpu().numpy(), ju[0].cpu().numpy(), v

    def _strain_pieces(self, atoms, relaxed: bool):
        """The raw second derivatives ``elastic.elastic_tensor`` assembles: (dvirial [6, 6], outs [6, N, 3], volume,
        Hessian [3N, 3N] or None), from the six Voigt strain products and, when ``relaxed``, the Hessian."""
        from . import elastic
        species, pos, cell, pbc, numbers = self._inputs(atoms)
        vol = abs(np.linalg.det(cell))
        if not pbc.all() or not vol > 0:
            raise ValueError('the elastic tensor needs a cell periodic in all three directions with a volume > 0')
        if relaxed:
            hessian = self.get_hessian(atoms)      # leaves the engine on the atoms' graph and forward
        else:
            hessian = None
            self.engine.set_positions(species, pos, cell, pbc)
            self.engine.compute()
            self._remember(pos, cell, pbc, numbers)
        outs, dvir = [], []
        for eps in elastic.voigt_strains():
            o, d = self.engine.hvp_strain(None, eps[None])
            outs.append(o)
            dvir.append(d[0])
        torch = self.engine.torch
        return torch.stack(dvir).cpu().numpy(), torch.stack(outs).double().cpu().numpy(), vol, hessian
