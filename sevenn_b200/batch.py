"""Several structures in one pass of the engine (SURVEY §8 f.4: the batched callers of the hot path).

The reference evaluates a batch as one disjoint-union graph: ``AtomGraphSequential`` with
``is_batch_data`` (``sevenn/nn/sequential.py:99-108,143``), per-graph energy from ``AtomReduce``
(``nn/linear.py:127-141``) and per-graph stress from the per-atom virial scattered by ``batch``
(``nn/force_output.py:216-228``).  The engine works on any CSR graph, so a batch is the concatenation
of the per-structure graphs with node offsets.  ``BatchedEvaluator`` builds it structure by structure from
host arrays, with torch segment sums for the per-structure results.  ``DeviceBatch`` keeps a batch on the
device: one batched neighbour list (``s7b_engine_set_positions_batch``) and per-structure energy / virial
reduced in fp64 by a kernel (``s7b_engine_system_results``).  ``SevenNetModel`` mirrors the TorchSim adapter ``sevenn/torchsim.py:56-292``:
same constructor keywords, ``forward(state) -> {'energy' [B], 'forces' [n,3], 'stress' [B,3,3]}``
with the sign / Voigt handling of ``torchsim.py:286-290``.  ``torch_sim`` is not installed here, so
``state`` is duck-typed: ``positions, row_vector_cell (or cell), pbc, atomic_numbers, system_idx``.
``SevenNetD3Model`` adds D3 dispersion of the whole batch (``d3.D3Batch``).
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from .engine import B200Engine, _host


class BatchedEvaluator:
    def __init__(self, engine: B200Engine):
        self.engine = engine

    def set_batch(self, systems: Sequence[dict]):
        """systems: dicts with ``species`` (indices) or ``numbers`` (atomic numbers), ``positions``
        [n,3], ``cell`` [3,3] and ``pbc``.  Builds every neighbour list on the device
        (``s7b_engine_set_positions_host``) and installs the union graph."""
        eng, torch = self.engine, self.engine.torch
        tm = eng.spec.type_map
        rowptrs, srcs, evs, species, counts, offs = [], [], [], [], [], [0]
        e_off = 0
        for s in systems:
            if 'species' in s:
                sp = np.asarray(s['species'], dtype=np.int32)
            else:
                try:
                    sp = np.array([tm[int(z)] for z in s['numbers']], dtype=np.int32)
                except KeyError as e:
                    raise ValueError(f'atomic number {e} is not known to this model') from None
            eng.set_positions(sp, s['positions'], s.get('cell'), s.get('pbc', False))
            rp, src, ev = eng.graph_arrays()
            rowptrs.append(rp[(1 if rowptrs else 0):].to(torch.int64) + e_off)
            srcs.append(src.to(torch.int64) + offs[-1])
            evs.append(ev.clone())
            species.append(torch.as_tensor(sp, device=eng.device))
            counts.append(len(sp))
            offs.append(offs[-1] + len(sp))
            e_off += int(src.shape[0])
        if not counts:
            raise ValueError('empty batch')
        cat = torch.cat
        self.counts = counts
        self.system_idx = torch.repeat_interleave(torch.arange(len(counts), device=eng.device),
                                                  torch.tensor(counts, device=eng.device))
        eng.set_graph_csr(cat(species).to(torch.int32).contiguous(), cat(rowptrs).to(torch.int32).contiguous(),
                          cat(srcs).to(torch.int32).contiguous(), cat(evs).contiguous(), offs[-1])
        return self

    def compute(self, systems: Optional[Sequence[dict]] = None) -> dict:
        """-> dict of device tensors: energy [B] f64, atomic_energy [n], forces [n,3], virial [B,6] f64
        (= -sum r (x) f per structure, order xx,yy,zz,xy,yz,zx), n_edges."""
        if systems is not None:
            self.set_batch(systems)
        eng, torch = self.engine, self.engine.torch
        eng.compute()
        B = len(self.counts)
        ae = eng.buffer('atomic_energy', shape=(eng.n_local,)).clone()
        energy = torch.zeros(B, dtype=torch.float64, device=eng.device).index_add_(0, self.system_idx, ae.double())
        forces = eng.buffer('forces', shape=(eng.n_nodes, 3)).clone()
        virial = torch.zeros(B, 6, dtype=torch.float64, device=eng.device)
        if eng.n_edges:
            g = eng._graph
            fe = eng.buffer('edge_force', shape=(eng.n_edges, 3)).double()
            ev = g['edge_vec'].double()
            v6 = ev[:, [0, 1, 2, 0, 1, 2]] * fe[:, [0, 1, 2, 1, 2, 0]]
            virial.index_add_(0, self.system_idx[g['src'].long()], -v6)
        return dict(energy=energy, atomic_energy=ae, forces=forces, virial=virial, n_edges=eng.n_edges)

    def split(self, out: dict) -> List[dict]:
        """Per-structure numpy results."""
        res, a = [], 0
        ae, f = out['atomic_energy'].cpu().numpy(), out['forces'].cpu().numpy()
        e, v = out['energy'].cpu().numpy(), out['virial'].cpu().numpy()
        for b, n in enumerate(self.counts):
            res.append(dict(energy=float(e[b]), energies=ae[a:a + n], forces=f[a:a + n], virial=v[b]))
            a += n
        return res


class DeviceBatch:
    """Structures given as flat device-resident arrays, the layout of a TorchSim state, evaluated in one engine
    pass without a host copy of the positions: only the atom counts, cells and pbc (O(B) values) cross to the
    host, with one readback per call for the checks."""

    def __init__(self, engine: B200Engine):
        self.engine = engine
        torch = engine.torch
        tm = engine.spec.type_map
        lut = torch.full((max(tm) + 1,), -1, dtype=torch.int32)
        for z, s in tm.items():
            lut[z] = s
        self._lut = lut.to(engine.device)

    def set_batch(self, numbers, positions, cells, pbc, system_idx):
        """numbers [n] atomic numbers, positions [n,3], cells [B,3,3] (rows = lattice vectors), pbc (bool, [3] or
        [B,3]), system_idx [n] (sorted structure index of every atom): torch tensors on any device, or numpy
        arrays.  Builds the union graph on the device."""
        eng, torch = self.engine, self.engine.torch
        dev = eng.device
        z = torch.as_tensor(numbers).to(dev, torch.int64).reshape(-1)
        si = torch.as_tensor(system_idx).to(dev, torch.int64).reshape(-1)
        cells = torch.as_tensor(cells).detach().to('cpu', torch.float64).reshape(-1, 3, 3)
        B, n = int(cells.shape[0]), int(z.shape[0])
        if B < 1:
            raise ValueError('empty batch')
        if si.shape[0] != n:
            raise ValueError(f'system_idx has {si.shape[0]} entries for {n} atoms')
        lut = self._lut
        known = (z >= 0) & (z < lut.shape[0])
        species = torch.where(known, lut[z.clamp(0, lut.shape[0] - 1)], -1)
        # one readback: any unknown atomic number, the first one, system_idx unsorted, out of range; then atom_ptr [B+1]
        flags = torch.zeros(4, dtype=torch.int64, device=dev)
        if n > 0:
            bad = species < 0
            flags[0] = bad.any()
            flags[1] = z[bad.to(torch.int8).argmax()]
            flags[2] = (si[1:] < si[:-1]).any()
            flags[3] = (si.min() < 0) | (si.max() >= B)
        counts = torch.bincount(si.clamp(0, B - 1), minlength=B)
        h = torch.cat([flags, torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(counts, 0)]).cpu().numpy()
        if h[0]:
            raise ValueError(f'atomic number {int(h[1])} is not known to this model')
        if h[2]:
            raise ValueError('system_idx must be sorted')
        if h[3]:
            raise ValueError(f'system_idx must lie in [0, {B}): one structure per cell')
        self.atom_ptr = h[4:]
        eng.set_positions_batch(species, positions, self.atom_ptr, cells, pbc)
        return self

    def compute(self, numbers, positions, cells, pbc, system_idx) -> dict:
        """-> dict of device tensors, as ``BatchedEvaluator.compute``: energy [B] f64 (fp64 sum of the per-atom
        energies), atomic_energy [n], forces [n,3], virial [B,6] f64 (= -sum r (x) f per structure, order
        xx,yy,zz,xy,yz,zx), n_edges."""
        self.set_batch(numbers, positions, cells, pbc, system_idx)
        eng = self.engine
        eng.compute()
        energy, virial = eng.system_results()
        ae = eng.buffer('atomic_energy', shape=(eng.n_local,)).clone()
        forces = eng.buffer('forces', shape=(eng.n_nodes, 3)).clone()
        return dict(energy=energy, atomic_energy=ae, forces=forces, virial=virial, n_edges=eng.n_edges)

    def heat_flux(self, velocities, masses=None, convective: bool = True, d3=None):
        """Heat flux of every structure of the batch of the last ``compute``, [B, 3] float64 device tensor
        (``sevenn_b200.heat_flux``'s definition, DESIGN.md §8.3): J_pot + J_conv, J_pot = sum_j sum_i
        (r_j - r_i) (dU_j/dr_i . v_i) over the structure's atoms j and every atom and periodic image i that U_j depends
        on, J_conv = sum_j (U_j + m_j |v_j|^2 / 2) v_j.  velocities [n, 3], masses [n] (needed when ``convective``),
        numpy or torch, in the atom order of ``compute``.  Units: eV A x (the unit of v); with ASE's units (v in
        A/(ASE time), m in amu) m v^2 / 2 is in eV.  ``convective=False`` gives J_pot alone.  One tangent-forward pass
        over the whole batch.  ``d3`` (a ``d3.D3Batch`` whose last ``compute`` was on the same structures, as
        ``SevenNetD3Model.forward`` leaves it) adds D3 dispersion's J_pot and sum_j U_j v_j (DESIGN.md §8.4); the
        kinetic part is counted once."""
        eng, torch = self.engine, self.engine.torch
        if d3 is not None and (d3.atom_ptr is None or not np.array_equal(np.asarray(d3.atom_ptr), np.asarray(self.atom_ptr))):
            raise ValueError('d3: its last compute was not on the structures of this batch (atom_ptr differs)')
        jpot, ju = eng.heat_flux(velocities)
        if d3 is not None:
            jp3, ju3 = d3.heat_flux(velocities)
            jpot, ju = jpot + jp3, ju + ju3
        if not convective:
            return jpot
        if masses is None:
            raise ValueError('the convective flux needs the masses (or pass convective=False)')
        from .heat_flux import kinetic_flux
        jk = kinetic_flux(_host(velocities), _host(masses), self.atom_ptr)
        return jpot + ju + torch.as_tensor(jk, dtype=torch.float64, device=jpot.device)

    def centroid_virials(self, d3=None):
        """Per-atom centroid virial of every atom of the batch of the last ``compute``, [n, 3, 3] float64 device tensor
        in eV, in the atom order of ``compute`` (``B200Engine.centroid_virial``, DESIGN.md §8.5).  The union graph has
        no edge between structures, so each row is its structure's alone: summed over a structure's atoms it is that
        structure's virial, and contracted with its velocities its J_pot.  ``d3`` (a ``d3.D3Batch`` whose last
        ``compute`` was on the same structures, as ``SevenNetD3Model.forward`` leaves it) adds D3 dispersion's rows
        (``D3Batch.centroid_virials``, DESIGN.md §8.6); without it D3 is not included."""
        if d3 is not None and (d3.atom_ptr is None or not np.array_equal(np.asarray(d3.atom_ptr), np.asarray(self.atom_ptr))):
            raise ValueError('d3: its last compute was not on the structures of this batch (atom_ptr differs)')
        wc = self.engine.centroid_virial()
        if d3 is not None:
            wc = wc + d3.centroid_virials()
        return wc

    def elastic_tensors(self, numbers, positions, cells, pbc, system_idx, relaxed: bool = True, d3=None) -> np.ndarray:
        """Elastic tensors of every structure, [B, 6, 6] float64 in eV/A^3 (``SevenNetCalculator.get_elastic_tensor``'s
        definition, units and Voigt order, per structure; inputs as ``compute``).  Every structure must be periodic in
        all three directions with a volume > 0.  C0 and Lambda of all structures come from six batched strain
        products (``B200Engine.hvp_strain``).  The union graph has no edge between structures, so with ``relaxed``
        every structure's Hessian comes from 3 max_b(n_b) more products: product k puts a unit tangent on direction
        k % 3 of local atom k // 3 of every structure at once.  ``d3`` (a ``d3.D3Batch``) adds D3 dispersion: its
        strain products and Hessian blocks, from the same tangents (D3 has no pair between structures either), are
        added to the network's before each structure's tensor is assembled."""
        from . import elastic
        torch = self.engine.torch
        c = torch.as_tensor(cells).detach().to('cpu', torch.float64).reshape(-1, 3, 3).numpy()
        B = c.shape[0]
        vol = np.abs(np.linalg.det(c))
        pb = np.broadcast_to(np.asarray(_host(pbc), dtype=bool), (B, 3))
        if not pb.all() or not (vol > 0).all():
            raise ValueError('elastic tensors need every cell periodic in all three directions with a volume > 0')
        self.set_batch(numbers, positions, c, pbc, system_idx)
        eng = self.engine
        eng.compute()
        ap = np.asarray(self.atom_ptr, dtype=np.int64)
        counts = np.diff(ap)
        if d3 is not None:
            d3.compute(numbers, positions, c, pbc, atom_ptr=ap)
        outs, dvir = [], []
        for eps in elastic.voigt_strains():
            o, d = eng.hvp_strain(None, np.repeat(eps[None], B, axis=0))
            if d3 is not None:
                o3, d3v = d3.hvp_strain(None, np.repeat(eps[None], B, axis=0))
                o, d = o.double() + o3, d + d3v
            outs.append(o)
            dvir.append(d)
        outs = torch.stack(outs).double().cpu().numpy()            # [6, n, 3]
        dvir = torch.stack(dvir).cpu().numpy()                     # [6, B, 6]
        hess = [np.zeros((3 * int(m), 3 * int(m))) for m in counts] if relaxed else None
        if relaxed and eng.n_nodes:
            base = torch.as_tensor(ap[:-1], device=eng.device)
            cnt = torch.as_tensor(counts, device=eng.device)
            rows = []
            for k in range(3 * int(counts.max())):
                v = torch.zeros(eng.n_nodes, 3, dtype=torch.float32, device=eng.device)
                v[base[cnt > k // 3] + k // 3, k % 3] = 1.0
                row = eng.hvp_strain(v, None)[0]
                rows.append(row if d3 is None else row.double() + d3.hvp_strain(v, None)[0])
            rows = torch.stack(rows).double().cpu().numpy()         # [3 max n_b, n, 3]
            for b in range(B):
                m = int(counts[b])
                hess[b][:] = rows[:3 * m, ap[b]:ap[b + 1]].reshape(3 * m, 3 * m)
        return np.stack([elastic.elastic_tensor(dvir[:, b], outs[:, ap[b]:ap[b + 1]], vol[b],
                                                hess[b] if relaxed else None) for b in range(B)])


class SevenNetModel:
    """TorchSim-style model wrapper (``sevenn/torchsim.py:56``): ``model(state)`` evaluates all systems of
    the state in one engine pass."""

    def __init__(self, model='7net-0', *, modal=None, neighbor_list_fn=None, enable_cueq=False,
                 enable_flash=False, enable_oeq=False, compute_atomic_virial=False, device='auto',
                 dtype=None, radial: str = 'table'):
        import torch
        if compute_atomic_virial:   # torchsim.py:112-116
            raise NotImplementedError('compute_atomic_virial is not supported for SevenNet TorchSim interface.')
        if modal is not None:
            raise NotImplementedError('multi-fidelity models are out of scope')
        if enable_cueq or enable_flash or enable_oeq:
            raise ValueError('enable_cueq/flash/oeq select other accelerators; this model always runs the sevenn_b200 engine')
        if neighbor_list_fn is not None:
            raise ValueError('the neighbour list is built by the engine on the device; neighbor_list_fn is not used')
        if dtype is not None and dtype is not torch.float32:   # torchsim.py:135-139
            raise ValueError(f'SevenNet currently only supports {torch.float32}, but received different dtype: {dtype}')
        dev = torch.device('cuda' if device == 'auto' else device)
        if dev.type != 'cuda':
            raise RuntimeError('sevenn_b200 has no CPU path; pass a CUDA device')
        from .calculator import resolve_model
        meta, arrays = resolve_model(model) if isinstance(model, str) else model
        self.engine = B200Engine(meta, arrays, radial=radial, device=dev.index)
        self._device, self._dtype = self.engine.device, torch.float32
        self.cutoff = torch.tensor(self.engine.spec.cutoff)
        self.type_map = self.engine.spec.type_map
        self.modal = None
        self.implemented_properties = ['energy', 'forces', 'stress']
        self._batch = DeviceBatch(self.engine)

    @property
    def device(self):
        return self._device

    @property
    def dtype(self):
        return self._dtype

    def _cells(self, state):
        """host float64 [B,3,3] cells of the state, rows = lattice vectors"""
        torch = self.engine.torch
        cells = getattr(state, 'row_vector_cell', None)
        if cells is None:   # SimState.cell holds column vectors
            cells = torch.as_tensor(state.cell).transpose(-1, -2)
        return torch.as_tensor(cells).detach().to('cpu', torch.float64).reshape(-1, 3, 3).numpy()

    def _stress(self, virial, cells):
        """[B,3,3] stress from the virial [B,6] (xx,yy,zz,xy,yz,zx) and the cells"""
        torch = self.engine.torch
        vol = torch.as_tensor(np.abs(np.linalg.det(cells)), device=self._device)
        s = (virial / vol[:, None])                             # 'inferred_stress', (xx,yy,zz,xy,yz,zx)
        v = -s[:, [0, 1, 2, 4, 5, 3]]                           # ASE Voigt, sign of torchsim.py:286-290
        return torch.stack([torch.stack([v[:, 0], v[:, 5], v[:, 4]], -1),
                            torch.stack([v[:, 5], v[:, 1], v[:, 3]], -1),
                            torch.stack([v[:, 4], v[:, 3], v[:, 2]], -1)], -2)

    def forward(self, state, **kwargs):
        cells = self._cells(state)
        out = self._batch.compute(state.atomic_numbers, state.positions, cells, state.pbc, state.system_idx)
        stress = self._stress(out['virial'], cells)
        return {'energy': out['energy'].to(self._dtype), 'forces': out['forces'], 'stress': stress.to(self._dtype)}

    __call__ = forward


class SevenNetD3Model(SevenNetModel):
    """``SevenNetModel`` + D3 dispersion (``d3.D3Batch``), the batched counterpart of ``d3.SevenNetD3Calculator``:
    ``model(state)`` evaluates the network and D3 of all systems of the state on the current stream and returns
    their sums, energy [B], forces [n,3] and stress [B,3,3] (fp64 sums, returned in float32).  The stress of both
    terms uses the state's cells.  A structure without a cell (all zeros) gets ``D3Calculator``'s generated cell for
    the D3 term (``self.d3.cells``); its energy and forces are those of the isolated structure, but it has no volume,
    so its stress is not finite (inf / nan), as in ``SevenNetModel``.  Keywords: those of ``SevenNetModel`` and of
    ``SevenNetD3Calculator``'s D3 part."""

    def __init__(self, model='7net-0', *, damping_type: str = 'damp_bj', functional_name: str = 'pbe',
                 vdw_cutoff: float = 9000, cn_cutoff: float = 1600, **kwargs):
        super().__init__(model, **kwargs)
        from .d3 import D3Batch
        self.d3 = D3Batch(damping_type, functional_name, vdw_cutoff, cn_cutoff, device=self._device.index)

    def forward(self, state, **kwargs):
        cells = self._cells(state)
        out = self._batch.compute(state.atomic_numbers, state.positions, cells, state.pbc, state.system_idx)
        d3 = self.d3.compute(state.atomic_numbers, state.positions, cells, state.pbc, atom_ptr=self._batch.atom_ptr)
        stress = self._stress(out['virial'] + d3['virial'], cells)
        return {'energy': (out['energy'] + d3['energy']).to(self._dtype),
                'forces': (out['forces'].double() + d3['forces']).to(self._dtype), 'stress': stress.to(self._dtype)}

    __call__ = forward

    def elastic_tensors(self, state, relaxed: bool = True) -> np.ndarray:
        """Elastic tensors of the network plus D3 energy of every structure of the state, [B, 6, 6] float64 in eV/A^3
        (``DeviceBatch.elastic_tensors`` with this model's ``D3Batch``)."""
        return self._batch.elastic_tensors(state.atomic_numbers, state.positions, self._cells(state), state.pbc,
                                           state.system_idx, relaxed, d3=self.d3)

    def heat_flux(self, state, velocities, convective: bool = True):
        """Heat flux of the network plus D3 energy of every structure of the state, [B, 3] float64 device tensor
        (``DeviceBatch.heat_flux`` with this model's ``D3Batch``): the network's and D3's J_pot and sum_j U_j v_j,
        plus the kinetic part once, with the masses from ``state.masses``.  velocities [n, 3] in the state's atom
        order.  Runs the network's and D3's forward on the state first."""
        cells = self._cells(state)
        self._batch.compute(state.atomic_numbers, state.positions, cells, state.pbc, state.system_idx)
        self.d3.compute(state.atomic_numbers, state.positions, cells, state.pbc, atom_ptr=self._batch.atom_ptr)
        return self._batch.heat_flux(velocities, state.masses if convective else None, convective, d3=self.d3)

    def centroid_virials(self, state):
        """Per-atom centroid virial of the network plus D3 energy of every atom of the state, [n, 3, 3] float64 device
        tensor in eV, in the state's atom order (``DeviceBatch.centroid_virials`` with this model's ``D3Batch``).  Runs
        the network's and D3's forward on the state first."""
        cells = self._cells(state)
        self._batch.compute(state.atomic_numbers, state.positions, cells, state.pbc, state.system_idx)
        self.d3.compute(state.atomic_numbers, state.positions, cells, state.pbc, atom_ptr=self._batch.atom_ptr)
        return self._batch.centroid_virials(d3=self.d3)
