"""D3 dispersion front-end: ``D3Calculator`` / ``SevenNetD3Calculator`` with the constructor and result
keys of the reference (``sevenn/calculator.py:236-314, 387-618``) on top of the cell-list CUDA kernels of
``csrc/d3_kernels.cuh`` (C ABI ``s7b_d3_*``), plus the multi-GPU driver the reference does not have
(its D3 is single-GPU and limited to 46 340 atoms, ``docs/source/user_guide/d3.md:7,53``), and ``D3Batch``: many
structures in one pass from device-resident arrays, the layout of a TorchSim state (``batch.SevenNetD3Model``).

Unlike the reference binding there is no LAMMPS-frame rotation: the library takes lattice vectors in any
orientation, so forces and the virial come back in the caller's frame.
"""
from __future__ import annotations

import ctypes
import json
import os
from typing import Optional

import numpy as np

from .engine import _host, check, load_library

_PARAMS = None
AU_TO_ANG = 0.52917726
AU_TO_EV = 27.21138505


def d3_tables():
    """Grimme's D3 reference tables, converted from the reference's ``pair_d3_pars.h`` by
    ``tools/convert_d3_params.py`` (``weights/d3_params.npz``)."""
    global _PARAMS
    if _PARAMS is None:
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'weights', 'd3_params.npz')
        f = np.load(path)
        p = {k: f[k] for k in ('r0ab', 'c6ref', 'cnref', 'mxc', 'r2r4', 'rcov')}
        p['functionals'] = json.loads(bytes(f['functionals']).decode())
        _PARAMS = p
    return _PARAMS


class D3Engine:
    """One D3 evaluator on one GPU (thin ctypes host of ``s7b_d3_*``)."""

    def __init__(self, damping_type: str = 'damp_bj', functional_name: str = 'pbe', vdw_cutoff: float = 9000.0,
                 cn_cutoff: float = 1600.0, device: Optional[int] = None):
        import torch
        if not torch.cuda.is_available():
            raise NotImplementedError('CPU + D3 is not implemented')       # same message class as calculator.py:421
        self.torch = torch
        self.lib = load_library()
        self.device = torch.device('cuda', torch.cuda.current_device() if device is None else device)
        damping_type, functional_name = damping_type.lower(), functional_name.lower()
        if damping_type not in ('damp_bj', 'damp_zero'):
            raise ValueError('Error: Invalid damping type.')
        T = d3_tables()
        if functional_name not in T['functionals'][damping_type]:
            raise ValueError(f'Functional name unknown: {functional_name}')
        p = T['functionals'][damping_type][functional_name]
        self.damping = 1 if damping_type == 'damp_bj' else 0
        self.par = dict(s6=p['s6'], s8=p['s18'], a1=p['rs6'], a2=p['rs18'], alp6=p['alp'], alp8=p['alp'] + 2.0)
        self.rthr, self.cnthr = float(vdw_cutoff), float(cn_cutoff)
        self._h = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            check(self.lib.s7b_d3_create(ctypes.byref(self._h)))
        self._numbers = None
        self.n, self.B = 0, 1

    def __del__(self):
        try:
            if getattr(self, '_h', None) is not None and self._h.value:
                self.lib.s7b_d3_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def _set_damping(self):
        check(self.lib.s7b_d3_set_damping(self._h, self.damping, self.par['s6'], self.par['s8'], self.par['a1'],
                                          self.par['a2'], self.par['alp6'], self.par['alp8'], self.rthr, self.cnthr))

    def set_system(self, numbers, positions, cell, pbc=(True, True, True)):
        """numbers [n] atomic numbers, positions [n,3] and cell rows in Angstrom."""
        numbers = np.asarray(numbers, dtype=np.int64)
        uniq = list(dict.fromkeys(numbers.tolist()))            # order of first appearance, as calculator.py:484-492
        if self._numbers != uniq:
            T = d3_tables()
            z = np.array(uniq) - 1
            f8 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
            rcov, r2r4 = f8(T['rcov'][z]), f8(T['r2r4'][z])
            r0, c6 = f8(T['r0ab'][np.ix_(z, z)]), f8(T['c6ref'][np.ix_(z, z)])
            cr, mxc = f8(T['cnref'][z]), np.ascontiguousarray(T['mxc'][z], dtype=np.int32)
            with self.torch.cuda.device(self.device):
                check(self.lib.s7b_d3_set_params(self._h, len(uniq), rcov.ctypes.data, r2r4.ctypes.data, r0.ctypes.data,
                                                 c6.ctypes.data, cr.ctypes.data, mxc.ctypes.data))
                self._set_damping()
            self._numbers = uniq
        lut = {zz: i for i, zz in enumerate(uniq)}
        types = np.ascontiguousarray([lut[int(a)] for a in numbers], dtype=np.int32)
        pos = np.ascontiguousarray(positions, dtype=np.float64).reshape(-1, 3)
        c = np.ascontiguousarray(cell, dtype=np.float64).reshape(3, 3)
        pb = np.ascontiguousarray(np.broadcast_to(np.asarray(pbc, dtype=bool), (3,)).astype(np.int32))
        self.n, self.B = len(types), 1
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_d3_set_system(self._h, self.n, types.ctypes.data, pos.ctypes.data, c.ctypes.data, pb.ctypes.data, self._stream()))
        return self

    def run_stage(self, stage: int, i_begin: int = 0, i_end: Optional[int] = None):
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_d3_run_stage(self._h, stage, i_begin, self.n if i_end is None else i_end, self._stream()))

    def buffer(self, name: str, dtype='f8', shape=None):
        from .engine import _DevView
        n = ctypes.c_size_t()
        ptr = self.lib.s7b_d3_buffer(self._h, name.encode(), ctypes.byref(n))
        shp = (n.value,) if shape is None else tuple(shape)
        return self.torch.as_tensor(_DevView(ptr, shp, '<' + dtype), device=self.device)

    def results(self):
        """(energy eV, forces [n,3] eV/A in the caller's atom order, sigma6 eV = sum f (x) r: xx,yy,zz,xy,xz,yz)"""
        e, s = np.zeros(1), np.zeros(6)
        f = np.zeros((self.n, 3))
        with self.torch.cuda.device(self.device):
            check(self.lib.s7b_d3_results_host(self._h, e.ctypes.data, f.ctypes.data, s.ctypes.data, self._stream()))
        return float(e[0]), f, s

    def compute(self, numbers, positions, cell, pbc=(True, True, True)):
        self.set_system(numbers, positions, cell, pbc)
        for stage in (1, 2, 3):
            self.run_stage(stage)
        return self.results()

    def hvp_strain(self, v=None, strain=None):
        """Second derivatives of the D3 energy along positions and a homogeneous strain together (C ABI
        ``s7b_d3_hvp_strain``): along r -> (I + s eps_b) r + s v for the atoms and cell of every structure b, with the
        forward of the last three stages over all atoms held.  v [n, 3] (Angstrom, caller's atom order) or None
        (zero); strain [B, 3, 3] (general 3x3, applied as eps . r) or None (zero), B = the structure count of the last
        ``D3Batch.compute``, else 1; numpy or torch (any device).  Returns (H v + Lambda eps [n, 3] in eV/A^2 x A resp.
        eV/A, Lambda = d2E/dr de; dW [B, 6], the tangent of the virial in eV, order xx,yy,zz,xy,yz,zx, the order and
        sign of ``B200Engine.hvp_strain``'s), float64 device tensors."""
        torch = self.torch
        n, B = self.n, self.B
        if v is not None:
            v = torch.as_tensor(v).to(self.device, torch.float64).contiguous()
            if v.numel() != 3 * n:
                raise ValueError(f'v has {tuple(v.shape)}, expected [{n}, 3] (atoms)')
        if strain is not None:
            strain = torch.as_tensor(strain).to(self.device, torch.float64).contiguous()
            if strain.numel() != 9 * B:
                raise ValueError(f'strain has {tuple(strain.shape)}, expected [{B}, 3, 3] (one per structure)')
        out = torch.empty(n, 3, dtype=torch.float64, device=self.device)
        dvir = torch.empty(B, 6, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.s7b_d3_hvp_strain(self._h, None if v is None else v.data_ptr(),
                                             None if strain is None else strain.data_ptr(), out.data_ptr(),
                                             dvir.data_ptr(), self._stream()))
        return out, dvir

    def hvp(self, v):
        """H v = (d2E/dr dr) v of the D3 energy, [n, 3] float64 device tensor in eV/A^2 x A: ``hvp_strain(v)[0]``."""
        return self.hvp_strain(v)[0]

    def atomic_energies(self):
        """D3's atomic energies U_j = -1/2 sum_{k,tau} C6_jk g(r_jk) of the last pair stage (self images included; they
        sum to the energy), [n] float64 device tensor in eV, caller's atom order"""
        torch = self.torch
        out = torch.zeros(self.n, dtype=torch.float64, device=self.device)
        if self.n:
            order = self.buffer('order', dtype='i4').long()
            out[order] = self.buffer('eatom') * AU_TO_EV
        return out

    def heat_flux(self, v):
        """Heat flux of D3's atomic energies (C ABI ``s7b_d3_heat_flux``, DESIGN.md §8.4) with the forward of the last
        three stages over all atoms held.  v [n, 3] velocities (Angstrom x any time unit, caller's atom order), numpy or
        torch (any device).  Returns (jpot, ju), [B, 3] float64 device tensors, B = the structure count of the last
        ``D3Batch.compute``, else 1: jpot = sum_j sum_i (r_j - r_i) (dU_j/dr_i . v_i) over every atom and periodic
        image i that U_j depends on, ju = sum_j U_j v_j (U_j = ``atomic_energies``).  Units: eV A x (the unit of v).
        Two cell-list passes; a periodic cell needs no unfolding."""
        torch = self.torch
        n, B = self.n, self.B
        v = torch.as_tensor(v).to(self.device, torch.float64).contiguous()
        if v.numel() != 3 * n or (v.dim() == 2 and v.shape[1] != 3) or v.dim() > 2:
            raise ValueError(f'v has {tuple(v.shape)}, expected [{n}, 3] (atoms)')
        jpot = torch.empty(B, 3, dtype=torch.float64, device=self.device)
        ju = torch.empty(B, 3, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.s7b_d3_heat_flux(self._h, v.data_ptr(), jpot.data_ptr(), ju.data_ptr(), self._stream()))
        return jpot, ju

    def centroid_virial(self):
        """Per-atom centroid virial of D3's atomic energies (C ABI ``s7b_d3_centroid_virial``, DESIGN.md §8.6) with the
        forward of the last three stages over all atoms held: [n, 3, 3] float64 device tensor in eV, caller's atom
        order, Wc_i[a, b] = sum_j sum_i' (r_j - r_i')_a dU_j/dr_i',b over atom i and its periodic images i'
        (U_j = ``atomic_energies``).  sum_i Wc_i over a structure is its virial, and sum_i Wc_i v_i is ``heat_flux(v)``'s
        jpot for any v.  Not symmetric: row a is the flux direction, column b the velocity direction.  Two cell-list
        passes; a periodic cell needs no unfolding."""
        torch = self.torch
        out = torch.empty(self.n, 3, 3, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            check(self.lib.s7b_d3_centroid_virial(self._h, out.data_ptr(), self._stream()))
        return out


def _rank_range(n, world, rank):
    """(chunk, lo, hi): rank's contiguous slice [lo, hi) of n bin-sorted atoms cut into `world` chunks (the last may
    be short or empty)"""
    chunk = (n + world - 1) // world
    return chunk, min(rank * chunk, n), min((rank + 1) * chunk, n)


def _gather_range(engine, name, width, lo, hi, chunk, group, dtype='f8'):
    """all-gather the rows [lo, hi) of every rank into the engine's device buffer `name` ([n] or [n, width] of
    `dtype`), in place: each rank's slice is padded to `chunk` rows for the collective"""
    import torch
    import torch.distributed as dist
    world, n = dist.get_world_size(group), engine.n
    buf = engine.buffer(name, dtype=dtype, shape=(n, width) if width > 1 else (n,))
    padded = torch.zeros((world * chunk,) + tuple(buf.shape[1:]), dtype=buf.dtype, device=buf.device)
    mine = torch.zeros((chunk,) + tuple(buf.shape[1:]), dtype=buf.dtype, device=buf.device)
    mine[:hi - lo] = buf[lo:hi]
    dist.all_gather_into_tensor(padded, mine, group=group)
    buf.copy_(padded[:n])


def distributed_d3(engine: D3Engine, numbers, positions, cell, pbc=(True, True, True), group=None):
    """The same system on every rank (positions replicated: the 50 A interaction range is of the order of the
    box), each rank evaluating a contiguous slice of the bin-sorted atoms; ``cn`` and ``dc6i`` are
    all-gathered between the stages (NCCL), energy / virial all-reduced, forces all-gathered.
    Returns (energy, forces [n,3], sigma6) on every rank.  The engine keeps the range forward for
    ``distributed_d3_centroid_virials`` and ``distributed_d3_heat_flux``."""
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    engine.set_system(numbers, positions, cell, pbc)
    chunk, lo, hi = _rank_range(engine.n, world, rank)
    engine.run_stage(1, lo, hi)
    _gather_range(engine, 'cn', 1, lo, hi, chunk, group)
    engine.run_stage(2, lo, hi)
    _gather_range(engine, 'dc6i', 1, lo, hi, chunk, group)
    engine.run_stage(3, lo, hi)
    _gather_range(engine, 'force', 3, lo, hi, chunk, group)
    for name in ('energy', 'sigma'):
        dist.all_reduce(engine.buffer(name), group=group)
    return engine.results()


def distributed_d3_centroid_virials(engine: D3Engine, group=None):
    """``D3Engine.centroid_virial`` after ``distributed_d3`` on the same group (C ABI ``s7b_d3_centroid_pass``,
    DESIGN.md §8.8): each rank runs both passes on its slice of the bin-sorted atoms, with the packed neighbour
    record (16 B per atom) all-gathered between them and the rows (72 B per atom) after them.  Returns [n, 3, 3]
    float64 device tensor in eV, caller's atom order, the same on every rank and bit for bit that of the one-GPU
    call.  Collective."""
    import torch
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = engine.n
    chunk, lo, hi = _rank_range(n, world, rank)
    with torch.cuda.device(engine.device):
        check(engine.lib.s7b_d3_centroid_pass(engine._h, 1, lo, hi, engine._stream()))
        _gather_range(engine, 'ct_nb', 4, lo, hi, chunk, group, dtype='f4')
        check(engine.lib.s7b_d3_centroid_pass(engine._h, 2, lo, hi, engine._stream()))
        _gather_range(engine, 'ct_out', 9, lo, hi, chunk, group)
    out = torch.empty(n, 9, dtype=torch.float64, device=engine.device)
    if n:
        out[engine.buffer('order', dtype='i4').long()] = engine.buffer('ct_out', shape=(n, 9))
    return out.reshape(n, 3, 3)


def distributed_d3_heat_flux(engine: D3Engine, v, group=None):
    """``D3Engine.heat_flux(v)`` after ``distributed_d3`` on the same group (C ABI ``s7b_d3_heat_flux_pass``,
    DESIGN.md §8.8): each rank runs both passes on its slice of the bin-sorted atoms, with the packed neighbour
    record (32 B per atom) all-gathered between them and the per-atom terms (48 B per atom) after them; every rank
    then sums all n rows in the one-GPU order.  v [n, 3] every atom's velocity (Angstrom x any time unit, caller's
    atom order), numpy or torch.  Returns (jpot, ju), [3] float64 device tensors in eV A x (the unit of v), the same
    on every rank and bit for bit those of the one-GPU call.  Collective."""
    import torch
    import torch.distributed as dist
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = engine.n
    v = torch.as_tensor(v).to(engine.device, torch.float64).contiguous()
    if v.numel() != 3 * n or (v.dim() == 2 and v.shape[1] != 3) or v.dim() > 2:
        raise ValueError(f'v has {tuple(v.shape)}, expected [{n}, 3] (atoms)')
    chunk, lo, hi = _rank_range(n, world, rank)
    jpot = torch.empty(1, 3, dtype=torch.float64, device=engine.device)
    ju = torch.empty(1, 3, dtype=torch.float64, device=engine.device)
    with torch.cuda.device(engine.device):
        check(engine.lib.s7b_d3_heat_flux_pass(engine._h, 1, v.data_ptr(), lo, hi, engine._stream()))
        _gather_range(engine, 'fx_nb', 8, lo, hi, chunk, group, dtype='f4')
        check(engine.lib.s7b_d3_heat_flux_pass(engine._h, 2, None, lo, hi, engine._stream()))
        _gather_range(engine, 'fx_out', 6, lo, hi, chunk, group)
        check(engine.lib.s7b_d3_heat_flux_sums(engine._h, jpot.data_ptr(), ju.data_ptr(), engine._stream()))
    return jpot[0], ju[0]


def batch_inputs(torch, device, numbers, positions, cells, pbc, system_idx=None, atom_ptr=None, max_cutoff=None):
    """Host logic of ``D3Batch.compute``: (numbers int32 [n] and positions float64 [n,3] on ``device``, atom_ptr int32
    [B+1], cells float64 [B,3,3], pbc int32 [B,3]; the last three on the host).  atom_ptr is taken as given, else
    derived from system_idx (one readback), else the batch is one structure.  A non-empty structure with an
    all-zero cell gets ``D3Calculator``'s cell: an orthogonal box of its extent + max_cutoff + 1 A, periodic; the
    extents are a device min / max, read back only when such a structure is present."""
    z = torch.as_tensor(numbers).detach().to(device, torch.int32).contiguous().reshape(-1)
    pos = torch.as_tensor(positions).detach().to(device, torch.float64).contiguous().reshape(-1, 3)
    c = np.array(_host(cells), dtype=np.float64).reshape(-1, 3, 3)
    B, n = int(c.shape[0]), int(z.shape[0])
    if B < 1:
        raise ValueError('empty batch')
    if pos.shape[0] != n:
        raise ValueError(f'numbers ({n}) and positions ({pos.shape[0]}) need the same number of rows')
    pb = np.array(np.broadcast_to(np.asarray(_host(pbc), dtype=bool), (B, 3)))
    if atom_ptr is not None:
        ap = np.array(_host(atom_ptr), dtype=np.int64).ravel()
        if ap.shape[0] != B + 1 or ap[0] != 0 or ap[-1] != n or (np.diff(ap) < 0).any():
            raise ValueError(f'atom_ptr must be non-decreasing, [B+1] = [{B + 1}], from 0 to {n}')
    elif system_idx is not None:
        si = torch.as_tensor(system_idx).detach().to(device, torch.int64).reshape(-1)
        if si.shape[0] != n:
            raise ValueError(f'system_idx has {si.shape[0]} entries for {n} atoms')
        flags = torch.zeros(2, dtype=torch.int64, device=device)
        if n > 0:                 # one readback: unsorted, out of range, then atom_ptr
            flags[0] = (si[1:] < si[:-1]).any()
            flags[1] = (si.min() < 0) | (si.max() >= B)
        counts = torch.bincount(si.clamp(0, B - 1), minlength=B)
        h = torch.cat([flags, torch.zeros(1, dtype=torch.int64, device=device), torch.cumsum(counts, 0)]).cpu().numpy()
        if h[0]:
            raise ValueError('system_idx must be sorted')
        if h[1]:
            raise ValueError(f'system_idx must lie in [0, {B}): one structure per cell')
        ap = h[2:]
    elif B == 1:
        ap = np.array([0, n])
    else:
        raise ValueError('a batch of several structures needs system_idx or atom_ptr')
    zero = np.flatnonzero((c.reshape(B, 9) == 0).all(1) & (ap[1:] > ap[:-1]))
    if zero.size:
        sys = torch.repeat_interleave(torch.arange(B, device=device), torch.as_tensor(np.diff(ap), device=device))
        idx = sys[:, None].expand(-1, 3)
        lo = torch.full((B, 3), np.inf, dtype=torch.float64, device=device).scatter_reduce(0, idx, pos, 'amin')
        hi = torch.full((B, 3), -np.inf, dtype=torch.float64, device=device).scatter_reduce(0, idx, pos, 'amax')
        zi = torch.as_tensor(zero, device=device)
        lohi = torch.stack([lo[zi], hi[zi]], 1).cpu().numpy()
        for k, b in enumerate(zero):       # D3Calculator.calculate, for this structure alone
            c[b] = np.eye(3) * (lohi[k, 1] - lohi[k, 0] + max_cutoff + 1.0)
            pb[b] = True
    return z, pos, np.ascontiguousarray(ap, dtype=np.int32), c, np.ascontiguousarray(pb.astype(np.int32))


class D3Batch:
    """D3 of B structures in one pass on one GPU (C ABI ``s7b_d3_set_system_batch``): atomic numbers and positions
    stay on the device, the full element tables are uploaded once, every structure has its own cell list and at most
    16 elements (any number in the batch).  Damping and functional as ``D3Engine``; ``engine`` is that D3Engine,
    whose ``buffer`` views show the per-atom values of the last batch (bin-sorted order, ``order`` maps them)."""

    def __init__(self, damping_type: str = 'damp_bj', functional_name: str = 'pbe', vdw_cutoff: float = 9000.0,
                 cn_cutoff: float = 1600.0, device: Optional[int] = None):
        self.engine = eng = D3Engine(damping_type, functional_name, vdw_cutoff, cn_cutoff, device=device)
        self.torch, self.device = eng.torch, eng.device
        self.max_cutoff = np.sqrt(max(eng.rthr, eng.cnthr)) * AU_TO_ANG        # D3Calculator's zero-cell rule
        T = d3_tables()
        f8 = lambda a: np.ascontiguousarray(a, dtype=np.float64)
        self._tables = [f8(T['rcov']), f8(T['r2r4']), f8(T['r0ab']), f8(T['c6ref']), f8(T['cnref']),
                        np.ascontiguousarray(T['mxc'], dtype=np.int32)]
        with self.torch.cuda.device(self.device):
            check(eng.lib.s7b_d3_set_element_tables(eng._h, *[a.ctypes.data for a in self._tables]))
            eng._set_damping()
        self.cells = self.pbc = self.atom_ptr = None

    def compute(self, numbers, positions, cells, pbc, system_idx=None, atom_ptr=None) -> dict:
        """numbers [n] atomic numbers, positions [n,3] (Angstrom, float32 or float64), cells [B,3,3] (rows), pbc
        ([3] or [B,3]), and system_idx [n] (sorted) or atom_ptr [B+1]: torch tensors on any device, or numpy arrays.
        -> dict of float64 device tensors: energy [B] (eV), forces [n,3] (eV/A), virial [B,6] (eV; xx,yy,zz,xy,yz,zx,
        the order and sign of ``DeviceBatch``'s virial).  ``self.cells`` / ``self.pbc`` hold the cells used."""
        torch, eng = self.torch, self.engine
        z, pos, ap, c, pb = batch_inputs(torch, self.device, numbers, positions, cells, pbc, system_idx, atom_ptr,
                                         self.max_cutoff)
        B, n = len(ap) - 1, int(ap[-1])
        self.cells, self.pbc = c, pb.astype(bool)
        cc = np.ascontiguousarray(c.reshape(B, 9))
        energy = torch.empty(B, dtype=torch.float64, device=self.device)
        forces = torch.empty(n, 3, dtype=torch.float64, device=self.device)
        virial = torch.empty(B, 6, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            st = eng._stream()
            check(eng.lib.s7b_d3_set_system_batch(eng._h, B, ap.ctypes.data, z.data_ptr(), pos.data_ptr(), cc.ctypes.data,
                                                  pb.ctypes.data, st))
            eng.n, eng.B = n, B
            self.atom_ptr = ap
            for stage in (1, 2, 3):
                check(eng.lib.s7b_d3_run_stage(eng._h, stage, 0, n, st))
            check(eng.lib.s7b_d3_system_results(eng._h, energy.data_ptr(), forces.data_ptr(), virial.data_ptr(), st))
        return dict(energy=energy, forces=forces, virial=virial)

    def hvp_strain(self, v=None, strain=None):
        """``D3Engine.hvp_strain`` on the last batch: v [n, 3] (Angstrom) or None, strain [B, 3, 3] (one per
        structure of ``atom_ptr``) or None -> (out [n, 3], dW [B, 6]), float64 device tensors.  D3 has no pair between
        the structures of a batch, so each structure's products are those of the structure alone."""
        if self.atom_ptr is None:
            raise RuntimeError('no batch: call compute first')
        return self.engine.hvp_strain(v, strain)

    def heat_flux(self, v):
        """``D3Engine.heat_flux`` on the last batch: v [n, 3] velocities -> (jpot [B, 3], ju [B, 3]), float64 device
        tensors.  Each structure's flux is that of the structure alone."""
        if self.atom_ptr is None:
            raise RuntimeError('no batch: call compute first')
        return self.engine.heat_flux(v)

    def centroid_virials(self):
        """``D3Engine.centroid_virial`` on the last batch: [n, 3, 3] float64 device tensor in eV, in the atom order of
        ``compute``.  Each row is that of its structure alone."""
        if self.atom_ptr is None:
            raise RuntimeError('no batch: call compute first')
        return self.engine.centroid_virial()


try:
    from ase.calculators.calculator import Calculator as _Base, all_changes as _all_changes
except Exception:   # ASE absent (as in the build container): duck-typed base, as sevenn_b200.calculator does
    _all_changes = ['positions', 'numbers', 'cell', 'pbc']

    class _Base:
        implemented_properties: list = []

        def __init__(self, **kwargs):
            self.results, self.atoms = {}, None

        def calculate(self, atoms=None, properties=None, system_changes=_all_changes):
            self.atoms = atoms


class D3Calculator(_Base):
    """ASE-style calculator of the D3 correction; constructor and ``results`` keys of
    ``sevenn/calculator.py:387-618`` (``free_energy, energy, forces, stress``)."""
    implemented_properties = ['free_energy', 'energy', 'forces', 'stress']

    def __init__(self, damping_type: str = 'damp_bj', functional_name: str = 'pbe', vdw_cutoff: float = 9000,
                 cn_cutoff: float = 1600, **kwargs):
        device = kwargs.pop('device', None)
        super().__init__(**kwargs)
        self.rthr, self.cnthr = vdw_cutoff, cn_cutoff
        self.engine = D3Engine(damping_type, functional_name, vdw_cutoff, cn_cutoff, device=device)
        self._engine_inputs = None     # (numbers, positions, cell, pbc) of the engine's current forward

    def _remember(self, numbers, pos, cell, pbc):
        self._engine_inputs = tuple(np.array(a, copy=True) for a in (numbers, pos, cell, pbc))

    def _inputs(self, atoms):
        """(numbers, positions, cell, pbc, generated) that ``calculate`` evaluates ``atoms`` with; a structure without
        a cell gets an orthogonal cell large enough, periodic (``generated``), and ``atoms`` is not modified."""
        cell = np.asarray(atoms.get_cell(), dtype=np.float64).reshape(3, 3)
        pbc = np.asarray(atoms.get_pbc(), dtype=bool)
        pos = np.asarray(atoms.get_positions(), dtype=np.float64)
        generated = cell.sum() == 0      # calculator.py:534-547: periodic "for minus positions"
        if generated:
            max_cutoff = np.sqrt(max(self.rthr, self.cnthr)) * AU_TO_ANG
            cell = np.eye(3) * (pos.max(axis=0) - pos.min(axis=0) + max_cutoff + 1.0)
            pbc = np.array([True, True, True])
        return np.asarray(atoms.get_atomic_numbers()), pos, cell, pbc, generated

    def calculate(self, atoms=None, properties=None, system_changes=_all_changes):
        super().calculate(atoms, properties, system_changes)
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        numbers, pos, cell, pbc, generated = self._inputs(atoms)
        if generated:
            print('Warning: D3Calculator requires a cell.\nWarning: An orthogonal cell large enough is generated.')
            atoms.set_cell(cell)
            atoms.set_pbc(pbc)
        energy, forces, s = self.engine.compute(numbers, pos, cell, pbc)
        self._remember(numbers, pos, cell, pbc)
        vol = abs(np.linalg.det(cell))
        stress = -np.array([s[0], s[1], s[2], s[5], s[4], s[3]]) / vol        # calculator.py:515-526 + /volume (:608)
        self.results = {'free_energy': energy, 'energy': energy, 'forces': forces, 'stress': stress}
        return self.results

    def _forward(self, atoms):
        """the three stages on ``atoms`` (``calculate``'s cell rule, ``atoms`` unmodified), held for the products"""
        numbers, pos, cell, pbc, _ = self._inputs(atoms)
        self.engine.set_system(numbers, pos, cell, pbc)
        for stage in (1, 2, 3):
            self.engine.run_stage(stage)
        self._remember(numbers, pos, cell, pbc)

    def _forward_if_changed(self, atoms):
        """Leave the engine on the forward of ``atoms``: the three stages run only when numbers, positions, cell or
        pbc (as ``calculate`` evaluates them) differ from those of the engine's current forward"""
        numbers, pos, cell, pbc, _ = self._inputs(atoms)
        last = self._engine_inputs
        if last is None or not all(np.array_equal(a, b) for a, b in zip(last, (numbers, pos, cell, pbc))):
            self._forward(atoms)

    def _flux_parts(self, atoms):
        """(J_pot [3], sum_j U_j v_j [3], velocities [n, 3]) of ``atoms``; the three stages run only when numbers,
        positions, cell or pbc (as ``calculate`` evaluates them) differ from those of the engine's current forward"""
        self._forward_if_changed(atoms)
        v = np.asarray(atoms.get_velocities(), dtype=np.float64).reshape(-1, 3)
        jpot, ju = self.engine.heat_flux(v)
        return jpot[0].cpu().numpy(), ju[0].cpu().numpy(), v

    def get_heat_flux(self, atoms=None, convective: bool = True) -> np.ndarray:
        """Energy-barycentre heat flux of the D3 energy of ``atoms`` (default: the calculator's atoms), [3] float64
        (``SevenNetCalculator.get_heat_flux``'s definition and units, DESIGN.md §8.4): J_pot + sum_j (U_j + m_j |v_j|^2
        / 2) v_j with D3's atomic energies U_j (``D3Engine.atomic_energies``).  Velocities and masses come from
        ``atoms``; ``convective=False`` gives J_pot alone.  A structure without a cell is evaluated in ``calculate``'s
        generated cell (``atoms`` is not modified).  The three stages run only when positions, numbers, cell or pbc
        differ from those of the last D3 forward; ``results`` is not touched."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        jpot, ju, v = self._flux_parts(atoms)
        if not convective:
            return jpot
        from .heat_flux import kinetic_flux
        return jpot + ju + kinetic_flux(v, atoms.get_masses())[0]

    def get_centroid_virials(self, atoms=None) -> np.ndarray:
        """Per-atom centroid virial of the D3 energy of ``atoms`` (default: the calculator's atoms), [N, 3, 3] float64
        in eV (``D3Engine.centroid_virial``, DESIGN.md §8.6): Wc_i[a, b] = sum_j sum_i' (r_j - r_i')_a dU_j/dr_i',b with
        D3's atomic energies U_j.  sum_i Wc_i is the virial and sum_i Wc_i v_i is ``get_heat_flux(convective=False)``.  A
        structure without a cell is evaluated in ``calculate``'s generated cell (``atoms`` is not modified).  The three
        stages run only when positions, numbers, cell or pbc differ from those of the last D3 forward; ``results`` is
        not touched."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        self._forward_if_changed(atoms)
        return self.engine.centroid_virial().cpu().numpy()

    def get_hessian(self, atoms=None) -> np.ndarray:
        """Hessian d2E/dr dr of the D3 energy of ``atoms`` (default: the calculator's atoms), [3N, 3N] float64 in
        eV/A^2, row 3i + a = H e_(i,a), from 3N Hessian-vector products (``D3Engine.hvp``).  A periodic cell gives the
        Gamma-point (supercell) Hessian; a structure without a cell is evaluated in ``calculate``'s generated cell
        (``atoms`` is not modified).  Not symmetrised (the two triangles agree to the fp32 error of the pair
        arithmetic); ``.reshape(N, 3, N, 3)`` gives the force constants.  ``results`` is not touched."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        self._forward(atoms)
        eng, torch = self.engine, self.engine.torch
        n = eng.n
        eye = torch.eye(3 * n, dtype=torch.float64, device=eng.device)
        rows = [eng.hvp(eye[k].reshape(n, 3)).reshape(-1) for k in range(3 * n)]
        if not rows:
            return np.zeros((0, 0))
        return torch.stack(rows).cpu().numpy()

    def _strain_pieces(self, atoms, relaxed: bool):
        """The raw second derivatives ``elastic.elastic_tensor`` assembles: (dvirial [6, 6], outs [6, N, 3], volume,
        Hessian [3N, 3N] or None), from the six Voigt strain products and, when ``relaxed``, the Hessian."""
        cell = np.asarray(atoms.get_cell(), dtype=np.float64).reshape(3, 3)
        vol = abs(np.linalg.det(cell))
        if not np.asarray(atoms.get_pbc(), dtype=bool).all() or not vol > 0:
            raise ValueError('the elastic tensor needs a cell periodic in all three directions with a volume > 0')
        from . import elastic
        if relaxed:
            hessian = self.get_hessian(atoms)          # leaves the engine on the atoms' forward
        else:
            hessian = None
            self._forward(atoms)
        outs, dvir = [], []
        for eps in elastic.voigt_strains():
            o, d = self.engine.hvp_strain(None, eps[None])
            outs.append(o)
            dvir.append(d[0])
        torch = self.engine.torch
        return torch.stack(dvir).cpu().numpy(), torch.stack(outs).cpu().numpy(), vol, hessian

    def get_elastic_tensor(self, atoms=None, relaxed: bool = True) -> np.ndarray:
        """Elastic tensor d2E/de de / V of the D3 energy of ``atoms`` (default: the calculator's atoms), [6, 6] float64
        in eV/A^3, ASE Voigt order, engineering strains: ``SevenNetCalculator.get_elastic_tensor``'s definitions,
        units and refusals (``sevenn_b200.elastic``).  Six strain products (``D3Engine.hvp_strain``), plus the Hessian
        (3N products) when ``relaxed``.  All three directions must be periodic."""
        from . import elastic
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        return elastic.elastic_tensor(*self._strain_pieces(atoms, relaxed))


class SevenNetD3Calculator(_Base):
    """``SevenNetCalculator`` + ``D3Calculator`` summed (the reference builds an ASE SumCalculator,
    ``sevenn/calculator.py:236-314``; without ASE the two result dicts are added here)."""
    implemented_properties = ['free_energy', 'energy', 'energies', 'forces', 'stress']

    def __init__(self, model='7net-0', file_type: str = 'checkpoint', device='auto', modal=None, enable_cueq=False,
                 enable_flash=False, enable_oeq=False, sevennet_config=None, damping_type: str = 'damp_bj',
                 functional_name: str = 'pbe', vdw_cutoff: float = 9000, cn_cutoff: float = 1600, **kwargs):
        from .calculator import SevenNetCalculator
        super().__init__()
        self.d3_calc = D3Calculator(damping_type=damping_type, functional_name=functional_name, vdw_cutoff=vdw_cutoff,
                                    cn_cutoff=cn_cutoff)
        self.sevennet_calc = SevenNetCalculator(model=model, file_type=file_type, device=device, modal=modal,
                                                enable_cueq=enable_cueq, enable_flash=enable_flash, enable_oeq=enable_oeq,
                                                sevennet_config=sevennet_config, **kwargs)

    def calculate(self, atoms=None, properties=None, system_changes=_all_changes):
        super().calculate(atoms, properties, system_changes)
        a = self.sevennet_calc.calculate(atoms, properties, system_changes)
        b = self.d3_calc.calculate(atoms, properties, system_changes)
        out = dict(a)
        for k in ('free_energy', 'energy', 'forces'):
            out[k] = a[k] + b[k]
        if 'stress' in a:
            out['stress'] = a['stress'] + b['stress']
        self.results = out
        return out

    def get_hessian(self, atoms=None) -> np.ndarray:
        """Hessian of the network plus D3 energy, [3N, 3N] float64 in eV/A^2: ``SevenNetCalculator.get_hessian`` +
        ``D3Calculator.get_hessian``, summed in fp64."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        return self.sevennet_calc.get_hessian(atoms) + self.d3_calc.get_hessian(atoms)

    def get_elastic_tensor(self, atoms=None, relaxed: bool = True) -> np.ndarray:
        """Elastic tensor of the network plus D3 energy, [6, 6] float64 in eV/A^3 (``SevenNetCalculator.
        get_elastic_tensor``'s definitions).  The two terms' strain products and Hessians are summed before the
        assembly: the relaxed-ion tensor C0 - Lambda^T H+ Lambda / V is not linear in (Lambda, H), so it is not the
        sum of the two terms' relaxed-ion tensors."""
        from . import elastic
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        dv_a, outs_a, vol, h_a = self.sevennet_calc._strain_pieces(atoms, relaxed)
        dv_b, outs_b, _, h_b = self.d3_calc._strain_pieces(atoms, relaxed)
        return elastic.elastic_tensor(dv_a + dv_b, outs_a + outs_b, vol, h_a + h_b if relaxed else None)

    def get_heat_flux(self, atoms=None, convective: bool = True) -> np.ndarray:
        """Energy-barycentre heat flux of the network plus D3 energy, [3] float64 (``SevenNetCalculator.
        get_heat_flux``'s definition and units): the atomic energies are the network's plus D3's, so J_pot and
        sum_j U_j v_j are the sums of the two terms', and the kinetic part sum_j m_j |v_j|^2 / 2 v_j is added once.
        Each term's forward runs only when the atoms changed since its last one; ``results`` is not touched."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        jp_a, ju_a, v = self.sevennet_calc._flux_parts(atoms)
        jp_b, ju_b, _ = self.d3_calc._flux_parts(atoms)
        if not convective:
            return jp_a + jp_b
        from .heat_flux import kinetic_flux
        return jp_a + jp_b + ju_a + ju_b + kinetic_flux(v, atoms.get_masses())[0]

    def get_centroid_virials(self, atoms=None) -> np.ndarray:
        """Per-atom centroid virial of the network plus D3 energy, [N, 3, 3] float64 in eV (``SevenNetCalculator.
        get_centroid_virials``'s definition): the atomic energies are the network's plus D3's, so Wc is the sum of
        the two terms', in fp64.  Each term's forward runs only when the atoms changed since its last one; ``results``
        is not touched."""
        atoms = atoms if atoms is not None else self.atoms
        if atoms is None:
            raise ValueError('No atoms to evaluate')
        return self.sevennet_calc.get_centroid_virials(atoms) + self.d3_calc.get_centroid_virials(atoms)
