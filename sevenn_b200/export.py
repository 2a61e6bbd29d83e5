"""Flat binary export of a prepared model for non-Python hosts (LAMMPS-style C++ callers).

File layout (little endian), consumed by ``examples/host_entry.cpp``:
    magic    8 bytes  b'S7BMODEL'
    version  int32    1
    desc     sizeof(S7bModelDesc) bytes, exactly the C struct of include/sevenn_b200.h
    n_arrays int32
    n_types  int32, then n_types x (atomic number int32, species index int32)
    then per array: name char[32] (NUL padded), layer int32, numel int64, numel x float32
The arrays are the ones ``sevenn_b200.engine.prepare_params`` produces (normalisations folded in,
radial tables packed), i.e. exactly what ``s7b_engine_set_param`` takes.
"""
from __future__ import annotations

import struct

import numpy as np

from .engine import default_table_knots, model_desc, prepare_params
from .spec import build_spec


def export_flat(path: str, meta: dict, arrays, radial: str = 'table', knots=None, radial_mlp: bool = False) -> None:
    """``radial_mlp``: a 'table' file also carries the radial MLP (mlp0..2 of every layer), which the second-order
    passes evaluate in both radial modes (s7b_engine_hvp, s7b_engine_heat_flux, s7b_engine_centroid_virial; a LAMMPS
    run whose compute centroid/stress/atom makes pair_style e3gnn/b200 fill cvatom).  An 'mlp' file always has it."""
    spec = build_spec(meta)
    knots = (knots or default_table_knots(spec)) if radial == 'table' else 0
    params = prepare_params(spec, arrays, radial, knots)
    if radial == 'table' and radial_mlp:
        params.update({k: v for k, v in prepare_params(spec, arrays, 'mlp', 0).items() if k[0] in ('mlp0', 'mlp1', 'mlp2')})
    d = model_desc(spec, knots)
    with open(path, 'wb') as f:
        f.write(b'S7BMODEL')
        f.write(struct.pack('<i', 1))
        f.write(bytes(d))
        f.write(struct.pack('<i', len(params)))
        f.write(struct.pack('<i', len(spec.type_map)))
        for z, idx in sorted(spec.type_map.items()):
            f.write(struct.pack('<ii', int(z), int(idx)))
        for (name, layer), arr in params.items():
            a = np.ascontiguousarray(arr, dtype=np.float32)
            f.write(name.encode().ljust(32, b'\0'))
            f.write(struct.pack('<iq', int(layer), int(a.size)))
            f.write(a.tobytes())
