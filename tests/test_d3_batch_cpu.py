"""CPU checks of ``d3.D3Batch``'s host logic (``d3.batch_inputs``): atom_ptr from system_idx or as given, the
argument errors raised before the library is called, and ``D3Calculator``'s cell for structures without one.  The
virial's order and sign are checked on the GPU (tests/test_d3_batch_gpu.py), where they are computed."""
import numpy as np
import pytest
import torch

import d3_cells as C

MAX_CUT = np.sqrt(9000.0) * 0.52917726


def _inputs(*args, **kw):
    from sevenn_b200.d3 import batch_inputs
    return batch_inputs(torch, torch.device('cpu'), *args, max_cutoff=MAX_CUT, **kw)


def _batch():
    z_m, pos_m, _, _ = C.molecule()
    numbers = np.concatenate([[11, 17], z_m, [8]])
    pos = np.concatenate([[[0.0, 0.0, 0.0], [2.8, 0.1, 0.0]], pos_m, [[1.0, 2.0, 3.0]]])
    cells = np.stack([np.eye(3) * 5.6, np.zeros((3, 3)), np.zeros((3, 3)), np.eye(3) * 7.0])   # 2: empty, no cell
    si = np.repeat([0, 1, 3], [2, len(z_m), 1])
    return numbers, pos, cells, si


def test_atom_ptr_and_generated_cells():
    numbers, pos, cells, si = _batch()
    z, p, ap, c, pb = _inputs(torch.tensor(numbers), torch.tensor(pos, dtype=torch.float32), cells, False,
                              system_idx=torch.tensor(si))
    assert np.array_equal(ap, [0, 2, 32, 32, 33]) and ap.dtype == np.int32
    assert z.dtype == torch.int32 and p.dtype == torch.float64
    # the molecule gets D3Calculator's cell, computed from the positions it was given (float32 -> float64)
    pm = torch.tensor(pos, dtype=torch.float32).double().numpy()[2:32]
    want = np.eye(3) * (pm.max(axis=0) - pm.min(axis=0) + MAX_CUT + 1.0)
    assert np.array_equal(c[1], want) and pb[1].all()
    assert not c[2].any() and not pb[2].any()                             # the empty structure keeps its zeros
    assert np.array_equal(c[0], cells[0]) and not pb[0].any()
    # the same from atom_ptr, and a one-structure batch needs neither
    _, _, ap2, c2, _ = _inputs(numbers, pos, cells, False, atom_ptr=[0, 2, 32, 32, 33])
    assert np.array_equal(ap2, ap)
    _, _, ap1, _, _ = _inputs(numbers[:2], pos[:2], cells[:1], True)
    assert np.array_equal(ap1, [0, 2])


def test_errors_before_the_library_is_called():
    numbers, pos, cells, si = _batch()
    with pytest.raises(ValueError, match='sorted'):
        _inputs(numbers, pos, cells, True, system_idx=si[::-1].copy())
    with pytest.raises(ValueError, match=r'\[0, 4\)'):
        _inputs(numbers, pos, cells, True, system_idx=np.where(si == 3, 4, si))
    with pytest.raises(ValueError, match='entries'):
        _inputs(numbers, pos, cells, True, system_idx=si[:-1])
    with pytest.raises(ValueError, match='atom_ptr'):
        _inputs(numbers, pos, cells, True, atom_ptr=[0, 2, 32, 33])
    with pytest.raises(ValueError, match='atom_ptr'):
        _inputs(numbers, pos, cells, True, atom_ptr=[0, 2, 32, 31, 33])
    with pytest.raises(ValueError, match='system_idx or atom_ptr'):
        _inputs(numbers, pos, cells, True)
    with pytest.raises(ValueError, match='same number of rows'):
        _inputs(numbers, pos[:-1], cells, True, system_idx=si)
