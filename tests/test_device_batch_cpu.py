"""CPU checks of ``batch.DeviceBatch``'s host logic with an engine stand-in that records what reaches
``set_positions_batch``: the species lookup, atom_ptr from system_idx, pbc broadcasting and the errors that must be
raised before the engine is called."""
import numpy as np
import pytest
import torch

from helpers import model_weights, species_of


class RecordingEngine:
    torch = torch
    device = torch.device('cpu')

    def __init__(self):
        from sevenn_b200.spec import build_spec
        self.meta, _ = model_weights('sevennet_0')
        self.spec = build_spec(self.meta)
        self.calls = []

    def set_positions_batch(self, species, positions, atom_ptr, cells, pbc):
        self.calls.append((species, positions, np.asarray(atom_ptr), cells, pbc))


def _batch():
    numbers = np.array([11, 17, 8, 1, 1, 14])
    system_idx = np.array([0, 0, 1, 1, 1, 3])            # structure 2 is empty
    pos = np.arange(18, dtype=np.float64).reshape(6, 3)
    cells = np.stack([np.eye(3) * (5 + b) for b in range(4)])
    return numbers, pos, cells, system_idx


def test_species_and_atom_ptr():
    from sevenn_b200.batch import DeviceBatch
    eng = RecordingEngine()
    numbers, pos, cells, si = _batch()
    DeviceBatch(eng).set_batch(torch.tensor(numbers), torch.tensor(pos, dtype=torch.float32), cells, True, torch.tensor(si))
    sp, p, ap, c, pbc = eng.calls[-1]
    assert np.array_equal(sp.numpy(), species_of(eng.meta, numbers))
    assert np.array_equal(ap, [0, 2, 5, 5, 6])
    assert p.dtype == torch.float32 and c.shape == (4, 3, 3) and pbc is True


def test_errors_before_the_engine_is_called():
    from sevenn_b200.batch import DeviceBatch
    eng = RecordingEngine()
    numbers, pos, cells, si = _batch()
    db = DeviceBatch(eng)
    z = numbers.copy()
    z[4] = 118
    with pytest.raises(ValueError, match='atomic number 118'):
        db.set_batch(z, pos, cells, True, si)
    z[4] = -3
    with pytest.raises(ValueError, match='atomic number -3'):
        db.set_batch(z, pos, cells, True, si)
    with pytest.raises(ValueError, match='sorted'):
        db.set_batch(numbers, pos, cells, True, si[::-1].copy())
    with pytest.raises(ValueError, match=r'\[0, 4\)'):
        db.set_batch(numbers, pos, cells, True, np.array([0, 0, 1, 1, 1, 4]))
    with pytest.raises(ValueError, match='entries'):
        db.set_batch(numbers, pos, cells, True, si[:-1])
    assert eng.calls == []
