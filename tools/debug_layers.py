"""GPU debugging aid: run the engine stage by stage and report, for every intermediate the
oracle also produces, the max abs difference (engine vs fp64 oracle), and the first stage that
diverges.  Usage:
    python tools/debug_layers.py [sevennet_0|sevennet_l3i5] [table|mlp] [ncell]
"""
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from helpers import first_divergence, format_stage_errors, model_weights, oracle, species_of, stage_errors  # noqa: E402
from sevenn_b200.engine import B200Engine  # noqa: E402
from sevenn_b200.neighbors import build_graph, diamond_si  # noqa: E402


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else 'sevennet_0'
    radial = sys.argv[2] if len(sys.argv) > 2 else 'table'
    nc = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    meta, arrays = model_weights(name)
    pos, cell, z = diamond_si(nc, nc, nc)
    ei, ev = build_graph(pos, cell, True, 5.0)
    species = species_of(meta, z)
    ref = oracle(name).forward(species, ei, ev, volume=abs(np.linalg.det(cell)), keep=True)
    errors = stage_errors(B200Engine(meta, arrays, radial=radial), arrays, species, ei, ev, ref)
    print(format_stage_errors(errors))
    print('first divergence:', first_divergence(errors))


if __name__ == '__main__':
    main()
