"""The tile rule of the sparse box3d tower (csrc/tower_tiles.cu, mirrored by tools/tower_coverage.py tile_lists): tower layer
i of `depth` must compute every pixel that reaches a sparse-predictor read through the remaining layers' 3x3 receptive fields.
Brute force: propagate the predictor's 3x3 reads backwards through the tower one 3x3 conv at a time, then cover the needed
pixels with conv tiles."""
import importlib.util
import os

import numpy as np
import pytest

_spec = importlib.util.spec_from_file_location(
    "tower_coverage", os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools", "tower_coverage.py"))
tower_coverage = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(tower_coverage)


def _grow(mask):  # pixels a 3x3 zero-padded conv reads to produce `mask`
    H, W = mask.shape
    p = np.pad(mask, 1)
    return np.any([p[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], axis=0)


def _brute_force(cands, H, W, depth, th, tw):
    need = np.zeros((H, W), bool)
    for y, x in cands:
        need[y, x] = True
    need = _grow(need)  # the predictor's 3x3 reads of the last tower layer's output
    tiles_x = -(-W // tw)
    out = [None] * depth
    for i in reversed(range(depth)):
        ys, xs = np.nonzero(need)
        out[i] = np.unique((ys // th) * tiles_x + xs // tw)
        need = _grow(need)  # what layer i reads of layer i - 1
    return out


@pytest.mark.parametrize("H,W,depth,th,tw,n,seed", [
    (56, 100, 4, 16, 8, 30, 0),    # tiles cut by the map edge in both directions
    (13, 21, 4, 16, 8, 5, 1),      # map smaller than a few tiles
    (64, 64, 2, 16, 8, 12, 2),
    (30, 37, 1, 8, 16, 9, 3),      # generic tile shape
    (100, 160, 6, 16, 8, 60, 4),
    (40, 40, 4, 16, 8, 0, 5),      # no candidates
])
def test_tile_rule_matches_receptive_field(H, W, depth, th, tw, n, seed):
    rng = np.random.default_rng(seed)
    cands = np.stack([rng.integers(0, H, n), rng.integers(0, W, n)], 1)
    # candidates on every border and corner of the map
    cands = np.concatenate([cands, [[0, 0], [H - 1, W - 1], [0, W - 1], [H - 1, 0], [H // 2, 0], [0, W // 2]]]) if n else cands
    got = tower_coverage.tile_lists(cands, H, W, depth, th, tw)
    want = _brute_force(cands, H, W, depth, th, tw)
    assert len(got) == depth
    for i in range(depth):
        assert np.array_equal(got[i], want[i]), f"layer {i}"
