"""The rule of the sparse box2d tower (csrc/tower_tiles.cu, mirrored by tools/tower_coverage.py), on the CPU:

  * the d + 1 tile lists (tower layers at dilation d .. 1, the predictor at dilation 0) cover every pixel that reaches a
    read of the decode through the predictor's and the tower's 3x3 receptive fields (brute-force propagation);
  * the seed set P (some class passes the threshold alone, class_passes in csrc/detect.cuh) holds every pixel the oracle's
    decode keeps as a pre-NMS candidate, with the threshold on the product and without it;
  * the inequality that makes this hold with THRESH_WITH_CTR: float32(cs * sigmoid(x)) <= cs."""
import copy
import importlib.util
import os

import numpy as np
import pytest
import torch

_spec = importlib.util.spec_from_file_location(
    "tower_coverage", os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tools", "tower_coverage.py"))
tower_coverage = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(tower_coverage)


def _grow(mask):  # pixels a 3x3 zero-padded conv reads to produce `mask`
    H, W = mask.shape
    p = np.pad(mask, 1)
    return np.any([p[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)], axis=0)


def _brute_force(seeds, H, W, d, th, tw):
    need = np.zeros((H, W), bool)
    for y, x in seeds:
        need[y, x] = True  # the decode reads the predictor's output at the seeds only
    tiles_x = -(-W // tw)
    out = [None] * (d + 1)
    for i in reversed(range(d + 1)):
        ys, xs = np.nonzero(need)
        out[i] = np.unique((ys // th) * tiles_x + xs // tw)
        need = _grow(need)  # what list i's conv reads of the layer before it
    return out


@pytest.mark.parametrize("H,W,d,th,tw,n,seed", [
    (56, 100, 4, 16, 8, 30, 0),    # tiles cut by the map edge in both directions
    (13, 21, 4, 16, 8, 5, 1),      # map smaller than a few tiles
    (64, 64, 2, 16, 8, 12, 2),
    (30, 37, 1, 8, 16, 9, 3),      # generic tile shape, one tower conv
    (100, 160, 6, 16, 8, 200, 4),  # many seeds
    (40, 40, 4, 16, 8, 0, 5),      # empty P
])
def test_box2d_tile_rule_matches_receptive_field(H, W, d, th, tw, n, seed):
    rng = np.random.default_rng(seed)
    seeds = np.stack([rng.integers(0, H, n), rng.integers(0, W, n)], 1)
    seeds = np.concatenate([seeds, [[0, 0], [H - 1, W - 1], [0, W - 1], [H - 1, 0], [H // 2, 0], [0, W // 2]]]) if n else seeds
    got = tower_coverage.tile_lists(seeds, H, W, d + 1, th, tw, reach=d)
    want = _brute_force(seeds, H, W, d, th, tw)
    assert len(got) == d + 1
    for i in range(d + 1):
        assert np.array_equal(got[i], want[i]), f"list {i}"


@pytest.mark.parametrize("with_ctr", [True, False])
def test_oracle_candidates_lie_in_the_seed_set(with_ctr):
    """DLA-34 golden case: every pre-NMS candidate pixel of the fp32 oracle's decode passes the class-only threshold."""
    from dd3d_b200.config import get_cfg
    from dd3d_b200.synthetic import make_state_dict
    from oracle.dd3d_oracle import DD3DOracle
    from oracle.gen_golden import CASES, case_inputs

    cfg = copy.deepcopy(get_cfg("dla34", CASES["dla34"][0]))
    cfg.DD3D.FCOS2D.INFERENCE.THRESH_WITH_CTR = with_ctr
    C, thresh = int(cfg.DD3D.NUM_CLASSES), float(cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH)
    inputs = case_inputs("dla34")
    with torch.no_grad():
        _, inter = DD3DOracle(cfg, make_state_dict(cfg), threads=1).forward(inputs, return_intermediates=True)
    total = 0
    for b in range(len(inputs)):
        det = inter["pre_nms"][b]
        for l, m in enumerate(inter["maps"]["logits"]):
            h, w = m.shape[-2:]
            P = {int(y) * w + int(x) for y, x in tower_coverage.class_pass_pixels(m[b], C, thresh)}
            pix = det["pixel"][det["level"] == l].tolist()
            total += len(pix)
            assert set(pix) <= P, f"image {b} level {l}: a candidate outside P"
    assert total > 0


def test_centerness_product_never_exceeds_the_class_score():
    """float32(cs * sigmoid(x)) <= cs for a dense sweep of x (both infinities, the fp32 extremes, the region where sigmoid
    rounds to 1) and random class scores cs in [0, 1], including 0, 1 and subnormals; sigmoid in fp32 as the kernels do."""
    f = np.float32
    x = np.concatenate([np.linspace(-120, 120, 48001, dtype=f), np.linspace(15, 20, 5001, dtype=f),
                        np.array([-np.inf, np.inf, np.finfo(f).max, -np.finfo(f).max, 0, -0.0], dtype=f)])
    with np.errstate(over="ignore"):
        sig = (f(1) / (f(1) + np.exp(-x))).astype(f)
    assert sig.dtype == f and (sig <= 1).all() and (sig >= 0).all()
    rng = np.random.default_rng(0)
    cs = np.concatenate([rng.random(400, dtype=f), np.array([0, 1, 1e-40, np.nextafter(f(1), f(0)), 0.05], dtype=f)])
    prod = cs[:, None] * sig[None, :]
    assert prod.dtype == f
    assert (prod <= cs[:, None]).all()
