"""The 8x8 tile lists of the sparse towers (csrc/tower_tiles.cu, mirrored by tools/tower_coverage.py) and the work-list pair
tile that computes them (conv_igemm_kernel<..., PAIR, LIST>).

CPU: the 8x8 lists of both towers and the box2d predictor's 16x8 list, which the kernel derives from the 8x8 distances, equal
a brute-force receptive-field propagation; on the DLA-34 golden case every oracle candidate (box3d tower) and every pixel of P
(box2d tower) is covered, dilated as far as each layer needs.
GPU (-m gpu): dd3d_op_conv2d_tiles8x8 under the exact-arithmetic contract -- listed, ragged and padding tiles, units with 1,
2, 3 and 4 real tiles -- on a 0xFF-poisoned output: listed pixels equal the float64 reference and the dense pair-tile conv bit
for bit, no other byte changes."""
import copy
import ctypes as C
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


def _tiles(need, th, tw):
    ys, xs = np.nonzero(need)
    return np.unique((ys // th) * (-(-need.shape[1] // tw)) + xs // tw)


def _needed(seeds, H, W, n, first_grow):
    """need[i], i < n: the pixels list i must compute, walking back from the last list (the seeds, grown once more for the
    box3d tower, whose sparse predictor reads 3x3 neighbourhoods) one 3x3 conv at a time."""
    need = np.zeros((H, W), bool)
    for y, x in seeds:
        need[y, x] = True
    if first_grow:
        need = _grow(need)
    out = [None] * n
    for i in reversed(range(n)):
        out[i] = need
        need = _grow(need)
    return out


CASES = [
    (56, 100, 4, 30, 0),    # tiles cut by the map edge in both directions
    (13, 21, 4, 5, 1),      # map smaller than a few tiles
    (45, 70, 2, 12, 2),     # odd number of 8x8 tile rows: the last 16x8 predictor tile has one half
    (100, 160, 6, 200, 3),  # many seeds
    (40, 40, 4, 0, 4),      # no seeds
]


def _seeds(H, W, n, seed):
    rng = np.random.default_rng(seed)
    s = np.stack([rng.integers(0, H, n), rng.integers(0, W, n)], 1)
    edges = [[0, 0], [H - 1, W - 1], [0, W - 1], [H - 1, 0], [H // 2, 0], [0, W // 2]]
    return np.concatenate([s, edges]) if n else s


@pytest.mark.parametrize("H,W,depth,n,seed", CASES)
def test_box3d_8x8_lists_match_receptive_field(H, W, depth, n, seed):
    cands = _seeds(H, W, n, seed)
    got = tower_coverage.tile_lists(cands, H, W, depth, 8, 8)
    want = [_tiles(m, 8, 8) for m in _needed(cands, H, W, depth, True)]
    for i in range(depth):
        assert np.array_equal(got[i], want[i]), f"layer {i}"


@pytest.mark.parametrize("H,W,d,n,seed", CASES)
def test_box2d_8x8_lists_and_16x8_predictor_match_receptive_field(H, W, d, n, seed):
    seeds = _seeds(H, W, n, seed)
    need = _needed(seeds, H, W, d + 1, False)
    got = tower_coverage.tile_lists(seeds, H, W, d + 1, 8, 8, reach=d)[:d]
    for i in range(d):
        assert np.array_equal(got[i], _tiles(need[i], 8, 8)), f"tower layer {i}"
    pred = tower_coverage.predictor_tiles(seeds, H, W)
    assert np.array_equal(pred, _tiles(need[d], 16, 8)), "predictor"
    # the same list as the 16x8 distances give directly
    assert np.array_equal(pred, tower_coverage.tile_lists(seeds, H, W, 1, 16, 8, reach=0)[0])


def _covered(lists, H, W, th, tw):
    m = np.zeros((-(-H // th) * th, -(-W // tw) * tw), bool)
    tiles_x = -(-W // tw)
    for t in lists:
        m[(t // tiles_x) * th:(t // tiles_x + 1) * th, (t % tiles_x) * tw:(t % tiles_x + 1) * tw] = True
    return m[:H, :W]


def _dilate(yx, H, W, r):
    m = np.zeros((H, W), bool)
    for y, x in yx:
        m[max(y - r, 0):y + r + 1, max(x - r, 0):x + r + 1] = True
    return m


def test_oracle_seeds_are_covered_at_every_layer():
    """DLA-34 golden case, fp32 oracle: layer i of the box3d tower lists every pixel within depth - i of a pre-NMS candidate,
    layer i of the box2d tower every pixel within d - i of P, and the box2d predictor every pixel of P."""
    from dd3d_b200.config import get_cfg
    from dd3d_b200.synthetic import make_state_dict
    from oracle.dd3d_oracle import DD3DOracle
    from oracle.gen_golden import CASES as GOLDEN, case_inputs

    cfg = copy.deepcopy(get_cfg("dla34", GOLDEN["dla34"][0]))
    C_, thresh = int(cfg.DD3D.NUM_CLASSES), float(cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH)
    d3, d2 = int(cfg.DD3D.FCOS3D.NUM_CONVS), int(cfg.DD3D.FCOS2D.NUM_BOX_CONVS)
    inputs = case_inputs("dla34")
    with torch.no_grad():
        _, inter = DD3DOracle(cfg, make_state_dict(cfg), threads=1).forward(inputs, return_intermediates=True)
    seen = 0
    for b in range(len(inputs)):
        det = inter["pre_nms"][b]
        for l, m in enumerate(inter["maps"]["logits"]):
            h, w = m.shape[-2:]
            pix = det["pixel"][det["level"] == l].numpy()
            cands = np.stack([pix // w, pix % w], 1)
            for i, t in enumerate(tower_coverage.tile_lists(cands, h, w, d3, 8, 8)):
                assert not (_dilate(cands, h, w, d3 - i) & ~_covered(t, h, w, 8, 8)).any(), f"box3d {b} {l} {i}"
            P = tower_coverage.class_pass_pixels(m[b], C_, thresh)
            for i, t in enumerate(tower_coverage.tile_lists(P, h, w, d2 + 1, 8, 8, reach=d2)[:d2]):
                assert not (_dilate(P, h, w, d2 - i) & ~_covered(t, h, w, 8, 8)).any(), f"box2d {b} {l} {i}"
            pred = _covered(tower_coverage.predictor_tiles(P, h, w), h, w, 16, 8)
            assert not (_dilate(P, h, w, 0) & ~pred).any(), f"box2d predictor {b} {l}"
            seen += len(cands) + len(P)
    assert seen > 0


# ------------------------------------------------------------------------------------------------ GPU: work-list conv
@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    import gpu_ops
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["int", "round"])
def test_conv2d_tiles8x8_exact(mode, act):
    """Units of four 8x8 tiles of one image: scattered tiles, the ragged bottom-right tile, and units with 1, 2, 3 and 4 real
    tiles padded with the out-of-image tile T, over two n-blocks and a K tail; an empty list writes nothing."""
    import exact_ops as X
    import gpu_ops
    from dd3d_b200 import lib

    L = lib.load()
    B, H, W, cin, cout = 2, 45, 70, 160, 256
    tiles_x, tiles_y = (W + 7) // 8, (H + 7) // 8
    T = tiles_x * tiles_y  # 54
    g = X._gen(46)
    x = X.operand((B, H, W, cin), mode, 9 * cin, g).to(gpu_ops.ACT).cuda()
    w = X.operand((cout, cin, 3, 3), mode, 9 * cin, g)
    scale, bias = X.epilogue(cout, mode, 9 * cin, g)
    ref = X.conv_ref64(x, w, scale, bias, 1, relu=True)
    d_w = gpu_ops.pack_conv_weight(w).to(gpu_ops.ACT).cuda()
    d_sc, d_bi = gpu_ops.pad16(scale, 1.0).cuda(), gpu_ops.pad16(bias, 0.0).cuda()
    units = [(0, [0, 5, T - 1, 13]), (0, [20, T, T, T]), (1, [3, 9, T, T]), (1, [10, 11, 12, T]), (1, [T - 1, 0, 40, 41])]
    listed = [(b, t) for b, ts in units for t in ts]
    o0, op = 64, cout + 128
    assert L.dd3d_set_conv_policy(b"pair_tile", 1) == 0
    try:
        dense = gpu_ops.conv2d(x, w, scale, bias, 1, True)
    finally:
        L.dd3d_set_conv_policy(b"pair_tile", -1)
    X.assert_exact(dense, ref, "dense pair-tile conv")
    for entries in (listed, []):
        tiles = torch.tensor([(b << 16) | t for b, t in entries] or [0], dtype=torch.int64).to(torch.int32).cuda()
        count = torch.tensor([len(entries)], dtype=torch.int32).cuda()
        out = torch.full((B, H, W, op), -1, dtype=torch.int16, device="cuda").view(gpu_ops.ACT)  # 0xFF bytes
        st = L.dd3d_op_conv2d_tiles8x8(gpu_ops._p(x), B, H, W, cin, cin, gpu_ops._p(d_w), cout, gpu_ops._p(d_sc),
                                       gpu_ops._p(d_bi), 1, C.c_void_p(out.data_ptr() + 2 * o0), op, gpu_ops._p(tiles),
                                       gpu_ops._p(count), gpu_ops._stream())
        assert st == 0
        torch.cuda.synchronize()
        mask = torch.zeros(B, H, W, dtype=torch.bool, device="cuda")
        for b, t in entries:
            if t == T:
                continue
            y0, x0 = (t // tiles_x) * 8, (t % tiles_x) * 8
            sl = (b, slice(y0, y0 + 8), slice(x0, x0 + 8))
            X.assert_exact(out[sl][..., o0:o0 + cout], ref[sl], f"listed tile {t} of image {b}")
            assert torch.equal(out[sl][..., o0:o0 + cout], dense[sl]), f"tile {t} of image {b} differs from the dense conv"
            mask[sl] = True
        raw = out.view(torch.int16)
        assert (raw[~mask] == -1).all(), "an unlisted pixel was written"
        assert (raw[..., :o0] == -1).all() and (raw[..., o0 + cout:] == -1).all()

