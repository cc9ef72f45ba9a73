"""The 256 x 128 pair tile of the halo conv (-m gpu; conv_igemm_kernel.cuh PAIR, policy "pair_tile"): two 16x8 tiles share
every weight tile, the K order of each output element is unchanged, so its outputs must be bit-identical to the 128-pixel
tile's, and equal to torch within one rounding of the storage type."""
import pytest
import torch

import gpu_ops
from dd3d_b200 import lib
from oracle.gen_golden import case_inputs
from test_e2e_gpu import _model
from test_kernels_gpu import _check_bf16, _rand_act, act  # noqa: F401  (act: fixture over bf16 / fp16)

pytestmark = pytest.mark.gpu


# cin, cout, H, W, B, residual.  Every shape keeps the halo variant (its 16x8 tiling costs at most 10 % more tiles than the
# best generic tiling); "tiles" = 16x8 tiles per image, odd counts leave the last pair's second sub-tile outside the image.
PAIR_CASES = [
    (256, 256, 32, 48, 2, False),   # tower conv, exact tiles, 12 tiles, 2 n-blocks
    (128, 128, 48, 40, 1, True),    # VoVNet stage 2 / BasicBlock + residual, 15 tiles (odd)
    (160, 512, 30, 50, 3, False),   # K tail (2.5 k-blocks), ragged map, 4 n-blocks, 14 tiles
    (256, 128, 16, 24, 3, True),    # 3 tiles (odd) per image, several images, residual
    (128, 256, 45, 77, 2, False),   # ragged map, 30 tiles
    (256, 256, 15, 17, 2, True),    # map smaller than a pair: 3 tiles, residual
]


@pytest.mark.parametrize("cin,cout,H,W,B,res", PAIR_CASES)
def test_conv_pair_tile_is_bit_identical(cin, cout, H, W, B, res, act):
    L = lib.load()
    g = torch.Generator().manual_seed(cin + cout + H + W)
    x = _rand_act(B, H, W, cin, seed=cin + W)
    w = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9)**0.5
    scale = 0.5 + torch.rand(cout, generator=g)
    bias = torch.randn(cout, generator=g) * 0.5
    residual = _rand_act(B, H, W, cout, seed=7) if res else None
    outs = []
    try:
        for mode in (1, 0):
            assert L.dd3d_set_conv_policy(b"pair_tile", mode) == 0
            outs.append(gpu_ops.conv2d(x, w, scale, bias, 1, True, residual, False))
    finally:
        L.dd3d_set_conv_policy(b"pair_tile", -1)
    assert torch.equal(outs[0], outs[1]), "pair tile and 128-pixel tile differ"
    ref = gpu_ops.conv2d_ref(x.cpu(), w, scale, bias, 1, True, None if residual is None else residual.cpu(), False)
    _check_bf16(outs[0], ref, f"pair-tile conv {cin}->{cout} {H}x{W}")


@pytest.mark.parametrize("arch", ["dla34", "v2_99"])
def test_engine_pair_tile_is_bit_identical(arch):
    """Whole forwards with the pair tile on every eligible layer (policy 1: the small golden shapes would otherwise keep most
    launches on the 128-pixel tile by the fill rule) against none (policy 0): FPN and head maps bit-identical."""
    L = lib.load()
    inputs = case_inputs(arch)
    snaps = []
    try:
        for mode in (0, 1):
            assert L.dd3d_set_conv_policy(b"pair_tile", mode) == 0
            _, _, model = _model(arch)
            model.set_engine_option("sparse_box3d", 0)
            model(inputs)
            torch.cuda.synchronize()
            n_pair = sum(1 for c in model.get_conv_info() if c is not None and c["pair"])
            assert (n_pair > 0) == (mode == 1), f"pair-tile launches with policy {mode}: {n_pair}"
            snaps.append([model.get_tensor(n).float().cpu().clone()
                          for l in range(5) for n in (f"p{l}", f"cls{l}", f"box{l}", f"b3d{l}")])
            del model
    finally:
        L.dd3d_set_conv_policy(b"pair_tile", -1)
    for a, b in zip(*snaps):
        assert torch.equal(a, b)
