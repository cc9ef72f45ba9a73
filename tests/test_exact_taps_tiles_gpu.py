"""Exact arithmetic of the work-list taps-in-N conv (-m gpu, both storage types), the sparse box2d tower's predictor, through
dd3d_op_conv2d_taps_tiles, under the contract of tests/test_exact_kernels_gpu.py: on the integer operands of tests/exact_ops.py
every listed output equals RN_storage(float64 reference) -- the float64 value itself for fp32 outputs -- with no tolerance,
and equals the dense taps-in-N conv bit for bit."""
import ctypes as C

import pytest
import torch

import exact_ops as X
import gpu_ops
from dd3d_b200 import lib

pytestmark = pytest.mark.gpu

SENTINEL = 7.0


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


def _launch(x, d_w, d_sc, d_bi, B, H, W, cin, cout, out, o0, out_pitch, out_f32, tiles, count):
    eb = out.element_size()
    return lib.load().dd3d_op_conv2d_taps_tiles(gpu_ops._p(x), B, H, W, cin, cin, gpu_ops._p(d_w), cout, gpu_ops._p(d_sc),
                                                gpu_ops._p(d_bi), 0, C.c_void_p(out.data_ptr() + eb * o0), out_pitch,
                                                int(out_f32), gpu_ops._p(tiles), gpu_ops._p(count), gpu_ops._stream())


@pytest.mark.parametrize("out_f32", [True, False])
@pytest.mark.parametrize("cin,cout", [(256, 5), (160, 15)])
@pytest.mark.parametrize("mode", ["int", "round"])
def test_conv2d_taps_tiles_exact(mode, cin, cout, out_f32, act):
    """The listed 16x8 tiles -- scattered, the ragged bottom-right tile, the out-of-image padding tile -- equal the float64
    reference (and, with fp32 outputs, the dense taps-in-N conv bit for bit; dd3d_op_conv2d has no 16-bit output of fewer
    than 16 channels); the padding channels up to 16 hold zeros; every other pixel and the neighbouring channels keep their
    sentinel; an empty list writes nothing.  (256, 5) is the box2d predictor's shape; (160, 15) has a K tail."""
    B, H, W = 2, 45, 70
    tiles_x, tiles_y = (W + 7) // 8, (H + 15) // 16
    T = tiles_x * tiles_y  # 27: the padding tile T is listed as in the engine's odd-length lists
    g = X._gen(46 + cin + cout)
    x = (X.operand((B, H, W, cin), mode, 9 * cin, g)).to(gpu_ops.ACT).cuda()
    w = X.operand((cout, cin, 3, 3), mode, 9 * cin, g)
    scale, bias = X.epilogue(cout, mode, 9 * cin, g)
    ref = X.conv_ref64(x, w, scale, bias, 1)
    d_w = gpu_ops.pack_conv_weight(w).cuda()
    d_sc, d_bi = gpu_ops.pad16(scale, 1.0).cuda(), gpu_ops.pad16(bias, 0.0).cuda()
    dense = gpu_ops.conv2d(x, w, scale, bias, 1, False, out_f32=True) if out_f32 else None
    if out_f32:
        X.assert_exact(dense[..., :cout], ref, "dense taps-in-N conv")
    o0, op = (4, 24) if out_f32 else (8, 32)
    dtype = torch.float32 if out_f32 else gpu_ops.ACT
    listed = [(0, 0), (0, 5), (0, T - 1), (0, 13), (1, 3), (1, T), (1, 9), (1, 10)]
    for entries in (listed, []):
        tiles = torch.tensor([(b << 16) | t for b, t in entries] or [0], dtype=torch.int64).to(torch.int32).cuda()
        count = torch.tensor([len(entries)], dtype=torch.int32).cuda()
        out = torch.full((B, H, W, op), SENTINEL, dtype=dtype, device="cuda")
        assert _launch(x, d_w, d_sc, d_bi, B, H, W, cin, cout, out, o0, op, out_f32, tiles, count) == 0
        torch.cuda.synchronize()
        mask = torch.zeros(B, H, W, dtype=torch.bool, device="cuda")
        for b, t in entries:
            if t == T:
                continue
            y0, x0 = (t // tiles_x) * 16, (t % tiles_x) * 8
            sl = (b, slice(y0, y0 + 16), slice(x0, x0 + 8))
            X.assert_exact(out[sl][..., o0:o0 + cout], ref[sl], f"listed tile {t} of image {b}")
            assert (out[sl][..., o0 + cout:o0 + 16].float() == 0).all(), f"tile {t} of image {b}: padding channels"
            if out_f32:
                assert torch.equal(out[sl][..., o0:o0 + 16], dense[sl][..., :16]), f"tile {t} of image {b} differs from the dense conv"
            mask[sl] = True
        assert (out[~mask].float() == SENTINEL).all(), "an unlisted pixel was written"
        assert (out[..., :o0].float() == SENTINEL).all() and (out[..., o0 + 16:].float() == SENTINEL).all()


def test_conv2d_taps_tiles_rejects_bad_arguments():
    L = lib.load()
    x = torch.zeros(1, 16, 8, 64, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(16, 9, 64, dtype=torch.bfloat16, device="cuda")
    v = torch.zeros(16, device="cuda")
    out = torch.zeros(1, 16, 8, 32, device="cuda")
    tiles = torch.zeros(1, dtype=torch.int32, device="cuda")
    count = torch.zeros(1, dtype=torch.int32, device="cuda")
    p = gpu_ops._p
    for cout, pitch, f32 in ((17, 16, 1), (0, 16, 1), (5, 18, 1), (5, 12, 0), (5, 8, 1)):
        st = L.dd3d_op_conv2d_taps_tiles(p(x), 1, 16, 8, 64, 64, p(w), cout, p(v), p(v), 0, p(out), pitch, f32, p(tiles),
                                         p(count), gpu_ops._stream())
        assert st == -1, (cout, pitch, f32, st)
