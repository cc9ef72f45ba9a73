"""Exact arithmetic of the grouped 3x3 conv (dd3d_op_conv2d_grouped, the block-diagonal mode of the implicit-GEMM kernel)
on the integer operands of tests/exact_ops.py: every output must equal RN_storage(float64 grouped conv) with no tolerance,
for channels per group 2..32 (groups 32 and 64), 64..2048 channels, stride 1 and 2, ragged, 1-pixel-wide and multi-tile
maps, channel-sliced input and output.  The packing / comparison pair is checked on the CPU first: a weight shifted into
the neighbouring group must fail the comparison."""
import ctypes as C

import pytest
import torch

import exact_ops as X
import gpu_ops
from dd3d_b200 import lib

MODES = ["int", "round"]


def pack_grouped(w, dtype=torch.float32):
    """[C][cpg][3][3] -> [C][9][64]: row co holds its group's cpg input channels at (co // cpg) * cpg % 64, zeros elsewhere
    (the layout dd3d_op_conv2d_grouped takes, csrc/engine.cu grouped_conv_layer)."""
    C_, cpg = w.shape[:2]
    out = torch.zeros(C_, 9, 64, dtype=torch.float32)
    for co in range(C_):
        c0 = (co // cpg) * cpg % 64
        out[co, :, c0:c0 + cpg] = w[co].reshape(cpg, 9).t()
    return out.to(dtype)


def block_diag_ref64(x_nchw, packed, stride):
    """What the block-diagonal kernel computes from a packed weight: output channel co of n-block j is the dense 3x3 conv of
    input channels [64 j, 64 j + 64) with row co of `packed` (float64, NCHW)."""
    C_ = packed.shape[0]
    dense = torch.zeros(C_, C_, 3, 3, dtype=torch.float64)
    for co in range(C_):
        j = co // 64
        dense[co, 64 * j:64 * j + 64] = packed[co].double().t().reshape(64, 3, 3)
    return X._conv64(x_nchw, dense, stride)


def grouped_ref64(x_nhwc, w, scale, bias, stride, relu, groups):
    """float64 NHWC relu(grouped_conv(x, w) * scale + bias) on the same 16-bit operands."""
    acc = X._conv64(x_nhwc.permute(0, 3, 1, 2), w, stride, groups)
    dev = acc.device
    y = acc * scale.double().to(dev).view(1, -1, 1, 1) + bias.double().to(dev).view(1, -1, 1, 1)
    if relu:
        y = y.clamp(min=0)
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("shift", [0, 1])
def test_packing_negative_control(shift):
    """CPU: the block-diagonal product of the packed weights equals the grouped conv exactly; the same weights with one
    group's input channels moved into the neighbouring group's columns fail assert_exact."""
    g = X._gen(7)
    C_, groups, cpg = 128, 32, 4
    x = X.operand((2, 9, 11, C_), "round", 9 * cpg, g)
    w = X.operand((C_, cpg, 3, 3), "round", 9 * cpg, g)
    w[5] = torch.where(w[5] == 0, torch.ones_like(w[5]), w[5])  # row 5 has no zero weight: a shift always shows
    ones, zeros = torch.ones(C_), torch.zeros(C_)
    ref = grouped_ref64(x, w, ones, zeros, 1, False, groups)
    packed = pack_grouped(w)
    if shift:
        packed[5] = torch.roll(packed[5], cpg, dims=1)  # row 5 (group 1) reads group 2's input channels
    got = block_diag_ref64(x.permute(0, 3, 1, 2), packed, 1).permute(0, 2, 3, 1).float()
    if shift:
        with pytest.raises(AssertionError, match="elements differ"):
            X.assert_exact(got, ref, "shifted group")
    else:
        X.assert_exact(got, ref, "block-diagonal packing")


def _grouped(x, c0, C_, packed, groups, stride, scale, bias, relu, out_pitch, o0):
    """dd3d_op_conv2d_grouped on channels [c0, c0 + C_) of x; writes channels [o0, o0 + C_) of a NaN-poisoned buffer."""
    B, H, W, pitch = x.shape
    Ho, Wo = H // stride, W // stride
    out = torch.full((B, Ho, Wo, out_pitch), float("nan"), dtype=x.dtype, device="cuda")
    st = lib.load().dd3d_op_conv2d_grouped(
        C.c_void_p(x.data_ptr() + 2 * c0), B, H, W, C_, pitch, gpu_ops._p(packed), groups, stride, gpu_ops._p(scale),
        gpu_ops._p(bias), int(relu), C.c_void_p(out.data_ptr() + 2 * o0), out_pitch, gpu_ops._stream())
    assert st == 0, f"dd3d_op_conv2d_grouped failed: {st}"
    torch.cuda.synchronize()
    return out


# C, groups, stride, B, H, W, relu, channel slices.  Channels per group 2, 4, 8, 16, 32 with 32 groups and 4 .. 32 with 64
# groups (DLA-X-102-64); ragged maps, 1-pixel-wide maps, maps smaller than a tile and maps with many tiles per CTA.
CASES = [
    (64, 32, 1, 2, 24, 40, True, False),
    (64, 32, 2, 1, 96, 160, True, True),
    (128, 32, 2, 1, 30, 44, False, True),
    (128, 32, 1, 2, 48, 80, True, False),
    (256, 32, 1, 1, 17, 1, True, True),
    (256, 32, 2, 2, 2, 34, False, False),
    (512, 32, 2, 2, 12, 20, True, False),
    (512, 32, 1, 1, 1, 29, False, True),
    (1024, 32, 1, 1, 9, 13, False, True),
    (1024, 32, 2, 1, 20, 2, True, False),
    (256, 64, 2, 1, 14, 22, True, True),
    (512, 64, 1, 2, 16, 8, True, False),
    (1024, 64, 1, 1, 7, 33, False, True),
    (2048, 64, 1, 1, 6, 10, True, True),
    (2048, 64, 2, 1, 12, 8, False, False),
]

# policies of a stride-1 case: the default and the weight-stationary variant off (it applies to a single n-block, C = 64)
POLICIES = [{}, {"wstat": 0}]


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(int(v)) for v in c))
def test_grouped_conv_exact(case, mode, act):
    C_, groups, stride, B, H, W, relu, slices = case
    cpg = C_ // groups
    K = 9 * cpg  # the real dot-product length of one output
    g = X._gen(C_ * 3 + groups + H)
    c0, pitch = (32, C_ + 96) if slices else (0, C_)  # input: a slice of a wider buffer
    o0, out_pitch = (64, C_ + 192) if slices else (0, C_)  # output: a slice of a root concat
    x = X.operand((B, H, W, pitch), mode, K, g).to(gpu_ops.ACT).cuda()
    w = X.operand((C_, cpg, 3, 3), mode, K, g)
    scale, bias = X.epilogue(C_, mode, K, g)
    ref = grouped_ref64(x[..., c0:c0 + C_], w, scale, bias, stride, relu, groups)
    packed = pack_grouped(w, gpu_ops.ACT).cuda()
    what = f"grouped {C_}/{groups} s{stride} {B}x{H}x{W} relu={relu} slices={slices} {mode} {act}"
    for pol in (POLICIES if stride == 1 else ({}, )):
        try:
            for n, v in pol.items():
                assert lib.load().dd3d_set_conv_policy(n.encode(), v) == 0
            out = _grouped(x, c0, C_, packed, groups, stride, scale.cuda(), bias.cuda(), relu, out_pitch, o0)
        finally:
            for n in pol:
                lib.load().dd3d_set_conv_policy(n.encode(), -1)
        X.assert_exact(out[..., o0:o0 + C_], ref, f"{what} {pol}")
        if slices:  # channels outside the written slice keep the NaN poison
            assert torch.isnan(out[..., :o0].float()).all() and torch.isnan(out[..., o0 + C_:].float()).all(), what


@pytest.mark.gpu
def test_grouped_conv_refuses_bad_shapes():
    """C not a multiple of 64, channels per group not dividing 64, odd maps at stride 2: DD3D_ERR_INVALID, no launch."""
    L = lib.load()
    x = torch.zeros(1, 10, 10, 192, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(192, 9, 64, dtype=torch.bfloat16, device="cuda")
    sb = torch.ones(192, device="cuda")
    out = torch.zeros(1, 10, 10, 192, dtype=torch.bfloat16, device="cuda")
    for C_, groups, H, W, stride in ((96, 32, 10, 10, 1), (192, 8, 10, 10, 1), (192, 32, 9, 10, 2), (192, 32, 10, 10, 3)):
        st = L.dd3d_op_conv2d_grouped(gpu_ops._p(x), 1, H, W, C_, 192, gpu_ops._p(w), groups, stride, gpu_ops._p(sb),
                                      gpu_ops._p(sb), 0, gpu_ops._p(out), 192, gpu_ops._stream())
        assert st == -1, (C_, groups, H, W, stride, st)
