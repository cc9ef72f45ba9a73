"""Exact-operand checking for the GEMM-shaped kernels (tests/test_exact_kernels_gpu.py, tests/test_exact_operands.py).

Every conv kernel here sums fp32 products of 16-bit operands.  With integer operands whose sum of |products| stays below
2^20 at every output, that fp32 sum is exact in any summation order (and with 4 bits of slack for the tensor core's
alignment of the products to the largest exponent), and so is the epilogue fma(acc, scale, bias) (+ residual) when the scale
is a power of two and bias / residual are small integers.  A correct kernel then stores exactly RN_storage(ref64) -- one
round-to-nearest-even to bf16 / fp16 of the float64 reference -- or ref64 itself for fp32 outputs, at every element, with
no tolerance.  A single missing, duplicated or misplaced product changes the output.

Two operand modes:
  "int":   inputs and weights in {-1, 0, +1} (about half nonzero), scale in {1/2, 1, 2}, bias / residual small integers:
           the outputs are small multiples of 1/2, mostly exact in the storage type;
  "round": integers in [-m, m] with m <= 15 chosen so that K * m^2 < 2^20, and a power-of-two scale that brings the output
           below 2^14: the exact sum has more significant bits than the storage type, which checks that the epilogue rounds
           once, to nearest even, after fma(acc, scale, bias), the residual add and the ReLU.

Plain Python + torch; nothing here needs a GPU to import."""
import math

import torch
import torch.nn.functional as F

EXACT_BITS = 20  # every output's sum of |products| stays below 2^EXACT_BITS (in units of the integer grid)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def int_range(K, mode):
    """Largest |value| of the operands of a K-term dot product in `mode`."""
    if mode == "int":
        return 1
    return max(1, min(15, math.isqrt((2**EXACT_BITS - 1) // K)))


def operand(shape, mode, K, g):
    """fp32 CPU tensor of integers: ternary ("int", about half nonzero) or uniform in [-m, m] ("round")."""
    if mode == "int":
        mag = (torch.rand(shape, generator=g) < 0.5).float()
        sign = torch.randint(0, 2, shape, generator=g).float() * 2 - 1
        return mag * sign
    m = int_range(K, mode)
    return torch.randint(-m, m + 1, shape, generator=g).float()


def epilogue(cout, mode, K, g):
    """(scale, bias) fp32 [cout]: power-of-two scales, small integer biases."""
    if mode == "int":
        scale = 2.0**torch.randint(-1, 2, (cout, ), generator=g).float()
        bias = torch.randint(-3, 4, (cout, ), generator=g).float()
    else:
        m = int_range(K, mode)
        shift = max(0, math.ceil(math.log2(K * m * m)) - 14)
        scale = 2.0**(-shift - torch.randint(0, 2, (cout, ), generator=g).float())
        bias = torch.randint(-8, 9, (cout, ), generator=g).float()
    return scale, bias


def residual(shape, g):
    return torch.randint(-8, 9, shape, generator=g).float()


def _assert_integer(t, what):
    assert torch.equal(t, torch.round(t)), f"{what}: operands must be integers"


def _conv64(x_nchw, w, stride, groups=1):
    """float64 conv of integer operands + the check that every output's sum of |products| is below 2^EXACT_BITS."""
    x, w = x_nchw.double(), w.double().to(x_nchw.device)
    _assert_integer(x, "conv input")
    _assert_integer(w, "conv weight")
    pad = (w.shape[-1] - 1) // 2
    with torch.backends.cudnn.flags(enabled=False):  # plain float64 GEMM on the GPU: no transform-domain algorithm
        acc = F.conv2d(x, w, None, stride, pad, 1, groups)
        mag = F.conv2d(x.abs(), w.abs(), None, stride, pad, 1, groups)
    assert float(mag.max()) < 2**EXACT_BITS, f"operands exceed the exactness bound: {float(mag.max())}"
    _assert_integer(acc, "float64 reference sum")
    return acc


def conv_ref64(x_nhwc, w, scale, bias, stride=1, relu=False, res=None, res_up2=False, in_slice=None):
    """float64 NHWC reference of dd3d_op_conv2d on the SAME 16-bit operands: relu(conv(x, w) * scale + bias + residual).
    x_nhwc / res: 16-bit NHWC (any device; res = the 2x coarser map when res_up2); w: [cout, cin, k, k] integers."""
    c0, cin = in_slice if in_slice is not None else (0, x_nhwc.shape[-1])
    x = x_nhwc[..., c0:c0 + cin].permute(0, 3, 1, 2)
    acc = _conv64(x, w, stride)
    dev = acc.device
    y = acc * scale.double().to(dev).view(1, -1, 1, 1) + bias.double().to(dev).view(1, -1, 1, 1)
    if res is not None:
        r = res.double().permute(0, 3, 1, 2).to(dev)
        if res_up2:
            r = r.repeat_interleave(2, 2).repeat_interleave(2, 3)
        y = y + r
    if relu:
        y = y.clamp(min=0)
    return y.permute(0, 2, 3, 1).contiguous()


def dwconv_ref64(x_nhwc, w, stride):
    """Depthwise 3x3, padding 1, no bias: x [B, H, W, C] 16-bit, w [C, 1, 3, 3] integers -> float64 NHWC."""
    C_ = x_nhwc.shape[-1]
    return _conv64(x_nhwc.permute(0, 3, 1, 2), w, stride, groups=C_).permute(0, 2, 3, 1).contiguous()


def stem_ref64(x_nhwc3, w, scale, bias, stride):
    """Cin = 3 stem (7x7/1 or 3x3/2, padding (k-1)/2) + affine + ReLU: float64 NHWC."""
    acc = _conv64(x_nhwc3.permute(0, 3, 1, 2), w, stride)
    dev = acc.device
    y = acc * scale.double().to(dev).view(1, -1, 1, 1) + bias.double().to(dev).view(1, -1, 1, 1)
    return y.clamp(min=0).permute(0, 2, 3, 1).contiguous()


def dla_front_ref64(x_nhwc3, layers, dtype):
    """DLA-34 base_layer (7x7/1) -> level0 (3x3/1) -> level1 (3x3/2), each conv * scale + bias, ReLU; the two intermediate
    maps rounded to the storage type `dtype` like the kernel's; returns the float64 level1 output (NHWC)."""
    y = x_nhwc3
    for i, (w, sc, bi) in enumerate(layers):
        y = stem_ref64(y, w, sc, bi, 2 if i == 2 else 1)
        if i < 2:
            y = y.float().to(dtype)
    return y


def b3d_rows_ref64(levels, weights, scales, biases, fin_pix, counts, topk, n_pad):
    """Gathered box3d predictor: rows[b][l][s] = (3x3 conv of level l at pixel fin_pix[b][l][s]) * scale_l + bias_l for
    s < counts[b][l] (zero padding outside the map), float64 [B, 5, topk, n_pad], NaN elsewhere.
    levels[l]: 16-bit [B, H, W, 256]; weights[l]: [n_pad, 256, 3, 3] integers."""
    B = levels[0].shape[0]
    rows = torch.full((B, len(levels), topk, n_pad), float("nan"), dtype=torch.float64)
    for l, x in enumerate(levels):
        dense = _conv64(x.permute(0, 3, 1, 2), weights[l], 1).cpu()  # [B, n_pad, H, W]
        dense = dense * scales[l].double().view(1, -1, 1, 1) + biases[l].double().view(1, -1, 1, 1)
        W = x.shape[2]
        for b in range(B):
            n = min(int(counts[b][l]), topk)
            pix = torch.as_tensor(fin_pix[b][l][:n], dtype=torch.long)
            rows[b, l, :n] = dense[b, :, pix // W, pix % W].t()
    return rows


def storage_round(ref64, dtype):
    """RN_storage(ref64): one round-to-nearest-even of the exact value to `dtype` (float32 for fp32 outputs).  The operands
    keep ref64 exactly representable in fp32, so the float64 -> fp32 step is exact and only the last step rounds."""
    r32 = ref64.float()
    assert torch.equal(r32.double(), ref64.to(r32.device)), "reference not exactly representable in fp32"
    return r32 if dtype == torch.float32 else r32.to(dtype)


def assert_exact(out, ref64, what):
    """out (16-bit or fp32, [..., C]) must equal RN_storage(ref64) at every element, compared as values (-0 == +0).
    On failure names the mismatch count and the first mismatching index (b, y, x, c), its value and the reference."""
    want = storage_round(ref64.to(out.device), out.dtype)
    bad = ~(out.float() == want.float())
    if bool(bad.any()):
        n = int(bad.sum())
        idx = tuple(int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements differ; first at {idx} (b, y, x, c): "
                             f"got {float(out[idx])!r}, want {float(want[idx])!r} (exact {float(ref64[idx])!r})")
