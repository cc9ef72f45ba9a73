"""CPU checks of the exact-operand scheme of tests/exact_ops.py: the generated operands keep every fp32 sum exact in any
order, and assert_exact catches the small arithmetic defects the GPU tests (tests/test_exact_kernels_gpu.py) are meant to
find -- a negative control that needs no kernel."""
import numpy as np
import pytest
import torch

import exact_ops as X

DTYPES = [torch.bfloat16, torch.float16]
MANTISSA = {torch.bfloat16: 7, torch.float16: 10}

# K = cin * k * k of every conv case of the GPU matrix and of the real layers (cin up to 2144 for 1x1, 1056 for 3x3)
_KS = sorted({c * k * k for c in (3, 16, 32, 48, 64, 80, 128, 160, 256, 512, 768, 1056, 1280, 2144) for k in (1, 3)} |
             {9, 147, 2304, 9 * 2144})


@pytest.mark.parametrize("mode", ["int", "round"])
def test_operands_meet_exactness_bound(mode):
    """Worst case over every K: the sum of |products| of one output, times the largest scale, plus the largest bias and
    residual, is below 2^20 -- an integer / dyadic value that fp32 (24 bits) holds exactly with 4 bits to spare; and the
    epilogue keeps fp16 outputs finite."""
    for K in _KS:
        m = X.int_range(K, mode)
        assert K * m * m < 2**X.EXACT_BITS, (K, m)
        g = X._gen(K)
        scale, bias = X.epilogue(64, mode, K, g)
        assert torch.equal(torch.log2(scale), torch.round(torch.log2(scale))), "scales must be powers of two"
        worst = K * m * m * float(scale.max()) + float(bias.abs().max()) + 8
        assert worst < (2**22 if mode == "int" else 2**15), (K, worst)
        if mode == "round":
            assert m >= 2, "round mode needs operands beyond the ternary grid"


def _case(mode, cin, cout, k, stride, H, W, seed, res=0):
    g = X._gen(seed)
    K = cin * k * k
    x = X.operand((2, H, W, cin), mode, K, g)
    w = X.operand((cout, cin, k, k), mode, K, g)
    scale, bias = X.epilogue(cout, mode, K, g)
    Ho, Wo = H // stride, W // stride
    r = None if res == 0 else X.residual((2, Ho, Wo, cout) if res == 1 else (2, Ho // 2, Wo // 2, cout), g)
    return x, w, scale, bias, r


# (cin, cout, k, stride, H, W, res): samples of every conv form of the GPU matrix
_CASES = [(64, 32, 3, 1, 9, 11, 0), (160, 16, 3, 1, 6, 7, 1), (48, 32, 3, 2, 10, 12, 0), (1056, 16, 1, 1, 4, 6, 0),
          (2144, 16, 1, 1, 4, 6, 2), (256, 16, 3, 1, 5, 5, 0)]


@pytest.mark.parametrize("mode", ["int", "round"])
@pytest.mark.parametrize("case", _CASES, ids=lambda c: "x".join(map(str, c)))
def test_fp32_sum_in_any_order_equals_float64(mode, case):
    """For sampled outputs: the fp32 sum of the products in several random orders, then the fp32 epilogue, equals the float64
    reference bit for bit -- the property that makes every kernel's tiling and K order irrelevant."""
    cin, cout, k, stride, H, W, res = case
    x, w, scale, bias, r = _case(mode, cin, cout, k, stride, H, W, seed=cin + H, res=res)
    ref = X.conv_ref64(x, w, scale, bias, stride, relu=False, res=r, res_up2=res == 2)
    pad = (k - 1) // 2
    xp = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (pad, pad, pad, pad)).double()
    rng = np.random.default_rng(cin)
    Ho, Wo = H // stride, W // stride
    for _ in range(12):
        b, oy, ox, co = int(rng.integers(2)), int(rng.integers(Ho)), int(rng.integers(Wo)), int(rng.integers(cout))
        patch = xp[b, :, oy * stride:oy * stride + k, ox * stride:ox * stride + k]
        prods = (patch * w[co].double()).flatten().numpy().astype(np.float32)
        exact = float(prods.astype(np.float64).sum())
        for _ in range(4):
            acc = np.cumsum(rng.permutation(prods), dtype=np.float32)[-1]
            assert float(acc) == exact
            y = np.float32(acc) * np.float32(scale[co]) + np.float32(bias[co])
            if r is not None:
                y = y + np.float32(r[b, oy >> (res == 2), ox >> (res == 2), co])
            assert float(y) == float(ref[b, oy, ox, co])


def _rtz(v64, dtype):
    """Round toward zero to the 16-bit type (the defect the checker must catch)."""
    p = MANTISSA[dtype]
    a = v64.abs()
    e = torch.floor(torch.log2(a.clamp(min=2.0**-30)))
    ulp = 2.0**(e - p)
    return (torch.sign(v64) * torch.floor(a / ulp) * ulp).float().to(dtype)


def _fails(out, ref):
    with pytest.raises(AssertionError, match=r"first at \("):
        X.assert_exact(out, ref, "corrupted")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", ["int", "round"])
def test_checker_catches_defects(mode, dtype):
    """Negative control: outputs computed with one of four small defects fail assert_exact against the true reference,
    while the correct output passes."""
    cin, cout, H, W = 64, 32, 9, 10
    x, w, scale, bias, _ = _case(mode, cin, cout, 3, 1, H, W, seed=5)
    x = x.to(dtype)
    r = X.residual((2, H, W, cout), X._gen(6)).to(dtype)
    ref = X.conv_ref64(x, w, scale, bias, 1, relu=True, res=r)
    X.assert_exact(X.storage_round(ref, dtype), ref, "correct")
    neg0 = X.storage_round(ref, dtype).clone()
    neg0[ref == 0] = -0.0
    X.assert_exact(neg0, ref, "signed zero")  # compared as values: -0 == +0

    # (1) one product dropped at one pixel: the first output with |ref| < 64 whose (0, 0) tap of channel 0 is nonzero
    xd = x.double()
    pre = X.conv_ref64(x, w, scale, bias, 1, relu=False, res=r)
    hit = None
    for (b, oy, ox, co) in (pre.abs() < 64).nonzero().tolist():
        if oy > 0 and ox > 0 and xd[b, oy - 1, ox - 1, 0] * w[co, 0, 0, 0] != 0:
            hit = (b, oy, ox, co)
            break
    assert hit is not None
    b, oy, ox, co = hit
    drop = pre.clone()
    drop[b, oy, ox, co] -= float(xd[b, oy - 1, ox - 1, 0] * w[co, 0, 0, 0]) * float(scale[co])
    _fails(X.storage_round(drop, dtype), pre)

    # (2) bias added after the 16-bit rounding
    acc = X.conv_ref64(x, w, scale, torch.zeros(cout), 1, relu=False)
    late = (X.storage_round(acc, dtype).double() + bias.double() + r.double()).clamp(min=0)
    late = late.float().to(dtype)
    if mode == "round":
        _fails(late, ref)
    else:  # ternary sums are exact in the storage type: rounding early is harmless there, which is why "round" exists
        X.assert_exact(late, ref, "int mode, late bias")

    # (3) round toward zero instead of to nearest even
    if mode == "round":
        _fails(_rtz(ref, dtype), ref)

    # (4) residual read one row off
    r_off = torch.roll(r, 1, dims=1)
    _fails(X.storage_round(X.conv_ref64(x, w, scale, bias, 1, relu=True, res=r_off), dtype), ref)


def test_checker_catches_fp32_defects():
    """fp32 outputs (predictors, sparse box3d rows) must equal the float64 value itself: one dropped product fails."""
    x, w, scale, bias, _ = _case("round", 256, 16, 3, 1, 5, 6, seed=9)
    ref = X.conv_ref64(x, w, scale, bias)
    X.assert_exact(ref.float(), ref, "correct fp32")
    bad = ref.clone()
    bad[1, 2, 3, 4] -= float(scale[4])
    _fails(bad.float(), ref)


def test_reference_forms():
    """The depthwise, stem, DLA chain and gathered-predictor references agree with the plain conv reference they restate."""
    g = X._gen(3)
    x = X.operand((1, 7, 9, 16), "round", 9, g)
    wd = X.operand((16, 1, 3, 3), "round", 9, g)
    dense = torch.zeros(16, 16, 3, 3)
    for c in range(16):
        dense[c, c] = wd[c, 0]
    for s in (1, 2):
        a = X.dwconv_ref64(x, wd, s)
        b = X.conv_ref64(x, dense, torch.ones(16), torch.zeros(16), s) if s == 1 else None
        if b is not None:
            assert torch.equal(a, b)
        assert a.shape[1:3] == ((7 - 1) // s + 1, (9 - 1) // s + 1)
    lv = [X.operand((2, h, w_, 256), "int", 2304, g) for h, w_ in ((5, 7), (3, 4), (1, 1), (1, 6), (2, 1))]
    ws = [X.operand((16, 256, 3, 3), "int", 2304, g) for _ in range(5)]
    sc = [torch.ones(16) * 2 for _ in range(5)]
    bi = [torch.arange(16).float() for _ in range(5)]
    pix = [[[0, 34, 6, 34] if l == 0 else [0] for l in range(5)] for _ in range(2)]
    cnt = [[4 if l == 0 else 1 for l in range(5)], [0, 1, 1, 1, 1]]
    rows = X.b3d_rows_ref64(lv, ws, sc, bi, pix, cnt, 8, 16)
    full = X.conv_ref64(lv[0], ws[0], sc[0], bi[0])
    assert torch.equal(rows[0, 0, 1], full[0, 4, 6]) and torch.equal(rows[0, 0, 3], full[0, 4, 6])
    assert torch.isnan(rows[0, 0, 4:]).all() and torch.isnan(rows[1, 0]).all()
