"""Kernel-level parity (-m gpu): every CUDA kernel is called through the C ABI and compared with a plain fp32 torch
reference of the same op on the SAME bf16-rounded operands (CPU, so no TF32 / cuDNN heuristics are involved).

Tolerances: conv outputs are bf16 -> |err| <= 2^-8 * |y| + small abs (one bf16 rounding of an fp32-accumulated value);
fp32-out convs 2e-4 relative to the output scale; pooling / preprocess bit-exact; decode / NMS per-field fp32 tolerances
with set-equality of the selected candidates."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_ops
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from oracle.dd3d_oracle import DD3DOracle, batched_nms_restated  # checker only
from util import quat_dist

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    """Runs the test once per 16-bit storage type of the engine (dd3d_model_desc.act_dtype)."""
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


def _rand_act(B, H, W, C, seed, pitch=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, pitch or C, generator=g)
    return x.to(gpu_ops.ACT).cuda()


def _check_bf16(out, ref, what):
    """One rounding of an fp32-accumulated value to the storage type: 2^-8 (bf16) / 2^-11 (fp16) relative, doubled for
    accumulation-order differences next to a rounding boundary, plus a small absolute term."""
    fp16 = out.dtype == torch.float16
    out = out.float().cpu()
    ref = ref.cpu()
    err = (out - ref).abs()
    tol = (2.0**-10 * ref.abs() + 3e-3) if fp16 else (2.0**-7 * ref.abs() + 2e-2)
    bad = (err > tol)
    assert not bad.any(), f"{what}: {int(bad.sum())} / {bad.numel()} mismatches, max err {err.max():.4f}"


# cin, cout, k, stride, H, W, B, relu, residual(0 none / 1 same / 2 up2)
CONV_CASES = [
    (256, 256, 3, 1, 16, 24, 2, True, 0),     # tower conv, exact tiles
    (256, 256, 3, 1, 15, 25, 2, True, 0),     # ragged map (p6 of V2-99): partial tiles, TMA clipping
    (256, 256, 3, 1, 3, 10, 3, True, 0),      # p7 of DLA-34: map smaller than one tile
    (128, 128, 3, 1, 24, 40, 1, True, 1),     # BasicBlock conv2 + residual
    (64, 64, 3, 1, 32, 32, 1, True, 0),
    (160, 160, 3, 1, 20, 28, 1, True, 0),     # ragged channels (K tail zero-filled by TMA), N=160
    (224, 224, 3, 1, 10, 14, 2, True, 0),
    (192, 192, 3, 1, 12, 20, 1, True, 0),
    (16, 16, 3, 1, 32, 64, 1, True, 0),       # DLA level0: C < 64
    (16, 32, 3, 2, 32, 64, 1, True, 0),       # DLA level1: stride 2, C=16
    (32, 64, 3, 2, 32, 48, 2, True, 0),
    (64, 128, 3, 2, 24, 40, 1, True, 0),      # stride-2, parity-split TMA view
    (256, 256, 3, 2, 30, 50, 1, False, 0),    # top_block.p6 (bias, no relu) on an odd-tiled map
    (768, 256, 1, 1, 16, 24, 1, True, 0),     # OSA concat 1x1
    (1056, 512, 1, 1, 12, 20, 1, True, 0),    # 2 N-blocks, ragged K (1056 = 16.5 chunks)
    (2144, 1024, 1, 1, 6, 10, 1, True, 0),    # 4 N-blocks
    (1280, 512, 1, 1, 6, 20, 2, True, 0),     # DLA root
    (512, 256, 1, 1, 12, 20, 1, False, 2),    # FPN lateral + nearest-2x top-down add
    (32, 64, 1, 1, 16, 16, 1, False, 0),      # DLA project
]


@pytest.mark.parametrize("cin,cout,k,stride,H,W,B,relu,res", CONV_CASES)
def test_conv_bf16(cin, cout, k, stride, H, W, B, relu, res, act):
    g = torch.Generator().manual_seed(cin * 131 + cout + k + H)
    x = _rand_act(B, H, W, cin, seed=cin + H)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k)**0.5
    scale = 0.5 + torch.rand(cout, generator=g)
    bias = torch.randn(cout, generator=g) * 0.5
    Ho, Wo = H // stride, W // stride
    residual = None
    if res == 1:
        residual = _rand_act(B, Ho, Wo, cout, seed=5)
    elif res == 2:
        residual = _rand_act(B, Ho // 2, Wo // 2, cout, seed=6)
    out = gpu_ops.conv2d(x, w, scale, bias, stride, relu, residual, res == 2)
    ref = gpu_ops.conv2d_ref(x.cpu(), w, scale, bias, stride, relu, None if residual is None else residual.cpu(), res == 2)
    _check_bf16(out, ref, f"conv {cin}->{cout} k{k} s{stride} {H}x{W}")


def test_conv_concat_slices(act):
    """Input = channel slice of a wider buffer, output written into a slice of another (the free-concat trick)."""
    g = torch.Generator().manual_seed(3)
    x = _rand_act(1, 16, 24, 0, seed=11, pitch=448)
    w = torch.randn(128, 160, 3, 3, generator=g) / (160 * 9)**0.5
    scale, bias = torch.ones(128), torch.zeros(128)
    out = gpu_ops.conv2d(x, w, scale, bias, relu=True, in_slice=(128, 160), out_pitch=320, out_offset=64)
    ref = gpu_ops.conv2d_ref(x.cpu(), w, scale, bias, relu=True, in_slice=(128, 160))
    _check_bf16(out[..., 64:192], ref, "slice conv")
    # neighbours of the slice must be untouched (sentinel 7.0)
    assert (out[..., :64].float() == 7.0).all() and (out[..., 192:].float() == 7.0).all()


@pytest.mark.parametrize("cout", [15, 110, 55])
def test_conv_f32_predictor(cout, act):
    g = torch.Generator().manual_seed(cout)
    x = _rand_act(2, 15, 25, 256, seed=cout)
    w = torch.randn(cout, 256, 3, 3, generator=g) / 48.0
    scale = 0.5 + torch.rand(cout, generator=g)
    bias = torch.randn(cout, generator=g)
    out = gpu_ops.conv2d(x, w, scale, bias, out_f32=True)
    ref = gpu_ops.conv2d_ref(x.cpu(), w, scale, bias)
    err = (out[..., :cout].cpu() - ref).abs().max().item()
    assert err < 2e-4 * max(1.0, ref.abs().max().item()), err
    assert torch.isfinite(out).all()


def test_conv_linearity_large():
    """Size-independent property at a BASELINE-scale map (240x400x256, K=2304): conv(a*x) == a*conv(x) exactly for a
    power-of-two a, and a full-size run equals the small-tile reference on a crop."""
    g = torch.Generator().manual_seed(9)
    x = _rand_act(1, 240, 400, 256, seed=21)
    w = torch.randn(256, 256, 3, 3, generator=g) / 48.0
    scale, bias = torch.ones(256), torch.zeros(256)
    y1 = gpu_ops.conv2d(x, w, scale, bias)
    y2 = gpu_ops.conv2d((x.float() * 2).to(torch.bfloat16), w, scale, bias)
    assert torch.equal((y1.float() * 2), y2.float())
    crop = x[:, 100:120, 200:232].contiguous()
    ref = gpu_ops.conv2d_ref(crop.cpu(), w, scale, bias)
    _check_bf16(y1[:, 101:119, 201:231], ref[:, 1:-1, 1:-1], "crop of the large map")


def test_stem_s2_mma_and_preprocess(act):
    L = lib.load()
    g = torch.Generator().manual_seed(4)
    B, Hs, Ws, Hp, Wp = 2, 50, 70, 64, 128
    img = torch.randint(0, 256, (B, 3, Hs, Ws), generator=g, dtype=torch.uint8)
    sizes = torch.tensor([[50, 70], [41, 66]], dtype=torch.int32)
    mean = torch.tensor([103.53, 116.28, 123.675])
    std = torch.tensor([57.375, 57.12, 58.395])
    out4 = torch.empty(B, Hp, Wp, 4, dtype=gpu_ops.ACT, device="cuda")
    d_img, d_sizes = img.cuda(), sizes.cuda()  # keep the device tensors alive across the async launch
    st = L.dd3d_op_preprocess(gpu_ops._p(d_img), lib.IMG_U8, gpu_ops._p(d_sizes), gpu_ops._p(out4), B, Hs, Ws,
                              Hp, Wp, (C.c_float * 3)(*mean.tolist()), (C.c_float * 3)(*std.tolist()), gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    ref = torch.zeros(B, 3, Hp, Wp)
    for b in range(B):
        h, w = sizes[b].tolist()
        ref[b, :, :h, :w] = (img[b, :, :h, :w].float() - mean.view(3, 1, 1)) / std.view(3, 1, 1)
    ref = ref.to(gpu_ops.ACT)
    assert torch.equal(out4[..., :3].cpu(), ref.permute(0, 2, 3, 1))
    assert (out4[..., 3].float() == 0).all()
    # VoVNet stem_1 (3x3 / stride 2, 3 -> 64) on the register-fragment kernel (csrc/stem_mma.cu), written into a channel slice
    wq = (torch.randn(64, 3, 3, 3, generator=g) / 27**0.5).to(gpu_ops.ACT).float()
    scale = 0.5 + torch.rand(64, generator=g)
    bias = torch.randn(64, generator=g) * 0.2
    wm = torch.zeros(64, 3, 4, 4)
    wm[:, :, :3, :3] = wq.permute(0, 2, 3, 1)
    wm = wm.to(gpu_ops.ACT).cuda()
    sb = torch.cat([scale, bias]).cuda()
    out = torch.full((B, Hp // 2, Wp // 2, 96), 7.0, dtype=gpu_ops.ACT, device="cuda")
    st = L.dd3d_op_stem_s2_mma(gpu_ops._p(out4), gpu_ops._p(wm), gpu_ops._p(sb), gpu_ops._p(out), 96, B, Hp, Wp,
                               gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    y = F.conv2d(ref.float(), wq, None, 2, 1)
    y = F.relu(y * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)).permute(0, 2, 3, 1)
    _check_bf16(out[..., :64], y, "stem_1 (mma.sync)")
    assert (out[..., 64:].float() == 7.0).all()


def test_stem_s2_mma_ragged_and_multi_tile(act):
    """csrc/stem_mma.cu on shapes with partial tiles in both directions, odd sizes (ceil(H/2) outputs) and more tiles than
    CTAs (persistent loop, both input buffers), against fp32 torch on the same 16-bit operands."""
    L = lib.load()
    g = torch.Generator().manual_seed(21)
    for B, H, W in ((1, 38, 90), (2, 33, 75), (3, 384, 640)):
        x4 = torch.zeros(B, H, W, 4)
        x4[..., :3] = torch.randn(B, H, W, 3, generator=g)
        x4 = x4.to(gpu_ops.ACT)
        w = (torch.randn(64, 3, 3, 3, generator=g) / 27**0.5).to(gpu_ops.ACT).float()
        scale, bias = 0.5 + torch.rand(64, generator=g), torch.randn(64, generator=g) * 0.2
        wm = torch.zeros(64, 3, 4, 4)
        wm[:, :, :3, :3] = w.permute(0, 2, 3, 1)
        d_in, d_w, d_sb = x4.cuda(), wm.to(gpu_ops.ACT).cuda(), torch.cat([scale, bias]).cuda()
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        pitch = 72 if B == 1 else 64  # 72: not a multiple of 16 channels -> the 2 x 128-bit store path instead of 256-bit stores
        out = torch.full((B, Ho, Wo, pitch), 7.0, dtype=gpu_ops.ACT, device="cuda")
        assert L.dd3d_op_stem_s2_mma(gpu_ops._p(d_in), gpu_ops._p(d_w), gpu_ops._p(d_sb), gpu_ops._p(out), pitch, B, H, W,
                                     gpu_ops._stream()) == 0
        torch.cuda.synchronize()
        y = F.conv2d(x4[..., :3].float().permute(0, 3, 1, 2), w, None, 2, 1)
        y = F.relu(y * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)).permute(0, 2, 3, 1)
        assert y.shape[1:3] == (Ho, Wo)
        _check_bf16(out[..., :64], y, f"stem_1 mma {B}x{H}x{W}")
        assert (out[..., 64:].float() == 7.0).all()


@pytest.mark.parametrize("B,H,W,out_pitch,pool_pitch", [(2, 64, 128, 32, 32), (1, 44, 76, 48, 40), (3, 128, 256, 32, 0)])
def test_dla_front_fused_vs_fp32_chain(B, H, W, out_pitch, pool_pitch, act):
    """csrc/dla_front.cu (base_layer -> level0 -> level1 -> 2x2 max-pool in one kernel, dla.py:271-283,346-350,235) against
    fp32 torch on the same 16-bit operands with every intermediate rounded to the storage type.  Shapes: exact tiles;
    partial tiles in both directions with channel-sliced outputs; several tiles per CTA (persistent loop, both input
    buffers)."""
    L = lib.load()
    g = torch.Generator().manual_seed(11)
    x4 = torch.zeros(B, H, W, 4)
    x4[..., :3] = torch.randn(B, H, W, 3, generator=g)
    x4[:, H - 5:, :, :] = 0  # padded rows / columns of a ragged batch are exactly zero
    x4[:, :, W - 7:, :] = 0
    x4 = x4.to(gpu_ops.ACT)
    layers = []
    for cout, cin, k in ((16, 3, 7), (16, 16, 3), (32, 16, 3)):
        w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k * k)**0.5).to(gpu_ops.ACT).float()
        layers.append((w, 0.5 + torch.rand(cout, generator=g), torch.randn(cout, generator=g) * 0.2))
    # ---- fp32 reference chain, intermediates rounded like the engine's 16-bit storage
    y = x4[..., :3].float().permute(0, 3, 1, 2)
    for i, (w, sc, bi) in enumerate(layers):
        y = F.conv2d(y, w, None, 2 if i == 2 else 1, (w.shape[-1] - 1) // 2)
        y = F.relu(y * sc.view(1, -1, 1, 1) + bi.view(1, -1, 1, 1))
        if i < 2:
            y = y.to(gpu_ops.ACT).float()
    ref = y.permute(0, 2, 3, 1)
    # ---- packed weights (include/dd3d_b200.h dd3d_op_dla_front)
    w0 = torch.zeros(16, 7, 8, 4)
    w0[:, :, :7, :3] = layers[0][0].permute(0, 2, 3, 1)
    w1 = layers[1][0].permute(0, 2, 3, 1).reshape(16, 9, 16)
    w2 = layers[2][0].permute(0, 2, 3, 1).reshape(32, 9, 16)
    dw = [t.contiguous().to(gpu_ops.ACT).cuda() for t in (w0, w1, w2)]
    dsb = [torch.cat([sc, bi]).cuda() for _, sc, bi in layers]
    d_in = x4.cuda()
    out = torch.full((B, H // 2, W // 2, out_pitch), 7.0, dtype=gpu_ops.ACT, device="cuda")
    pool = torch.full((B, H // 4, W // 4, pool_pitch), 7.0, dtype=gpu_ops.ACT, device="cuda") if pool_pitch else None
    st = L.dd3d_op_dla_front(gpu_ops._p(d_in), gpu_ops._p(dw[0]), gpu_ops._p(dw[1]), gpu_ops._p(dw[2]), gpu_ops._p(dsb[0]),
                             gpu_ops._p(dsb[1]), gpu_ops._p(dsb[2]), gpu_ops._p(out), out_pitch, gpu_ops._p(pool), pool_pitch,
                             B, H, W, gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    _check_bf16(out[..., :32], ref, "fused DLA front vs fp32 chain")
    assert (out[..., 32:].float() == 7.0).all(), "channels beyond the 32 outputs must not be written"
    if pool is not None:
        pref = F.max_pool2d(out[..., :32].float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        assert torch.equal(pool[..., :32].float(), pref), "pooled copy != max-pool of the kernel's own level1 output"
        assert (pool[..., 32:].float() == 7.0).all()


@pytest.mark.parametrize("ksize,H,W", [(2, 24, 40), (3, 24, 40), (3, 15, 25)])
def test_maxpool(ksize, H, W, act):
    L = lib.load()
    x = _rand_act(2, H, W, 0, seed=8, pitch=96)
    Cc = 64
    ref = F.max_pool2d(x[..., 16:16 + Cc].float().permute(0, 3, 1, 2), ksize, 2, ceil_mode=(ksize == 3)).permute(0, 2, 3, 1)
    out = torch.zeros(2, ref.shape[1], ref.shape[2], 128, dtype=gpu_ops.ACT, device="cuda")
    st = L.dd3d_op_maxpool(C.c_void_p(x.data_ptr() + 32), C.c_void_p(out.data_ptr() + 64), 2, H, W, Cc, 96, 128, ksize,
                           gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    assert torch.equal(out[..., 32:32 + Cc].float().cpu(), ref.cpu())  # bit-exact
    assert (out[..., :32] == 0).all() and (out[..., 96:] == 0).all()


@pytest.mark.parametrize("Cc,H,W,ident", [(256, 24, 40, False), (768, 15, 25, True), (1024, 8, 13, True)])
def test_ese(Cc, H, W, ident, act):
    L = lib.load()
    g = torch.Generator().manual_seed(Cc)
    B = 2
    x = _rand_act(B, H, W, Cc, seed=Cc)
    idt = _rand_act(B, H, W, 0, seed=Cc + 1, pitch=Cc + 64) if ident else None
    fw = torch.randn(Cc, Cc, generator=g) / Cc**0.5
    fb = torch.randn(Cc, generator=g)
    out = torch.zeros(B, H, W, Cc, dtype=gpu_ops.ACT, device="cuda")
    scratch = torch.empty(L.dd3d_op_ese_scratch_bytes(B, H * W, Cc) // 4, dtype=torch.float32, device="cuda")
    d_fw, d_fb = fw.cuda(), fb.cuda()
    st = L.dd3d_op_ese(gpu_ops._p(x), Cc, gpu_ops._p(d_fw), gpu_ops._p(d_fb), gpu_ops._p(idt), Cc + 64 if ident else 0,
                       gpu_ops._p(out), Cc, gpu_ops._p(scratch), B, H * W, Cc, gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    xf = x.float().cpu()
    gate = F.relu6(xf.mean(dim=(1, 2)) @ fw.T + fb + 3.0) / 6.0
    ref = xf * gate[:, None, None, :]
    if ident:
        ref = ref + idt[..., :Cc].float().cpu()
    _check_bf16(out, ref, "eSE")


# ------------------------------------------------------------------------------------------------ decode + NMS
def _run_detect(desc, maps, K, sizes, level_hw, strides, topk):
    L = lib.load()
    B = K.shape[0]
    cls = [m.cuda() for m in maps["cls"]]
    box = [m.cuda() for m in maps["box"]]
    b3d = [m.cuda() for m in maps["b3d"]]
    arr = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    scratch = torch.empty(L.dd3d_op_detect_scratch_bytes(B, topk), dtype=torch.uint8, device="cuda")
    pre = torch.zeros(B, 5 * topk, 24, dtype=torch.float32, device="cuda")
    pre_n = torch.zeros(B, 5, dtype=torch.int32, device="cuda")
    out = torch.zeros(B, desc.out_cap, 24, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    flags = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    hw = (C.c_int32 * 10)(*[v for p in level_hw for v in p])
    st = (C.c_int32 * 5)(*strides)
    Kd, sd = K.reshape(B, 9).contiguous().cuda(), sizes.cuda()
    r = L.dd3d_op_detect_flags(C.byref(desc), B, hw, st, arr(cls), arr(box), arr(b3d), cls[0].shape[-1],
                               b3d[0].shape[-1], gpu_ops._p(Kd), gpu_ops._p(sd), gpu_ops._p(scratch), gpu_ops._p(pre),
                               gpu_ops._p(pre_n), gpu_ops._p(out), gpu_ops._p(cnt), gpu_ops._p(flags), gpu_ops._stream())
    assert r == 0
    torch.cuda.synchronize()
    assert int(flags) == 0, f"overflow flags {int(flags)}"
    return pre.cpu(), pre_n.cpu(), out.cpu(), cnt.cpu()


def _oracle_maps(maps, Cn, level_hw, B):
    """Engine-layout head maps -> the per-level NCHW tensors the oracle's decode_level consumes."""
    o = dict(logits=[], centerness=[], box2d_reg=[], quat=[], ctr=[], depth=[], size=[], conf=[])
    for l, (h, w) in enumerate(level_hw):
        cls = maps["cls"][l].reshape(B, h, w, -1).permute(0, 3, 1, 2)
        box = maps["box"][l].reshape(B, h, w, -1).permute(0, 3, 1, 2)
        b3 = maps["b3d"][l].reshape(B, h, w, -1).permute(0, 3, 1, 2)
        o["logits"].append(cls[:, :Cn])
        o["box2d_reg"].append(box[:, 0:4])
        o["centerness"].append(box[:, 4:5])
        o["quat"].append(b3[:, 0:4 * Cn])
        o["ctr"].append(b3[:, 4 * Cn:6 * Cn])
        o["depth"].append(b3[:, 6 * Cn:7 * Cn])
        o["size"].append(b3[:, 7 * Cn:10 * Cn])
        o["conf"].append(b3[:, 10 * Cn:11 * Cn])
    return o


@pytest.mark.parametrize("arch,rate,seed", [("v2_99", -3.0, 0), ("v2_99", -0.5, 1), ("dla34", -2.0, 2), ("dla34", -9.0, 3)])
def test_decode_and_nms_vs_oracle(arch, rate, seed):
    """Random head maps; `rate` = logit bias: -0.5 floods the levels far beyond PRE_NMS_TOPK (exact top-k path),
    -9 yields no candidate at all (empty path)."""
    _decode_case(arch, rate, seed, {})


@pytest.mark.parametrize("arch,rate,seed,dominant", [("dla34", -1.0, 5, 4), ("v2_99", -0.5, 6, 2)])
def test_nms_one_dominant_class_vs_oracle(arch, rate, seed, dominant):
    """The multi-CTA NMS path (class-major sort -> IoU bit matrix on all SMs -> per-class scan, csrc/nms.cu) where one class
    holds nearly all candidates (the DLA-34 bench batch: 616 of 623): class segments of many 64-box blocks, long suppression
    chains across blocks; kept set AND order must equal the oracle's batched_nms."""
    _decode_case(arch, rate, seed, {}, dominant=dominant)


@pytest.mark.parametrize("arch,rate,seed", [("v2_99", -0.5, 1), ("dla34", -2.0, 2)])
def test_decode_and_nms_single_cta_path_vs_oracle(arch, rate, seed):
    """The same decode + NMS cases through the one-CTA-per-image NMS kernel (the path the TTA merge uses; the default
    engine path is the multi-CTA one: sort / IoU bit matrix / per-class scan / finish)."""
    L = lib.load()
    try:
        assert L.dd3d_set_conv_policy(b"nms_class_parallel", 0) == 0
        _decode_case(arch, rate, seed, {})
    finally:
        L.dd3d_set_conv_policy(b"nms_class_parallel", -1)


@pytest.mark.parametrize("flags", [
    dict(FEATURE_LOCATIONS_OFFSET="half"), dict(PREDICT_DISTANCE=True), dict(PREDICT_ALLOCENTRIC_ROT=False),
    dict(SCALE_DEPTH_BY_FOCAL_LENGTHS=False),
    dict(FEATURE_LOCATIONS_OFFSET="half", PREDICT_DISTANCE=True, PREDICT_ALLOCENTRIC_ROT=False)], ids=lambda f: "+".join(f))
def test_decode_flags_vs_oracle(flags):
    """The decode switches of dd3d_model_desc (feature-location offset, PREDICT_DISTANCE, egocentric quaternions, no
    focal-length depth scaling; fcos3d.py:36-47, core.py:38) against the oracle, which test_cpu_oracle pins against the
    reference for the same switches."""
    _decode_case("dla34", -2.0, 11, flags)


def _decode_case(arch, rate, seed, flags, dominant=None):
    ds = "nuscenes" if arch == "v2_99" else "kitti_3d"
    cfg = get_cfg(arch, ds)
    for k, v in flags.items():
        if k == "FEATURE_LOCATIONS_OFFSET":
            cfg.DD3D.FEATURE_LOCATIONS_OFFSET = v
        else:
            cfg.DD3D.FCOS3D[k] = v
    desc = lib.desc_from_cfg(cfg)
    Cn = cfg.DD3D.NUM_CLASSES
    B = 2
    strides = [4, 8, 16, 32, 64] if arch == "v2_99" else [8, 16, 32, 64, 128]
    Himg, Wimg = 256, 448
    level_hw = [((Himg + s - 1) // s, (Wimg + s - 1) // s) for s in strides]
    g = torch.Generator().manual_seed(seed)
    cp, p3 = (Cn + 15) // 16 * 16, (11 * Cn + 15) // 16 * 16
    maps = dict(cls=[], box=[], b3d=[])
    for (h, w), s in zip(level_hw, strides):
        n = B * h * w
        cls = torch.randn(n, cp, generator=g) * 1.5 + rate
        if dominant is not None:  # nearly every candidate in ONE class: thousands of same-class boxes per image
            cls -= 6.0
            cls[:, dominant] += 8.0
        maps["cls"].append(cls)
        box = torch.zeros(n, 16)
        box[:, :4] = torch.rand(n, 4, generator=g) * 4 * s + s
        box[:, 4] = torch.randn(n, generator=g) + 1.0
        maps["box"].append(box)
        b3 = torch.randn(n, p3, generator=g)
        b3[:, 6 * Cn:7 * Cn] = b3[:, 6 * Cn:7 * Cn] * 10 + 20  # depth
        maps["b3d"].append(b3)
    K = torch.tensor([[[700.0, 0.5, 224.0], [0, 690.0, 128.0], [0, 0, 1]]]).repeat(B, 1, 1)
    K[1, 0, 0] = 1266.4
    sizes = torch.tensor([[Himg, Wimg, Himg, Wimg], [Himg - 10, Wimg - 20, 2 * (Himg - 10), 2 * (Wimg - 20)]],
                         dtype=torch.int32)
    topk = cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK
    pre, pre_n, out, cnt = _run_detect(desc, maps, K, sizes, level_hw, strides, topk)

    orc = DD3DOracle(cfg, {})
    omaps = _oracle_maps(maps, Cn, level_hw, B)
    inv_K = torch.linalg.inv(K)
    for b in range(B):
        per_level = [orc.decode_level(omaps, l, b, inv_K[b]) for l in range(5)]
        for l, d in enumerate(per_level):
            n = int(pre_n[b, l])
            assert n == d["box2d"].shape[0], (b, l, n, d["box2d"].shape[0])
            if n == 0:
                continue
            got = pre[b, l * topk:l * topk + n]
            gi = got.view(torch.int32)
            # candidate SET equality on (pixel*C + class); topk(sorted=False) has set semantics
            idx_ref = (d["pixel"] * Cn + d["cls"]).numpy()
            idx_got = gi[:, 20].numpy()
            assert set(idx_got.tolist()) == set(idx_ref.tolist()), (b, l)
            o_ref, o_got = np.argsort(idx_ref), np.argsort(idx_got)
            got = got[o_got]
            np.testing.assert_allclose(got[:, 0:4], d["box2d"][o_ref], rtol=1e-6, atol=1e-4)
            np.testing.assert_allclose(got[:, 4], d["score"][o_ref], rtol=1e-5)
            np.testing.assert_allclose(got[:, 5], d["score3d"][o_ref], rtol=1e-5)
            assert quat_dist(got[:, 8:12], d["quat"][o_ref]).max() < 1e-4
            np.testing.assert_allclose(got[:, 12:14], d["proj_ctr"][o_ref], rtol=1e-5, atol=1e-3)
            np.testing.assert_allclose(got[:, 14], d["depth"][o_ref], rtol=1e-4)
            np.testing.assert_allclose(got[:, 15:18], d["size"][o_ref], rtol=1e-4, atol=1e-6)
        det = {k: torch.cat([d[k] for d in per_level], 0) for k in per_level[0]}
        img = (int(sizes[b, 0]), int(sizes[b, 1]))
        osz = (int(sizes[b, 2]), int(sizes[b, 3]))
        ref = orc.nms_topk_postprocess(dict(det), img, osz)
        n = int(cnt[b])
        assert n == ref["box2d"].shape[0], (b, n, ref["box2d"].shape[0])
        if n:
            got = out[b, :n]
            gi = got.view(torch.int32)
            assert np.array_equal(gi[:, 6].numpy(), ref["cls"].numpy())
            assert np.array_equal(gi[:, 7].numpy(), ref["level"].numpy())
            assert np.array_equal(gi[:, 20].numpy(), (ref["pixel"] * Cn + ref["cls"]).numpy())  # same order
            np.testing.assert_allclose(got[:, 0:4], ref["box2d"], rtol=1e-5, atol=1e-3)
            np.testing.assert_allclose(got[:, 5], ref["score3d"], rtol=1e-5)


@pytest.mark.parametrize("cin,cout,H,W,B,f32", [(256, 14, 30, 50, 2, True), (256, 5, 15, 25, 3, True), (256, 16, 48, 160, 1, True),
                                                  (16, 16, 64, 96, 2, False), (64, 16, 33, 70, 1, False), (160, 11, 9, 9, 2, True)])
def test_conv_taps_in_n_matches_per_tap_kernel(cin, cout, H, W, B, f32, act):
    """The taps-in-N kernel (nine taps as GEMM columns + shifted sum from shared memory) against the per-tap implicit GEMM
    on the same operands: same fp32 products, different summation order -> equal within fp32 rounding of the accumulation
    (relative to the output scale), ragged maps / partial tiles / K tails / zero padding included; and against torch."""
    L = lib.load()
    g = torch.Generator().manual_seed(cin + cout + H)
    x = _rand_act(B, H, W, cin, seed=cin + W)
    w = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9)**0.5
    scale = 0.5 + torch.rand(cout, generator=g)
    bias = torch.randn(cout, generator=g) * 0.5
    outs = []
    try:
        for mode in (1, 0):
            assert L.dd3d_set_conv_policy(b"taps", mode) == 0
            outs.append(gpu_ops.conv2d(x, w, scale, bias, 1, not f32, None, False, out_f32=f32))
    finally:
        L.dd3d_set_conv_policy(b"taps", -1)
    a, b = outs[0].float().cpu(), outs[1].float().cpu()
    ref = gpu_ops.conv2d_ref(x.cpu(), w, scale, bias, 1, not f32)
    if f32:
        tol = 2e-5 * max(1.0, ref.abs().max().item())
        assert (a[..., :cout] - b[..., :cout]).abs().max().item() < tol
        assert (a[..., :cout] - ref).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())
        assert torch.isfinite(a).all()
    else:
        _check_bf16(outs[0], ref, "taps-in-N 16-bit output")
        assert (a != b).float().mean().item() < 2e-3  # isolated 1-ulp storage flips only


@pytest.mark.parametrize("cin,cout,H,W,B,res", [(64, 64, 192, 320, 4, 0), (64, 64, 45, 77, 2, 1), (48, 64, 33, 40, 1, 0), (64, 32, 64, 64, 3, 0)])
def test_conv_weight_stationary_is_bit_identical(cin, cout, H, W, B, res, act):
    """3x3 stride-1 layers whose whole weight tensor fits next to the activation patches (<= 64 -> 64 channels: DLA-34 level2,
    VoVNet stem_2) keep it resident in shared memory and run 5 A patches deep (conv_igemm.cu, ConvParams::wstat) instead of
    re-streaming it per tile: same MMAs in the same order -> bit-identical to the streaming variant, on maps with many tiles
    per CTA (the A ring wraps), ragged maps, a K tail (48 channels) and a residual; and equal to torch within one rounding."""
    L = lib.load()
    g = torch.Generator().manual_seed(cin + cout + H)
    x = _rand_act(B, H, W, cin, seed=cin + W)
    w = torch.randn(cout, cin, 3, 3, generator=g) / (cin * 9)**0.5
    scale = 0.5 + torch.rand(cout, generator=g)
    bias = torch.randn(cout, generator=g) * 0.5
    residual = _rand_act(B, H, W, cout, seed=5) if res else None
    outs = []
    try:
        for mode in (1, 0):
            assert L.dd3d_set_conv_policy(b"wstat", mode) == 0
            outs.append(gpu_ops.conv2d(x, w, scale, bias, 1, True, residual, False))
    finally:
        L.dd3d_set_conv_policy(b"wstat", -1)
    assert torch.equal(outs[0], outs[1]), "weight-stationary and streaming variants differ"
    ref = gpu_ops.conv2d_ref(x.cpu(), w, scale, bias, 1, True, None if residual is None else residual.cpu(), False)
    _check_bf16(outs[0], ref, f"wstat conv {cin}->{cout} {H}x{W}")
