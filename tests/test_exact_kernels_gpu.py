"""Exact arithmetic of every GEMM-shaped kernel (-m gpu, both storage types): on the integer operands of tests/exact_ops.py
the fp32 sums have no rounding error in any order, so each kernel output must equal RN_storage(float64 reference) -- fp32
outputs the float64 value itself -- at every element, with no tolerance.  Covers dd3d_op_conv2d over every compiled
block_n and policy variant and at the real layer shapes of three backbones, the depthwise conv, both stems, the fused DLA
front end, the sparse box3d predictor and the work-list conv of the sparse tower; and checks that the benchmark batch
(V2-99, 32 x 900 x 1600) gives every image the detections it gets alone."""
import ctypes as C

import pytest
import torch

import exact_ops as X
import gpu_ops
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_inputs, make_state_dict

pytestmark = pytest.mark.gpu

MODES = ["int", "round"]


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


def _policy(name, value):
    assert lib.load().dd3d_set_conv_policy(name.encode(), value) == 0


def _dev(t):
    return t.to(gpu_ops.ACT).cuda()


# ------------------------------------------------------------------------------------------------ dd3d_op_conv2d
# cin, cout, k, stride, B, H, W, relu, residual (0 none / 1 same / 2 nearest-2x), fp32 out, channel slices.
# Every block_n 16..256 (the four conv_igemm_n*.cu units) plus 384 (2 x 192), 512 and 1024; K tails (48, 80, 160, 1056,
# 2144); exact tiles, ragged maps, maps smaller than a tile, 1 x W, H x 1, and maps with many tiles per CTA.
CONV_CASES = [
    (16, 16, 3, 1, 2, 32, 64, True, 0, False, False),
    (48, 32, 3, 1, 1, 33, 40, False, 1, False, False),
    (64, 48, 3, 2, 2, 24, 40, True, 0, False, False),
    (80, 64, 3, 1, 3, 45, 77, True, 1, False, False),
    (160, 80, 1, 1, 1, 16, 24, False, 2, False, False),
    (1056, 96, 1, 1, 1, 12, 20, True, 0, False, False),
    (16, 112, 3, 1, 1, 3, 10, False, 0, False, False),
    (64, 128, 3, 1, 2, 40, 64, True, 1, False, True),
    (2144, 144, 1, 1, 1, 6, 10, False, 0, False, False),
    (160, 160, 3, 1, 1, 1, 37, True, 0, False, False),
    (48, 176, 3, 2, 1, 30, 2, False, 0, False, False),
    (80, 192, 3, 1, 1, 29, 1, True, 1, False, False),
    (64, 208, 1, 1, 2, 16, 24, False, 1, False, True),
    (1056, 224, 3, 1, 1, 10, 14, True, 0, False, False),
    (16, 240, 3, 2, 1, 20, 28, False, 2, False, False),
    (256, 256, 3, 1, 2, 15, 25, True, 0, False, False),
    (160, 384, 3, 1, 1, 24, 40, True, 1, False, False),
    (2144, 512, 1, 1, 1, 8, 12, False, 2, False, False),
    (1056, 1024, 1, 1, 1, 6, 10, True, 0, False, True),
    (256, 15, 3, 1, 2, 15, 25, False, 0, True, False),
    (256, 55, 3, 1, 1, 9, 9, False, 0, True, False),
    (256, 110, 3, 1, 1, 30, 50, False, 0, True, False),
    (160, 11, 3, 1, 2, 9, 9, False, 0, True, False),
    (256, 256, 3, 1, 1, 120, 200, True, 0, False, False),
    (64, 64, 3, 1, 2, 192, 320, True, 0, False, False),
]

# dd3d_set_conv_policy settings a 3x3 stride-1 case runs under: the default, the pair tile forced on / off, the weight-
# stationary and taps-in-N variants off.  Each run must match the reference on its own.
POLICIES = [{}, {"pair_tile": 1}, {"pair_tile": 0}, {"wstat": 0}, {"taps": 0}]


def _conv_exact(cin, cout, k, stride, B, H, W, relu, res, f32, slices, mode, seed, policies=({}, )):
    g = X._gen(seed)
    K = cin * k * k
    c0, pitch = (16, cin + 48) if slices else (0, cin)
    x = _dev(X.operand((B, H, W, pitch), mode, K, g))
    w = X.operand((cout, cin, k, k), mode, K, g)
    scale, bias = X.epilogue(cout, mode, K, g)
    Ho, Wo = H // stride, W // stride
    r = None
    if res:
        r = _dev(X.residual((B, Ho, Wo, cout) if res == 1 else (B, Ho // 2, Wo // 2, cout), g))
    ref = X.conv_ref64(x, w, scale, bias, stride, relu, r, res == 2, in_slice=(c0, cin))
    o0, op = (64, cout + 128) if slices else (0, None)
    what = f"conv {cin}->{cout} k{k} s{stride} {B}x{H}x{W} relu={relu} res={res} f32={f32} {mode} {gpu_ops.ACT}"
    for pol in policies:
        try:
            for n, v in pol.items():
                _policy(n, v)
            out = gpu_ops.conv2d(x, w, scale, bias, stride, relu, r, res == 2, out_f32=f32, in_slice=(c0, cin),
                                 out_pitch=op, out_offset=o0)
        finally:
            for n in pol:
                _policy(n, -1)
        if f32:
            X.assert_exact(out[..., :cout], ref, f"{what} {pol}")
        else:
            X.assert_exact(out[..., o0:o0 + cout], ref, f"{what} {pol}")
            if slices:  # neighbouring channels keep the sentinel 7.0
                assert (out[..., :o0].float() == 7.0).all() and (out[..., o0 + cout:].float() == 7.0).all(), what


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "-".join(str(int(v)) for v in c))
def test_conv2d_exact(case, mode, act):
    cin, cout, k, stride = case[:4]
    policies = POLICIES if (k == 3 and stride == 1) else ({}, )
    _conv_exact(*case, mode=mode, seed=cin * 7 + cout + case[5], policies=policies)


def test_conv2d_stride2_odd_map_is_refused(act):
    """Stride 2 takes even maps only (the parity-split view): odd sizes return DD3D_ERR_INVALID before any launch."""
    L = lib.load()
    x = torch.zeros(1, 9, 10, 64, dtype=gpu_ops.ACT, device="cuda")
    w = torch.zeros(64, 9, 64, dtype=gpu_ops.ACT, device="cuda")
    sb = torch.ones(64, device="cuda")
    out = torch.zeros(1, 5, 5, 64, dtype=gpu_ops.ACT, device="cuda")
    for H, W in ((9, 10), (10, 9)):
        st = L.dd3d_op_conv2d(gpu_ops._p(x), 1, H, W, 64, 64, gpu_ops._p(w), 64, 3, 2, gpu_ops._p(sb), gpu_ops._p(sb), 0, None,
                              0, 0, gpu_ops._p(out), 64, 0, gpu_ops._stream())
        assert st == -1, (H, W, st)


# ------------------------------------------------------------------------------------------------ real layer shapes
REAL_MODELS = [("dla34", "kitti_3d", 384, 1280, 721.5), ("v2_99", "nuscenes", 900, 1600, 1266.4),
               ("v2_19_slim_dw", "nuscenes", 900, 1600, 1266.4)]


def _layer_shapes(arch, ds, H, W, focal, act):
    """Distinct (k, stride, cin, cout, Ho, Wo, fp32 out) of every conv of the engine's B = 1 plan, with the output map of
    each segment (op<i>:<s> views); fp32 predictors take the head level sizes."""
    cfg = get_cfg(arch, ds, act_dtype=act)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    model.set_engine_option("sparse_box3d", 0)  # the dense box3d predictor is a conv op of the plan
    model(make_inputs(1, H, W, focal))
    torch.cuda.synchronize()
    levels = [tuple(model.get_tensor(f"cls{l}").shape[1:3]) for l in range(5)]
    shapes = set()
    for i, c in enumerate(model.get_conv_info()):
        if c is None:
            continue
        k = 3 if c["taps"] == 9 else 1
        views = []
        for s in range(5):
            try:
                views.append(model.get_tensor(f"op{i}" if s == 0 else f"op{i}:{s}"))
            except RuntimeError:
                break
        if views:
            for v in views:
                shapes.add((k, c["stride"], c["cin"], v.shape[-1], v.shape[1], v.shape[2], False))
        else:
            for h, w in levels:
                shapes.add((k, c["stride"], c["cin"], c["cout_pad"], h, w, True))
    del model
    torch.cuda.empty_cache()
    return sorted(shapes)


@pytest.mark.parametrize("arch,ds,H,W,focal", REAL_MODELS, ids=[m[0] for m in REAL_MODELS])
def test_real_layer_shapes_exact(arch, ds, H, W, focal, act):
    """Every distinct conv of DLA-34 at 384x1280 and of V2-99 / V2-19-slim-dw at 900x1600 (B = 1), once at its real map
    size through dd3d_op_conv2d in exact-integer mode."""
    shapes = _layer_shapes(arch, ds, H, W, focal, act)
    assert len(shapes) > 10
    for n, (k, stride, cin, cout, Ho, Wo, f32) in enumerate(shapes):
        _conv_exact(cin, cout, k, stride, 1, Ho * stride, Wo * stride, False, 0, f32, False, "int", seed=n)


# ------------------------------------------------------------------------------------------------ depthwise 3x3
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("C_,B,H,W", [(8, 2, 37, 45), (64, 1, 1, 1), (72, 2, 1, 9), (160, 1, 7, 1), (224, 3, 30, 41)])
def test_dwconv3x3_exact(C_, B, H, W, stride, mode, act):
    g = X._gen(C_ + H + stride)
    c0, pitch = 16, C_ + 48
    x = _dev(X.operand((B, H, W, pitch), mode, 9, g))
    w = X.operand((C_, 1, 3, 3), mode, 9, g)
    w9 = _dev(w.reshape(C_, 9).t().contiguous())
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    oc0, out_pitch = 8, C_ + 32
    out = torch.full((B, Ho, Wo, out_pitch), float("nan"), dtype=gpu_ops.ACT, device="cuda")
    st = lib.load().dd3d_op_dwconv3x3(C.c_void_p(x.data_ptr() + 2 * c0), B, H, W, C_, pitch, gpu_ops._p(w9), stride,
                                      C.c_void_p(out.data_ptr() + 2 * oc0), out_pitch, gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    X.assert_exact(out[..., oc0:oc0 + C_], X.dwconv_ref64(x[..., c0:c0 + C_], w, stride), f"dwconv C={C_} {H}x{W} s{stride}")
    assert torch.isnan(out[..., :oc0].float()).all() and torch.isnan(out[..., oc0 + C_:].float()).all()


# ------------------------------------------------------------------------------------------------ stems
def _input4(B, H, W, mode, K, g):
    x4 = torch.zeros(B, H, W, 4)
    x4[..., :3] = X.operand((B, H, W, 3), mode, K, g)
    return _dev(x4)


@pytest.mark.parametrize("mode", MODES)
def test_stem_s2_mma_exact(mode, act):
    """dd3d_op_stem_s2_mma (csrc/stem_mma.cu): odd sizes, partial tiles, a pitch with the 128-bit store path, and more
    tiles than CTAs."""
    L = lib.load()
    for B, H, W, pitch in ((1, 38, 90, 72), (2, 33, 75, 64), (3, 384, 640, 64)):
        g = X._gen(H + W)
        x4 = _input4(B, H, W, mode, 27, g)
        w = X.operand((64, 3, 3, 3), mode, 27, g)
        scale, bias = X.epilogue(64, mode, 27, g)
        wm = torch.zeros(64, 3, 4, 4)
        wm[:, :, :3, :3] = w.permute(0, 2, 3, 1)
        d_w, d_sb = _dev(wm), torch.cat([scale, bias]).cuda()
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        out = torch.full((B, Ho, Wo, pitch), 7.0, dtype=gpu_ops.ACT, device="cuda")
        assert L.dd3d_op_stem_s2_mma(gpu_ops._p(x4), gpu_ops._p(d_w), gpu_ops._p(d_sb), gpu_ops._p(out), pitch, B, H, W,
                                     gpu_ops._stream()) == 0
        torch.cuda.synchronize()
        X.assert_exact(out[..., :64], X.stem_ref64(x4[..., :3], w, scale, bias, 2), f"stem_s2_mma {B}x{H}x{W} {mode}")
        assert (out[..., 64:].float() == 7.0).all()


@pytest.mark.parametrize("B,H,W,out_pitch,pool_pitch", [(2, 64, 128, 32, 32), (1, 44, 76, 48, 40), (3, 128, 256, 32, 0)])
def test_dla_front_exact(B, H, W, out_pitch, pool_pitch, act):
    """dd3d_op_dla_front (csrc/dla_front.cu): ternary operands keep every layer's sum an integer, so the float64 chain that
    rounds the two intermediate maps to the storage type is bit-exact; the pooled copy is the max-pool of the output."""
    L = lib.load()
    g = X._gen(H + W)
    x4 = _input4(B, H, W, "int", 147, g)
    layers = []
    for cout, cin, k in ((16, 3, 7), (16, 16, 3), (32, 16, 3)):
        w = X.operand((cout, cin, k, k), "int", cin * k * k, g)
        scale = 2.0**torch.randint(0, 2, (cout, ), generator=g).float()  # integer intermediates: scales 1 and 2
        layers.append((w, scale, torch.randint(-3, 4, (cout, ), generator=g).float()))
    ref = X.dla_front_ref64(x4[..., :3], layers, gpu_ops.ACT)
    w0 = torch.zeros(16, 7, 8, 4)
    w0[:, :, :7, :3] = layers[0][0].permute(0, 2, 3, 1)
    w1 = layers[1][0].permute(0, 2, 3, 1).reshape(16, 9, 16)
    w2 = layers[2][0].permute(0, 2, 3, 1).reshape(32, 9, 16)
    dw = [_dev(t.contiguous()) for t in (w0, w1, w2)]
    dsb = [torch.cat([sc, bi]).cuda() for _, sc, bi in layers]
    out = torch.full((B, H // 2, W // 2, out_pitch), 7.0, dtype=gpu_ops.ACT, device="cuda")
    pool = torch.full((B, H // 4, W // 4, pool_pitch), 7.0, dtype=gpu_ops.ACT, device="cuda") if pool_pitch else None
    assert L.dd3d_op_dla_front(gpu_ops._p(x4), gpu_ops._p(dw[0]), gpu_ops._p(dw[1]), gpu_ops._p(dw[2]), gpu_ops._p(dsb[0]),
                               gpu_ops._p(dsb[1]), gpu_ops._p(dsb[2]), gpu_ops._p(out), out_pitch, gpu_ops._p(pool), pool_pitch,
                               B, H, W, gpu_ops._stream()) == 0
    torch.cuda.synchronize()
    X.assert_exact(out[..., :32], ref, f"DLA front {B}x{H}x{W}")
    assert (out[..., 32:].float() == 7.0).all()
    if pool is not None:
        pref = torch.nn.functional.max_pool2d(out[..., :32].float().permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
        assert torch.equal(pool[..., :32].float(), pref)
        assert (pool[..., 32:].float() == 7.0).all()


# ------------------------------------------------------------------------------------------------ sparse box3d predictor
# (H, W) of the five levels: ragged, 1 x W and 1 x 1 maps
B3D_LEVELS = [(23, 40), (12, 20), (6, 10), (1, 5), (1, 1)]
B3D_TOPK = 300  # three 128-row CTAs per (image, level), the last one partial


def _b3d_candidates(B, C_, counts, g):
    """fin pixels and entries [B][5][topk]: every level starts with its four corners and border midpoints, then one pixel
    several times with different classes, then random pixels; the slots past the count hold pixel 0."""
    pix = [[None] * 5 for _ in range(B)]
    fin = torch.zeros(B, 5, B3D_TOPK, 2, dtype=torch.int64)
    for b in range(B):
        for l, (H, W) in enumerate(B3D_LEVELS):
            edge = [0, W - 1, (H - 1) * W, H * W - 1, W // 2, (H - 1) * W + W // 2, (H // 2) * W, (H // 2) * W + W - 1]
            rnd = torch.randint(0, H * W, (B3D_TOPK, ), generator=g).tolist()
            p = (edge + [rnd[0]] * 4 + rnd)[:B3D_TOPK]
            n = min(counts[b][l], B3D_TOPK)
            p = p[:n] + [0] * (B3D_TOPK - n)
            cls = torch.randint(0, C_, (B3D_TOPK, ), generator=g)
            fin[b, l, :, 0] = torch.randint(0, 2**31, (B3D_TOPK, ), generator=g)
            fin[b, l, :, 1] = torch.tensor(p) * C_ + cls
            pix[b][l] = p[:n]
    return pix, fin.to(torch.int32)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("per_level", [False, True], ids=["shared", "per_level"])
@pytest.mark.parametrize("n_pad,C_", [(16, 10), (64, 5), (112, 10)], ids=["agnostic", "kitti", "nuscenes"])
def test_b3d_sparse_exact(n_pad, C_, per_level, mode, act):
    """dd3d_op_b3d_sparse (csrc/b3d_sparse.cu): exact fp32 rows for candidates on every border and corner, 1 x 1 and 1 x W
    levels, counts 0, 1, 127, 128, 129, topk and beyond, repeated pixels with several classes, both n-tile instances,
    shared and per-level weights; rows at or past the count and columns past n_pad keep their NaN sentinel."""
    L = lib.load()
    B = 2
    g = X._gen(n_pad + per_level)
    counts = [[B3D_TOPK, 129, 128, 1, 127], [127, 0, B3D_TOPK + 7, 129, 128]]
    pix, fin = _b3d_candidates(B, C_, counts, g)
    pitches = [256 + 8 * (l % 2) for l in range(5)]
    levels = [_dev(X.operand((B, H, W, pitches[l]), mode, 2304, g)) for l, (H, W) in enumerate(B3D_LEVELS)]
    ws, scs, bis = [], [], []
    for l in range(5):
        if per_level or l == 0:
            w = X.operand((n_pad, 256, 3, 3), mode, 2304, g)
        ws.append(w)
        sc, bi = X.epilogue(n_pad, mode, 2304, g)
        scs.append(sc)
        bis.append(bi)
    d_w = [_dev(gpu_ops.pack_conv_weight(w)) for w in ws]
    d_sc, d_bi = [s.cuda() for s in scs], [b.cuda() for b in bis]
    d_fin, d_cnt = fin.cuda(), torch.tensor(counts, dtype=torch.int32).cuda()
    out_pitch = n_pad + 8
    rows = torch.full((B, 5, B3D_TOPK, out_pitch), float("nan"), device="cuda")
    ptrs = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    hw = (C.c_int32 * 10)(*[v for p in B3D_LEVELS for v in p])
    st = L.dd3d_op_b3d_sparse(ptrs(levels), hw, (C.c_int32 * 5)(*pitches), ptrs(d_w), ptrs(d_sc), ptrs(d_bi), gpu_ops._p(d_fin),
                              gpu_ops._p(d_cnt), B, C_, B3D_TOPK, n_pad, gpu_ops._p(rows), out_pitch, gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    ref = X.b3d_rows_ref64([x[..., :256] for x in levels], ws, scs, bis, pix, counts, B3D_TOPK, n_pad)
    for b in range(B):
        for l in range(5):
            n = min(counts[b][l], B3D_TOPK)
            X.assert_exact(rows[b, l, :n, :n_pad], ref[b, l, :n].cuda(), f"b3d rows image {b} level {l} (slot, channel)")
            assert torch.isnan(rows[b, l, n:]).all(), f"image {b} level {l}: rows past the count were written"
    assert torch.isnan(rows[..., n_pad:]).all(), "columns past n_pad were written"


def test_b3d_sparse_refuses_bad_widths(act):
    """n_pad must be a multiple of 8 in [8, 112] and out_pitch >= n_pad: anything else returns DD3D_ERR_INVALID unlaunched."""
    L = lib.load()
    x = torch.zeros(1, 2, 2, 256, dtype=gpu_ops.ACT, device="cuda")
    w = torch.zeros(128, 9, 256, dtype=gpu_ops.ACT, device="cuda")
    sb = torch.zeros(128, device="cuda")
    fin = torch.zeros(1, 5, 4, 2, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, 5, dtype=torch.int32, device="cuda")
    rows = torch.zeros(1, 5, 4, 128, device="cuda")
    five = lambda t: (C.c_void_p * 5)(*([t.data_ptr()] * 5))  # noqa: E731
    hw = (C.c_int32 * 10)(*([2] * 10))
    pitch = (C.c_int32 * 5)(*([256] * 5))
    for n_pad, out_pitch in ((120, 128), (12, 16), (0, 16), (64, 32)):
        st = L.dd3d_op_b3d_sparse(five(x), hw, pitch, five(w), five(sb), five(sb), gpu_ops._p(fin), gpu_ops._p(cnt), 1, 5, 4,
                                  n_pad, gpu_ops._p(rows), out_pitch, gpu_ops._stream())
        assert st == -1, (n_pad, out_pitch, st)


# ------------------------------------------------------------------------------------------------ work-list conv
@pytest.mark.parametrize("mode", MODES)
def test_conv2d_tiles_exact(mode, act):
    """dd3d_op_conv2d_tiles (the pair tile in work-list mode, the sparse box3d tower's conv): the listed 16x8 tiles -- scattered,
    the ragged bottom-right tile, the out-of-image padding tile -- equal the float64 reference and the dense pair-tile conv
    bit for bit; every other pixel and the neighbouring channels keep their sentinel; an empty list writes nothing."""
    L = lib.load()
    B, H, W, cin, cout = 2, 45, 70, 160, 256
    tiles_x, tiles_y = (W + 7) // 8, (H + 15) // 16
    T = tiles_x * tiles_y  # 27: odd, so the padding tile T is a real case
    g = X._gen(45)
    x = _dev(X.operand((B, H, W, cin), mode, 9 * cin, g))
    w = X.operand((cout, cin, 3, 3), mode, 9 * cin, g)
    scale, bias = X.epilogue(cout, mode, 9 * cin, g)
    ref = X.conv_ref64(x, w, scale, bias, 1, relu=True)
    d_w, d_sc, d_bi = _dev(gpu_ops.pack_conv_weight(w)), gpu_ops.pad16(scale, 1.0).cuda(), gpu_ops.pad16(bias, 0.0).cuda()
    listed = [(0, 0), (0, 5), (0, T - 1), (0, 13), (1, 3), (1, T), (1, 9), (1, 10)]
    o0, op = 64, cout + 128
    try:
        _policy("pair_tile", 1)
        dense = gpu_ops.conv2d(x, w, scale, bias, 1, True)
    finally:
        _policy("pair_tile", -1)
    X.assert_exact(dense, ref, "dense pair-tile conv")
    for entries in (listed, []):
        tiles = torch.tensor([(b << 16) | t for b, t in entries] or [0], dtype=torch.int64).to(torch.int32).cuda()
        count = torch.tensor([len(entries)], dtype=torch.int32).cuda()
        out = torch.full((B, H, W, op), 7.0, dtype=gpu_ops.ACT, device="cuda")
        st = L.dd3d_op_conv2d_tiles(gpu_ops._p(x), B, H, W, cin, cin, gpu_ops._p(d_w), cout, gpu_ops._p(d_sc), gpu_ops._p(d_bi),
                                    1, C.c_void_p(out.data_ptr() + 2 * o0), op, gpu_ops._p(tiles), gpu_ops._p(count),
                                    gpu_ops._stream())
        assert st == 0
        torch.cuda.synchronize()
        mask = torch.zeros(B, H, W, dtype=torch.bool, device="cuda")
        for b, t in entries:
            if t == T:
                continue
            y0, x0 = (t // tiles_x) * 16, (t % tiles_x) * 8
            sl = (b, slice(y0, y0 + 16), slice(x0, x0 + 8))
            X.assert_exact(out[sl][..., o0:o0 + cout], ref[sl], f"listed tile {t} of image {b}")
            assert torch.equal(out[sl][..., o0:o0 + cout], dense[sl]), f"tile {t} of image {b} differs from the dense conv"
            mask[sl] = True
        assert (out[~mask].float() == 7.0).all(), "an unlisted pixel was written"
        assert (out[..., :o0].float() == 7.0).all() and (out[..., o0 + cout:].float() == 7.0).all()


# ------------------------------------------------------------------------------------------------ benchmark batch
def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _dets(o):
    inst = o["instances"]
    b3 = inst.pred_boxes3d
    return (_bits(torch.cat([inst.pred_boxes.tensor, inst.scores[:, None], inst.scores_3d[:, None], b3.quat, b3.size, b3.tvec],
                            1)), inst.pred_classes.cpu(), inst.fpn_levels.cpu())


def test_benchmark_batch_matches_single_images():
    """The bench.py workload (V2-99, bf16, B = 32, 900x1600, make_inputs(32, ..., seed_base=1)), where several buffers
    exceed 2^31 bytes: images 0, 17 and 31 (the highest offsets) give bit-identical detections inside the batch and alone."""
    cfg = get_cfg("v2_99", "nuscenes", act_dtype="bf16")
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    batch = model(make_inputs(32, 900, 1600, 1266.4, seed_base=1))
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    got = {k: _dets(batch[k]) for k in (0, 17, 31)}
    del batch
    for k in (0, 17, 31):
        alone = _dets(model(make_inputs(1, 900, 1600, 1266.4, seed_base=1 + k))[0])
        assert got[k][0].shape[0] > 0, f"image {k}: no detections"
        for a, b in zip(got[k], alone):
            assert a.shape == b.shape and torch.equal(a, b), f"image {k}: batch of 32 and alone differ"
