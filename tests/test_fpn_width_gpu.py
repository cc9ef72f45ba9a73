"""GPU suite (-m gpu) for FE.FPN.OUT_CHANNELS: every case of oracle/fpn_width_oracle.py end to end against the emulating
oracle (bf16 and fp16) and the reference's own fp32 forward, the sparse box3d predictor at every width exact against a
float64 reference, the GroupNorm kernels of the 320-, 384- and 448-channel heads, and the sparse predictor / towers on and
off at every width."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import exact_ops as X
import gpu_ops
import parity_lib as PL
from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import FPN_WIDTHS
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.fpn_width_oracle import FPN_WIDTH_CASES, case_cfg, case_inputs
from util import quat_dist

pytestmark = pytest.mark.gpu


def _inputs(case):
    if FPN_WIDTH_CASES[case][2] == "NuscenesDD3D":
        return make_nusc_inputs(1, 128, 192, 1266.4)
    return case_inputs(case)


def _model(cfg):
    nusc = cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D"
    m = (NuscenesDD3DB200 if nusc else DD3DB200)(cfg).to("cuda")
    m.load_state_dict(make_state_dict(cfg))
    if nusc:
        m.sample_aggregate_in_inference = False  # per-image detections, as the oracle returns them
    return m


# ------------------------------------------------------------------------------------------------ end to end
# Matched detections against the storage-emulating oracle (tests/parity_lib.py field errors).  The BN / no-norm bounds are
# the head-norm suite's; the bf16 GN cases take its GN bounds (GroupNorm normalises the raw conv output the conv stored at
# 16 bits, so a bf16 rounding is amplified by |mean| / std of its group).  At width 64 a group has 2 channels, and one H100
# run measured size 4.9e-2, score 1.7e-2 and score3d 1.0e-2 (dla34_gn_64, bf16); those three GN bounds are about 1.4x that.
_BOUNDS = {"box": 1.3e-2, "size": 2.6e-2, "depth": 8e-3, "score": 8e-3, "score3d": 8e-3}
_BOUNDS_GN_BF16 = {"box": 5.5e-2, "size": 7e-2, "depth": 1.7e-2, "score": 2.5e-2, "score3d": 1.4e-2}


@pytest.mark.parametrize("act_dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("case", list(FPN_WIDTH_CASES))
def test_forward_vs_emulating_oracle(case, act_dtype):
    cfg = case_cfg(case, act_dtype=act_dtype)
    model = _model(cfg)
    inputs = _inputs(case)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    ref = DD3DOracle(cfg, make_state_dict(cfg), emulate=act_dtype, threads=1).forward(inputs)
    gn = act_dtype == "bf16" and cfg.FE.FPN.NORM == "GN"
    bounds = _BOUNDS_GN_BF16 if gn else _BOUNDS
    worst = {f: 0.0 for f in bounds}
    for b, (o, r) in enumerate(zip(out, ref)):
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_oracle(r)
        rep, ia, ib = PL.compare_sets(a, e)
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        for f in bounds:
            if len(errs[f]):
                worst[f] = max(worst[f], float(errs[f].max()))
        if len(ia):
            assert quat_dist(a["quat"][ia], e["quat"][ib]).max() < 1e-1
    print(f"\n{case} {act_dtype}: worst {worst}")
    for f, bound in bounds.items():
        assert worst[f] < bound, f"{f}: {worst[f]} >= {bound}"


@pytest.mark.parametrize("case", [c for c, v in FPN_WIDTH_CASES.items() if v[2] == "DD3D"])
def test_forward_vs_reference_golden(case):
    g = np.load(os.path.join(GOLDEN_DIR, "golden_fpn_width.npz"))
    g = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(case + "/")}
    cfg = case_cfg(case)
    out = _model(cfg)(case_inputs(case))
    gn = cfg.FE.FPN.NORM == "GN"
    for b, o in enumerate(out):
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_golden(g, b)
        assert tuple(o["instances"].image_size) == tuple(g[f"image_size{b}"].tolist())
        rep, ia, ib = PL.compare_sets(a, e)
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        if len(ia):
            print(f"\n{case} image {b}: box {errs['box'].max():.3e} size {errs['size'].max():.3e}")
            assert errs["box"].max() < (8e-2 if gn else 1.6e-2)


# ------------------------------------------------------------------------------------------------ sparse box3d predictor
_LEVELS = [(23, 40), (12, 20), (6, 10), (1, 5), (1, 1)]
_TOPK = 300


def _b3d_case(cin, n_pad, C_, mode, g):
    from test_exact_kernels_gpu import _b3d_candidates  # noqa: PLC0415  (fin / pixel layout shared with the 256 test)
    B = 2
    counts = [[_TOPK, 129, 128, 1, 127], [127, 0, _TOPK + 7, 129, 128]]
    pix, fin = _b3d_candidates(B, C_, counts, g)
    pitches = [cin + 8 * (l % 2) for l in range(5)]
    K = 9 * cin
    levels = [X.operand((B, H, W, pitches[l]), mode, K, g).to(gpu_ops.ACT).cuda() for l, (H, W) in enumerate(_LEVELS)]
    ws = [X.operand((n_pad, cin, 3, 3), mode, K, g) for _ in range(5)]
    sb = [X.epilogue(n_pad, mode, K, g) for _ in range(5)]
    return B, counts, pix, fin, pitches, levels, ws, sb


def _run_b3d(fn, cin, B, C_, counts, fin, pitches, levels, ws, sb, n_pad):
    L = lib.load()
    d_w = [gpu_ops.pack_conv_weight(w).cuda() for w in ws]
    d_sc, d_bi = [s.cuda() for s, _ in sb], [b.cuda() for _, b in sb]
    d_fin, d_cnt = fin.cuda(), torch.tensor(counts, dtype=torch.int32).cuda()
    rows = torch.full((B, 5, _TOPK, n_pad + 8), float("nan"), device="cuda")
    ptrs = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    hw = (C.c_int32 * 10)(*[v for p in _LEVELS for v in p])
    args = [ptrs(levels), hw, (C.c_int32 * 5)(*pitches), ptrs(d_w), ptrs(d_sc), ptrs(d_bi), gpu_ops._p(d_fin),
            gpu_ops._p(d_cnt), B, C_, _TOPK, n_pad, gpu_ops._p(rows), n_pad + 8]
    st = getattr(L, fn)(*(args + ([cin] if fn.endswith("_c") else []) + [gpu_ops._stream()]))
    assert st == 0
    torch.cuda.synchronize()
    return rows


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


@pytest.mark.parametrize("n_pad,C_", [(64, 5), (112, 10)], ids=["kitti", "nuscenes"])
@pytest.mark.parametrize("cin", [64, 128, 192, 320, 448, 512])
def test_b3d_sparse_c_exact(cin, n_pad, C_, act):
    """dd3d_op_b3d_sparse_c: exact fp32 rows at every width (integer operands: no rounding in any order); rows past the count
    and columns past n_pad keep their NaN sentinel."""
    g = X._gen(cin + n_pad)
    B, counts, pix, fin, pitches, levels, ws, sb = _b3d_case(cin, n_pad, C_, "round", g)
    rows = _run_b3d("dd3d_op_b3d_sparse_c", cin, B, C_, counts, fin, pitches, levels, ws, sb, n_pad)
    ref = X.b3d_rows_ref64([x[..., :cin] for x in levels], ws, [s for s, _ in sb], [b for _, b in sb], pix, counts, _TOPK,
                           n_pad)
    for b in range(B):
        for l in range(5):
            n = min(counts[b][l], _TOPK)
            X.assert_exact(rows[b, l, :n, :n_pad], ref[b, l, :n].cuda(), f"cin {cin} image {b} level {l}")
            assert torch.isnan(rows[b, l, n:]).all()
    assert torch.isnan(rows[..., n_pad:]).all()


@pytest.mark.parametrize("n_pad,C_", [(64, 5), (112, 10)], ids=["kitti", "nuscenes"])
def test_b3d_sparse_c_at_256_is_b3d_sparse(n_pad, C_, act):
    """Non-integer operands: at 256 channels the two entry points give the same bits."""
    g = torch.Generator().manual_seed(256 + n_pad)
    B, counts, pix, fin, pitches, levels, ws, sb = _b3d_case(256, n_pad, C_, "round", X._gen(n_pad))
    levels = [torch.randn(x.shape, generator=g).to(gpu_ops.ACT).cuda() for x in levels]
    ws = [torch.randn(w.shape, generator=g) / 48.0 for w in ws]
    a = _run_b3d("dd3d_op_b3d_sparse", 256, B, C_, counts, fin, pitches, levels, ws, sb, n_pad)
    b = _run_b3d("dd3d_op_b3d_sparse_c", 256, B, C_, counts, fin, pitches, levels, ws, sb, n_pad)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_b3d_sparse_c_refuses_bad_widths():
    L = lib.load()
    x = torch.zeros(1, 2, 2, 576, dtype=gpu_ops.ACT, device="cuda")
    w = torch.zeros(64, 9, 576, dtype=gpu_ops.ACT, device="cuda")
    sb = torch.zeros(64, device="cuda")
    fin = torch.zeros(1, 5, 4, 2, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, 5, dtype=torch.int32, device="cuda")
    rows = torch.zeros(1, 5, 4, 64, device="cuda")
    five = lambda t: (C.c_void_p * 5)(*([t.data_ptr()] * 5))  # noqa: E731
    hw = (C.c_int32 * 10)(*([2] * 10))
    for cin, pitch in ((96, 96), (0, 64), (576, 576), (128, 64)):
        st = L.dd3d_op_b3d_sparse_c(five(x), hw, (C.c_int32 * 5)(*([pitch] * 5)), five(w), five(sb), five(sb),
                                    gpu_ops._p(fin), gpu_ops._p(cnt), 1, 5, 4, 64, gpu_ops._p(rows), 64, cin,
                                    gpu_ops._stream())
        assert st == -1, (cin, pitch, st)


# ------------------------------------------------------------------------------------------------ GroupNorm cpg 10 / 12 / 14
def _gn_c(x, C_, gamma, beta, relu, out, scratch):
    B, H, W, pitch = x.shape
    st = lib.load().dd3d_op_group_norm_c(C.c_void_p(x.data_ptr()), B, H, W, C_, 0, pitch, C.c_void_p(gamma.data_ptr()),
                                         C.c_void_p(beta.data_ptr()), int(relu), C.c_void_p(out.data_ptr()), 0, out.shape[-1],
                                         C.c_void_p(scratch.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("H,W,offset", [(240, 400, 40.0), (37, 45, 0.0)])
@pytest.mark.parametrize("C_", [320, 384, 448])
def test_group_norm_new_widths_vs_float64(C_, H, W, offset, dtype):
    """GroupNorm(32, C) at cpg 10, 12, 14 within one 16-bit rounding of float64 F.group_norm (the bound of the 256-channel
    kernel test), channels past C untouched, and bit-identical over a 0xFF-poisoned scratch."""
    gpu_ops.set_act_dtype(dtype)
    try:
        act = gpu_ops.ACT
        g = torch.Generator().manual_seed(C_ + H)
        B, pitch = 2, C_ + 8
        x = (offset + torch.randn(B, H, W, pitch, generator=g) * torch.linspace(0.5, 2.0, pitch)).to(act).cuda()
        gamma, beta = (0.5 + torch.rand(C_, generator=g)).cuda(), (0.2 * torch.randn(C_, generator=g)).cuda()
        scratch = torch.zeros(lib.load().dd3d_op_group_norm_scratch_bytes(B, H, W), dtype=torch.uint8, device="cuda")
        got = _gn_c(x, C_, gamma, beta, True, torch.full((B, H, W, pitch), float("nan"), dtype=act, device="cuda"), scratch)
        assert torch.isnan(got[..., C_:].float()).all()
        scratch.fill_(255)
        again = _gn_c(x, C_, gamma, beta, True, torch.empty_like(got), scratch)
        assert torch.equal(got[..., :C_].contiguous().view(torch.int16), again[..., :C_].contiguous().view(torch.int16))
        cpg = C_ // 32
        xd = x[..., :C_].double().cpu()
        ref = F.group_norm(xd.permute(0, 3, 1, 2), 32, gamma.double().cpu(), beta.double().cpu(), 1e-5).permute(0, 2, 3, 1)
        xg = xd.reshape(B, H * W, 32, cpg)
        s = gamma.double().cpu().view(32, cpg) / (xg.var((1, 3), unbiased=False) + 1e-5).sqrt()[:, :, None]
        b_ = beta.double().cpu().view(32, cpg) - xg.mean((1, 3))[:, :, None] * s
        slack = 2.0**-20 * ((xg.abs() * s[:, None].abs()) + b_[:, None].abs()).reshape(B, H, W, C_)
        ref = ref.clamp(min=0)
        y = got[..., :C_].double().cpu()
        ulp = ref.abs().clamp(min=2.0**-14) * (2.0**-7 if dtype == "bf16" else 2.0**-10)
        assert ((y - ref).abs() <= ulp * 1.01 + slack + 1e-7).all(), (y - ref).abs().max().item()
    finally:
        gpu_ops.set_act_dtype("bf16")


# ------------------------------------------------------------------------------------------------ sparse paths per width
@pytest.fixture
def _pair_tile():
    L = lib.load()
    assert L.dd3d_set_conv_policy(b"pair_tile", 1) == 0
    yield
    L.dd3d_set_conv_policy(b"pair_tile", -1)


def _dets(out):
    res = []
    for o in out:
        inst = o["instances"]
        b3 = inst.pred_boxes3d
        two = torch.cat([inst.pred_boxes.tensor, inst.scores[:, None]], 1).contiguous().view(torch.int32).cpu()
        three = torch.cat([inst.scores_3d[:, None], b3.quat, b3.size, b3.tvec], 1).cpu()
        res.append((two, inst.pred_classes.cpu().clone(), inst.fpn_levels.cpu().clone(), three))
    return res


def _run_opts(cfg, inputs, **opts):
    model = _model(cfg)
    for k, v in opts.items():
        model.set_engine_option(k, v)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    n = model.launches_per_forward()
    del model
    return _dets(out), n


@pytest.mark.parametrize("width", FPN_WIDTHS)
def test_sparse_paths_at_every_width(width, _pair_tile):
    """DLA-34 at every width: the sparse box2d / box3d towers are bit-identical to the dense towers where they run (widths
    that 128 divides: their extra launches) and absent elsewhere (same launches: the dense fallback).  The sparse box3d
    predictor sums in another fp32 order than the dense one, and the NMS is keyed on the 3-D score: its detections match
    the dense predictor's to that rounding."""
    cfg = get_cfg("dla34", "kitti_3d", fpn_channels=width)
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.03
    inputs = make_inputs(2, 192, 320, 721.5)
    off = dict(sparse_box3d=0, sparse_tower=0, sparse_box2d_tower=0)
    dense, n_dense = _run_opts(cfg, inputs, **off)
    assert sum(len(d[0]) for d in dense) > 0
    pair = width % 128 == 0
    box2d, n_box2d = _run_opts(cfg, inputs, **dict(off, sparse_box2d_tower=1))
    assert n_box2d == n_dense + (2 if pair else 0), (n_box2d, n_dense)  # seed + tile-list launches
    sp3, n_sp3 = _run_opts(cfg, inputs, **dict(off, sparse_box3d=1))
    tower, n_tower = _run_opts(cfg, inputs, **dict(off, sparse_box3d=1, sparse_tower=1))
    assert n_tower == n_sp3 + (1 if pair else 0), (n_tower, n_sp3)
    for i, (d, b, s, t) in enumerate(zip(dense, box2d, sp3, tower)):
        for k in range(4):
            assert torch.equal(d[k], b[k]), f"width {width} image {i}: sparse box2d tower differs"
            assert torch.equal(s[k], t[k]), f"width {width} image {i}: sparse box3d tower differs"
        kd = [(int(l), int(c), *d[0][j, :4].tolist()) for j, (c, l) in enumerate(zip(d[1], d[2]))]
        ks = {(int(l), int(c), *s[0][j, :4].tolist()): j for j, (c, l) in enumerate(zip(s[1], s[2]))}
        ia = [j for j, k in enumerate(kd) if k in ks]
        assert len(ia) >= len(kd) - 2 and abs(len(ks) - len(kd)) <= 2, f"width {width} image {i}: {len(ia)} of {len(kd)}"
        ib = [ks[kd[j]] for j in ia]
        assert torch.allclose(d[3][ia], s[3][ib], rtol=1e-4, atol=1e-4), f"width {width} image {i}: 3-D fields"
