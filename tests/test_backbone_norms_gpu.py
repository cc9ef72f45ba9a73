"""GPU suite (-m gpu) for FE.BACKBONE.NORM and the GroupNorm kernel at every VoVNet channel count: dd3d_op_group_norm_c
against float64 F.group_norm on channel slices of concat buffers, its 256-channel bit-identity with dd3d_op_group_norm, and
the cases of oracle/backbone_norm_oracle.py end to end against the emulating oracle and the reference's own fp32 forward."""
import ctypes as C
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gpu_ops
from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.backbone_norm_oracle import BACKBONE_NORM_CASES, case_cfg, case_inputs
from oracle.dd3d_oracle import DD3DOracle
from util import det_key, match_by_key, quat_dist

pytestmark = pytest.mark.gpu

CHANNELS = [64, 128, 160, 192, 224, 256, 512, 768, 1024]


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _gn_c(x, c0, C_, gamma, beta, relu, out, out_c0, scratch):
    B, H, W, pitch = x.shape
    st = lib.load().dd3d_op_group_norm_c(C.c_void_p(x.data_ptr()), B, H, W, C_, c0, pitch, C.c_void_p(gamma.data_ptr()),
                                         C.c_void_p(beta.data_ptr()), int(relu), C.c_void_p(out.data_ptr()), out_c0,
                                         out.shape[-1], C.c_void_p(scratch.data_ptr()), _stream())
    torch.cuda.synchronize()
    return st


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("Cn", CHANNELS)
@pytest.mark.parametrize("H,W,offset", [(75, 130, 30.0), (9, 13, 0.0)])
def test_group_norm_c_vs_float64(dtype, Cn, H, W, offset):
    """A C-channel slice at offset c0 of a wider buffer (the OSA concat layout), normalised in place with ReLU, and into a
    slice of another buffer: within one 16-bit rounding plus the fp32 slack of test_group_norm_vs_float64; every channel
    outside the slice untouched; bit-identical over a poisoned scratch."""
    gpu_ops.set_act_dtype(dtype)
    try:
        act = gpu_ops.ACT
        g = torch.Generator().manual_seed(Cn * 31 + H)
        B, c0 = 2, 64
        pitch = c0 + Cn + 40
        x = (offset + torch.randn(B, H, W, pitch, generator=g) * torch.linspace(0.5, 2.0, pitch)).to(act).cuda()
        gamma = (0.5 + torch.rand(Cn, generator=g)).cuda()
        beta = (0.2 * torch.randn(Cn, generator=g)).cuda()
        scratch = torch.zeros(lib.load().dd3d_op_group_norm_scratch_bytes(B, H, W), dtype=torch.uint8, device="cuda")
        x0 = x.clone()
        out = torch.full((B, H, W, Cn + 16), float("nan"), dtype=act, device="cuda")
        assert _gn_c(x, c0, Cn, gamma, beta, True, out, 8, scratch) == 0
        assert torch.equal(x.view(torch.int16), x0.view(torch.int16)), "the input was modified"
        assert torch.isnan(out[..., :8].float()).all() and torch.isnan(out[..., 8 + Cn:].float()).all()
        got = out[..., 8:8 + Cn].clone()
        scratch.fill_(255)
        assert _gn_c(x, c0, Cn, gamma, beta, True, x, c0, scratch) == 0  # in place
        assert torch.equal(x[..., c0:c0 + Cn].contiguous().view(torch.int16), got.contiguous().view(torch.int16))
        assert torch.equal(x[..., :c0].view(torch.int16), x0[..., :c0].view(torch.int16))
        assert torch.equal(x[..., c0 + Cn:].view(torch.int16), x0[..., c0 + Cn:].view(torch.int16))
        xd = x0[..., c0:c0 + Cn].double()
        ref = F.group_norm(xd.permute(0, 3, 1, 2), 32, gamma.double(), beta.double(), 1e-5).permute(0, 2, 3, 1).clamp(min=0)
        cpg = Cn // 32
        xg = xd.reshape(B, H * W, 32, cpg)
        s = gamma.double().view(32, cpg) / (xg.var((1, 3), unbiased=False) + 1e-5).sqrt()[:, :, None]
        b_ = beta.double().view(32, cpg) - xg.mean((1, 3))[:, :, None] * s
        slack = 2.0**-20 * ((xg.abs() * s[:, None].abs()) + b_[:, None].abs()).reshape(B, H, W, Cn)
        ulp = ref.abs().clamp(min=2.0**-14) * (2.0**-7 if dtype == "bf16" else 2.0**-10)
        y = got.double()
        assert ((y - ref).abs() <= ulp * 1.01 + slack + 1e-7).all(), (y - ref).abs().max().item()
    finally:
        gpu_ops.set_act_dtype("bf16")


@pytest.mark.parametrize("H,W", [(120, 200), (5, 7)])
def test_group_norm_c_256_is_bit_identical_to_group_norm(H, W):
    g = torch.Generator().manual_seed(H)
    B = 3
    x = (7.0 + torch.randn(B, H, W, 264, generator=g)).to(torch.bfloat16).cuda()
    gamma = (0.5 + torch.rand(256, generator=g)).cuda()
    beta = (0.2 * torch.randn(256, generator=g)).cuda()
    scratch = torch.zeros(lib.load().dd3d_op_group_norm_scratch_bytes(B, H, W), dtype=torch.uint8, device="cuda")
    a = torch.empty(B, H, W, 256, dtype=torch.bfloat16, device="cuda")
    st = lib.load().dd3d_op_group_norm(C.c_void_p(x.data_ptr()), B, H, W, 264, C.c_void_p(gamma.data_ptr()),
                                       C.c_void_p(beta.data_ptr()), 1, None, 0, 0, C.c_void_p(a.data_ptr()), 256,
                                       C.c_void_p(scratch.data_ptr()), _stream())
    assert st == 0
    b = torch.empty_like(a)
    assert _gn_c(x, 0, 256, gamma, beta, True, b, 0, scratch) == 0
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_group_norm_c_refusals():
    x = torch.zeros(1, 4, 4, 256, dtype=torch.bfloat16, device="cuda")
    gam = torch.ones(256, device="cuda")
    sc = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    assert _gn_c(x, 0, 96, gam, gam, False, x, 0, sc) == -1   # 3 channels per group: not a VoVNet / head count
    assert _gn_c(x, 0, 112, gam, gam, False, x, 0, sc) == -1  # 112 = 32 x 3.5
    assert _gn_c(x, 4, 128, gam, gam, False, x, 4, sc) == -1   # offset not a multiple of 8
    assert _gn_c(x, 192, 128, gam, gam, False, x, 0, sc) == -1  # slice past the pitch


def _model(case, act_dtype="bf16"):
    cfg = case_cfg(case, act_dtype=act_dtype)
    sd = make_state_dict(cfg)
    m = DD3DB200(cfg).to("cuda")
    m.load_state_dict(sd)
    return cfg, sd, m


def _keys_inst(inst):
    return [det_key(l, p, c) for l, p, c in zip(inst.fpn_levels.cpu(), inst.locations.cpu(), inst.pred_classes.cpu())]


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


# The BN bounds of tests/test_head_norms_gpu.py.  Box errors are relative to max(box side, 16 px): without a backbone norm
# the synthetic weights give boxes only a few pixels high, whose 0.1 px storage-level differences (NVIDIA H100 80GB HBM3,
# 400 W power limit, bf16 dla34_none: at most 0.12 px on boxes 2-16 px high) would otherwise read as 6 %.
_BOX_FLOOR = 16.0
_BN = {"fpn": 1e-2, "box": 1.3e-2, "score": 8e-3, "size": 2.6e-2, "depth": 8e-3, "golden_box": 1.6e-2, "golden_match": 0.9}
# GroupNorm backbones with bf16 storage: every GN layer normalises a raw conv output that was rounded to bf16, and that
# rounding is amplified by |mean| / std of its group (tests/test_head_norms_gpu.py, GN heads); through 23-99 GN layers the
# engine's 1-ulp fp32 differences from the emulating oracle flip more roundings than with GN heads.  Measured on an NVIDIA
# H100 80GB HBM3 (700 W power limit), bf16, against the emulating oracle: FPN rel L2 2.28e-2 (v2_39_gn), 2.34e-2
# (v2_19_dw_gn), 1.62e-2 (v2_99_gn); boxes up to 2.35e-2, scores 7.8e-3, depths 1.05e-2, 3-D sizes 3.8e-2 (v2_99_gn),
# 5.9e-2 (v2_39_gn) and 6.5e-2 (v2_19_dw_gn).  Against the
# reference: v2_99_gn boxes 1.5e-2 with 95-97 of 100 matched, v2_19_dw_gn boxes 2.3e-2 with 44-45 of 47-49, v2_39_gn 33 of 38
# matched in image 0 (87 %).  The FPN, size and golden match bounds come from the worst measured values (1.4x, 1.4x, 0.8);
# the other bounds are the GN-head bounds of that file, the golden box bound its dla34_gn one.  With fp16 storage the same cases stay within the BN bounds (FPN 3.1e-3,
# boxes 2.0e-3 against the emulating oracle) and match the reference to the BN bounds (test_gn_fp16_vs_reference_golden).
_GN_BF16 = {"fpn": 3.3e-2, "box": 5.5e-2, "score": 1.5e-2, "size": 9.1e-2, "depth": 1.7e-2, "golden_box": 8e-2,
            "golden_match": 0.8}


def _bounds(case, act_dtype="bf16"):
    return _GN_BF16 if act_dtype == "bf16" and case_cfg(case).FE.BACKBONE.NORM == "GN" else _BN


_E2E = [(c, "bf16") for c in BACKBONE_NORM_CASES] + [("dla34_none", "fp16"), ("v2_39_gn", "fp16"), ("v2_99_gn", "fp16")]


@pytest.mark.parametrize("case,act_dtype", _E2E)
def test_forward_vs_emulating_oracle(case, act_dtype):
    cfg, sd, model = _model(case, act_dtype)
    inputs = case_inputs(case)
    model.set_engine_option("sparse_box3d", 0)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    ref, inter = DD3DOracle(cfg, sd, emulate=act_dtype, threads=1).forward(inputs, return_intermediates=True)
    bd = _bounds(case, act_dtype)
    fpn = max(_rel_l2(model.get_tensor(f"p{l}").float().cpu().permute(0, 3, 1, 2), inter["features"][l]) for l in range(5))
    print(f"\n{case} {act_dtype}: FPN rel L2 {fpn:.3e}")
    assert fpn < bd["fpn"]
    for b, (o, r) in enumerate(zip(out, ref)):
        inst = o["instances"]
        kr = [det_key(l, p, c) for l, p, c in zip(r["level"], r["loc"], r["cls"])]
        ia, ib = match_by_key(_keys_inst(inst), kr)
        assert len(ib) >= 0.9 * len(kr) - 1, f"image {b}: matched {len(ib)} of {len(kr)}"
        if len(ia) == 0:
            continue
        gb, rb = inst.pred_boxes.tensor.cpu()[ia], r["box2d"][ib]
        size = torch.stack([rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]], 1).clamp(min=_BOX_FLOOR).repeat(1, 2)
        b3 = inst.pred_boxes3d
        e = {"box": ((gb - rb).abs() / size).max().item(),
             "score": max((inst.scores_3d.cpu()[ia] - r["score3d"][ib]).abs().max().item(),
                          (inst.scores.cpu()[ia] - r["score"][ib]).abs().max().item()),
             "size": ((b3.size.cpu()[ia] - r["size"][ib]).abs() / r["size"][ib]).max().item(),
             "depth": ((b3.depth.cpu()[ia, 0] - r["depth"][ib]).abs() / r["depth"][ib]).max().item()}
        print(f"{case} {act_dtype} image {b}: matched {len(ib)} of {len(kr)}, " + ", ".join(f"{k} {v:.3e}" for k, v in e.items()))
        for k, v in e.items():
            assert v < bd[k], (k, v)
        assert quat_dist(b3.quat.cpu()[ia], r["quat"][ib]).max() < 1e-1


def _vs_golden(case, act_dtype):
    g = np.load(os.path.join(GOLDEN_DIR, "golden_backbone_norms.npz"))
    _, _, model = _model(case, act_dtype)
    bd = _bounds(case, act_dtype)
    out = model(case_inputs(case))
    for b, o in enumerate(out):
        inst = o["instances"]
        p = f"{case}/"
        assert tuple(inst.image_size) == tuple(g[f"{p}image_size{b}"].tolist())
        kg = [det_key(l, q, c) for l, q, c in zip(g[f"{p}levels{b}"], g[f"{p}locations{b}"], g[f"{p}classes{b}"])]
        ia, ib = match_by_key(_keys_inst(inst), kg)
        print(f"\n{case} {act_dtype} vs reference image {b}: matched {len(ib)} of {len(kg)}")
        assert len(ib) >= bd["golden_match"] * len(kg) - 1, f"image {b}: matched {len(ib)} of {len(kg)}"
        if len(ia) == 0:
            continue
        gb, rb = inst.pred_boxes.tensor.cpu()[ia], torch.tensor(g[f"{p}boxes{b}"])[ib]
        size = torch.stack([rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]], 1).clamp(min=_BOX_FLOOR).repeat(1, 2)
        e = ((gb - rb).abs() / size).max().item()
        print(f"{case} {act_dtype} vs reference image {b}: box {e:.3e}")
        assert e < bd["golden_box"]


@pytest.mark.parametrize("case", list(BACKBONE_NORM_CASES))
def test_forward_vs_reference_golden(case):
    _vs_golden(case, "bf16")


@pytest.mark.parametrize("case", [c for c in BACKBONE_NORM_CASES if c.endswith("_gn")])
def test_gn_fp16_vs_reference_golden(case):
    """With fp16 storage the GN backbones hold the BN bounds against the reference's fp32 forward."""
    _vs_golden(case, "fp16")


def _dets(out):
    return [torch.cat([o["instances"].pred_boxes.tensor, o["instances"].scores_3d[:, None],
                       o["instances"].pred_boxes3d.quat], 1).cpu() for o in out]


@pytest.mark.parametrize("backbone,norm", [("dla34", "BN"), ("v2_99", "SyncBN")])
def test_bn_checkpoint_matches_frozen_bit_for_bit(backbone, norm):
    """A BatchNorm2d-keyed checkpoint holding the FrozenBN checkpoint's values gives bit-identical detections."""
    inputs = case_inputs("dla34_bn")
    res = []
    for n in ("FrozenBN", norm):
        cfg = get_cfg(backbone, "nuscenes")
        cfg.FE.BACKBONE.NORM = n
        cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.02  # candidates from the synthetic weights at this size
        m = DD3DB200(cfg).to("cuda")
        m.load_state_dict(make_state_dict(cfg))
        res.append(_dets(m(inputs)))
    assert sum(len(x) for x in res[0]) > 0
    for a, b in zip(*res):
        assert torch.equal(a, b)


@pytest.mark.parametrize("case", ["dla34_none", "v2_19_dw_gn", "v2_39_gn"])
def test_plan_ignores_workspace_contents(case):
    """A plan over a zeroed and over a 0xFF-poisoned workspace: bit-identical detections, through the fused DLA front end,
    the stem kernel and the eSE pass with the new norms."""
    res = []
    for fill in (0, 255):
        _, _, model = _model(case)
        L = lib.load()
        h = model._engine()
        lib.check(L.dd3d_set_option(h, b"workspace_fill", fill), h)
        res.append(_dets(model(case_inputs(case))))
    assert sum(len(x) for x in res[0]) > 0
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_engine_backbone_norm_refusals():
    """DLA-34 and the slim VoVNets have no GN backbone and a VoVNet needs a norm; the call is refused after dd3d_finalize."""
    L = lib.load()
    for backbone, norm in (("dla34", lib.NORM_GN), ("v2_39", lib.NORM_NONE), ("v2_19_slim", lib.NORM_GN),
                           ("v2_19_slim_dw", lib.NORM_GN), ("dla34", 7)):
        d = lib.desc_from_cfg(get_cfg(backbone, "kitti_3d"))
        h = C.c_void_p()
        lib.check(L.dd3d_create(C.byref(d), C.byref(h)))
        try:
            assert L.dd3d_set_backbone_norm(h, norm) == -1
        finally:
            L.dd3d_destroy(h)
    _, _, model = _model("dla34_none")
    h = model._engine()
    assert L.dd3d_set_backbone_norm(h, lib.NORM_BN_SHARED) < 0


def test_gn_plan_has_one_group_norm_per_backbone_norm():
    """V-39 GN: the 39 GroupNorm layers of the reference are 39 GN ops (category 5 with the relu), beside the DLA-34-free
    default heads; the default V-39 plan has none."""
    res = {}
    for case in ("v2_39_syncbn", "v2_39_gn"):
        _, _, model = _model(case)
        model.set_profile(True)
        model(case_inputs(case))
        res[case] = [c for c, _, _ in model.get_op_times()].count("relu")
    assert res == {"v2_39_syncbn": 0, "v2_39_gn": 39}


def test_nuscenes_with_gn_backbone():
    """NuscenesDD3DB200 with a GN V-39 against the bf16-emulating oracle."""
    from dd3d_b200.meta_arch import NuscenesDD3DB200
    from dd3d_b200.synthetic import make_nusc_inputs
    from util import rel_err
    cfg = case_cfg("v2_39_gn", meta_arch="NuscenesDD3D")
    sd = make_state_dict(cfg)
    model = NuscenesDD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    inputs = make_nusc_inputs(1, 128, 192, 1266.4)
    out = model(inputs)
    assert model.overflow_flags() == 0
    emu = DD3DOracle(cfg, sd, emulate="bf16", threads=1).forward(inputs)
    matched = total = attr_same = 0
    worst = 0.0
    for o, e in zip(out, emu):
        inst = o["instances"]
        ka = _keys_inst(inst)
        kb = [det_key(l, loc, c) for l, loc, c in zip(e["level"], e["loc"], e["cls"])]
        ia, ib = match_by_key(ka, kb)
        matched += len(ia)
        total += max(len(ka), len(kb))
        if len(ia):
            worst = max(worst, rel_err(inst.pred_boxes.tensor.cpu()[ia], e["box2d"][ib], floor=32.0))
            attr_same += int((inst.pred_attributes.cpu()[ia] == e["attr"][ib]).sum())
            assert rel_err(inst.pred_speeds.cpu()[ia], e["speed"][ib], floor=1.0) < 5e-2
    print(f"\nNuscenesDD3D v2_39_gn: matched {matched} of {total}, box {worst:.3e}")
    assert worst < _GN_BF16["box"]
    assert total > 0 and matched >= 0.9 * total
    assert attr_same >= 0.9 * matched
