"""GPU suite (-m gpu) for the VoVNetV2-eSE family: the depthwise 3x3 kernel (csrc/dwconv.cu) against torch, the 384-channel
conv tile, and every variant end to end against the emulating oracle and the reference's own fp32 forward, with the bounds
of tests/test_e2e_gpu.py."""
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
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_nusc_inputs, make_state_dict
from oracle import bev_nms_oracle
from oracle.dd3d_oracle import pose_of
from oracle.vovnet_oracle import VOVNET_ARCHS, VOVNET_CASE, VoVNetOracle, case_inputs
from util import det_key, match_by_key, quat_dist, rel_err

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _keys_inst(inst):
    return [det_key(l, p, c) for l, p, c in zip(inst.fpn_levels.cpu(), inst.locations.cpu(), inst.pred_classes.cpu())]


def _model(arch, act_dtype="bf16", meta_arch="DD3D"):
    cfg = get_cfg(arch, VOVNET_CASE[0], act_dtype=act_dtype, meta_arch=meta_arch)
    sd = make_state_dict(cfg)
    m = (NuscenesDD3DB200 if meta_arch == "NuscenesDD3D" else DD3DB200)(cfg).to("cuda")
    m.load_state_dict(sd)
    return cfg, sd, m


# ------------------------------------------------------------------------------------------------ depthwise kernel
def _dwconv(x, c0, C_, w9, stride, out_pitch, out_c0):
    """dd3d_op_dwconv3x3 on channels [c0, c0 + C_) of x ([B, H, W, pitch]); writes channels [out_c0, out_c0 + C_) of a
    NaN-poisoned [B, Ho, Wo, out_pitch] buffer."""
    B, H, W, pitch = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = torch.full((B, Ho, Wo, out_pitch), float("nan"), dtype=x.dtype, device="cuda")
    st = lib.load().dd3d_op_dwconv3x3(C.c_void_p(x.data_ptr() + 2 * c0), B, H, W, C_, pitch, C.c_void_p(w9.data_ptr()), stride,
                                      C.c_void_p(out.data_ptr() + 2 * out_c0), out_pitch,
                                      C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("C_", [64, 80, 112, 224])
def test_dwconv3x3_vs_torch(dtype, stride, C_):
    gpu_ops.set_act_dtype(dtype)
    try:
        act = gpu_ops.ACT
        g = torch.Generator().manual_seed(C_ * 10 + stride)
        B, H, W = 3, 37, 45  # odd sizes: partial tiles on both axes
        c0, pitch = 16, C_ + 48  # channel slice of a wider (pitched) buffer
        x = torch.randn(B, H, W, pitch, generator=g).to(act).cuda()
        w = (torch.randn(C_, 1, 3, 3, generator=g) / 3.0).to(act)
        w9 = w.reshape(C_, 9).t().contiguous().cuda()
        out_pitch, oc0 = C_ + 32, 8
        got = _dwconv(x, c0, C_, w9, stride, out_pitch, oc0)
        again = _dwconv(x, c0, C_, w9, stride, out_pitch, oc0)
        assert torch.equal(got.view(torch.int16), again.view(torch.int16)), "two launches differ"
        ref = F.conv2d(x[..., c0:c0 + C_].float().permute(0, 3, 1, 2), w.float().cuda(), None, stride, 1, 1, C_)
        ref = ref.permute(0, 2, 3, 1)
        y = got[..., oc0:oc0 + C_].float()
        assert not torch.isnan(y).any()
        # within one rounding of the 16-bit type (fp32 sums in a different order may straddle a rounding boundary)
        ulp = ref.abs().clamp(min=2.0**-14) * (2.0**-7 if dtype == "bf16" else 2.0**-10)
        assert ((y - ref).abs() <= ulp * 1.01 + 1e-6).all()
        # channels outside the written slice stay untouched
        assert torch.isnan(got[..., :oc0].float()).all() and torch.isnan(got[..., oc0 + C_:].float()).all()
    finally:
        gpu_ops.set_act_dtype("bf16")


# ------------------------------------------------------------------------------------------------ 384-channel conv
@pytest.mark.parametrize("k", [1, 3])
def test_conv_384_output_channels(k):
    g = torch.Generator().manual_seed(384 + k)
    B, H, W, cin = 2, 24, 40, 96
    x = torch.randn(B, H, W, cin, generator=g).to(torch.bfloat16).cuda()
    w = torch.randn(384, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    scale, bias = 0.5 + torch.rand(384, generator=g), 0.1 * torch.randn(384, generator=g)
    got = gpu_ops.conv2d(x, w, scale, bias, relu=True).float()
    ref = gpu_ops.conv2d_ref(x, w, scale, bias, relu=True)
    assert (got - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()


def test_slim_model_uses_block_n_192():
    _, _, model = _model("v2_19_slim")
    model(case_inputs("v2_19_slim"))
    info = model.get_conv_info()
    wide = [r for r in info if r is not None and r["cout_pad"] == 384]
    assert wide and all(r["block_n"] == 192 for r in wide), wide


# ------------------------------------------------------------------------------------------------ end to end
_E2E = [(a, "bf16") for a in VOVNET_ARCHS] + [("v2_19_slim_dw", "fp16"), ("v2_57", "fp16")]


@pytest.mark.parametrize("arch,act_dtype", _E2E)
def test_forward_vs_emulating_oracle(arch, act_dtype):
    cfg, sd, model = _model(arch, act_dtype)
    inputs = case_inputs(arch)
    model.set_engine_option("sparse_box3d", 0)  # the stage-level check needs the dense 3-D maps
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    ref, inter = VoVNetOracle(cfg, sd, emulate=act_dtype, threads=1).forward(inputs, return_intermediates=True)
    x = model.get_tensor("input")[..., :3].float().cpu().permute(0, 3, 1, 2)
    assert torch.equal(x, inter["batch"])
    for l in range(5):
        f = model.get_tensor(f"p{l}").float().cpu().permute(0, 3, 1, 2)
        e = _rel_l2(f, inter["features"][l])
        assert e < 1e-2, f"FPN level {l}: rel L2 {e}"
        m = inter["maps"]
        cls = model.get_tensor(f"cls{l}").cpu().permute(0, 3, 1, 2)
        box = model.get_tensor(f"box{l}").cpu().permute(0, 3, 1, 2)
        b3d = model.get_tensor(f"b3d{l}").cpu().permute(0, 3, 1, 2)
        ref3d = torch.cat([m["quat"][l], m["ctr"][l], m["depth"][l], m["size"][l], m["conf"][l]], 1)
        for name, got, want in (("cls", cls, m["logits"][l]), ("reg", box[:, :4], m["box2d_reg"][l]),
                                ("ctr", box[:, 4:5], m["centerness"][l]), ("b3d", b3d, ref3d)):
            e = _rel_l2(got, want)
            # 1.5e-2 for V2-99; the small centerness map of level 0 measured 1.57e-2 (V-57) and 1.66e-2 (V-39) here
            assert e < (2.5e-2 if name == "ctr" else 1.5e-2), f"{name} level {l}: rel L2 {e}"
    for b, (o, r) in enumerate(zip(out, ref)):
        inst = o["instances"]
        kr = [det_key(l, p, c) for l, p, c in zip(r["level"], r["loc"], r["cls"])]
        ia, ib = match_by_key(_keys_inst(inst), kr)
        assert len(ib) >= 0.9 * len(kr) - 1, f"image {b}: matched {len(ib)} of {len(kr)}"
        if len(ia) == 0:
            continue
        gb, rb = inst.pred_boxes.tensor.cpu()[ia], r["box2d"][ib]
        size = torch.stack([rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]], 1).clamp(min=1.0).repeat(1, 2)
        assert ((gb - rb).abs() / size).max() < 1.3e-2
        # V2-99 bounds, except where a variant measured above them across two H100 runs (scores_3d 4.1e-3 for V-57 bf16,
        # quaternion 7.0e-2 for V-19-slim-dw): the storage emulation turns 1-ulp fp32 differences into 16-bit flips
        assert (inst.scores_3d.cpu()[ia] - r["score3d"][ib]).abs().max() < 8e-3
        assert (inst.scores.cpu()[ia] - r["score"][ib]).abs().max() < 8e-3
        b3 = inst.pred_boxes3d
        assert quat_dist(b3.quat.cpu()[ia], r["quat"][ib]).max() < 1e-1
        assert ((b3.size.cpu()[ia] - r["size"][ib]).abs() / r["size"][ib]).max() < 2.6e-2
        assert ((b3.depth.cpu()[ia, 0] - r["depth"][ib]).abs() / r["depth"][ib]).max() < 8e-3
        assert (b3.tvec.cpu()[ia] - r["tvec"][ib]).abs().max() < 0.05 * r["tvec"][ib].abs().max()


@pytest.mark.parametrize("arch", VOVNET_ARCHS)
def test_forward_vs_reference_golden(arch):
    g = np.load(os.path.join(GOLDEN_DIR, "golden_vovnet.npz"))
    _, _, model = _model(arch)
    out = model(case_inputs(arch))
    for b, o in enumerate(out):
        inst = o["instances"]
        p = f"{arch}/"
        assert tuple(inst.image_size) == tuple(g[f"{p}image_size{b}"].tolist())
        kg = [det_key(l, q, c) for l, q, c in zip(g[f"{p}levels{b}"], g[f"{p}locations{b}"], g[f"{p}classes{b}"])]
        ia, ib = match_by_key(_keys_inst(inst), kg)
        assert len(ib) >= 0.9 * len(kg) - 1, f"image {b}: matched {len(ib)} of {len(kg)}"
        if len(ia) == 0:
            continue
        gb, rb = inst.pred_boxes.tensor.cpu()[ia], torch.tensor(g[f"{p}boxes{b}"])[ib]
        size = torch.stack([rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]], 1).clamp(min=1.0).repeat(1, 2)
        assert ((gb - rb).abs() / size).max() < 1.6e-2


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def test_depthwise_plan_ignores_workspace_contents():
    """A v2_19_dw plan over a zeroed and over a 0xFF-poisoned workspace: bit-identical detections and op outputs."""
    res = []
    for fill in (0, 255):
        cfg, sd, model = _model("v2_19_dw")
        L = lib.load()
        h = model._engine()
        lib.check(L.dd3d_set_option(h, b"workspace_fill", fill), h)
        out = model(case_inputs("v2_19_dw"))
        torch.cuda.synchronize()
        snap = []
        for i in range(L.dd3d_num_ops(h)):
            try:
                snap.append(_bits(model.get_tensor(f"op{i}")))
            except RuntimeError:  # fp32 predictor ops have no 16-bit output view
                snap.append(None)
        res.append((out, snap))
    (a, sa), (b, sb) = res
    assert len(sa) == len(sb)
    for i, (x, y) in enumerate(zip(sa, sb)):
        assert (x is None) == (y is None)
        assert x is None or torch.equal(x, y), f"op {i} depends on the workspace contents"
    for x, y in zip(a, b):
        assert torch.equal(x["instances"].pred_boxes.tensor.cpu(), y["instances"].pred_boxes.tensor.cpu())
        assert torch.equal(x["instances"].scores_3d.cpu(), y["instances"].scores_3d.cpu())


def test_nuscenes_sample_aggregation_v2_39():
    """NuscenesDD3DB200 with V-39: per-image detections against the bf16-emulating oracle, and the sample aggregation
    exactly (the oracle's aggregation on the model's own pre-aggregation detections) -- the head / BEV path does not
    depend on the backbone."""
    cfg, sd, model = _model("v2_39", meta_arch="NuscenesDD3D")
    H, W = 128, 192
    inputs = make_nusc_inputs(1, H, W, 1266.4)
    for x in inputs:
        x["height"], x["width"] = 2 * H, 2 * W
    out = model(inputs)
    assert model.overflow_flags() == 0

    def as_dict(inst):
        b3 = inst.pred_boxes3d
        d = dict(level=inst.fpn_levels.cpu(), loc=inst.locations.cpu(), cls=inst.pred_classes.cpu(),
                 box2d=inst.pred_boxes.tensor.cpu(), score3d=inst.scores_3d.cpu(), score=inst.scores.cpu(),
                 quat=b3.quat.cpu(), tvec=b3.tvec.cpu(), size=b3.size.cpu(), attr=inst.pred_attributes.cpu(),
                 speed=inst.pred_speeds.cpu())
        if inst.has("pred_boxes3d_global"):
            d["quat_global"], d["tvec_global"] = inst.pred_boxes3d_global.quat.cpu(), inst.pred_boxes3d_global.tvec.cpu()
        return d

    got = [as_dict(o["instances"]) for o in out]
    model.sample_aggregate_in_inference = False
    pre = [as_dict(o["instances"]) for o in model(inputs)]
    model.sample_aggregate_in_inference = True
    assert sum(p["score3d"].shape[0] for p in pre) > 0
    ref = bev_nms_oracle.sample_aggregate(pre, [0] * 6, [pose_of(x) for x in inputs], cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH,
                                          cfg.DD3D.NUSC.INFERENCE.MAX_NUM_DETS_PER_SAMPLE)
    for gd, r in zip(got, ref):
        assert torch.equal(gd["score3d"], r["score3d"])
        assert quat_dist(gd["quat_global"], r["quat_global"]).max().item() < 1e-5 if len(gd["score3d"]) else True
        np.testing.assert_allclose(gd["tvec_global"].numpy(), r["tvec_global"].numpy(), rtol=1e-5, atol=1e-4)
    emu = VoVNetOracle(cfg, sd, emulate="bf16", threads=1).forward(inputs)
    matched = total = 0
    for gd, e in zip(got, emu):
        ka = [det_key(l, loc, c) for l, loc, c in zip(gd["level"], gd["loc"], gd["cls"])]
        kb = [det_key(l, loc, c) for l, loc, c in zip(e["level"], e["loc"], e["cls"])]
        ia, ib = match_by_key(ka, kb)
        matched += len(ia)
        total += max(len(ka), len(kb))
        if len(ia):
            assert rel_err(gd["box2d"][ia], e["box2d"][ib], floor=32.0) < 2e-2  # measured 5.9e-3 and 1.1e-2 on two H100 runs
    assert matched >= 0.9 * total
