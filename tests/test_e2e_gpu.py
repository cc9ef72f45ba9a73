"""End-to-end parity (-m gpu): DD3DB200.forward (C ABI -> sm_90a kernels) vs the CPU oracle on identical inputs.

Tolerances (see DESIGN.md "Numerics"; thresholds = the measured values of tools/parity_report.py x ~2): the engine
stores activations in bf16, so it is compared
  (a) with the oracle run in bf16-storage emulation on ONE thread (same rounding points; differences come only from fp32
      accumulation order -> isolated 1-ulp bf16 flips): relative L2 error of every FPN / head map <= 1e-2 / 1.5e-2 (measured
      7e-3 .. 1.0e-2), >= 90 % of the detections matched (measured 95.5 % / 98.8 %), boxes within 1.3e-2 of the box size
      (measured 6.5e-3), scores within 8e-3 (3.7e-3);
  (b) with the committed fp32 golden vectors of the REAL reference: >= 90 % of the reference detections reproduced (same
      level, location, class; measured 95.8 % / 100 %) with boxes within 1.6e-2 of the box size (measured 8e-3).
The fp32 decode / NMS kernels themselves are held to <= 1e-4 in tests/test_kernels_gpu.py, and at the BASELINE shapes to
exact sets / order in tests/test_parity_full_gpu.py (which also covers the fp16 storage type)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_inputs, make_state_dict
from oracle.dd3d_oracle import DD3DOracle  # checker only
from oracle.gen_golden import CASES, case_inputs
from util import det_key, match_by_key, quat_dist

pytestmark = pytest.mark.gpu


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _model(arch):
    cfg = get_cfg(arch, CASES[arch][0])
    sd = make_state_dict(cfg)
    m = DD3DB200(cfg).to("cuda")
    m.load_state_dict(sd)
    return cfg, sd, m


def _keys_inst(inst):
    return [det_key(l, p, c) for l, p, c in zip(inst.fpn_levels.cpu(), inst.locations.cpu(), inst.pred_classes.cpu())]


@pytest.mark.parametrize("arch", ["dla34", "v2_99"])
def test_forward_vs_emulating_oracle(arch):
    cfg, sd, model = _model(arch)
    inputs = case_inputs(arch)
    model.set_engine_option("sparse_box3d", 1)  # sparse box3d predictor (csrc/b3d_sparse.cu); the detections below come from it
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    model.set_engine_option("sparse_box3d", 0)  # the stage-level check needs the dense 3-D maps
    out_dense = model(inputs)
    torch.cuda.synchronize()
    for o, od in zip(out, out_dense):
        assert _keys_inst(o["instances"]) == _keys_inst(od["instances"]), "sparse and dense predictors: different detections"
        assert torch.equal(o["instances"].pred_boxes.tensor, od["instances"].pred_boxes.tensor)
        assert (o["instances"].scores_3d - od["instances"].scores_3d).abs().max() < 2e-5 if len(o["instances"]) else True
    ref, inter = DD3DOracle(cfg, sd, emulate="bf16", threads=1).forward(inputs, return_intermediates=True)
    C = cfg.DD3D.NUM_CLASSES
    # ---- stage level: preprocessed input (bit exact), FPN outputs, head maps
    x = model.get_tensor("input")[..., :3].float().cpu().permute(0, 3, 1, 2)
    assert torch.equal(x, inter["batch"])
    for l in range(5):
        f = model.get_tensor(f"p{l}").float().cpu().permute(0, 3, 1, 2)
        e = _rel_l2(f, inter["features"][l])
        assert e < 1e-2, f"FPN level {l}: rel L2 {e}"
        cls = model.get_tensor(f"cls{l}").cpu().permute(0, 3, 1, 2)
        box = model.get_tensor(f"box{l}").cpu().permute(0, 3, 1, 2)
        b3d = model.get_tensor(f"b3d{l}").cpu().permute(0, 3, 1, 2)
        m = inter["maps"]
        ref3d = torch.cat([m["quat"][l], m["ctr"][l], m["depth"][l], m["size"][l], m["conf"][l]], 1)
        for name, got, want in (("cls", cls, m["logits"][l]), ("reg", box[:, :4], m["box2d_reg"][l]),
                                ("ctr", box[:, 4:5], m["centerness"][l]), ("b3d", b3d, ref3d)):
            e = _rel_l2(got, want)
            assert e < 1.5e-2, f"{name} level {l}: rel L2 {e}"
    # ---- detections
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
        assert (inst.scores_3d.cpu()[ia] - r["score3d"][ib]).abs().max() < 4e-3
        assert (inst.scores.cpu()[ia] - r["score"][ib]).abs().max() < 8e-3
        b3 = inst.pred_boxes3d
        assert quat_dist(b3.quat.cpu()[ia], r["quat"][ib]).max() < 6e-2
        assert ((b3.size.cpu()[ia] - r["size"][ib]).abs() / r["size"][ib]).max() < 2.6e-2
        assert ((b3.depth.cpu()[ia, 0] - r["depth"][ib]).abs() / r["depth"][ib]).max() < 8e-3
        assert (b3.tvec.cpu()[ia] - r["tvec"][ib]).abs().max() < 0.05 * r["tvec"][ib].abs().max()


@pytest.mark.parametrize("arch", ["dla34", "v2_99"])
def test_forward_vs_reference_golden(arch):
    g = np.load(os.path.join(GOLDEN_DIR, f"golden_{arch}.npz"))
    _, _, model = _model(arch)
    out = model(case_inputs(arch))
    for b, o in enumerate(out):
        inst = o["instances"]
        assert tuple(inst.image_size) == tuple(g[f"image_size{b}"].tolist())
        kg = [det_key(l, p, c) for l, p, c in zip(g[f"levels{b}"], g[f"locations{b}"], g[f"classes{b}"])]
        ia, ib = match_by_key(_keys_inst(inst), kg)
        assert len(ib) >= 0.9 * len(kg) - 1, f"image {b}: matched {len(ib)} of {len(kg)}"
        gb, rb = inst.pred_boxes.tensor.cpu()[ia], torch.tensor(g[f"boxes{b}"])[ib]
        size = torch.stack([rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]], 1).clamp(min=1.0).repeat(1, 2)
        assert ((gb - rb).abs() / size).max() < 1.6e-2


def test_host_path_equals_device_path_and_is_deterministic():
    _, _, model = _model("dla34")
    inputs = case_inputs("dla34")
    a = model(inputs)
    b = model.forward_host(inputs)
    c = model(inputs)
    for x, y, z in zip(a, b, c):
        ix, iy, iz = x["instances"], y["instances"], z["instances"]
        assert len(ix) == len(iy) == len(iz)
        assert torch.equal(ix.pred_boxes.tensor.cpu(), iy.pred_boxes.tensor.cpu())
        assert torch.equal(ix.pred_boxes.tensor.cpu(), iz.pred_boxes.tensor.cpu())
        assert torch.equal(ix.scores_3d.cpu(), iy.scores_3d.cpu())
        assert torch.equal(ix.pred_boxes3d.quat.cpu(), iz.pred_boxes3d.quat.cpu())


def test_postprocess_toggle_and_no_nms():
    cfg, sd, model = _model("dla34")
    inputs = case_inputs("dla34")
    full = model(inputs)
    model.postprocess_in_inference = False
    raw = model(inputs)
    # image 1 is rescaled x2 by postprocess: raw boxes * 2 (then clipped) == processed boxes for surviving detections
    assert tuple(raw[1]["instances"].image_size) == (171, 286)
    n = min(len(raw[1]["instances"]), len(full[1]["instances"]))
    if n and len(raw[1]["instances"]) == len(full[1]["instances"]):
        rb = raw[1]["instances"].pred_boxes.tensor * 2
        rb[:, 0::2].clamp_(0, 572)
        rb[:, 1::2].clamp_(0, 342)
        assert torch.allclose(rb, full[1]["instances"].pred_boxes.tensor, atol=1e-3)
    cfg2 = get_cfg("dla34", "kitti_3d")  # out_cap is sized for the no-NMS case at construction
    cfg2.DD3D.INFERENCE.DO_NMS = False
    model2 = DD3DB200(cfg2).to("cuda")
    model2.load_state_dict(sd)
    allc = model2(inputs)
    assert len(allc[0]["instances"]) >= len(full[0]["instances"])


def test_full_size_properties_v2_99():
    """BASELINE shape (900x1600 -> 960x1600), size-independent properties: batch independence (image i of a batch ==
    the same image alone, bit for bit), determinism, sortedness by scores_3d, <= POST_NMS_TOPK (+ties), boxes clipped."""
    cfg, sd, model = _model("v2_99")
    inputs = make_inputs(2, 900, 1600, 1266.4)
    both = model(inputs)
    again = model(inputs)
    single = model(inputs[1:])
    assert model.overflow_flags() == 0
    for x, y in zip(both, again):
        assert torch.equal(x["instances"].pred_boxes.tensor, y["instances"].pred_boxes.tensor)
    a, s = both[1]["instances"], single[0]["instances"]
    assert len(a) == len(s)
    assert torch.equal(a.pred_boxes.tensor, s.pred_boxes.tensor) and torch.equal(a.scores_3d, s.scores_3d)
    for o in both:
        inst = o["instances"]
        assert 0 < len(inst) <= 128
        s3 = inst.scores_3d
        assert (s3[:-1] >= s3[1:]).all()
        bx = inst.pred_boxes.tensor
        assert (bx[:, 0] >= 0).all() and (bx[:, 2] <= 1600).all() and (bx[:, 1] >= 0).all() and (bx[:, 3] <= 900).all()
        assert ((bx[:, 2] - bx[:, 0]) > 0).all() and ((bx[:, 3] - bx[:, 1]) > 0).all()
        q = inst.pred_boxes3d.quat
        assert (q.norm(dim=1) - 1).abs().max() < 1e-3
        d = inst.pred_boxes3d.depth
        assert (d >= 0.1).all() and (d <= 80.0).all()


@pytest.mark.gpu
def test_submit_wait_host_matches_forward_host():
    """Double-buffered host path: two different batches in flight on slots 0 / 1 give exactly the results of the serial
    dd3d_forward_host calls (same kernels, same stream order)."""
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_inputs, make_state_dict
    cfg = get_cfg("dla34", "kitti_3d")
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    batches = [make_inputs(2, 192, 320, 721.5, seed_base=1 + 7 * i) for i in range(3)]
    ref = [model.forward_host(b) for b in batches]
    got = []
    model.submit_host(batches[0], 0)
    for k in range(3):
        if k + 1 < 3:
            model.submit_host(batches[k + 1], (k + 1) & 1)
        got.append(model.wait_host(k & 1))
    with pytest.raises(RuntimeError):
        model.wait_host(0)  # nothing pending on the slot
    total = 0
    for r, g in zip(ref, got):
        for a, b in zip(r, g):
            ia, ib = a["instances"], b["instances"]
            assert len(ia) == len(ib)
            total += len(ia)
            assert torch.equal(ia.pred_boxes.tensor, ib.pred_boxes.tensor)
            assert torch.equal(ia.scores_3d, ib.scores_3d)
            assert torch.equal(ia.pred_boxes3d.vectorize(), ib.pred_boxes3d.vectorize())
    assert total > 10


HEAD_CASES = [dict(THRESH_WITH_CTR=False), dict(FCOS3D_USE_SCALE=False), dict(FCOS2D_USE_SCALE=False),
              dict(CLASS_AGNOSTIC_BOX3D=True), dict(PER_LEVEL_PREDICTORS=True), dict(BOX3D_ON=False),
              dict(THRESH_WITH_CTR=False, FCOS3D_USE_SCALE=False, FCOS2D_USE_SCALE=False, CLASS_AGNOSTIC_BOX3D=True,
                   PER_LEVEL_PREDICTORS=True)]


@pytest.mark.parametrize("flags", HEAD_CASES, ids=lambda f: "+".join(f))
def test_non_default_head_configs_vs_oracle(flags):
    """The head switches no shipped experiment changes (fcos2d.py:280-290,100-108; fcos3d.py:103-104,116,128-139,166,
    175-180,333-352; core.py:34-40,117-125) run on the engine; tests/test_cpu_oracle.py pins the oracle for the same
    switches against the reference executed in the build container."""
    from test_cpu_oracle import apply_head_flags
    cfg = apply_head_flags(get_cfg("dla34", "kitti_3d"), flags)
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.03
    sd = make_state_dict(cfg)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    inputs = make_inputs(2, 128, 256, 721.5, seed_base=7)
    model.set_engine_option("sparse_box3d", 1)  # per-level weights / class-agnostic N = 16 / no 3-D head on the sparse predictor
    out = model(inputs)
    torch.cuda.synchronize()
    model.set_engine_option("sparse_box3d", 0)
    out_dense = model(inputs)
    torch.cuda.synchronize()
    for o, od in zip(out, out_dense):
        assert _keys_inst(o["instances"]) == _keys_inst(od["instances"])
        if cfg.MODEL.BOX3D_ON and len(o["instances"]):
            assert (o["instances"].scores_3d - od["instances"].scores_3d).abs().max() < 2e-5
            assert (o["instances"].pred_boxes3d.size - od["instances"].pred_boxes3d.size).abs().max() < 1e-4
    ref, inter = DD3DOracle(cfg, sd, emulate="bf16", threads=1).forward(inputs, return_intermediates=True)
    C = cfg.DD3D.NUM_CLASSES
    for l in range(5):
        cls = model.get_tensor(f"cls{l}").cpu().permute(0, 3, 1, 2)
        box = model.get_tensor(f"box{l}").cpu().permute(0, 3, 1, 2)
        assert _rel_l2(cls, inter["maps"]["logits"][l]) < 1.5e-2
        assert _rel_l2(box[:, :4], inter["maps"]["box2d_reg"][l]) < 1.5e-2
        if cfg.MODEL.BOX3D_ON:
            m = inter["maps"]
            ref3d = torch.cat([m["quat"][l], m["ctr"][l], m["depth"][l], m["size"][l], m["conf"][l]], 1)
            b3d = model.get_tensor(f"b3d{l}").cpu().permute(0, 3, 1, 2)
            assert b3d.shape[1] == ref3d.shape[1] == 11 * (1 if cfg.DD3D.FCOS3D.CLASS_AGNOSTIC_BOX3D else C)
            assert _rel_l2(b3d, ref3d) < 1.5e-2
    total = 0
    for b, (o, r) in enumerate(zip(out, ref)):
        inst = o["instances"]
        assert inst.has("pred_boxes3d") == bool(cfg.MODEL.BOX3D_ON) and inst.has("scores_3d") == bool(cfg.MODEL.BOX3D_ON)
        kr = [det_key(l, p, c) for l, p, c in zip(r["level"], r["loc"], r["cls"])]
        ia, ib = match_by_key(_keys_inst(inst), kr)
        assert len(ib) >= 0.85 * len(kr) - 1, f"image {b}: matched {len(ib)} of {len(kr)}"
        total += len(ib)
        if len(ia) == 0:
            continue
        gb, rb = inst.pred_boxes.tensor.cpu()[ia], r["box2d"][ib]
        size = torch.stack([rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]], 1).clamp(min=1.0).repeat(1, 2)
        assert ((gb - rb).abs() / size).max() < 2e-2
        assert (inst.scores.cpu()[ia] - r["score"][ib]).abs().max() < 8e-3
        if cfg.MODEL.BOX3D_ON:
            assert (inst.scores_3d.cpu()[ia] - r["score3d"][ib]).abs().max() < 8e-3
            b3 = inst.pred_boxes3d
            assert ((b3.depth.cpu()[ia, 0] - r["depth"][ib]).abs() / r["depth"][ib]).max() < 1.5e-2
            assert ((b3.size.cpu()[ia] - r["size"][ib]).abs() / r["size"][ib]).max() < 4e-2
    assert total > 5


def test_dla_front_fusion_matches_layer_by_layer():
    """The fused DLA-34 front end (csrc/dla_front.cu, engine option "dla_front" = 1, the default) against the same engine
    with the three layers run one by one ("dla_front" = 0): same FPN maps up to isolated 1-ulp flips of the 16-bit
    intermediates (different fp32 accumulation order), same number of ops minus three."""
    cfg, sd, model = _model("dla34")
    inputs = case_inputs("dla34")
    model(inputs)
    torch.cuda.synchronize()
    n_fused = model.launches_per_forward()
    fused = [model.get_tensor(f"p{l}").float().cpu().clone() for l in range(5)]
    model.set_engine_option("dla_front", 0)
    model(inputs)
    torch.cuda.synchronize()
    assert model.launches_per_forward() == n_fused + 3  # stem + level0 + level1 + maxpool -> one launch
    for l in range(5):
        e = _rel_l2(fused[l], model.get_tensor(f"p{l}").float().cpu())
        assert e < 1.5e-2, f"FPN level {l}: fused vs layer-by-layer rel L2 {e}"  # measured 7.2e-3: early 1-ulp flips amplified by the random-weight net, same size as engine-vs-oracle
    model.set_engine_option("dla_front", 1)
    model(inputs)
    torch.cuda.synchronize()
    for l in range(5):
        assert torch.equal(fused[l], model.get_tensor(f"p{l}").float().cpu()), "fused path is not reproducible"


@pytest.mark.parametrize("arch", ["dla34", "v2_99"])
def test_conv_n_split_is_bit_identical(arch):
    """Under-filled conv launches split their N tile (engine.cu Builder::conv, policy "n_split"): the K order of every output
    element is unchanged, so FPN and head maps must be bit-identical to the unsplit plan (the small golden shapes leave most
    launches under-filled, so the split path is what runs by default here)."""
    from dd3d_b200 import lib
    L = lib.load()
    inputs = case_inputs(arch)
    snaps = []
    try:
        for mode in (0, 1):
            assert L.dd3d_set_conv_policy(b"n_split", mode) == 0
            _, _, model = _model(arch)
            model.set_engine_option("sparse_box3d", 0)
            model(inputs)
            torch.cuda.synchronize()
            snaps.append([model.get_tensor(n).float().cpu().clone() for l in range(5) for n in (f"p{l}", f"cls{l}", f"b3d{l}")])
            del model
    finally:
        L.dd3d_set_conv_policy(b"n_split", -1)
    for a, b in zip(*snaps):
        assert torch.equal(a, b)


def test_v2_99_stem_mma_matches_stem_tc():
    """VoVNet stem_1 on the register-fragment kernel (csrc/stem_mma.cu, default) against the wgmma im2col kernel
    (csrc/stem_tc.cu, engine option "stem_mma" = 0) inside the engine: same FPN maps up to isolated 1-ulp flips of the stem's
    16-bit outputs (different fp32 summation order), amplified like any other rounding by the random-weight network."""
    cfg, sd, model = _model("v2_99")
    inputs = case_inputs("v2_99")
    model(inputs)
    torch.cuda.synchronize()
    a = [model.get_tensor(f"p{l}").float().cpu().clone() for l in range(5)]
    model.set_engine_option("stem_mma", 0)
    model(inputs)
    torch.cuda.synchronize()
    for l in range(5):
        e = _rel_l2(a[l], model.get_tensor(f"p{l}").float().cpu())
        assert e < 1.5e-2, f"FPN level {l}: stem_mma vs stem_tc rel L2 {e}"


def test_v2_99_fused_ese_pool_is_bit_identical():
    """The eSE scale pass of a VoVNet stage's last module can also write the next stage's max-pooled input (engine option
    "ese_pool" = 1; off by default because it measured ~10 % slower than the two kernels): pure data movement around the same
    arithmetic -> every FPN and head map is bit-identical to the default graph, with three launches fewer."""
    cfg, sd, model = _model("v2_99")
    inputs = case_inputs("v2_99")
    model.set_engine_option("sparse_box3d", 0)
    model.set_engine_option("ese_pool", 1)
    model(inputs)
    torch.cuda.synchronize()
    n_fused = model.launches_per_forward()
    names = [f"{n}{l}" for l in range(5) for n in ("p", "cls", "box", "b3d")]
    a = {n: model.get_tensor(n).float().cpu().clone() for n in names}
    model.set_engine_option("ese_pool", 0)  # the default: separate pool kernels
    model(inputs)
    torch.cuda.synchronize()
    assert model.launches_per_forward() == n_fused + 3
    for n in names:
        assert torch.equal(a[n], model.get_tensor(n).float().cpu()), n
