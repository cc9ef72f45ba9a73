"""Test-time augmentation for NuscenesDD3D (nuscenes_dd3d_tta.py) and the DO_BEV_NMS branch of both TTA wrappers:
constructor / call contracts and build_tta_model on the CPU; on the GPU, NuscenesDD3DB200WithTTA's aggregation and the
merged-set BEV step against the oracle on the model's own detections, and the whole path against the bf16-emulating
oracle."""
import os

import numpy as np
import pytest
import torch

import nusc_tta_oracle as NT
from conftest import GOLDEN_DIR
from util import quat_dist, rel_err

NUSC_TTA = dict(H=128, W=192, orig=(256, 384), focal=1266.4, min_sizes=[128, 160, 192], ims_per_batch=4,
                pre_nms_thresh=0.01, max_dets=300, samples=2)


# fixtures written by tools/gen_nusc_tta_golden.py from the reference's own NuscenesDD3DWithTTA: name -> (DO_BEV_NMS, samples)
GOLDEN_CASES = {"nusc_tta_v2_99": (False, 2), "nusc_tta_bev_v2_99": (True, 1)}


def nusc_tta_case(do_bev_nms=False, samples=None):
    """(cfg, inputs): 2 samples x 6 cameras of synthetic V2-99 images, 3 scales x flip = 6 views per image in chunks of 4
    (so one image's views split across two engine calls), a low pre-NMS threshold and a per-call cap that binds.  With
    DO_BEV_NMS the BEV IoU threshold is lowered to 0.05 so that the BEV steps suppress, and every view runs in its own
    model call: the reference's per-view BEV NMS (nuscenes_sample_aggregate with dummy groups inside NuscenesDD3D.forward)
    concatenates the Instances of one call, and detectron2's Instances.cat asserts one image size, so the reference runs
    this branch only when a call holds views of a single scale."""
    from dd3d_b200.config import get_cfg
    from dd3d_b200.synthetic import make_nusc_inputs
    c = NUSC_TTA
    cfg = get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D")
    cfg.DD3D.INFERENCE.DO_POSTPROCESS = False
    cfg.DD3D.INFERENCE.DO_BEV_NMS = do_bev_nms
    cfg.TEST.IMS_PER_BATCH = c["ims_per_batch"]
    if do_bev_nms:
        cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH = 0.05
        cfg.TEST.IMS_PER_BATCH = 1
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = c["pre_nms_thresh"]
    cfg.DD3D.NUSC.INFERENCE.MAX_NUM_DETS_PER_SAMPLE = c["max_dets"]
    cfg.TEST.AUG.MIN_SIZES = list(c["min_sizes"])
    inputs = make_nusc_inputs(samples or c["samples"], c["H"], c["W"], c["focal"])
    for x in inputs:
        x["height"], x["width"] = c["orig"]
    return cfg, inputs


def _model(cfg, device="cuda"):
    from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from dd3d_b200.arch import is_nuscenes_arch
    model = (NuscenesDD3DB200 if is_nuscenes_arch(cfg) else DD3DB200)(cfg).to(device)
    model.load_state_dict(make_state_dict(cfg))
    return model


# ------------------------------------------------------------------------------------------------ CPU
def test_build_tta_model_mapping():
    from dd3d_b200.config import get_cfg
    from dd3d_b200.tta import DD3DB200WithTTA, NuscenesDD3DB200WithTTA, build_tta_model
    for name, cls in (("DD3D", DD3DB200WithTTA), ("DD3DB200", DD3DB200WithTTA), ("NuscenesDD3D", NuscenesDD3DB200WithTTA),
                      ("NuscenesDD3DB200", NuscenesDD3DB200WithTTA)):
        cfg = get_cfg("v2_99", "nuscenes", meta_arch=name.replace("B200", ""))
        cfg.MODEL.META_ARCHITECTURE = name
        cfg.DD3D.INFERENCE.DO_POSTPROCESS = False
        tta = build_tta_model(cfg, _model(cfg, "cpu"))
        assert type(tta) is cls
        assert tta.batch_size == cfg.TEST.IMS_PER_BATCH and tta.num_views == 2 * len(cfg.TEST.AUG.MIN_SIZES)
    cfg.MODEL.META_ARCHITECTURE = "GeneralizedRCNN"
    with pytest.raises(AssertionError, match="not available"):
        build_tta_model(cfg, None)


def test_nusc_tta_constructor_and_call_contracts():
    from dd3d_b200.tta import DD3DB200WithTTA, NuscenesDD3DB200WithTTA
    cfg, inputs = nusc_tta_case()
    model = _model(cfg, "cpu")
    tta = NuscenesDD3DB200WithTTA(cfg, model, world_size=2)
    assert tta.batch_size == NUSC_TTA["ims_per_batch"] // 2
    with pytest.raises(AssertionError, match="only supports"):
        DD3DB200WithTTA(cfg, model)
    from dd3d_b200.config import get_cfg
    kcfg = get_cfg("dla34", "kitti_3d")
    kcfg.DD3D.INFERENCE.DO_POSTPROCESS = False
    with pytest.raises(AssertionError, match="only supports"):
        NuscenesDD3DB200WithTTA(kcfg, _model(kcfg, "cpu"))
    model.postprocess_in_inference = True
    with pytest.raises(AssertionError, match="postprocess_in_inference"):
        NuscenesDD3DB200WithTTA(cfg, model)
    # get_group_idxs' error comes before any device work (the model here has no engine and no CUDA device)
    with pytest.raises(ValueError, match="Group sizes"):
        tta(inputs[:5])
    with pytest.raises(ValueError, match="Group sizes"):
        tta(inputs + inputs[:3])


@pytest.mark.parametrize("name", list(GOLDEN_CASES))
def test_nusc_tta_oracle_matches_reference_golden(name):
    """fp32 oracle == the reference's NuscenesDD3DWithTTA(NuscenesDD3D) on the fixture cases (tools/gen_nusc_tta_golden.py):
    the same detections in the same order per image, with attributes, speeds and global boxes."""
    from dd3d_b200.synthetic import make_state_dict
    from oracle.dd3d_oracle import DD3DOracle
    do_bev_nms, samples = GOLDEN_CASES[name]
    g = np.load(os.path.join(GOLDEN_DIR, f"{name}.npz"))
    cfg, inputs = nusc_tta_case(do_bev_nms=do_bev_nms, samples=samples)
    out = NT.nusc_tta_forward(DD3DOracle(cfg, make_state_dict(cfg)), inputs, cfg)
    total = 0
    for b, o in enumerate(out):
        n = g[f"scores_3d{b}"].shape[0]
        total += n
        assert o["score3d"].shape[0] == n, (b, o["score3d"].shape[0], n)
        assert tuple(g[f"image_size{b}"]) == (inputs[b]["height"], inputs[b]["width"])
        if not n:
            continue
        np.testing.assert_allclose(o["score3d"].numpy(), g[f"scores_3d{b}"], rtol=1e-4, atol=1e-6)
        assert np.array_equal(o["cls"].numpy(), g[f"classes{b}"])
        assert rel_err(o["box2d"], g[f"boxes{b}"], floor=16.0) < 1e-4
        assert quat_dist(o["quat"], g[f"quat{b}"]).max().item() < 1e-4
        assert rel_err(o["proj_ctr"], g[f"proj_ctr{b}"], floor=16.0) < 1e-4
        assert rel_err(o["depth"], g[f"depth{b}"].reshape(-1), floor=1.0) < 1e-4
        assert rel_err(o["inv_K"], g[f"inv_K{b}"], floor=1e-3) < 1e-3
        assert np.array_equal(o["attr"].numpy(), g[f"attr{b}"])
        assert rel_err(o["speed"], g[f"speed{b}"], floor=1.0) < 1e-4
        assert quat_dist(o["quat_global"], g[f"quat_global{b}"]).max().item() < 1e-4
        assert rel_err(o["tvec_global"], g[f"tvec_global{b}"], floor=1.0) < 1e-4
    if not do_bev_nms:  # the per-call cap binds across the two samples
        assert total == NUSC_TTA["max_dets"]
    assert total > 100


# ------------------------------------------------------------------------------------------------ GPU
def _as_dict(inst):
    b3 = inst.pred_boxes3d
    d = dict(box2d=inst.pred_boxes.tensor.cpu(), cls=inst.pred_classes.cpu(), score3d=inst.scores_3d.cpu(),
             score=inst.scores.cpu(), quat=b3.quat.cpu(), proj_ctr=b3.proj_ctr.cpu(), depth=b3.depth.cpu().reshape(-1),
             size=b3.size.cpu(), inv_K=b3.inv_intrinsics.cpu(), tvec=b3.tvec.cpu())
    if inst.has("pred_attributes"):
        d["attr"], d["speed"] = inst.pred_attributes.cpu(), inst.pred_speeds.cpu()
    if inst.has("pred_boxes3d_global"):
        d["quat_global"], d["tvec_global"] = inst.pred_boxes3d_global.quat.cpu(), inst.pred_boxes3d_global.tvec.cpu()
    return d


@pytest.mark.gpu
def test_nusc_tta_aggregation_exact_and_vs_emulating_oracle():
    from dd3d_b200.tta import NuscenesDD3DB200WithTTA
    from oracle.dd3d_oracle import DD3DOracle
    from dd3d_b200.synthetic import make_state_dict
    cfg, inputs = nusc_tta_case()
    model = _model(cfg)
    tta = NuscenesDD3DB200WithTTA(cfg, model)
    out = [_as_dict(o["instances"]) for o in tta(inputs)]
    assert tta.overflow_flags() == 0
    insts = tta(inputs)
    for o, x in zip(insts, inputs):
        inst = o["instances"]
        assert tuple(inst.image_size) == (x["height"], x["width"])
        assert not inst.has("locations") and not inst.has("fpn_levels")
    # (1) the aggregation step in isolation, on the wrapper's own merged per-image sets
    model.sample_aggregate_in_inference = False
    pre = [_as_dict(o["instances"]) for o in tta(inputs)]
    model.sample_aggregate_in_inference = True
    assert max(p["score3d"].shape[0] for p in pre) > 256  # beyond the one-CTA per-image BEV kernel
    assert sum(p["score3d"].shape[0] for p in pre[:6]) > 768  # beyond the one-CTA sample-aggregation kernel
    ref = NT.nusc_tta_forward(None, inputs, cfg, per_image=pre)
    assert sum(r["score3d"].shape[0] for r in ref) == NUSC_TTA["max_dets"]  # the per-call cap binds
    from oracle.dd3d_oracle import pose_of
    for got, r, x in zip(out, ref, inputs):
        assert torch.equal(got["score3d"], r["score3d"])
        assert torch.equal(got["attr"], r["attr"]) and torch.equal(got["speed"], r["speed"])
        if r["score3d"].numel():
            q64, t64 = NT.to_global_f64(r["quat"], r["tvec"], *pose_of(x))
            assert quat_dist(got["quat_global"].double(), q64).max().item() < 1e-5
            np.testing.assert_allclose(got["tvec_global"].double().numpy(), t64.numpy(), rtol=1e-5, atol=1e-4)
    # (2) the merged per-image sets vs the bf16-emulating oracle, matched by (class, rounded box)
    emu = DD3DOracle(cfg, make_state_dict(cfg), emulate_bf16=True)
    matched = total = 0
    for x, p in zip(inputs[:6], pre[:6]):
        e = NT.tta_forward(emu, x, cfg)
        n, m = p["score3d"].shape[0], e["score3d"].shape[0]
        assert abs(n - m) <= 0.1 * m

        def keys(box, cls):
            return [(int(c), ) + tuple(int(round(float(v) / 2.0)) for v in b) for b, c in zip(box, cls)]
        pos = {k: i for i, k in enumerate(keys(e["box2d"], e["cls"]))}
        pairs = [(i, pos[k]) for i, k in enumerate(keys(p["box2d"], p["cls"])) if k in pos]
        matched += len(pairs)
        total += m
        ia, ib = (torch.tensor(v) for v in zip(*pairs))
        assert rel_err(p["box2d"][ia], e["box2d"][ib], floor=16.0) < 0.1
        assert rel_err(p["depth"][ia], e["depth"][ib], floor=1.0) < 0.05
        assert rel_err(p["speed"][ia], e["speed"][ib], floor=1.0) < 0.1
        assert (p["attr"][ia] == e["attr"][ib]).float().mean().item() > 0.9
    assert matched >= 0.7 * total
    # (3) the whole path vs the fp32 reference golden, loosely (bf16 storage moves scores near the per-call cap)
    g = np.load(os.path.join(GOLDEN_DIR, "nusc_tta_v2_99.npz"))
    matched = total = 0
    for b, got in enumerate(out):
        kg = keys4(g[f"boxes{b}"], g[f"classes{b}"])
        pos = {k: i for i, k in enumerate(kg)}
        pairs = [(i, pos[k]) for i, k in enumerate(keys4(got["box2d"], got["cls"])) if k in pos]
        matched += len(pairs)
        total += len(kg)
        if pairs:
            ia, ib = (torch.tensor(v) for v in zip(*pairs))
            assert rel_err(got["score3d"][ia], g[f"scores_3d{b}"][ib], floor=0.05) < 0.2
            assert rel_err(got["tvec_global"][ia], g[f"tvec_global{b}"][ib], floor=1.0) < 0.1
    assert sum(o["score3d"].shape[0] for o in out) == total == NUSC_TTA["max_dets"]
    assert matched >= 0.5 * total, (matched, total)


def keys4(box, cls):
    return [(int(c), ) + tuple(int(round(float(v) / 4.0)) for v in b) for b, c in zip(box, cls)]


@pytest.mark.gpu
def test_nusc_tta_do_bev_nms_vs_reference_golden():
    """DO_BEV_NMS case of the wrapper vs the fp32 reference golden, loosely (bf16 storage)."""
    from dd3d_b200.tta import NuscenesDD3DB200WithTTA
    cfg, inputs = nusc_tta_case(do_bev_nms=True, samples=1)
    tta = NuscenesDD3DB200WithTTA(cfg, _model(cfg))
    out = [_as_dict(o["instances"]) for o in tta(inputs)]
    assert tta.overflow_flags() == 0
    g = np.load(os.path.join(GOLDEN_DIR, "nusc_tta_bev_v2_99.npz"))
    matched = total = 0
    for b, got in enumerate(out):
        n = g[f"scores_3d{b}"].shape[0]
        assert abs(got["score3d"].shape[0] - n) <= max(3, 0.15 * n)
        pos = {k: i for i, k in enumerate(keys4(g[f"boxes{b}"], g[f"classes{b}"]))}
        matched += sum(k in pos for k in keys4(got["box2d"], got["cls"]))
        total += n
    assert matched >= 0.6 * total, (matched, total)


@pytest.mark.gpu
@pytest.mark.parametrize("nusc", [False, True])
def test_tta_do_bev_nms_merged_step_exact(nusc):
    """DO_BEV_NMS: the merged-set BEV step (camera frame, per-detection intrinsics) == the oracle's bev_nms applied to the
    wrapper's own merged sets; the per-view BEV NMS inside the views' forwards is the existing kernel."""
    from dd3d_b200.tta import DD3DB200WithTTA, NuscenesDD3DB200WithTTA
    if nusc:
        cfg, inputs = nusc_tta_case(do_bev_nms=True)
        model = _model(cfg)
        model.sample_aggregate_in_inference = False
        tta = NuscenesDD3DB200WithTTA(cfg, model)
        run = lambda: [_as_dict(o["instances"]) for o in tta(inputs)]  # noqa: E731
    else:
        from oracle.gen_golden import tta_case
        cfg, x = tta_case()
        cfg.DD3D.INFERENCE.DO_BEV_NMS = True
        cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH = 0.05
        x["pose"] = ([0.9238795, 0.0, 0.3826834, 0.0], [3.0, -1.0, 2.0])
        model = _model(cfg)
        tta = DD3DB200WithTTA(cfg, model)
        run = lambda: [_as_dict(tta([x])[0]["instances"])]  # noqa: E731
    got = run()
    tta.merged_bev_nms_in_inference = False
    pre = run()
    tta.merged_bev_nms_in_inference = True
    assert tta.overflow_flags() == 0
    removed = 0
    for g, p in zip(got, pre):
        keep = NT.bev_nms_camera(p, cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH)
        removed += p["score3d"].shape[0] - keep.numel()
        assert torch.equal(g["score3d"], p["score3d"][keep])
        assert torch.equal(g["box2d"], p["box2d"][keep])
    assert removed > 0
