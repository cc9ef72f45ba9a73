"""GPU suite (-m gpu) for DD3D.IN_FEATURES: every case of oracle/in_features_oracle.py end to end against the emulating oracle
(bf16 and fp16, sparse box2d / box3d towers and sparse predictor on and off) and the reference's own fp32 forward, both
engine DO_BEV_NMS paths, DD3DB200WithTTA, the poisoned workspace and batch independence, and the FPN convs that no head reads
being absent."""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

import parity_lib as PL
from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_nusc_inputs, make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.in_features_oracle import IN_FEATURES_CASES, case_cfg, case_inputs
from util import quat_dist

pytestmark = pytest.mark.gpu

# The bounds of tests/test_fpn_width_gpu.py (BN heads).
_BOUNDS = {"box": 1.3e-2, "size": 2.6e-2, "depth": 8e-3, "score": 8e-3, "score3d": 8e-3}
_SPARSE = ("sparse_box3d", "sparse_tower", "sparse_box2d_tower")


def _inputs(case):
    if IN_FEATURES_CASES[case][2] == "NuscenesDD3D":
        return make_nusc_inputs(1, 128, 192, 1266.4)
    return case_inputs(case)


def _model(cfg, **opts):
    nusc = cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D"
    m = (NuscenesDD3DB200 if nusc else DD3DB200)(cfg).to("cuda")
    m.load_state_dict(make_state_dict(cfg))
    if nusc:
        m.sample_aggregate_in_inference = False  # per-image detections, as the oracle returns them
    for k, v in opts.items():
        m.set_engine_option(k, v)
    return m


@pytest.fixture
def _pair_tile():
    """The sparse towers run on the pair tile: force it, so that they run at these small shapes too."""
    L = lib.load()
    assert L.dd3d_set_conv_policy(b"pair_tile", 1) == 0
    yield
    L.dd3d_set_conv_policy(b"pair_tile", -1)


@functools.lru_cache(maxsize=None)
def _oracle(case, act_dtype):
    cfg = case_cfg(case, act_dtype=act_dtype)
    return DD3DOracle(cfg, make_state_dict(cfg), emulate=act_dtype, threads=1).forward(_inputs(case))


def _snap(out):
    return [torch.cat([o["instances"].pred_boxes.tensor, o["instances"].scores_3d[:, None], o["instances"].pred_boxes3d.quat,
                       o["instances"].pred_boxes3d.size, o["instances"].fpn_levels[:, None].float()], 1)
            .contiguous().view(torch.int32).cpu() for o in out]


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("sparse", [1, 0], ids=["sparse", "dense"])
@pytest.mark.parametrize("act_dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("case", list(IN_FEATURES_CASES))
def test_forward_vs_emulating_oracle(case, act_dtype, sparse, _pair_tile):
    cfg = case_cfg(case, act_dtype=act_dtype)
    model = _model(cfg, **{k: sparse for k in _SPARSE})
    inputs = _inputs(case)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    ref = _oracle(case, act_dtype)
    nl = len(IN_FEATURES_CASES[case][1])
    worst = {f: 0.0 for f in _BOUNDS}
    n = 0
    for b, (o, r) in enumerate(zip(out, ref)):
        lv = o["instances"].fpn_levels
        assert len(lv) == 0 or int(lv.max()) < nl  # the position, not the FPN index
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_oracle(r)
        rep, ia, ib = PL.compare_sets(a, e)  # keys include the level (the position)
        n += rep["n_ref"]
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        for f in _BOUNDS:
            if len(errs[f]):
                worst[f] = max(worst[f], float(errs[f].max()))
        if len(ia):
            assert quat_dist(a["quat"][ia], e["quat"][ib]).max() < 1e-1
    print(f"\n{case} {act_dtype} sparse={sparse}: {n} detections, launches {model.launches_per_forward()}, worst {worst}")
    assert n > 0
    for f, bound in _BOUNDS.items():
        assert worst[f] < bound, f"{f}: {worst[f]} >= {bound}"


@pytest.mark.parametrize("case", [c for c, v in IN_FEATURES_CASES.items() if v[2] == "DD3D"])
def test_forward_vs_reference_golden(case):
    g = np.load(os.path.join(GOLDEN_DIR, "golden_in_features.npz"))
    g = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(case + "/")}
    out = _model(case_cfg(case))(case_inputs(case))
    for b, o in enumerate(out):
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_golden(g, b)
        assert tuple(o["instances"].image_size) == tuple(g[f"image_size{b}"].tolist())
        rep, ia, ib = PL.compare_sets(a, e)
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        if len(ia):
            print(f"\n{case} image {b}: box {errs['box'].max():.3e} depth {errs['depth'].max():.3e}")
            assert errs["box"].max() < 1.6e-2
            assert errs["depth"].max() < 8e-3


# ------------------------------------------------------------------------------------------------ skipped FPN convs
def _ops(cfg, inputs):
    m = _model(cfg, **{k: 0 for k in _SPARSE})
    m(inputs)
    torch.cuda.synchronize()
    L = lib.load()
    n = L.dd3d_num_ops(m._handle)
    ws = L.dd3d_workspace_bytes(m._handle, len(inputs), 128, 192)
    return m, n, ws


@pytest.mark.parametrize("backbone,feats,absent,skipped", [
    ("v2_99", ["p3", "p4", "p5", "p6"], ["p0"], 2),  # fpn_lateral2 + fpn_output2
    ("dla34", ["p3", "p4", "p5", "p6"], ["p4"], 2),  # relu(P6) + top_block.p7
    ("dla34", ["p4"], ["p0", "p2", "p3", "p4"], 6),  # fpn_lateral3, fpn_output3 / 5, P6, relu(P6), P7
])
def test_unread_fpn_outputs_are_not_built(backbone, feats, absent, skipped):
    inputs = case_inputs("dla34_p4")
    _, n_all, ws_all = _ops(get_cfg(backbone), inputs)
    m, n, ws = _ops(get_cfg(backbone, in_features=feats), inputs)
    assert n == n_all - skipped, (n, n_all)
    assert ws < ws_all
    for l in range(5):
        name = f"p{l}"
        if name in absent:
            with pytest.raises(RuntimeError, match="not built"):
                m.get_tensor(name)
        else:
            assert m.get_tensor(name).shape[0] == len(inputs)
    for l in range(5):
        if l < len(feats):
            m.get_tensor(f"cls{l}")
        else:
            with pytest.raises(RuntimeError, match="unknown tensor"):
                m.get_tensor(f"cls{l}")


def test_setter_refusals_and_call_order():
    cfg = get_cfg("dla34")
    m = _model(cfg)
    h = m._engine()  # finalized
    L = lib.load()
    arr = lambda *v: (C.c_int32 * len(v))(*v)  # noqa: E731
    assert L.dd3d_set_in_features(h, arr(1, 2), 2) == -2  # DD3D_ERR_STATE after finalize
    d = lib.desc_from_cfg(cfg)
    h2 = C.c_void_p()
    assert L.dd3d_create(C.byref(d), C.byref(h2)) == 0
    try:
        assert L.dd3d_set_in_features(h2, arr(1, 1), 2) == -1
        assert b"repeated" in L.dd3d_last_error(h2)
        for v in ((5, ), (-1, ), (0, 1, 2, 3, 4, 0)):
            assert L.dd3d_set_in_features(h2, arr(*v), len(v)) == -1, v
        assert L.dd3d_set_in_features(h2, arr(0), 0) == -1
        assert L.dd3d_set_in_features(h2, arr(3, 0), 2) == 0
    finally:
        L.dd3d_destroy(h2)


def test_do_nms_off_holds_every_level_candidate():
    """Without the 2-D NMS every candidate of the L levels survives: the output buffer holds L * PRE_NMS_TOPK per image, and
    the engine returns as many candidates as the oracle's pre-NMS list holds, more than PRE_NMS_TOPK (no postprocess, which
    would drop the empty boxes)."""
    cfg = case_cfg("v2_99_p6_p3")
    cfg.DD3D.INFERENCE.DO_NMS = False
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.001  # p3 fills its PRE_NMS_TOPK, p6 adds its candidates
    topk = cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK
    m = _model(cfg)
    assert m._desc.out_cap == 2 * topk
    m.postprocess_in_inference = False
    out = m(case_inputs("v2_99_p6_p3"))
    assert m.overflow_flags() == 0
    _, inter = DD3DOracle(cfg, make_state_dict(cfg), emulate="bf16", threads=1).forward(
        case_inputs("v2_99_p6_p3"), return_intermediates=True)
    for o, r in zip(out, inter["pre_nms"]):
        n_pre = r["box2d"].shape[0]
        assert n_pre > topk
        assert len(o["instances"]) == n_pre
        assert int(o["instances"].fpn_levels.max()) == 1


# ------------------------------------------------------------------------------------------------ determinism
def test_poisoned_workspace_and_batch_independence():
    case = "v2_99_p6_p3"
    cfg = case_cfg(case)
    inputs = case_inputs(case)
    snaps = []
    for fill in (0x00, 0xFF):
        m = _model(cfg, workspace_fill=fill)
        snaps.append(_snap(m(inputs)))
        assert m.overflow_flags() == 0
        del m
    assert sum(len(s) for s in snaps[0]) > 0
    for a, b in zip(*snaps):
        assert torch.equal(a, b)
    m = _model(cfg)
    alone = _snap(m([inputs[0]]))[0]
    pair = _snap(m([inputs[0], inputs[0]]))
    assert torch.equal(alone, pair[0]) and torch.equal(alone, pair[1])


# ------------------------------------------------------------------------------------------------ engine DO_BEV_NMS
@pytest.mark.parametrize("path", [1, 2], ids=["one_cta", "multi_cta"])
def test_engine_bev_nms(path):
    """DO_BEV_NMS with and without the 2-D NMS on [p6, p3]: the BEV NMS op equals the reference BEV NMS
    (oracle/bev_nms_oracle.py) on the same engine's pre-BEV detections."""
    from oracle import bev_nms_oracle as BO
    from oracle.dd3d_oracle import DD3DOracle
    from test_bev_nms_large_gpu import BEV_THR, POSES, _inputs as bev_inputs
    cfg = get_cfg("dla34", in_features=["p6", "p3"])
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.03
    if path == 2:
        cfg.DD3D.INFERENCE.DO_NMS = False
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH = BEV_THR
    model = _model(cfg)
    assert lib.load().dd3d_bev_nms_path(C.byref(model._desc)) == path
    inputs = bev_inputs()
    out = model(inputs)
    assert model.last_overflow_flags == 0
    model.do_bev_nms = False
    model.postprocess_in_inference = False
    pre = model(inputs)
    removed, total = 0, 0
    for b, (o, q) in enumerate(zip(out, pre)):
        pi = q["instances"]
        assert int(pi.fpn_levels.max()) <= 1
        det = dict(quat=pi.pred_boxes3d.quat.cpu(), tvec=pi.pred_boxes3d.tvec.cpu(), size=pi.pred_boxes3d.size.cpu(),
                   score3d=pi.scores_3d.cpu(), cls=pi.pred_classes.cpu(), box2d=pi.pred_boxes.tensor.cpu())
        keep = BO.bev_nms_image(det, POSES[b][0], POSES[b][1], BEV_THR)
        removed += len(pi) - len(keep)
        total += len(pi)
        h, w = pi.image_size
        oh, ow = inputs[b].get("height", h), inputs[b].get("width", w)
        ref = DD3DOracle.postprocess({k: v[keep] for k, v in det.items()}, (h, w), (oh, ow))
        inst = o["instances"]
        assert len(inst) == ref["box2d"].shape[0]
        ka = np.lexsort((inst.pred_classes.cpu().numpy(), inst.scores_3d.cpu().numpy()))
        kb = np.lexsort((ref["cls"].numpy(), ref["score3d"].numpy()))
        assert torch.equal(inst.scores_3d.cpu()[ka], ref["score3d"][kb])
        assert torch.equal(inst.pred_classes.cpu()[ka], ref["cls"][kb])
        np.testing.assert_allclose(inst.pred_boxes.tensor.cpu().numpy()[ka], ref["box2d"].numpy()[kb], rtol=1e-6, atol=1e-4)
    assert total > 0 and removed > 0


# ------------------------------------------------------------------------------------------------ TTA
def test_tta_vs_emulating_oracle():
    """DD3DB200WithTTA on [p4, p5, p6, p7] against the bf16-emulating oracle's TTA, with tests/test_tta.py's matching rule and
    bounds; without the 2-D NMS the view capacity is 4 * PRE_NMS_TOPK."""
    from dd3d_b200.tta import DD3DB200WithTTA
    from oracle import tta_oracle as T
    from oracle.gen_golden import tta_case
    from util import rel_err
    cfg, x = tta_case()
    cfg.DD3D.IN_FEATURES = ["p4", "p5", "p6", "p7"]
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.01  # the fixture's 0.02 leaves no candidate without p3
    sd = make_state_dict(cfg)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    tta = DD3DB200WithTTA(cfg, model)
    inst = tta([x])[0]["instances"]
    assert tta.overflow_flags() == 0
    assert tuple(inst.image_size) == (x["height"], x["width"])
    emu = T.tta_forward(DD3DOracle(cfg, sd, emulate="bf16"), x, cfg.TEST.AUG.MIN_SIZES, cfg.TEST.AUG.MAX_SIZE,
                        cfg.TEST.AUG.FLIP, cfg.TEST.IMS_PER_BATCH, cfg.DD3D.FCOS2D.INFERENCE.NMS_THRESH)
    n, m = len(inst), emu["score3d"].shape[0]
    assert m > 0 and abs(n - m) <= 0.1 * m

    def keys(box, cls):
        return [(int(c), ) + tuple(int(round(float(v) / 2.0)) for v in b) for b, c in zip(box, cls)]
    ka, kb = keys(inst.pred_boxes.tensor.cpu(), inst.pred_classes.cpu()), keys(emu["box2d"], emu["cls"])
    pos = {k: i for i, k in enumerate(kb)}
    pairs = [(i, pos[k]) for i, k in enumerate(ka) if k in pos]
    assert len(pairs) >= 0.7 * m
    ia, ib = (torch.tensor(p) for p in zip(*pairs))
    assert rel_err(inst.pred_boxes.tensor.cpu()[ia], emu["box2d"][ib], floor=16.0) < 0.1
    assert rel_err(inst.scores_3d.cpu()[ia], emu["score3d"][ib], floor=0.05) < 0.2
    assert rel_err(inst.pred_boxes3d.depth.cpu()[ia].reshape(-1), emu["depth"][ib], floor=1.0) < 0.05
    assert quat_dist(inst.pred_boxes3d.quat.cpu()[ia], emu["quat"][ib]).median().item() < 0.05
    model.do_nms = False
    tta_large = DD3DB200WithTTA(cfg, model)
    tta_large([x])
    assert tta_large.overflow_flags() == 0
    assert model._desc.out_cap >= 4 * cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK
