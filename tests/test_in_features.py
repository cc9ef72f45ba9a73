"""CPU suite for DD3D.IN_FEATURES (the FPN outputs the heads run on): parameter inventory against the reference at every case of
oracle/in_features_oracle.py, the oracle against the reference's own forward, the unchanged default, the refusals and the new
C symbol."""
import ctypes
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import fpn_output_names, in_feature_levels, level_strides, param_specs
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.gen_golden import CASES, inventory_digest
from oracle.in_features_oracle import IN_FEATURES_CASES, case_cfg, case_inputs
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_CASES = [c for c, v in IN_FEATURES_CASES.items() if v[2] == "DD3D"]


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "in_features_inventory.json")) as f:
        return json.load(f)


def _mirror(cfg):
    return (NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200)(cfg)


@pytest.mark.parametrize("case", list(IN_FEATURES_CASES))
def test_param_specs_match_reference_inventory(case):
    shapes = {k: shape for k, (shape, _) in param_specs(case_cfg(case)).items()}
    assert inventory_digest(shapes) == _inventory()[case]


@pytest.mark.parametrize("case", list(IN_FEATURES_CASES))
def test_model_state_dict_keys_equal_generator_keys(case):
    cfg = case_cfg(case)
    sd = _mirror(cfg).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == _inventory()[case]
    assert set(sd) == set(make_state_dict(cfg))


@pytest.mark.parametrize("backbone", ["dla34", "v2_99"])
def test_per_level_modules_follow_the_list(backbone):
    """One tower BN and one Scale per listed level; scales_depth / offsets_depth keep one per MEAN_DEPTH_PER_LEVEL entry; the
    FPN keeps every conv (the reference still builds and runs all of them)."""
    feats = fpn_output_names(get_cfg(backbone))[1:3]
    cfg = get_cfg(backbone, in_features=feats, meta_arch="DD3D")
    cfg.DD3D.FCOS3D.PER_LEVEL_PREDICTORS = True
    s = param_specs(cfg)
    d = param_specs(get_cfg(backbone))
    assert [k for k in d if k.startswith("backbone.")] == [k for k in s if k.startswith("backbone.")]
    assert {int(k.split(".")[-2]) for k in s if ".cls_tower.0.norm." in k} == {0, 1}
    for name in ("scales_box2d_reg", "scales_proj_ctr", "scales_size", "scales_conf", "box3d_quat"):
        assert len({k.split(".")[2] for k in s if f".{name}." in k}) == 2, name
    for name in ("scales_depth", "offsets_depth"):
        assert len({k.split(".")[2] for k in s if f".{name}." in k}) == 5, name
    assert s["fcos3d_head.mean_depth_per_level"][0] == (5, )


@pytest.mark.parametrize("backbone", ["dla34", "v2_99"])
def test_default_is_every_fpn_output_in_order(backbone):
    """IN_FEATURES unset, empty or all five in order: the inventory, strides and generator stream of the parent."""
    dataset = CASES[backbone][0]
    with open(os.path.join(GOLDEN_DIR, "reference_live.json")) as f:
        digest = json.load(f)["inventory"][backbone]
    names = fpn_output_names(get_cfg(backbone))
    base = make_state_dict(get_cfg(backbone, dataset))
    for feats in (None, [], names):
        cfg = get_cfg(backbone, dataset, in_features=feats)
        assert in_feature_levels(cfg) == [0, 1, 2, 3, 4]
        assert level_strides(cfg) == ([8, 16, 32, 64, 128] if backbone == "dla34" else [4, 8, 16, 32, 64])
        assert inventory_digest({k: shape for k, (shape, _) in param_specs(cfg).items()}) == digest
        assert lib.in_features_from_cfg(cfg) is None  # no dd3d_set_in_features call: the parent's engine
        sd = make_state_dict(cfg)
        assert list(sd) == list(base) and all(np.array_equal(sd[k].numpy(), base[k].numpy()) for k in sd)


def test_strides_and_capacity_follow_the_list():
    cfg = get_cfg("v2_99", in_features=["p6", "p3"])
    assert in_feature_levels(cfg) == [4, 1]
    assert level_strides(cfg) == [64, 8]
    cfg.DD3D.INFERENCE.DO_NMS = False
    assert lib.max_candidates(cfg) == 2 * cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK
    assert lib.desc_from_cfg(cfg).out_cap == 2000
    arr, n = lib.in_features_from_cfg(cfg)
    assert n == 2 and list(arr) == [4, 1]


@pytest.mark.parametrize("case", DD3D_CASES)
def test_oracle_matches_reference_golden(case):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/in_features_oracle.py --golden): detections, fpn_levels
    (the position) and the 3-D fields, whose depth takes scales_depth / offsets_depth by position."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_in_features.npz"))
    cfg = case_cfg(case)
    out = DD3DOracle(cfg, make_state_dict(cfg)).forward(case_inputs(case))
    total = 0
    for b, o in enumerate(out):
        p = f"{case}/"
        assert o["box2d"].shape[0] == g[f"{p}boxes{b}"].shape[0]
        total += o["box2d"].shape[0]
        assert np.array_equal(o["cls"].numpy(), g[f"{p}classes{b}"])
        assert np.array_equal(o["level"].numpy(), g[f"{p}levels{b}"])
        assert g[f"{p}levels{b}"].max(initial=0) < len(IN_FEATURES_CASES[case][1])
        np.testing.assert_allclose(o["loc"].numpy(), g[f"{p}locations{b}"], rtol=0, atol=0)
        np.testing.assert_allclose(o["box2d"].numpy(), g[f"{p}boxes{b}"], rtol=1e-4, atol=1e-3)
        np.testing.assert_allclose(o["score"].numpy(), g[f"{p}scores{b}"], rtol=1e-4)
        np.testing.assert_allclose(o["score3d"].numpy(), g[f"{p}scores_3d{b}"], rtol=1e-4)
        if o["box2d"].shape[0]:
            assert quat_dist(o["quat"], g[f"{p}quat{b}"]).max() < 1e-4
        np.testing.assert_allclose(o["depth"].numpy(), g[f"{p}depth{b}"].reshape(-1), rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(o["tvec"].numpy(), g[f"{p}tvec{b}"], rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(o["size"].numpy(), g[f"{p}size{b}"], rtol=1e-4)
    assert total > 0


def test_depth_offset_is_taken_by_position():
    """[p6, p3]: the p3 head (position 1) uses offsets_depth.1 / scales_depth.1 -- not entry 1 of the FPN index (p3 is FPN
    output 0 of DLA-34).  Moving offsets_depth.1 moves exactly the position-1 pre-NMS depths."""
    cfg = case_cfg("dla34_p6_p3")
    cfg.DD3D.FCOS3D.MIN_DEPTH, cfg.DD3D.FCOS3D.MAX_DEPTH = -1e6, 1e6  # no clamp: the offset shows through unchanged
    sd = make_state_dict(cfg)
    inputs = case_inputs("dla34_p6_p3")
    _, a = DD3DOracle(cfg, sd).forward(inputs, return_intermediates=True)
    sd2 = dict(sd)
    sd2["fcos3d_head.offsets_depth.1.bias"] = sd["fcos3d_head.offsets_depth.1.bias"] + 7.0
    _, b = DD3DOracle(cfg, sd2).forward(inputs, return_intermediates=True)
    for da, db in zip(a["pre_nms"], b["pre_nms"]):
        on = da["level"] == 1
        assert on.any()
        assert np.array_equal(da["level"].numpy(), db["level"].numpy())
        assert np.array_equal(da["depth"][~on].numpy(), db["depth"][~on].numpy())
        assert not np.array_equal(da["depth"][on].numpy(), db["depth"][on].numpy())


@pytest.mark.parametrize("backbone,feats,missing", [("dla34", ["p2", "p3"], "p2"), ("v2_99", ["p3", "p7"], "p7"),
                                                     ("dla34", ["res4"], "res4")])
def test_unknown_name_raises_key_error(backbone, feats, missing):
    cfg = get_cfg(backbone, in_features=feats)
    with pytest.raises(KeyError, match=missing):
        param_specs(cfg)
    with pytest.raises(KeyError, match=missing):
        DD3DB200(cfg)


def test_repeated_level_raises_not_implemented():
    cfg = get_cfg("v2_99", in_features=["p3", "p4", "p3"])
    with pytest.raises(NotImplementedError, match="'p3'"):
        DD3DB200(cfg)


def test_new_symbol_is_declared_and_exported():
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"int dd3d_set_in_features\(dd3d_handle h, const int32_t\* h_fpn_levels, int n\);", hdr)
    assert hasattr(lib.load(), "dd3d_set_in_features")


def test_set_in_features_without_a_handle_is_refused():
    levels = (ctypes.c_int32 * 2)(1, 2)
    assert lib.load().dd3d_set_in_features(None, levels, 2) == -1
