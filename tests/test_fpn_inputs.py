"""CPU suite for FE.FPN.IN_FEATURES (the backbone outputs the FPN reads): parameter inventory against the reference at every case of
oracle/fpn_inputs_oracle.py, the oracle against the reference's own forward, the names / strides / head levels each list gives,
the refusals with the reference's exception types, the unchanged default and the new C symbol."""
import builtins
import ctypes
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import (check_fpn_inputs, fpn_inputs, fpn_output_names, in_feature_levels, level_strides, param_specs,
                            size_divisibility)
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.fpn_inputs_oracle import (FPN_INPUTS_CASES, FPN_INPUTS_REFUSED, case_cfg, case_inputs, refused_cfg,
                                      refused_key)
from oracle.gen_golden import inventory_digest
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_CASES = [c for c, v in FPN_INPUTS_CASES.items() if v[3] == "DD3D"]


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "fpn_inputs_inventory.json")) as f:
        return json.load(f)


def _mirror(cfg):
    return (NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200)(cfg)


@pytest.mark.parametrize("case", list(FPN_INPUTS_CASES))
def test_param_specs_match_reference_inventory(case):
    cfg = case_cfg(case)
    shapes = {k: shape for k, (shape, _) in param_specs(cfg).items()}
    assert inventory_digest(shapes) == _inventory()[case]
    sd = _mirror(cfg).state_dict()
    assert set(sd) == set(make_state_dict(cfg)) == set(shapes)


@pytest.mark.parametrize("backbone,fpn_in,names,strides", [
    ("dla34", ["level4", "level5"], ["p4", "p5", "p6", "p7"], [16, 32, 64, 128]),
    ("dla34", ["level2", "level3", "level4", "level5"], ["p2", "p3", "p4", "p5", "p6", "p7"], [4, 8, 16, 32, 64, 128]),
    ("dla_x_60", ["level5"], ["p5", "p6", "p7"], [32, 64, 128]),
    ("v2_99", ["stage3", "stage4", "stage5"], ["p3", "p4", "p5", "p6"], [8, 16, 32, 64]),
    ("v2_99", ["stem", "stage3", "stage4", "stage5"], ["p2", "p3", "p4", "p5", "p6"], [4, 8, 16, 32, 64]),
    ("v2_19_slim_dw", ["stage5"], ["p5", "p6"], [32, 64]),
])
def test_names_strides_and_levels_follow_the_list(backbone, fpn_in, names, strides):
    cfg = get_cfg(backbone, fpn_in_features=fpn_in)
    assert cfg.FE.BACKBONE.OUT_FEATURES == fpn_in and cfg.FE.FPN.IN_FEATURES == fpn_in
    assert fpn_output_names(cfg) == names
    assert size_divisibility(cfg) == (128 if backbone.startswith("dla") else 64)
    specs = param_specs(cfg)
    assert [k for k in specs if re.fullmatch(r"backbone\.fpn_lateral\d\.weight", k)] == \
        [f"backbone.fpn_lateral{n[1:]}.weight" for n in names[:len(fpn_in)]]
    if len(names) > 5:  # DLA level2..5: the heads take at most five of the six outputs
        with pytest.raises(NotImplementedError, match="6 head levels"):
            check_fpn_inputs(cfg)
        cfg = get_cfg(backbone, fpn_in_features=fpn_in, in_features=names[:5])
        assert in_feature_levels(cfg) == [0, 1, 2, 3, 4]
        assert level_strides(cfg) == strides[:5]
        assert list(lib.in_features_from_cfg(cfg)[0]) == [0, 1, 2, 3, 4]  # not "every output": sent to the engine
    else:
        assert in_feature_levels(cfg) == list(range(len(names)))
        assert level_strides(cfg) == strides
        assert lib.in_features_from_cfg(cfg) is None
    check_fpn_inputs(cfg)
    arr, n = lib.fpn_inputs_from_cfg(cfg)
    assert list(arr) == [lib.FPN_IN_STEM if f == "stem" else int(f[-1]) for f in fpn_in] and n == len(fpn_in)
    cfg = get_cfg(backbone, fpn_in_features=fpn_in, in_features=[names[-1], names[0]])
    assert level_strides(cfg) == [strides[-1], strides[0]]


@pytest.mark.parametrize("case", DD3D_CASES)
def test_oracle_matches_reference_golden(case):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/fpn_inputs_oracle.py --golden)."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_fpn_inputs.npz"))
    cfg = case_cfg(case)
    assert list(g[f"{case}/fpn_outputs"]) == fpn_output_names(cfg)
    out = DD3DOracle(cfg, make_state_dict(cfg)).forward(case_inputs(case))
    total = 0
    for b, o in enumerate(out):
        p = f"{case}/"
        assert o["box2d"].shape[0] == g[f"{p}boxes{b}"].shape[0]
        total += o["box2d"].shape[0]
        assert np.array_equal(o["cls"].numpy(), g[f"{p}classes{b}"])
        assert np.array_equal(o["level"].numpy(), g[f"{p}levels{b}"])
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


@pytest.mark.parametrize("backbone,out,fpn_in", FPN_INPUTS_REFUSED)
def test_lists_the_reference_cannot_build_raise_its_error(backbone, out, fpn_in):
    """Unknown outputs, strides that do not double, no p5 for the top block: the reference's exception type and message
    (recorded from its own DD3D by oracle/fpn_inputs_oracle.py --golden), raised at construction."""
    name, msg = _inventory()["refused"][refused_key(backbone, out, fpn_in)]
    with pytest.raises(getattr(builtins, name)) as e:
        DD3DB200(refused_cfg(backbone, out, fpn_in))
    assert str(e.value) == msg


@pytest.mark.parametrize("backbone,fpn_in,in_features,match", [
    ("dla34", ["level1", "level2", "level3", "level4", "level5"], ["p1", "p2"], r"\['level1'\] below stride 4"),
    ("dla34", ["level0", "level1", "level2", "level3", "level4", "level5"], ["p3"], r"\['level0', 'level1'\] below stride 4"),
    ("dla34", ["level2", "level3", "level4", "level5"], None, "6 head levels"),
])
def test_engine_refusals_are_not_implemented(backbone, fpn_in, in_features, match):
    cfg = get_cfg(backbone, fpn_in_features=fpn_in, in_features=in_features)
    param_specs(cfg)  # the reference builds these
    with pytest.raises(NotImplementedError, match=match):
        DD3DB200(cfg)


@pytest.mark.parametrize("backbone", ["dla34", "v2_99", "dla_x_46_c", "v2_19_slim_dw"])
def test_default_list_is_the_parent_graph(backbone):
    """The builder's list, given or not: the same inventory order, generator stream and descs, and no dd3d_set_fpn_inputs call."""
    base_cfg = get_cfg(backbone)
    default = [n for n, _ in fpn_inputs(base_cfg)]
    assert default == list(base_cfg.FE.BACKBONE.OUT_FEATURES)
    cfg = get_cfg(backbone, fpn_in_features=default)
    assert list(param_specs(cfg).items()) == list(param_specs(base_cfg).items())
    a, b = make_state_dict(cfg), make_state_dict(base_cfg)
    assert list(a) == list(b) and all(np.array_equal(a[k].numpy(), b[k].numpy()) for k in a)
    assert bytes(lib.desc_from_cfg(cfg)) == bytes(lib.desc_from_cfg(base_cfg))
    assert bytes(lib.layout_from_cfg(cfg)) == bytes(lib.layout_from_cfg(base_cfg))
    assert lib.fpn_inputs_from_cfg(cfg) is None and lib.in_features_from_cfg(cfg) is None


def test_new_symbol_is_declared_and_exported():
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"int dd3d_set_fpn_inputs\(dd3d_handle h, const int32_t\* h_inputs, int n\);", hdr)
    assert re.search(r"#define DD3D_FPN_IN_STEM 1\b", hdr) and re.search(r"#define DD3D_FPN_MAX_OUTPUTS 6\b", hdr)
    assert hasattr(lib.load(), "dd3d_set_fpn_inputs")


def test_set_fpn_inputs_without_a_handle_is_refused():
    arr = (ctypes.c_int32 * 2)(4, 5)
    assert lib.load().dd3d_set_fpn_inputs(None, arr, 2) == -1
    assert lib.load().dd3d_set_fpn_inputs(None, None, 2) == -1
