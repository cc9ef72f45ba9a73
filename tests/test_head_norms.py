"""CPU suite for the FPN / FCOS head structure keys (FCOS2D.NORM, FCOS3D.NORM, FE.FPN.NORM, the tower depths and
FE.FPN.FUSE_TYPE): parameter inventory against the reference, the oracle against the reference's own forward, the default
layout's bit-identity with DD3DOracle, the cfg -> dd3d_layout_desc round trip and the refusals."""
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import param_specs
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.gen_golden import inventory_digest
from oracle.head_norm_oracle import HEAD_NORM_CASES, HeadNormOracle, case_cfg, case_inputs
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CASES = list(HEAD_NORM_CASES)


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "head_norms_inventory.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", CASES)
def test_param_specs_match_reference_inventory(case):
    shapes = {k: shape for k, (shape, _) in param_specs(case_cfg(case)).items()}
    assert inventory_digest(shapes) == _inventory()[case]


@pytest.mark.parametrize("case", CASES)
def test_model_state_dict_keys_equal_generator_keys(case):
    cfg = case_cfg(case)
    sd = DD3DB200(cfg).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == _inventory()[case]
    assert set(sd) == set(make_state_dict(cfg))


def test_norm_keys_of_each_mode():
    """GN: one affine per conv, no running stats; SyncBN: one BN per conv (with num_batches_tracked); "": conv biases."""
    s = param_specs(case_cfg("dla34_gn"))
    assert s["fcos2d_head.cls_tower.0.norm.weight"][1] == "gn_w" and "fcos2d_head.cls_tower.0.norm.running_mean" not in s
    assert s["backbone.fpn_lateral3.norm.bias"][1] == "gn_b"
    s = param_specs(case_cfg("dla34_syncbn_depth"))
    assert "fcos2d_head.cls_tower.0.norm.num_batches_tracked" in s and "fcos2d_head.cls_tower.0.norm.0.weight" not in s
    assert "fcos2d_head.cls_tower.2.weight" not in s and "fcos2d_head.box2d_tower.2.weight" in s
    assert "fcos3d_head.box3d_tower.0.norm.4.num_batches_tracked" in s and "fcos3d_head.box3d_tower.1.weight" not in s
    assert "backbone.fpn_output3.norm.num_batches_tracked" in s
    s = param_specs(case_cfg("dla34_none"))
    assert "fcos2d_head.cls_tower.0.bias" in s and "backbone.fpn_output3.bias" in s
    assert not any(".norm" in k and ("tower" in k or "fpn_" in k) for k in s)
    s = param_specs(case_cfg("dla34_no_towers"))
    assert not any("_tower." in k for k in s)


@pytest.mark.parametrize("backbone", ["dla34", "v2_99"])
def test_defaults_keep_the_inventory_and_generator_stream(backbone):
    """The default layout's keys, order and generated tensors do not change with the new keys (pinned by the parent's
    inventory and golden tests as well)."""
    cfg = get_cfg(backbone, "kitti_3d")
    specs = list(param_specs(cfg))
    towers = [k for k in specs if "_tower." in k]
    assert len([k for k in towers if k.endswith(".weight") and ".norm" not in k]) == 12
    assert all(re.search(r"_tower\.\d\.(weight|norm\.\d\.)", k) for k in towers)
    assert not any(k.startswith("backbone.fpn_") and k.endswith("num_batches_tracked") for k in specs)


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_golden(case):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/head_norm_oracle.py --golden), the bounds of the V2-99 and
    VoVNet fixtures."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_head_norms.npz"))
    cfg = case_cfg(case)
    out = HeadNormOracle(cfg, make_state_dict(cfg)).forward(case_inputs(case))
    total = 0
    for b, o in enumerate(out):
        p = f"{case}/"
        assert o["box2d"].shape[0] == g[f"{p}boxes{b}"].shape[0]
        total += o["box2d"].shape[0]
        assert np.array_equal(o["cls"].numpy(), g[f"{p}classes{b}"])
        assert np.array_equal(o["level"].numpy(), g[f"{p}levels{b}"])
        np.testing.assert_allclose(o["box2d"].numpy(), g[f"{p}boxes{b}"], rtol=1e-4, atol=1e-3)
        np.testing.assert_allclose(o["score"].numpy(), g[f"{p}scores{b}"], rtol=1e-4)
        np.testing.assert_allclose(o["score3d"].numpy(), g[f"{p}scores_3d{b}"], rtol=1e-4)
        if o["box2d"].shape[0]:
            assert quat_dist(o["quat"], g[f"{p}quat{b}"]).max() < 1e-4
        np.testing.assert_allclose(o["tvec"].numpy(), g[f"{p}tvec{b}"], rtol=1e-3, atol=1e-3)
        np.testing.assert_allclose(o["size"].numpy(), g[f"{p}size{b}"], rtol=1e-4)
    assert total > 0


@pytest.mark.parametrize("backbone", ["dla34", "v2_99"])
def test_head_norm_oracle_is_dd3d_oracle_on_defaults(backbone):
    from oracle.dd3d_oracle import DD3DOracle
    cfg = get_cfg(backbone, "nuscenes")
    sd = make_state_dict(cfg)
    inputs = case_inputs("dla34_gn")
    a, ia = DD3DOracle(cfg, sd, emulate="bf16", threads=1).forward(inputs, return_intermediates=True)
    b, ib = HeadNormOracle(cfg, sd, emulate="bf16", threads=1).forward(inputs, return_intermediates=True)
    assert all(x.equal(y) for x, y in zip(ia["features"], ib["features"]))
    for k, v in ia["maps"].items():
        assert all(x.equal(y) for x, y in zip(v, ib["maps"][k])), k
    for x, y in zip(a, b):
        assert all(x[k].equal(y[k]) for k in x)


def test_layout_round_trip():
    d = lib.layout_from_cfg(get_cfg("dla34", "kitti_3d"))
    assert (d.fcos2d_norm, d.fcos3d_norm, d.fpn_norm) == (lib.NORM_BN_PER_LEVEL, lib.NORM_BN_PER_LEVEL, lib.NORM_BN_SHARED)
    assert (d.num_cls_convs, d.num_box2d_convs, d.num_box3d_convs, d.fpn_fuse_avg) == (4, 4, 4, 0)
    d = lib.layout_from_cfg(case_cfg("v2_99_gn_avg"))
    assert (d.fcos2d_norm, d.fcos3d_norm, d.fpn_norm, d.fpn_fuse_avg) == (lib.NORM_GN,) * 3 + (1, )
    d = lib.layout_from_cfg(case_cfg("dla34_none"))
    assert (d.fcos2d_norm, d.fcos3d_norm, d.fpn_norm) == (lib.NORM_NONE, ) * 3
    d = lib.layout_from_cfg(case_cfg("dla34_syncbn_depth"))
    assert (d.fcos2d_norm, d.fcos3d_norm, d.fpn_norm) == (lib.NORM_BN_SHARED, lib.NORM_BN_PER_LEVEL, lib.NORM_BN_SHARED)
    assert (d.num_cls_convs, d.num_box2d_convs, d.num_box3d_convs) == (2, 3, 1)
    d = lib.layout_from_cfg(case_cfg("dla34_no_towers"))
    assert (d.num_cls_convs, d.num_box2d_convs, d.num_box3d_convs, d.fpn_fuse_avg) == (0, 0, 0, 1)


def test_header_matches_python_mirror():
    import ctypes
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    for name, val in (("BN_PER_LEVEL", lib.NORM_BN_PER_LEVEL), ("BN_SHARED", lib.NORM_BN_SHARED), ("GN", lib.NORM_GN),
                      ("NONE", lib.NORM_NONE)):
        assert re.search(rf"DD3D_NORM_{name} = {val}\b", hdr), name
    body = hdr[hdr.index("typedef struct dd3d_layout_desc {"):]
    body = body[:body.index("} dd3d_layout_desc;")]
    assert re.findall(r"int32_t (\w+);", body) == [f for f, _ in lib.LayoutDesc._fields_]
    assert ctypes.sizeof(lib.LayoutDesc) == 4 * 7


def test_refusals():
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.DD3D.FCOS2D.NORM = "NaiveGN"
    with pytest.raises(KeyError):
        DD3DB200(cfg)
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.FE.FPN.NORM = "LN"
    with pytest.raises(KeyError):
        DD3DB200(cfg)
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.DD3D.FCOS3D.NORM = "GroupNorm"
    cfg.DD3D.FCOS3D.NUM_CONVS = 0  # the reference looks the norm up only per conv; the engine refuses it regardless
    with pytest.raises(KeyError):
        DD3DB200(cfg)
    for key in ("FCOS2D", "FCOS3D"):
        cfg = get_cfg("dla34", "kitti_3d")
        cfg.DD3D[key].USE_DEFORMABLE = True
        with pytest.raises(ValueError, match="Not supported yet."):
            DD3DB200(cfg)


def test_engine_refuses_bad_layouts_before_the_device():
    """dd3d_set_layout checks its values on the host; without a handle it is refused outright."""
    import ctypes as C
    L = lib.load()
    d = lib.layout_from_cfg(get_cfg("dla34", "kitti_3d"))
    assert L.dd3d_set_layout(None, C.byref(d)) == -1
    assert L.dd3d_set_layout(None, None) == -1
