"""CPU suite for FE.BACKBONE.NORM: the parameter inventory against the reference's for each (backbone, norm) case, the
reference's errors at DD3DB200(cfg), strict loading of BN / SyncBN checkpoints, the oracle against the reference's own forward,
and the shipped configs' inventory and synthetic stream."""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import ARCH_KEYS, param_specs
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.backbone_norm_oracle import BACKBONE_NORM_CASES, case_cfg, case_inputs
from oracle.dd3d_oracle import DD3DOracle
from oracle.gen_golden import inventory_digest
from util import quat_dist

CASES = list(BACKBONE_NORM_CASES)


def _cfg(backbone, norm):
    cfg = get_cfg(backbone, "kitti_3d")
    cfg.FE.BACKBONE.NORM = norm
    return cfg


@pytest.mark.parametrize("case", CASES)
def test_param_specs_match_reference_inventory(case):
    with open(os.path.join(GOLDEN_DIR, "backbone_norms_inventory.json")) as f:
        want = json.load(f)[case]
    shapes = {k: shape for k, (shape, _) in param_specs(case_cfg(case)).items()}
    assert inventory_digest(shapes) == want
    sd = DD3DB200(case_cfg(case)).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == want


def test_norm_keys_of_each_mode():
    """BN / SyncBN: BN keys with num_batches_tracked; FrozenBN: without; GN: an affine only; "": a bias on every DLA conv."""
    bn = param_specs(_cfg("dla34", "BN"))
    nbt = [k for k in bn if k.startswith("backbone.bottom_up") and k.endswith("num_batches_tracked")]
    assert len(nbt) == 37 and "backbone.bottom_up.base_layer.norm.num_batches_tracked" in bn
    assert len([k for k in param_specs(_cfg("v2_99", "SyncBN")) if k.startswith("backbone.bottom_up") and
                k.endswith("num_batches_tracked")]) == 99
    none = param_specs(_cfg("dla34", ""))
    assert none["backbone.bottom_up.base_layer.bias"] == ((16, ), "bias:relu")
    assert none["backbone.bottom_up.level2.tree1.conv2.bias"] == ((64, ), "bias:linear")
    assert not any(k.startswith("backbone.bottom_up") and ".norm" in k for k in none)
    assert len([k for k in none if k.startswith("backbone.bottom_up") and k.endswith(".bias")]) == 37
    gn = param_specs(_cfg("v2_39", "GN"))
    assert gn["backbone.bottom_up.stem.stem_1/norm.weight"] == ((64, ), "gn_w")
    assert not any(k.startswith("backbone.bottom_up") and "running" in k for k in gn)
    assert len([k for k in gn if k.startswith("backbone.bottom_up") and k.endswith("norm.weight")]) == 39
    assert len([k for k in param_specs(_cfg("v2_19_dw", "GN")) if k.startswith("backbone.bottom_up") and
                k.endswith("norm.weight")]) == 23


@pytest.mark.parametrize("backbone,norm,exc,msg", [
    ("dla34", "GN", ValueError, r"num_channels \(16\) must be divisible by num_groups \(32\)"),
    ("v2_19_slim", "GN", ValueError, r"num_channels \(112\) must be divisible by num_groups \(32\)"),
    ("v2_19_slim_dw", "GN", ValueError, r"num_channels \(112\) must be divisible by num_groups \(32\)"),
    ("v2_39", "", TypeError, "'NoneType' object is not callable"),
    ("v2_99", "", TypeError, "'NoneType' object is not callable"),
    ("dla34", "NaiveSyncBN", KeyError, "NaiveSyncBN"),
    ("v2_57", "LN", KeyError, "LN"),
])
def test_reference_errors_at_construction(backbone, norm, exc, msg):
    with pytest.raises(exc, match=msg):
        DD3DB200(_cfg(backbone, norm))


@pytest.mark.parametrize("backbone", ["v2_19", "v2_19_dw", "v2_39", "v2_57", "v2_99"])
def test_gn_vovnet_builds(backbone):
    """Every non-slim VoVNet takes GroupNorm(32, C): its layout asks the engine for the GN backbone."""
    assert DD3DB200(_cfg(backbone, "GN"))._backbone_norm == lib.NORM_GN


@pytest.mark.parametrize("backbone,norm", [("dla34", "BN"), ("dla34", "SyncBN"), ("v2_99", "BN"), ("v2_19_slim_dw", "SyncBN")])
def test_bn_checkpoint_loads_strictly_with_the_frozen_values(backbone, norm):
    """A BatchNorm2d-keyed state_dict loads strictly.  Its synthetic tensors are the FrozenBN ones (num_batches_tracked draws
    nothing from the generator), so the two checkpoints hold the same values."""
    cfg = _cfg(backbone, norm)
    sd = make_state_dict(cfg)
    frozen = make_state_dict(get_cfg(backbone, "kitti_3d"))
    extra = set(sd) - set(frozen)
    assert extra and all(k.endswith("num_batches_tracked") for k in extra) and set(frozen) <= set(sd)
    assert all(torch.equal(frozen[k], sd[k]) for k in frozen)
    res = DD3DB200(cfg).load_state_dict(sd)
    assert res.missing_keys == [] and res.unexpected_keys == []
    with pytest.raises(RuntimeError, match="unexpected"):
        DD3DB200(get_cfg(backbone, "kitti_3d")).load_state_dict(sd)


@pytest.mark.parametrize("backbone", ARCH_KEYS)
def test_backbone_norm_mapping(backbone):
    assert DD3DB200(get_cfg(backbone, "kitti_3d"))._backbone_norm == lib.NORM_BN_SHARED
    for norm in ("BN", "SyncBN"):
        assert DD3DB200(_cfg(backbone, norm))._backbone_norm == lib.NORM_BN_SHARED
    if backbone == "dla34":
        assert DD3DB200(_cfg(backbone, ""))._backbone_norm == lib.NORM_NONE


def test_engine_refuses_without_a_handle():
    assert lib.load().dd3d_set_backbone_norm(None, lib.NORM_NONE) == -1


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_golden(case):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/backbone_norm_oracle.py --golden)."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_backbone_norms.npz"))
    cfg = case_cfg(case)
    out = DD3DOracle(cfg, make_state_dict(cfg)).forward(case_inputs(case))
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


@pytest.mark.parametrize("backbone", ["dla34", "v2_99", "v2_19_slim_dw"])
def test_shipped_configs_keep_inventory_and_stream(backbone):
    """FrozenBN (the shipped experiments) keeps the parent's keys: no num_batches_tracked and no conv bias in the backbone,
    and the state_dict generator draws the same tensors in the same order (golden tests pin the values)."""
    cfg = get_cfg(backbone, "nuscenes")
    specs = param_specs(cfg)
    bb = [k for k in specs if k.startswith("backbone.bottom_up")]
    assert not any(k.endswith("num_batches_tracked") for k in bb)
    assert all(specs[k][1] != "bias:relu" and specs[k][1] != "bias:linear" for k in bb)
    cfg_frozen = get_cfg(backbone, "nuscenes")
    cfg_frozen.FE.BACKBONE.NORM = "FrozenBN"
    assert list(param_specs(cfg_frozen).items()) == list(specs.items())
