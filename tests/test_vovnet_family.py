"""CPU suite for the VoVNetV2-eSE family that FE.BACKBONE.NAME selects (reference vovnet.py:19-97): parameter inventory,
oracle against the reference's own forward, config and C-ABI arch round trip, and the name errors."""
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import VOVNET_SPECS, arch_of, param_specs
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.gen_golden import inventory_digest
from oracle.vovnet_oracle import VOVNET, VOVNET_ARCHS, VOVNET_CASE, VoVNetOracle, case_inputs
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NAMES = {"v2_19_slim_dw": "V-19-slim-dw-eSE", "v2_19_dw": "V-19-dw-eSE", "v2_19_slim": "V-19-slim-eSE", "v2_19": "V-19-eSE",
         "v2_39": "V-39-eSE", "v2_57": "V-57-eSE", "v2_99": "V-99-eSE"}


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "vovnet_inventory.json")) as f:
        return json.load(f)


def _cfg(arch):
    return get_cfg(arch, VOVNET_CASE[0])


@pytest.mark.parametrize("arch", VOVNET_ARCHS)
def test_param_specs_match_reference_inventory(arch):
    shapes = {k: shape for k, (shape, _) in param_specs(_cfg(arch)).items()}
    assert inventory_digest(shapes) == _inventory()[arch]


@pytest.mark.parametrize("arch", VOVNET_ARCHS)
def test_model_state_dict_keys_equal_inventory(arch):
    cfg = _cfg(arch)
    sd = DD3DB200(cfg).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == _inventory()[arch]
    assert set(sd) == set(make_state_dict(cfg))


def test_engine_spec_table_matches_python_copy():
    """csrc/engine.cu kVovSpecs (the engine's table) == arch.VOVNET_SPECS (pinned to the reference by the inventory)."""
    with open(os.path.join(ROOT, "dd3d_b200", "csrc", "engine.cu")) as f:
        src = f.read()
    table = src[src.index("kVovSpecs[] = {"):]
    table = table[:table.index("};")]
    rows = re.findall(r"\{DD3D_ARCH_(\w+), \{([\d, ]+)\}, \{([\d, ]+)\}, \{([\d, ]+)\}, (\d+), \{([\d, ]+)\}, (true|false)\}", table)
    ints = lambda s: tuple(int(v) for v in s.split(","))  # noqa: E731
    got = {a.lower(): (ints(st), ints(sc), ints(oc), int(nl), ints(nb), dw == "true") for a, st, sc, oc, nl, nb, dw in rows}
    want = {k: tuple(v[1:]) for k, v in VOVNET_SPECS.items()}
    assert got == want
    # and the oracle's restatement
    assert {v[0]: (v[1], v[2], v[3], v[4], v[5], v[6]) for v in VOVNET_SPECS.values()} == {
        n: (s["stem"], s["stage_ch"], s["out_ch"], s["layers"], s["blocks"], s["dw"]) for n, s in VOVNET.items()}
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    for key, val in lib.ARCH_IDS.items():
        assert re.search(rf"DD3D_ARCH_{key.upper()} = {val}\b", hdr), key


@pytest.mark.parametrize("arch", VOVNET_ARCHS)
def test_oracle_matches_reference_golden(arch):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/vovnet_oracle.py --golden), same bounds as for V2-99."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_vovnet.npz"))
    cfg = _cfg(arch)
    out = VoVNetOracle(cfg, make_state_dict(cfg)).forward(case_inputs(arch))
    total = 0
    for b, o in enumerate(out):
        p = f"{arch}/"
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


@pytest.mark.parametrize("arch", list(NAMES))
def test_cfg_and_desc_round_trip(arch):
    cfg = get_cfg(arch, "nuscenes")
    assert cfg.FE.BUILDER == "build_fcos_vovnet_fpn_backbone_p6"
    assert cfg.FE.BACKBONE.NAME == NAMES[arch]
    assert arch_of(cfg) == arch
    assert lib.desc_from_cfg(cfg).arch == lib.ARCH_IDS[arch]
    assert DD3DB200(cfg).backbone.size_divisibility == 64


def test_unknown_names():
    cfg = get_cfg("v2_39", "kitti_3d")
    cfg.FE.BACKBONE.NAME = "V-27-eSE"
    with pytest.raises(KeyError):
        arch_of(cfg)
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.FE.BACKBONE.NAME = "DLA-60"
    with pytest.raises(NotImplementedError, match="DLA-60"):
        arch_of(cfg)
    with pytest.raises(NotImplementedError):
        DD3DB200(cfg)


def test_v2_99_recipe_unchanged_by_the_family():
    """The synthetic generator stream of V2-99 does not depend on the other variants' entries."""
    a = make_state_dict(get_cfg("v2_99", "nuscenes"))
    assert list(a)[:4] == ["pixel_mean", "pixel_std", "backbone.bottom_up.stem.stem_1/conv.weight",
                           "backbone.bottom_up.stem.stem_1/norm.weight"]
    assert not any("dw_conv3x3" in k or "conv_reduction" in k for k in a)


def test_vovnet_oracle_is_the_v2_99_oracle_for_v2_99():
    """The generic VoVNet forward reproduces the V2-99 oracle bit for bit (storage emulation included)."""
    from oracle.dd3d_oracle import DD3DOracle
    from oracle.gen_golden import CASES
    from oracle.gen_golden import case_inputs as v99_inputs
    cfg = get_cfg("v2_99", CASES["v2_99"][0])
    sd = make_state_dict(cfg)
    batch = DD3DOracle(cfg, sd, emulate="bf16").preprocess(v99_inputs("v2_99"))[0]
    a = DD3DOracle(cfg, sd, emulate="bf16").backbone(batch)
    b = VoVNetOracle(cfg, sd, emulate="bf16").backbone(batch)
    assert all(x.equal(y) for x, y in zip(a, b))
