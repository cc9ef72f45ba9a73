"""CPU suite for the DLA-X networks that FE.BACKBONE.NAME selects (reference dla.py:104-441): parameter inventory, oracle
against the reference's own forward, config and C-ABI arch round trip, the engine's spec table, backbone norms and the names
that stay refused."""
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import DLA_SPECS, arch_of, param_specs
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.dd3d_oracle import DLA, DD3DOracle
from oracle.dla_oracle import DLA_X_ARCHS, case_cfg, case_inputs
from oracle.gen_golden import inventory_digest
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
NAMES = {"dla_x_46_c": "DLA-X-46-C", "dla_x_60_c": "DLA-X-60-C", "dla_x_60": "DLA-X-60", "dla_x_102": "DLA-X-102",
         "dla_x_102_64": "DLA-X-102-64"}


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "dla_x_inventory.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("arch", DLA_X_ARCHS)
def test_param_specs_match_reference_inventory(arch):
    shapes = {k: shape for k, (shape, _) in param_specs(case_cfg(arch)).items()}
    assert inventory_digest(shapes) == _inventory()[arch]


@pytest.mark.parametrize("arch", DLA_X_ARCHS)
def test_model_state_dict_keys_equal_inventory(arch):
    cfg = case_cfg(arch)
    sd = DD3DB200(cfg).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == _inventory()[arch]
    assert set(sd) == set(make_state_dict(cfg))


def test_grouped_conv_inventory():
    """conv2 of every BottleneckX is (width, width / cardinality, 3, 3); project only where tree1 is a block and in != out."""
    specs = param_specs(get_cfg("dla_x_102_64"))
    conv2 = {k: s for k, (s, _) in specs.items() if k.endswith(".conv2.weight") and ".bottom_up.level" in k}
    assert conv2 and all(s[0] == 64 * s[1] and s[2:] == (3, 3) for s in conv2.values())
    assert {s[0] for s in conv2.values()} == {256, 512, 1024, 2048}
    projects = sorted(k for k in specs if k.endswith("project.weight"))
    assert projects == ["backbone.bottom_up.level2.project.weight", "backbone.bottom_up.level3.tree1.tree1.project.weight",
                        "backbone.bottom_up.level4.tree1.tree1.tree1.project.weight", "backbone.bottom_up.level5.project.weight"]
    assert "backbone.top_block.p7.weight" in specs


def test_engine_spec_table_matches_python_copy():
    """csrc/engine.cu kDlaSpecs == arch.DLA_SPECS == the oracle's restatement; the header names every arch id."""
    with open(os.path.join(ROOT, "dd3d_b200", "csrc", "engine.cu")) as f:
        src = f.read()
    table = src[src.index("kDlaSpecs[] = {"):]
    table = table[:table.index("};")]
    rows = re.findall(r"\{DD3D_ARCH_(\w+), \{([\d, ]+)\}, \{([\d, ]+)\}, (true|false), (true|false), (\d+)\}", table)
    ints = lambda s: tuple(int(v) for v in s.split(","))  # noqa: E731
    got = {a.lower(): (ints(lv), ints(ch), bx == "true", rr == "true", int(c)) for a, lv, ch, bx, rr, c in rows}
    assert got == {k: tuple(v[1:]) for k, v in DLA_SPECS.items()}
    assert {v[0]: tuple(v[1:]) for v in DLA_SPECS.values()} == {
        n: (s["levels"], s["channels"], s["bottleneck_x"], s["root_residual"], s["cardinality"]) for n, s in DLA.items()}
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    for key in DLA_SPECS:
        assert re.search(rf"DD3D_ARCH_{key.upper()} = {lib.ARCH_IDS[key]}\b", hdr), key


@pytest.mark.parametrize("arch", DLA_X_ARCHS)
def test_oracle_matches_reference_golden(arch):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/dla_oracle.py --golden), the VoVNet family's bounds."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_dla_x.npz"))
    cfg = case_cfg(arch)
    out = DD3DOracle(cfg, make_state_dict(cfg)).forward(case_inputs(arch))
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
    cfg = get_cfg(arch, "kitti_3d")
    ref = get_cfg("dla34", "kitti_3d")
    assert cfg.FE.BACKBONE.NAME == NAMES[arch]
    cfg.FE.BACKBONE.NAME = "DLA-34"
    assert cfg == ref  # the dla34 entry with only FE.BACKBONE.NAME changed
    cfg.FE.BACKBONE.NAME = NAMES[arch]
    assert arch_of(cfg) == arch
    assert lib.desc_from_cfg(cfg).arch == lib.ARCH_IDS[arch]
    assert DD3DB200(cfg).backbone.size_divisibility == 128
    assert get_cfg(arch, "nuscenes").TEST.IMS_PER_BATCH == get_cfg("dla34", "nuscenes").TEST.IMS_PER_BATCH


@pytest.mark.parametrize("name", ["DLA-46-C", "DLA-60", "DLA-102", "DLA-169"])
def test_plain_bottleneck_names_refused(name):
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.FE.BACKBONE.NAME = name
    with pytest.raises(NotImplementedError, match=name):
        arch_of(cfg)
    with pytest.raises(NotImplementedError, match=name):
        DD3DB200(cfg)


@pytest.mark.parametrize("arch", ["dla_x_46_c", "dla_x_102_64"])
@pytest.mark.parametrize("norm", ["", "BN", "SyncBN"])
def test_backbone_norms_load_strictly(arch, norm):
    cfg = get_cfg(arch, "kitti_3d")
    cfg.FE.BACKBONE.NORM = norm
    specs = param_specs(cfg)
    conv2 = f"backbone.bottom_up.level2.tree1.conv2"
    assert (conv2 + ".bias" in specs) == (norm == "")
    assert (conv2 + ".norm.num_batches_tracked" in specs) == (norm != "")
    model = DD3DB200(cfg)
    assert model._backbone_norm == lib.BACKBONE_NORMS[norm]
    res = model.load_state_dict(make_state_dict(cfg))
    assert res.missing_keys == [] and res.unexpected_keys == []


@pytest.mark.parametrize("arch", DLA_X_ARCHS)
def test_group_norm_refused_like_the_reference(arch):
    """GroupNorm(32, 16) of the base_layer: nn.GroupNorm's ValueError, as for DLA-34."""
    cfg = get_cfg(arch, "kitti_3d")
    cfg.FE.BACKBONE.NORM = "GN"
    with pytest.raises(ValueError, match=r"num_channels \(16\)"):
        DD3DB200(cfg)


def test_dla34_inventory_unchanged_by_the_family():
    """The DLA-34 generator stream is the parent's: BasicBlocks only, its golden fixtures pin the values."""
    specs = param_specs(get_cfg("dla34", "kitti_3d"))
    assert not any(".conv3." in k for k in specs)
    assert list(specs)[2:5] == ["backbone.bottom_up.base_layer.weight", "backbone.bottom_up.base_layer.norm.weight",
                                "backbone.bottom_up.base_layer.norm.bias"]
