"""CPU suite for FE.FPN.OUT_CHANNELS (the width of the FPN and of every FCOS head): parameter inventory against the reference
at every case of oracle/fpn_width_oracle.py, the oracle against the reference's own forward, the unchanged 256-wide inventory
and generator stream, the refusals and the new C symbols."""
import hashlib
import json
import os
import re

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.arch import FPN_WIDTHS, param_specs
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.fpn_width_oracle import FPN_WIDTH_CASES, case_cfg, case_inputs
from oracle.gen_golden import CASES, inventory_digest
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_CASES = [c for c, v in FPN_WIDTH_CASES.items() if v[2] == "DD3D"]


def _inventory():
    with open(os.path.join(GOLDEN_DIR, "fpn_width_inventory.json")) as f:
        return json.load(f)


def _mirror(cfg):
    return (NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200)(cfg)


@pytest.mark.parametrize("case", list(FPN_WIDTH_CASES))
def test_param_specs_match_reference_inventory(case):
    shapes = {k: shape for k, (shape, _) in param_specs(case_cfg(case)).items()}
    assert inventory_digest(shapes) == _inventory()[case]


@pytest.mark.parametrize("case", list(FPN_WIDTH_CASES))
def test_model_state_dict_keys_equal_generator_keys(case):
    cfg = case_cfg(case)
    sd = _mirror(cfg).state_dict()
    assert inventory_digest({k: tuple(v.shape) for k, v in sd.items()}) == _inventory()[case]
    assert set(sd) == set(make_state_dict(cfg))


@pytest.mark.parametrize("width", FPN_WIDTHS)
def test_every_width_sizes_the_fpn_and_heads(width):
    """Every FPN, tower and predictor conv reads or writes `width` channels; nothing else changes."""
    s = param_specs(get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D", fpn_channels=width))
    d = param_specs(get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D"))
    assert list(s) == list(d)
    for k, (shape, kind) in s.items():
        if k.startswith(("backbone.fpn_", "backbone.top_block", "fcos2d_head.", "fcos3d_head.", "attr_logits", "speed")):
            want = tuple(width if v == 256 else v for v in d[k][0])
            if k.startswith("backbone.fpn_lateral") and k.endswith(".weight") and len(shape) == 4:
                want = (width, ) + d[k][0][1:]  # the backbone side keeps its own channels
            assert shape == want, k
        else:
            assert shape == d[k][0], k


# the parent's make_state_dict stream (SHA-256 over name + fp32 bytes, in order) of the default configs
_DEFAULT_STREAM = {
    "dla34": "aee368f85814be2fe36e91ad1ce6fd72c8a4b7d91f263b290d190351fef08612",
    "v2_99": "04806deee89e181e5af83cc4e97317378c7dd04784f633a4ec424ad4948e8d47",
}


@pytest.mark.parametrize("backbone", ["dla34", "v2_99"])
def test_width_256_inventory_and_generator_stream_are_unchanged(backbone):
    dataset = CASES[backbone][0]
    with open(os.path.join(GOLDEN_DIR, "reference_live.json")) as f:
        digest = json.load(f)["inventory"][backbone]
    for cfg in (get_cfg(backbone, dataset), get_cfg(backbone, dataset, fpn_channels=256)):
        assert cfg.FE.FPN.OUT_CHANNELS == 256
        assert inventory_digest({k: shape for k, (shape, _) in param_specs(cfg).items()}) == digest
        h = hashlib.sha256()
        for k, v in make_state_dict(cfg).items():
            h.update(k.encode())
            h.update(v.contiguous().numpy().tobytes())
        assert h.hexdigest() == _DEFAULT_STREAM[backbone]


@pytest.mark.parametrize("case", DD3D_CASES)
def test_oracle_matches_reference_golden(case):
    """Oracle (fp32) vs the reference's own DD3D.forward (oracle/fpn_width_oracle.py --golden), the bounds of the head-norm
    fixtures."""
    g = np.load(os.path.join(GOLDEN_DIR, "golden_fpn_width.npz"))
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


@pytest.mark.parametrize("width", [32, 96, 160, 576, 1024])
def test_unsupported_widths_raise_not_implemented(width):
    """Widths the reference builds and the engine does not: NotImplementedError naming the supported set."""
    cfg = get_cfg("dla34", "kitti_3d", fpn_channels=width)
    param_specs(cfg)  # the reference builds it
    with pytest.raises(NotImplementedError, match="64, 128, 192, 256, 320, 384, 448, 512"):
        DD3DB200(cfg)


@pytest.mark.parametrize("key", ["FE.FPN.NORM", "DD3D.FCOS2D.NORM", "DD3D.FCOS3D.NORM"])
def test_group_norm_on_a_width_32_does_not_divide(key):
    """GN on a width that 32 does not divide: nn.GroupNorm's ValueError, raised by the inventory before the width check."""
    for width in (80, 200):
        cfg = get_cfg("dla34", "kitti_3d", fpn_channels=width)
        node = cfg
        *parents, leaf = key.split(".")
        for p in parents:
            node = node[p]
        node[leaf] = "GN"
        with pytest.raises(ValueError, match=rf"num_channels \({width}\) must be divisible by num_groups \(32\)"):
            DD3DB200(cfg)


def test_width_refusal_order():
    """A GN width that 32 divides but the engine does not build (96) gets the NotImplementedError."""
    cfg = get_cfg("v2_99", "kitti_3d", fpn_channels=96)
    cfg.FE.FPN.NORM = "GN"
    with pytest.raises(NotImplementedError):
        DD3DB200(cfg)


def test_new_symbols_are_declared_and_exported():
    with open(os.path.join(ROOT, "include", "dd3d_b200.h")) as f:
        hdr = f.read()
    assert re.search(r"int dd3d_set_fpn_channels\(dd3d_handle h, int32_t channels\);", hdr)
    body = hdr[hdr.index("int dd3d_op_b3d_sparse_c("):]
    body = body[:body.index(";")]
    assert body.count(",") == 15 and "int cin" in body
    L = lib.load()
    for name in ("dd3d_set_fpn_channels", "dd3d_op_b3d_sparse_c", "dd3d_op_b3d_sparse"):
        assert hasattr(L, name)
    assert len(lib.SIGNATURES["dd3d_op_b3d_sparse_c"][1]) == len(lib.SIGNATURES["dd3d_op_b3d_sparse"][1]) + 1


def test_set_fpn_channels_without_a_handle_is_refused():
    assert lib.load().dd3d_set_fpn_channels(None, 128) == -1
