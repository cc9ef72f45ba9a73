"""Sparse box3d tower (-m gpu; csrc/tower_tiles.cu + the work-list pair tile of conv_igemm_kernel.cuh): the tower convs run
only on the tiles the sparse predictor's reads need, with the same kernel and K order per output element, so the detections
must be bit-identical to the dense tower's -- and must not depend on what the skipped pixels of the workspace hold.

The golden shapes are small, so the pair tile is forced on (policy "pair_tile" = 1; the fill rule would otherwise keep them
on the 128-pixel tile, which has no work-list mode) and option sparse_tower = 1 skips the head-size rule of the default."""
import copy

import pytest
import torch

from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict
from oracle.gen_golden import CASES, case_inputs
from oracle.head_norm_oracle import case_cfg as head_norm_cfg
from oracle.head_norm_oracle import case_inputs as head_norm_inputs

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _pair_tile():
    L = lib.load()
    assert L.dd3d_set_conv_policy(b"pair_tile", 1) == 0
    yield
    L.dd3d_set_conv_policy(b"pair_tile", -1)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _dets(out):
    res = []
    for o in out:
        inst = o["instances"]
        b3 = inst.pred_boxes3d
        res.append((_bits(torch.cat([inst.pred_boxes.tensor, inst.scores[:, None], inst.scores_3d[:, None], b3.quat, b3.size,
                                     b3.tvec], 1)), inst.pred_classes.cpu().clone(), inst.fpn_levels.cpu().clone()))
    return res


def _run(cfg, inputs, tower, fill=-1, nusc=False):
    model = (NuscenesDD3DB200 if nusc else DD3DB200)(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    model.set_engine_option("sparse_box3d", 1)
    model.set_engine_option("sparse_tower", tower)
    if fill >= 0:
        model.set_engine_option("workspace_fill", fill)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    n = model.launches_per_forward()
    del model
    return _dets(out), n


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        for u, v in zip(x, y):
            assert u.shape == v.shape and torch.equal(u, v), f"{what}: image {i} differs"


def _cfg(arch, thresh=None, depth=None):
    cfg = copy.deepcopy(get_cfg(arch, CASES[arch][0]))
    if thresh is not None:
        cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = thresh
    if depth is not None:
        cfg.DD3D.FCOS3D.NUM_CONVS = depth
    return cfg


# arch, PRE_NMS_THRESH (None: shipped 0.05), box3d tower depth (None: shipped 4).  dla34: ragged sizes in one batch + output
# rescale; v2_99: 128x192, level 1 has 3 tiles per image (odd: the pair padding).  Threshold 0: candidates at every border
# and in the padded rows of the ragged image; 0.9999: no candidate at all (empty tile lists).
CASES_SPARSE = [
    ("dla34", None, None), ("v2_99", None, None), ("dla34", 0.0, None), ("v2_99", 0.0, None), ("dla34", 0.9999, None),
    ("dla34", None, 2), ("v2_99", None, 2), ("v2_99", 0.0, 2),
]


@pytest.mark.parametrize("arch,thresh,depth", CASES_SPARSE)
def test_sparse_tower_is_bit_identical(arch, thresh, depth):
    cfg = _cfg(arch, thresh, depth)
    inputs = case_inputs(arch)
    dense, n_dense = _run(cfg, inputs, 0)
    sparse, n_sparse = _run(cfg, inputs, 1)
    assert n_sparse == n_dense + 1, "the sparse tower did not run (one tile-list launch per forward)"
    _assert_same(sparse, dense, f"{arch} thresh={thresh} depth={depth}")
    if thresh == 0.9999:
        assert sum(d[0].shape[0] for d in dense) == 0
    elif thresh is None and depth is None:  # the synthetic weights give detections at the shipped depth
        assert sum(d[0].shape[0] for d in dense) > 0


def test_sparse_tower_mixed_batch():
    """An image gives the same detections alone and inside a batch of other images (the tile lists are per image)."""
    cfg = _cfg("v2_99")
    imgs = make_inputs(3, 128, 192, 1266.4)
    alone, _ = _run(cfg, imgs[1:2], 1)
    batch, _ = _run(cfg, imgs, 1)
    dense, _ = _run(cfg, imgs, 0)
    _assert_same(batch, dense, "mixed batch")
    _assert_same(batch[1:2], alone, "image alone vs in a batch")


@pytest.mark.parametrize("arch", ["dla34", "v2_99"])
def test_sparse_tower_ignores_workspace_contents(arch):
    """Skipped tower pixels keep whatever the workspace held: zeroed and 0xFF-poisoned (NaN) arenas give the same bits."""
    cfg = _cfg(arch, 0.0 if arch == "dla34" else None)
    inputs = case_inputs(arch)
    a, _ = _run(cfg, inputs, 1, fill=0x00)
    b, _ = _run(cfg, inputs, 1, fill=0xFF)
    d, _ = _run(cfg, inputs, 0, fill=0xFF)
    _assert_same(a, b, "zeroed vs poisoned")
    _assert_same(b, d, "sparse vs dense")


def test_sparse_tower_nuscenes():
    cfg = copy.deepcopy(get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D"))
    inputs = make_nusc_inputs(1, 128, 192, 1266.4)
    for x in inputs:
        x["height"], x["width"] = 256, 384
    dense, n_dense = _run(cfg, inputs, 0, nusc=True)
    sparse, n_sparse = _run(cfg, inputs, 1, nusc=True)
    assert n_sparse == n_dense + 1
    _assert_same(sparse, dense, "NuscenesDD3D")


def test_gn_tower_stays_dense():
    """GroupNorm needs whole-map statistics: a GN box3d tower is built dense even with sparse_tower = 1."""
    cfg = head_norm_cfg("dla34_gn")
    inputs = head_norm_inputs("dla34_gn")
    dense, n_dense = _run(cfg, inputs, 0)
    sparse, n_sparse = _run(cfg, inputs, 1)
    assert n_sparse == n_dense
    _assert_same(sparse, dense, "GN layout")
