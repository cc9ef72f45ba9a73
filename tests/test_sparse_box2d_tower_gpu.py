"""Sparse box2d tower (-m gpu; tower_mark_kernel + tower_tiles_kernel of csrc/tower_tiles.cu, the work-list pair tile and the
work-list taps-in-N predictor): the box2d tower and its predictor run only on the tiles around the pixels where some class
passes the threshold alone, with the same kernels and K order per output element, so the detections must be bit-identical to
the dense tower's -- and must not depend on what the skipped pixels of the workspace hold.

The golden shapes are small, so the pair tile is forced on (policy "pair_tile" = 1; the fill rule would otherwise keep them
on the 128-pixel tile, which has no work-list mode) and option sparse_box2d_tower = 1 skips the head-size rule of the default.
The last test runs the benchmark workload with the default options."""
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


@pytest.fixture
def pair_tile():
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


def _run(cfg, inputs, box2d, tower=1, fill=-1, nusc=False, check_box_map=False):
    model = (NuscenesDD3DB200 if nusc else DD3DB200)(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    model.set_engine_option("sparse_box3d", 1)
    model.set_engine_option("sparse_tower", tower)
    model.set_engine_option("sparse_box2d_tower", box2d)
    if fill >= 0:
        model.set_engine_option("workspace_fill", fill)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    n = model.launches_per_forward()
    if check_box_map:  # a partly stale box map is never handed out
        with pytest.raises(RuntimeError, match="sparse_box2d_tower"):
            model.get_tensor("box0")
    del model
    return _dets(out), n


def _assert_same(a, b, what):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        for u, v in zip(x, y):
            assert u.shape == v.shape and torch.equal(u, v), f"{what}: image {i} differs"


def _cfg(arch, thresh=None, depth=None, with_ctr=True):
    cfg = copy.deepcopy(get_cfg(arch, CASES[arch][0]))
    if thresh is not None:
        cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = thresh
    if depth is not None:
        cfg.DD3D.FCOS2D.NUM_BOX_CONVS = depth
    cfg.DD3D.FCOS2D.INFERENCE.THRESH_WITH_CTR = with_ctr
    return cfg


# arch, PRE_NMS_THRESH (None: shipped 0.05), box2d tower depth (None: shipped 4), THRESH_WITH_CTR, sparse box3d tower.
# dla34: ragged sizes in one batch + output rescale; v2_99: 128x192, level 1 has 3 tiles per image (odd: the pair padding).
# Threshold 0: every pixel passes, so every tile is listed, borders and the padded rows of the ragged image included;
# 0.9999: no pixel passes (empty lists: zero work units, zero detections).
CASES_SPARSE = [
    ("dla34", None, None, True, 1), ("v2_99", None, None, True, 1), ("dla34", 0.0, None, True, 1),
    ("v2_99", 0.0, None, True, 1), ("dla34", 0.9999, None, True, 1), ("v2_99", 0.9999, None, True, 0),
    ("dla34", None, None, False, 1), ("v2_99", None, None, False, 0), ("dla34", None, 2, True, 1),
    ("v2_99", None, 2, False, 1), ("v2_99", 0.0, 2, True, 0), ("v2_99", None, None, True, 0),
]


@pytest.mark.parametrize("arch,thresh,depth,with_ctr,tower", CASES_SPARSE)
def test_sparse_box2d_tower_is_bit_identical(pair_tile, arch, thresh, depth, with_ctr, tower):
    cfg = _cfg(arch, thresh, depth, with_ctr)
    inputs = case_inputs(arch)
    dense, n_dense = _run(cfg, inputs, 0, tower)
    sparse, n_sparse = _run(cfg, inputs, 1, tower, check_box_map=True)
    assert n_sparse == n_dense + 2, "the sparse box2d tower did not run (seed + tile-list launches per forward)"
    _assert_same(sparse, dense, f"{arch} thresh={thresh} depth={depth} with_ctr={with_ctr} tower={tower}")
    if thresh == 0.9999:
        assert sum(d[0].shape[0] for d in dense) == 0
    elif thresh is None and depth is None:  # the synthetic weights give detections at the shipped depth
        assert sum(d[0].shape[0] for d in dense) > 0


def test_sparse_box2d_tower_mixed_batch(pair_tile):
    """An image gives the same detections alone and inside a batch of other images (the tile lists are per image)."""
    cfg = _cfg("v2_99")
    imgs = make_inputs(3, 128, 192, 1266.4)
    alone, _ = _run(cfg, imgs[1:2], 1)
    batch, _ = _run(cfg, imgs, 1)
    dense, _ = _run(cfg, imgs, 0)
    _assert_same(batch, dense, "mixed batch")
    _assert_same(batch[1:2], alone, "image alone vs in a batch")


@pytest.mark.parametrize("arch", ["dla34", "v2_99"])
def test_sparse_box2d_tower_ignores_workspace_contents(pair_tile, arch):
    """Skipped tower and box map pixels keep whatever the workspace held: zeroed and 0xFF-poisoned (NaN) arenas give the same
    bits, equal to the dense tower's."""
    cfg = _cfg(arch)
    inputs = case_inputs(arch)
    a, _ = _run(cfg, inputs, 1, fill=0x00)
    b, _ = _run(cfg, inputs, 1, fill=0xFF)
    d, _ = _run(cfg, inputs, 0, fill=0xFF)
    _assert_same(a, b, "zeroed vs poisoned")
    _assert_same(b, d, "sparse vs dense")


def test_sparse_box2d_tower_nuscenes(pair_tile):
    """NuscenesDD3D: the attribute and speed columns of the cls map are not class columns of the threshold."""
    cfg = copy.deepcopy(get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D"))
    inputs = make_nusc_inputs(1, 128, 192, 1266.4)
    for x in inputs:
        x["height"], x["width"] = 256, 384
    dense, n_dense = _run(cfg, inputs, 0, nusc=True)
    sparse, n_sparse = _run(cfg, inputs, 1, nusc=True)
    assert n_sparse == n_dense + 2
    _assert_same(sparse, dense, "NuscenesDD3D")


def test_gn_box2d_tower_stays_dense(pair_tile):
    """GroupNorm needs whole-map statistics: a GN FCOS2D head is built dense even with sparse_box2d_tower = 1."""
    cfg = head_norm_cfg("dla34_gn")
    inputs = head_norm_inputs("dla34_gn")
    dense, n_dense = _run(cfg, inputs, 0)
    sparse, n_sparse = _run(cfg, inputs, 1)
    assert n_sparse == n_dense
    _assert_same(sparse, dense, "GN layout")


def test_benchmark_batch_default_matches_dense_box2d_tower():
    """The bench.py workload (V2-99, bf16, B = 32, 900x1600, make_inputs(32, ..., seed_base=1)) with the default options,
    where the auto rule runs the sparse box2d tower, against sparse_box2d_tower = 0."""
    cfg = get_cfg("v2_99", "nuscenes", act_dtype="bf16")
    inputs = make_inputs(32, 900, 1600, 1266.4, seed_base=1)
    res = {}
    for opt in (2, 0):
        model = DD3DB200(cfg).to("cuda")
        model.load_state_dict(make_state_dict(cfg))
        model.set_engine_option("sparse_box2d_tower", opt)
        res[opt] = (_dets(model(inputs)), model.launches_per_forward())
        torch.cuda.synchronize()
        assert model.overflow_flags() == 0
        del model
        torch.cuda.empty_cache()
    assert res[2][1] == res[0][1] + 2, "the default options did not run the sparse box2d tower"
    assert sum(d[0].shape[0] for d in res[0][0]) > 0
    _assert_same(res[2][0], res[0][0], "benchmark batch")
