"""Large-set test-time augmentation (csrc/tta_large.cu, dd3d_op_tta_merge_large / dd3d_op_group_bev_nms_large), CPU side:
host refusals of the new operators, scratch linear in the number of boxes, and the wrappers' path choice from the config."""
from types import SimpleNamespace

import pytest

from dd3d_b200.config import get_cfg


def _lib():
    from dd3d_b200 import lib
    try:
        return lib.load()
    except RuntimeError:
        pytest.skip("the library is not built")


# ------------------------------------------------------------------------------------------------ refusals
def test_merged_cap_large_limits():
    L = _lib()
    assert L.dd3d_op_tta_merged_cap_large(16, 5750) == 92000
    assert L.dd3d_op_tta_merged_cap_large(10, 128) == 1280  # no clamp at 1024
    for A, cap in ((0, 10), (17, 10), (4, 0), (4, 5751)):
        assert L.dd3d_op_tta_merged_cap_large(A, cap) == -1
        assert L.dd3d_op_tta_merge_large_scratch_bytes(A, cap) == -1
    # the one-CTA merge keeps its clamp
    assert L.dd3d_op_tta_merged_cap(10, 128) == 1024


def test_merge_large_refuses_before_any_launch():
    """Out-of-range arguments return DD3D_ERR_INVALID on the host: no pointer is dereferenced, no CUDA call is made."""
    import ctypes as C
    from dd3d_b200 import lib
    L = _lib()
    views = (lib.TtaView * 17)()
    fake = C.c_void_p(256)
    for A, cap in ((0, 100), (17, 100), (4, 0), (4, 5751)):
        assert L.dd3d_op_tta_merge_large(fake, fake, views, A, cap, 0.5, 1, fake, fake, fake, fake, None) == -1
    assert L.dd3d_op_tta_merge_large(None, fake, views, 4, 100, 0.5, 1, fake, fake, fake, fake, None) == -1


def test_group_bev_nms_large_refuses_before_any_launch():
    import ctypes as C
    L = _lib()
    for B, cap, g in ((0, 10, 1), (257, 10, 1), (4, 0, 1), (4, 92001, 1), (4, 10, 0), (4, 10, 17)):
        assert L.dd3d_op_group_bev_nms_large_scratch_bytes(B, cap, g) == -1
    assert L.dd3d_op_group_bev_nms_large_scratch_bytes(16, 92000, 16) > 0
    # the existing op keeps its limits
    assert L.dd3d_op_group_bev_nms_scratch_bytes(1, 2048, 1) < 0
    fake = C.c_void_p(256)
    args = dict(num_views=1, pose_mode=1, num_groups=1, max_group_images=1, B=1, cap=100)

    def call(**kw):
        a = dict(args, **kw)
        return L.dd3d_op_group_bev_nms_large(fake, fake, fake, a["num_views"], None, a["pose_mode"], fake,
                                             a["num_groups"], a["max_group_images"], None, fake, fake, a["B"], a["cap"],
                                             0.3, 0, None)
    assert call(cap=92001) == -1
    assert call(B=257) == -1
    assert call(num_groups=2) == -1            # more groups than images
    assert call(num_views=0) == -1
    assert call(max_group_images=17) == -1
    assert call(pose_mode=0) == -1             # global mode without poses
    assert call(pose_mode=2) == -1


# ------------------------------------------------------------------------------------------------ scratch
@pytest.mark.parametrize("A", [1, 10, 16])
def test_merge_large_scratch_is_linear(A):
    L = _lib()
    for cap in (100, 500, 1000, 2875):
        one, two = L.dd3d_op_tta_merge_large_scratch_bytes(A, cap), L.dd3d_op_tta_merge_large_scratch_bytes(A, 2 * cap)
        assert 0 < one < two <= 2 * one
    # bytes per merged box stay bounded at the largest size: no A * cap squared term
    n = 16 * 5750
    assert L.dd3d_op_tta_merge_large_scratch_bytes(16, 5750) < 200 * n


@pytest.mark.parametrize("B,g", [(1, 1), (6, 6), (16, 16), (256, 1)])
def test_group_bev_nms_large_scratch_is_linear(B, g):
    L = _lib()
    fixed = B * 128 * 8 + 16 * 256  # per-segment bounds table + alignment
    for cap in (100, 1000, 5000, 46000):
        one = L.dd3d_op_group_bev_nms_large_scratch_bytes(B, cap, g)
        two = L.dd3d_op_group_bev_nms_large_scratch_bytes(B, 2 * cap, g)
        assert 0 < one < two <= 2 * one + fixed
    assert L.dd3d_op_group_bev_nms_large_scratch_bytes(16, 92000, 16) < 160 * 16 * 92000


# ------------------------------------------------------------------------------------------------ path choice
def _tta(cfg, wrapper_model=None):
    from dd3d_b200.tta import _DeviceTTA
    inf = cfg.DD3D.INFERENCE
    model = wrapper_model or SimpleNamespace(do_nms=bool(inf.DO_NMS), do_bev_nms=bool(inf.DO_BEV_NMS), only_box2d=False)
    return _DeviceTTA(cfg, model, 1)


@pytest.mark.parametrize("backbone,dataset,meta", [("dla34", "kitti_3d", "DD3D"), ("v2_99", "kitti_3d", "DD3D"),
                                                   ("dla34", "nuscenes", "NuscenesDD3D"),
                                                   ("v2_99", "nuscenes", "NuscenesDD3D")])
def test_shipped_configs_keep_the_one_cta_path(backbone, dataset, meta):
    cfg = get_cfg(backbone, dataset, meta_arch=meta)
    t = _tta(cfg)
    assert t.num_views == 10 and t.per_view_bound() == 100
    assert not t.large_path()
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True  # DO_BEV_NMS after the 2-D NMS: still within the one-CTA ops
    assert not _tta(cfg).large_path()


def test_large_path_choice():
    cfg = get_cfg("dla34", "kitti_3d")
    inf = cfg.DD3D.FCOS2D.INFERENCE
    inf.POST_NMS_TOPK = 102
    assert not _tta(cfg).large_path()  # 10 x 102 = 1020
    inf.POST_NMS_TOPK = 103
    assert _tta(cfg).large_path()      # 10 x 103 > 1024
    inf.POST_NMS_TOPK = 200
    assert _tta(cfg).large_path()
    inf.POST_NMS_TOPK = 100
    cfg.TEST.AUG.MIN_SIZES = [288, 320, 352, 384, 448, 512, 576, 640]
    t = _tta(cfg)
    assert t.num_views == 16 and t.large_path()  # 16 views x 100
    cfg.TEST.AUG.FLIP = False
    assert not _tta(cfg).large_path()            # 8 views x 100
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.DD3D.INFERENCE.DO_NMS = False
    t = _tta(cfg)
    assert t.per_view_bound() == 5000 and t.large_path()
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    assert _tta(cfg).large_path()
    # DO_BEV_NMS alone takes the large path even when the merged bound is small
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.DD3D.INFERENCE.DO_NMS, cfg.DD3D.INFERENCE.DO_BEV_NMS = False, True
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK = 10
    cfg.TEST.AUG.MIN_SIZES, cfg.TEST.AUG.FLIP = [320], False
    assert _tta(cfg).large_path()
    # the model's switches are read at call time, like the reference reads model.do_nms / do_bev_nms
    m = SimpleNamespace(do_nms=True, do_bev_nms=True, only_box2d=False)
    t = _tta(cfg, m)
    assert not t.large_path()
    m.do_nms = False
    assert t.large_path()
    m.only_box2d = True  # no 3-D boxes: no BEV NMS, and 1 view x 50 candidates fit the one-CTA merge
    assert not t.large_path()


# ------------------------------------------------------------------------------------------------ reference goldens
@pytest.mark.parametrize("name", ["tta_large_nonms", "tta_large_nonms_bev", "tta_large_post200", "tta_large_16views"])
def test_tta_large_oracle_matches_reference_golden(name):
    """fp32 oracle == the reference's DD3DWithTTA(DD3D) on the large-path cases (tools/gen_tta_large_golden.py): the same
    detections, in the same order wherever the reference's output order is defined by scores (every case but DO_NMS off
    without the BEV NMS, whose order is the per-level candidate order of each view)."""
    import os
    import numpy as np
    import nusc_tta_oracle as NT
    from conftest import GOLDEN_DIR
    from dd3d_b200.synthetic import make_state_dict
    from oracle import tta_large_oracle as TL
    from oracle.dd3d_oracle import DD3DOracle
    from util import quat_dist, rel_err
    g = np.load(os.path.join(GOLDEN_DIR, f"{name}.npz"))
    cfg, x = TL.case(name)
    out = TL.tta_forward(DD3DOracle(cfg, make_state_dict(cfg)), x, cfg, nms_rotated=NT.nms_rotated)
    n = g["scores_3d"].shape[0]
    assert out["score3d"].shape[0] == n and n > 100
    assert tuple(g["image_size"]) == (x["height"], x["width"])
    if name == "tta_large_nonms":
        o = TL.canonical_order(out["score3d"].numpy(), out["box2d"].numpy(), out["cls"].numpy())
        r = TL.canonical_order(g["scores_3d"], g["boxes"], g["classes"])
    else:
        o = r = np.arange(n)
        s = g["scores_3d"]
        assert np.all(s[:-1] >= s[1:])  # merged_instances[keep]: descending scores_3d
    np.testing.assert_allclose(out["score3d"].numpy()[o], g["scores_3d"][r], rtol=1e-4, atol=1e-6)
    assert np.array_equal(out["cls"].numpy()[o], g["classes"][r])
    assert rel_err(out["box2d"][o], TL.as_tensor(g["boxes"][r]), floor=16.0) < 1e-4
    assert quat_dist(out["quat"][o], TL.as_tensor(g["quat"][r])).max().item() < 1e-4
    assert rel_err(out["depth"][o], TL.as_tensor(g["depth"].reshape(-1)[r]), floor=1.0) < 1e-4
