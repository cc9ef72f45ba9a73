"""BEV NMS on thousands of boxes per image (DO_BEV_NMS with DO_NMS off or POST_NMS_TOPK <= 0): the oracle against the
reference's own forward, the rule that picks the BEV kernel, and the C ABI of the BEV NMS as an engine op."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from oracle import bev_nms_oracle as B
from oracle.dd3d_oracle import DD3DOracle
from oracle.gen_bev_golden import BEV_CASES, BEV_POSES, PRE_FIELDS, bev_case_cfg

ONE_CTA_MAX = 256  # boxes per image the one-CTA BEV kernel holds (kBevNmsMax)
NEW_SYMBOLS = ("dd3d_set_bev_nms", "dd3d_set_poses", "dd3d_set_host_poses", "dd3d_bev_nms_path",
               "dd3d_op_bev_nms_large_scratch_bytes", "dd3d_op_bev_nms_large")


def _golden():
    return np.load(os.path.join(GOLDEN_DIR, "bev_nms_large.npz"))


@pytest.mark.parametrize("case", list(BEV_CASES))
def test_oracle_matches_reference_forward(case):
    """Fixture written by oracle/gen_bev_golden.py from the reference's own DD3D.forward: its detections before the BEV
    step, pushed through the oracle's BEV NMS and detector_postprocess, are what its DO_BEV_NMS forward returned."""
    g = _golden()
    thr = float(g["thr"])
    entering = [len(g[f"{case}/pre_score3d{b}"]) for b in range(len(BEV_POSES))]
    assert max(entering) > ONE_CTA_MAX, entering  # beyond the one-CTA kernel
    for b, (pq, pt) in enumerate(BEV_POSES):
        det = {k: torch.as_tensor(g[f"{case}/pre_{k}{b}"]) for k in PRE_FIELDS}
        keep = B.bev_nms_image(det, pq, pt, thr)
        assert 0 < len(keep) < entering[b]  # the case suppresses
        h, w = (int(v) for v in g[f"{case}/pre_image_size{b}"])
        oh, ow = (int(v) for v in g[f"{case}/image_size{b}"])
        ref = DD3DOracle.postprocess({k: v[keep] for k, v in det.items()}, (h, w), (oh, ow))
        assert np.array_equal(ref["score3d"].numpy(), g[f"{case}/scores_3d{b}"])
        assert np.array_equal(ref["cls"].numpy(), g[f"{case}/classes{b}"])
        np.testing.assert_allclose(ref["box2d"].numpy(), g[f"{case}/boxes{b}"], rtol=1e-6, atol=1e-4)


def test_no_nms_input_is_not_score_sorted():
    """With DO_NMS off the BEV step sees the level-major candidate list: the kernel's own sort has to order it."""
    g = _golden()
    s = g["no_nms/pre_score3d0"]
    assert np.any(np.diff(s) > 0)


def test_bev_kernel_choice_rule():
    """One-CTA kernel for the score-sorted 2-D NMS output of at most 256 boxes, the multi-CTA kernels otherwise."""
    from dd3d_b200 import lib
    from dd3d_b200.config import get_cfg
    L = lib.load()
    d = lib.ModelDesc()
    for do_nms, post, want in [(1, 1, 1), (1, 100, 1), (1, 256, 1), (1, 257, 2), (1, 1000, 2), (1, 0, 2), (1, -1, 2),
                               (0, 100, 2), (0, 0, 2)]:
        d.do_nms, d.post_nms_topk = do_nms, post
        assert L.dd3d_bev_nms_path(C.byref(d)) == want, (do_nms, post)
    assert L.dd3d_bev_nms_path(None) < 0
    for name in BEV_CASES:
        assert L.dd3d_bev_nms_path(C.byref(lib.desc_from_cfg(bev_case_cfg(name)))) == 2
    cfg = get_cfg("dla34", "kitti_3d")
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    assert L.dd3d_bev_nms_path(C.byref(lib.desc_from_cfg(cfg))) == 1


def test_bev_abi_declared_and_exported():
    from dd3d_b200 import lib
    header = open(os.path.join(ROOT, "include", "dd3d_b200.h")).read()
    L = lib.load()
    for name in NEW_SYMBOLS:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert name in lib.SIGNATURES and hasattr(L, name), name
    # argument checks that need no device
    assert L.dd3d_set_bev_nms(None, 1, 0.05) < 0
    assert L.dd3d_set_poses(None, None) < 0
    assert L.dd3d_set_host_poses(None, 0, None) < 0
    assert L.dd3d_op_bev_nms_large_scratch_bytes(1, 5 * 1150 + 1) < 0
    assert L.dd3d_op_bev_nms_large_scratch_bytes(0, 100) < 0
    # the IoU bit matrix dominates: n * ceil(n / 64) words for n = 5 * PRE_NMS_TOPK (about 4.1 MB at n = 5750)
    one = L.dd3d_op_bev_nms_large_scratch_bytes(1, 5750)
    assert 5750 * 90 * 8 < one < 5e6
    assert L.dd3d_op_bev_nms_large_scratch_bytes(32, 5750) >= 32 * 5750 * 90 * 8
