"""TEST INFRASTRUCTURE ONLY -- CPU oracle of DD3DWithTTA on the configurations that need the large-set TTA path
(csrc/tta_large.cu), and the fixture cases whose reference outputs tools/gen_tta_large_golden.py writes to
tests/golden/tta_large_*.npz.

Restates tridet/modeling/dd3d/test_time_augmentation.py:_inference_one_image (:151-184) with every branch the model's
switches select, built on oracle/tta_oracle.py (views, inverse transforms, merged 2-D NMS) and tests/nusc_tta_oracle.py
(camera-frame bev_nms):
  * per view: the model's own forward -- with DO_NMS the 2-D NMS + POST_NMS_TOPK, without it every pre-NMS candidate
    (core.py:130-135); with DO_BEV_NMS the per-image BEV NMS on top (core.py:137-151, mask order);
  * merged: the union in view order, batched_nms on scores_3d with DO_NMS (:164-170), then with DO_BEV_NMS
    merged_instances[bev_nms(...)] -- survivors in descending scores_3d order, ties in concatenation order (:172-181).
"""
import numpy as np
import torch

from oracle import bev_nms_oracle as B
from oracle import tta_oracle as T
from oracle.dd3d_oracle import pose_of

# name: overrides of the TTA fixture (oracle/gen_golden.py tta_case: DLA-34 KITTI, 96x320 mapped from 94x313)
CASES = {
    "tta_large_nonms": dict(do_nms=False, do_bev_nms=False),
    "tta_large_nonms_bev": dict(do_nms=False, do_bev_nms=True),
    "tta_large_post200": dict(post_nms_topk=200, min_sizes=[64, 80, 96, 112, 128]),         # 10 views x 200
    "tta_large_16views": dict(min_sizes=[64, 72, 80, 88, 96, 112, 128, 144]),              # 16 views x 100
}
POSE = ((0.9238795, 0.0, 0.0, 0.3826834), (1.5, -2.0, 0.25))  # camera -> world (w, x, y, z), t: the BEV case's pose


def case(name):
    """(cfg, mapped dataset dict) of a large-path case.  With DO_BEV_NMS every view runs in its own model call: the
    reference's per-view BEV step concatenates the Instances of one call, and Instances.cat asserts one image size."""
    from oracle.gen_golden import tta_case
    c = CASES[name]
    cfg, x = tta_case()
    inf = cfg.DD3D.INFERENCE
    inf.DO_NMS = c.get("do_nms", True)
    inf.DO_BEV_NMS = c.get("do_bev_nms", False)
    if "post_nms_topk" in c:
        cfg.DD3D.FCOS2D.INFERENCE.POST_NMS_TOPK = c["post_nms_topk"]
    if "min_sizes" in c:
        cfg.TEST.AUG.MIN_SIZES = list(c["min_sizes"])
    if inf.DO_BEV_NMS:
        cfg.TEST.IMS_PER_BATCH = 1
        x["pose"] = (tuple(float(v) for v in POSE[0]), tuple(float(v) for v in POSE[1]))
    return cfg, x


def _with_fast_nms(nms_rotated, fn, *a):
    saved = B.nms_rotated
    if nms_rotated is not None:
        B.nms_rotated = nms_rotated
    try:
        return fn(*a)
    finally:
        B.nms_rotated = saved


def tta_forward(oracle, x, cfg, nms_rotated=None):
    """_inference_one_image with `oracle` (a DD3DOracle) as the model.  nms_rotated: a drop-in for
    bev_nms_oracle.nms_rotated (same kept indices, same order) that keeps large sets tractable."""
    import nusc_tta_oracle as NT
    aug, inf = cfg.TEST.AUG, cfg.DD3D.INFERENCE
    image = x["image"]
    h, w = int(image.shape[1]), int(image.shape[2])
    orig = (int(x.get("height", h)), int(x.get("width", w)))
    views = T.make_views(image, orig, x["intrinsics"], aug.MIN_SIZES, aug.MAX_SIZE, aug.FLIP)
    outs = []
    bs = cfg.TEST.IMS_PER_BATCH
    for a0 in range(0, len(views), bs):
        chunk = [dict({k: x[k] for k in ("pose", "extrinsics") if k in x}, image=v["image"], intrinsics=v["intrinsics"])
                 for v in views[a0:a0 + bs]]
        if inf.DO_NMS:
            outs.extend(_with_fast_nms(nms_rotated, oracle.forward, chunk, False, False))
            continue
        _, inter = oracle.forward(chunk, return_intermediates=True, do_postprocess=False)
        for b, det in enumerate(inter["pre_nms"]):  # no 2-D NMS: every candidate, level by level (core.py:130-131)
            det = dict(det)
            if inf.DO_BEV_NMS and det["quat"].shape[0]:
                keep = _with_fast_nms(nms_rotated, B.bev_nms_image, det, *pose_of(chunk[b]), inf.BEV_NMS_IOU_THRESH)
                det = {k: v[keep] for k, v in det.items()}
            outs.append(det)
    inverted = []
    for a, (v, det) in enumerate(zip(views, outs)):
        v["index"] = a
        inverted.append(T.invert_view(det, v, (h, w), orig))
    out = T.merge(inverted, cfg.DD3D.FCOS2D.INFERENCE.NMS_THRESH, do_nms=bool(inf.DO_NMS))
    out["tvec"] = NT.boxes3d_tvec(out)
    if inf.DO_BEV_NMS and out["score3d"].shape[0]:
        keep = _with_fast_nms(nms_rotated, NT.bev_nms_camera, out, inf.BEV_NMS_IOU_THRESH)
        out = {k: v[keep] for k, v in out.items()}
    return out


def golden_blob(inst):
    """The arrays a golden keeps of the reference's merged Instances."""
    b3 = inst.pred_boxes3d
    return dict(boxes=inst.pred_boxes.tensor.numpy(), scores=inst.scores.numpy(), scores_3d=inst.scores_3d.numpy(),
                classes=inst.pred_classes.numpy(), quat=b3.quat.numpy(), proj_ctr=b3.proj_ctr.numpy(),
                depth=b3.depth.numpy(), size=b3.size.numpy(), tvec=b3.tvec.numpy(), inv_K=b3.inv_intrinsics.numpy(),
                image_size=np.array(inst.image_size))


def canonical_order(score3d, box2d, cls):
    """Indices ordering a detection set by (rounded scores_3d descending, class, rounded box): compares sets whose order the config
    leaves to the per-level top-k (DO_NMS off without the BEV NMS keeps the candidate order of each view)."""
    s = np.round(np.asarray(score3d, dtype=np.float64), 4)  # fp32 restatements agree to ~1e-6: rounded keys
    b = np.round(np.asarray(box2d, dtype=np.float64), 1)
    c = np.asarray(cls, dtype=np.float64)
    return np.lexsort((b[:, 3], b[:, 2], b[:, 1], b[:, 0], c, -s))


def as_tensor(a):
    return torch.as_tensor(np.asarray(a))
