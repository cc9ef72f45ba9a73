"""TEST INFRASTRUCTURE -- generates tests/golden/bev_nms_large.npz by running the REAL reference DD3D.forward
(tridet/modeling/dd3d/core.py, imported unmodified under oracle/ref_standin.py) with DD3D.INFERENCE.DO_BEV_NMS on the
configurations whose BEV step sees more than 256 boxes per image: (a) DO_NMS False (all 5 * PRE_NMS_TOPK candidates of
an image enter it, level-major and unsorted) and (b) POST_NMS_TOPK 0 (every 2-D NMS survivor enters it).

    python -m oracle.gen_bev_golden

Per case and image the fixture holds what entered the BEV step (the same forward with the BEV NMS and the
postprocess off) and what the forward returned (BEV NMS, then detector_postprocess).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402
from oracle import ref_standin  # noqa: E402
from oracle.gen_golden import case_cfg, with_reference_poses  # noqa: E402

BEV_THRESH = 0.05  # low enough to suppress on the synthetic weights (the value the TTA BEV case uses)
# PRE_NMS_THRESH 0.02: more candidates pass the threshold than the default 0.05 lets through
BEV_CASES = {
    "no_nms": dict(DO_NMS=False, POST_NMS_TOPK=100, PRE_NMS_THRESH=0.02),
    "post_topk0": dict(DO_NMS=True, POST_NMS_TOPK=0, PRE_NMS_THRESH=0.02),
}
BEV_POSES = [([1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0]), ([0.9238795, 0.0, 0.3826834, 0.0], [3.0, -1.0, 2.0])]
PRE_FIELDS = ("quat", "tvec", "size", "score3d", "cls", "box2d")


def bev_case_cfg(name, bev=True, postprocess=True):
    c = BEV_CASES[name]
    cfg = case_cfg("dla34")
    cfg.DD3D.INFERENCE.DO_NMS = c["DO_NMS"]
    cfg.DD3D.FCOS2D.INFERENCE.POST_NMS_TOPK = c["POST_NMS_TOPK"]
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = c["PRE_NMS_THRESH"]
    cfg.DD3D.INFERENCE.DO_BEV_NMS = bev
    cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH = BEV_THRESH
    cfg.DD3D.INFERENCE.DO_POSTPROCESS = postprocess
    return cfg


def bev_case_inputs():
    """Two 192x320 DLA-34 inputs, the second with a 2x output size, one pose each.  Not ragged: the reference's BEV step
    concatenates the Instances of the whole batch (postprocessing.py:96), which requires one common image size."""
    inputs = make_inputs(2, 192, 320, 721.5)
    inputs[-1]["height"], inputs[-1]["width"] = 384, 640
    for x, p in zip(inputs, BEV_POSES):
        x["pose"] = p
    return inputs


def _run(cfg, inputs):
    model = ref_standin.build_reference_model(cfg).eval()
    model.load_state_dict(make_state_dict(cfg))
    with torch.no_grad():
        return [o["instances"] for o in model(inputs)]


def main():
    ref_standin.install()
    blob = {"thr": np.float32(BEV_THRESH), "cases": np.array(list(BEV_CASES))}
    for name in BEV_CASES:
        inputs = with_reference_poses(bev_case_inputs())
        pre = _run(bev_case_cfg(name, bev=False, postprocess=False), inputs)
        post = _run(bev_case_cfg(name), inputs)
        for b, (p, o) in enumerate(zip(pre, post)):
            b3 = p.pred_boxes3d
            vals = (b3.quat, b3.tvec, b3.size, p.scores_3d, p.pred_classes, p.pred_boxes.tensor)
            for k, v in zip(PRE_FIELDS, vals):
                blob[f"{name}/pre_{k}{b}"] = v.numpy()
            blob[f"{name}/pre_image_size{b}"] = np.array(p.image_size)
            blob[f"{name}/boxes{b}"] = o.pred_boxes.tensor.numpy()
            blob[f"{name}/scores_3d{b}"] = o.scores_3d.numpy()
            blob[f"{name}/classes{b}"] = o.pred_classes.numpy()
            blob[f"{name}/image_size{b}"] = np.array(o.image_size)
            print(name, "image", b, "boxes entering the BEV NMS", len(p), "returned", len(o))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "bev_nms_large.npz"), **blob)


if __name__ == "__main__":
    main()
