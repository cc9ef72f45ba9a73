"""Writes tests/golden/nusc_tta_v2_99.npz and tests/golden/nusc_tta_bev_v2_99.npz by running the reference's own
NuscenesDD3DWithTTA(NuscenesDD3D) (tridet/modeling/dd3d/nuscenes_dd3d_tta.py, imported unmodified under
oracle/ref_standin.py) in fp32 on the CPU, on the cases of tests/test_tta_nusc.py:

  nusc_tta_v2_99      2 samples x 6 cameras, 3 scales x flip, views split across engine calls, per-call cap binding
  nusc_tta_bev_v2_99  1 sample x 6 cameras with DD3D.INFERENCE.DO_BEV_NMS (per-view and merged-set BEV NMS)

    python tools/gen_nusc_tta_golden.py        (needs the reference sources, see oracle/ref_standin.py)

The stand-in's rotated NMS is bev_nms_oracle.nms_rotated, pure Python and quadratic in the boxes of the call; it is
swapped for tests/nusc_tta_oracle.nms_rotated, which returns the same kept indices in the same order (its bounding-circle
shortcut only skips pairs that are provably disjoint; tests/test_group_bev_nms.py pins the two against each other)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dd3d_b200.synthetic import make_state_dict  # noqa: E402
from oracle import bev_nms_oracle, ref_standin  # noqa: E402
from oracle.gen_golden import with_reference_poses  # noqa: E402
import nusc_tta_oracle  # noqa: E402
from test_tta_nusc import GOLDEN_CASES, nusc_tta_case  # noqa: E402


def run_reference(name):
    do_bev_nms, samples = GOLDEN_CASES[name]
    cfg, inputs = nusc_tta_case(do_bev_nms=do_bev_nms, samples=samples)
    ref_standin.install()
    from tridet.modeling.dd3d.nuscenes_dd3d_tta import NuscenesDD3DWithTTA
    model = ref_standin.build_reference_model(cfg).eval()
    model.load_state_dict(make_state_dict(cfg))
    model.postprocess_in_inference = False  # do_test(use_tta=True), scripts/train.py:204-209
    with torch.no_grad():
        outs = NuscenesDD3DWithTTA(cfg, model)(with_reference_poses(inputs))
    blob = {}
    for b, o in enumerate(outs):
        inst = o["instances"]
        b3, g3 = inst.pred_boxes3d, inst.pred_boxes3d_global
        blob.update({
            f"boxes{b}": inst.pred_boxes.tensor.numpy(), f"scores{b}": inst.scores.numpy(),
            f"scores_3d{b}": inst.scores_3d.numpy(), f"classes{b}": inst.pred_classes.numpy(),
            f"quat{b}": b3.quat.numpy(), f"proj_ctr{b}": b3.proj_ctr.numpy(), f"depth{b}": b3.depth.numpy(),
            f"size{b}": b3.size.numpy(), f"tvec{b}": b3.tvec.numpy(), f"inv_K{b}": b3.inv_intrinsics.numpy(),
            f"attr{b}": inst.pred_attributes.numpy(), f"speed{b}": inst.pred_speeds.numpy(),
            f"quat_global{b}": g3.quat.numpy(), f"tvec_global{b}": g3.tvec.numpy(),
            f"image_size{b}": np.array(inst.image_size),
        })
        print(name, "image", b, "detections", len(inst))
    return blob


def main():
    bev_nms_oracle.nms_rotated = nusc_tta_oracle.nms_rotated
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name in GOLDEN_CASES:
        np.savez_compressed(os.path.join(out_dir, f"{name}.npz"), **run_reference(name))


if __name__ == "__main__":
    main()
