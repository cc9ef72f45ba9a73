"""Writes tests/golden/tta_large_*.npz by running the reference's own DD3DWithTTA(DD3D)
(tridet/modeling/dd3d/test_time_augmentation.py, imported unmodified under oracle/ref_standin.py) in fp32 on the CPU, on
the cases of oracle/tta_large_oracle.py: DO_NMS off with and without DO_BEV_NMS, POST_NMS_TOPK 200 with 10 views, and 16
views at POST_NMS_TOPK 100.

    python tools/gen_tta_large_golden.py        (needs the reference sources, see oracle/ref_standin.py)

The stand-in's rotated NMS (bev_nms_oracle.nms_rotated, pure Python and quadratic) is swapped for
tests/nusc_tta_oracle.nms_rotated, which returns the same kept indices in the same order."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from dd3d_b200.synthetic import make_state_dict  # noqa: E402
from oracle import bev_nms_oracle, ref_standin  # noqa: E402
from oracle import tta_large_oracle as TL  # noqa: E402
from oracle.gen_golden import with_reference_poses  # noqa: E402
import nusc_tta_oracle  # noqa: E402


def run_reference(name):
    cfg, x = TL.case(name)
    ref_standin.install()
    from tridet.modeling.dd3d.test_time_augmentation import DD3DWithTTA
    model = ref_standin.build_reference_model(cfg).eval()
    model.load_state_dict(make_state_dict(cfg))
    if "pose" in x:
        x = with_reference_poses([x])[0]
    with torch.no_grad():
        inst = DD3DWithTTA(cfg, model)([x])[0]["instances"]
    print(name, "merged detections", len(inst))
    return TL.golden_blob(inst)


def main():
    bev_nms_oracle.nms_rotated = nusc_tta_oracle.nms_rotated
    out_dir = os.path.join(ROOT, "tests", "golden")
    names = sys.argv[1:] or list(TL.CASES)
    for name in names:
        np.savez_compressed(os.path.join(out_dir, f"{name}.npz"), **run_reference(name))


if __name__ == "__main__":
    main()
