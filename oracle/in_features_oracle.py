"""TEST INFRASTRUCTURE ONLY -- the cases and reference fixtures for DD3D.IN_FEATURES, the FPN outputs the heads run on:
``features = [features[f] for f in self.in_features]`` (core.py:25-26,82); every per-level module is sized by
``len(in_features)`` (fcos2d.py:35-36,68,77,102-108, fcos3d.py:60,86,104,128-134) and indexed by position, scales_depth /
offsets_depth by MEAN_DEPTH_PER_LEVEL (fcos3d.py:136-139, also by position); compute_locations takes the strides of the
selected levels (core.py:166-174) and ``fpn_levels`` is the position.

    python -m oracle.in_features_oracle --golden   # tests/golden/golden_in_features.npz + in_features_inventory.json
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.synthetic import make_state_dict  # noqa: E402
# DD3DOracle, by the name the code that imports the cases of this module uses for their oracle
from oracle.dd3d_oracle import DD3DOracle as InFeaturesOracle  # noqa: E402,F401
from oracle.gen_golden import PRE_NMS_THRESH as _THRESH  # noqa: E402
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields, set_key  # noqa: E402

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (as oracle/fpn_width_oracle.py)
IN_FEATURES_CASE = ("kitti_3d", 2, 128, 192, 721.5, (21, 34))
# name -> (backbone, DD3D.IN_FEATURES, meta-architecture, {cfg path: value}); PRE_NMS_THRESH is lowered where the synthetic
# weights give too few candidates.  [p6, p3] runs PER_LEVEL_PREDICTORS, so predictor l serves position l.
IN_FEATURES_CASES = {
    "dla34_p3_p6": ("dla34", ["p3", "p4", "p5", "p6"], "DD3D", {_THRESH: 0.012}),
    "dla34_p4": ("dla34", ["p4"], "DD3D", {_THRESH: 0.009}),
    "dla34_p6_p3": ("dla34", ["p6", "p3"], "DD3D", {"DD3D.FCOS3D.PER_LEVEL_PREDICTORS": True}),
    "v2_99_p3_p6": ("v2_99", ["p3", "p4", "p5", "p6"], "DD3D", {_THRESH: 0.03}),
    "v2_99_p4": ("v2_99", ["p4"], "DD3D", {_THRESH: 0.015}),
    "v2_99_p6_p3": ("v2_99", ["p6", "p3"], "DD3D", {_THRESH: 0.006}),
    "v2_99_p2_p5": ("v2_99", ["p2", "p3", "p4", "p5"], "DD3D", {_THRESH: 0.025}),
    "nusc_dla34_p4_p7": ("dla34", ["p4", "p5", "p6", "p7"], "NuscenesDD3D", {_THRESH: 0.013}),
}


def case_cfg(case, **kw):
    backbone, feats, meta_arch, keys = IN_FEATURES_CASES[case]
    dataset = "nuscenes" if meta_arch == "NuscenesDD3D" else IN_FEATURES_CASE[0]
    cfg = get_cfg(backbone, dataset, meta_arch=meta_arch, in_features=feats, **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    return ragged_inputs(*IN_FEATURES_CASE[1:])


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_in_features.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every DD3D case,
    fields "<case>/<field><image>" as in golden_fpn_width.npz; in_features_inventory.json: case -> inventory_digest of the
    reference's state_dict, for every case (NuscenesDD3D: inventory only, as in oracle/fpn_width_oracle.py)."""
    from oracle import ref_standin
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case, (_, _, meta_arch, _) in IN_FEATURES_CASES.items():
        cfg = case_cfg(case)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        if meta_arch != "DD3D":
            continue
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        blob.update(reference_fields(case, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_in_features.npz"), **blob)
    with open(os.path.join(out_dir, "in_features_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_in_features.npz and in_features_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
