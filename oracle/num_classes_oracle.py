"""TEST INFRASTRUCTURE ONLY -- the cases and reference fixtures for DD3D.NUM_CLASSES above the 16 the model desc
holds: the reference sizes cls_logits at C (fcos2d.py:96), the five box3d predictors at 4C / 2C / C / 3C / C (fcos3d.py:
103-124) and looks CANONICAL_BOX3D_SIZES up by predicted class (fcos3d.py:378).

    python -m oracle.num_classes_oracle --golden   # tests/golden/golden_num_classes.npz + num_classes_inventory.json

oracle/dd3d_oracle.py's DD3DOracle reads every class count from the state_dict and the cfg.
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
from oracle.gen_golden import PRE_NMS_THRESH as _THRESH  # noqa: E402
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields, set_key  # noqa: E402

# ragged fixture case: B, H, W, focal, crop (dh, dw) of the last image (as oracle/fpn_width_oracle.py)
NUM_CLASSES_CASE = (2, 128, 192, 1266.4, (21, 34))
# name -> (backbone, DD3D.NUM_CLASSES, meta-architecture, {cfg path: value}).  PRE_NMS_THRESH is lowered where the synthetic
# weights give too few candidates.
NUM_CLASSES_CASES = {
    "dla34_c26": ("dla34", 26, "DD3D", {_THRESH: 0.02}),
    "v2_19_slim_c128": ("v2_19_slim", 128, "DD3D", {}),
    "dla_x_46_c_c64_agnostic": ("dla_x_46_c", 64, "DD3D", {"DD3D.FCOS3D.CLASS_AGNOSTIC_BOX3D": True}),
    "dla34_c40_per_level": ("dla34", 40, "DD3D", {"DD3D.FCOS3D.PER_LEVEL_PREDICTORS": True, _THRESH: 0.02}),
    "nusc_dla34_c17": ("dla34", 17, "NuscenesDD3D", {_THRESH: 0.02}),
}


def canonical_sizes(n):
    """CANONICAL_BOX3D_SIZES of the synthetic n-class datasets: row c = (W, L, H) in metres from a fixed rule (no RNG),
    W in [0.6, 3.0), L in [0.8, 11.8), H in [0.9, 4.0), every row different."""
    return [[round(0.6 + (c * 0.173) % 2.4, 3), round(0.8 + (c * 0.619) % 11.0, 3), round(0.9 + (c * 0.291) % 3.1, 3)]
            for c in range(n)]


def num_classes_cfg(backbone, n, meta_arch="DD3D", **kw):
    """get_cfg(backbone, "nuscenes") with DD3D.NUM_CLASSES = n and the rows of canonical_sizes(n)."""
    cfg = get_cfg(backbone, "nuscenes", meta_arch=meta_arch, **kw)
    cfg.DD3D.NUM_CLASSES = n
    cfg.DD3D.FCOS3D.CANONICAL_BOX3D_SIZES = canonical_sizes(n)
    return cfg


def case_cfg(case, **kw):
    backbone, n, meta_arch, keys = NUM_CLASSES_CASES[case]
    cfg = num_classes_cfg(backbone, n, meta_arch, **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    return ragged_inputs(*NUM_CLASSES_CASE)


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_num_classes.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every DD3D case,
    fields "<case>/<field><image>" as in golden_fpn_width.npz; num_classes_inventory.json: case -> inventory_digest of the
    reference's state_dict, for every case (NuscenesDD3D: inventory only, as in oracle/fpn_width_oracle.py)."""
    from oracle import ref_standin
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case, (_, _, meta_arch, _) in NUM_CLASSES_CASES.items():
        cfg = case_cfg(case)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        if meta_arch != "DD3D":
            continue
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        blob.update(reference_fields(case, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_num_classes.npz"), **blob)
    with open(os.path.join(out_dir, "num_classes_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_num_classes.npz and num_classes_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
