"""TEST INFRASTRUCTURE ONLY -- the cases and reference fixtures for the FPN / FCOS head structure keys: DD3D.FCOS2D.NORM,
DD3D.FCOS3D.NORM, FE.FPN.NORM ("BN", "FrozenBN", "SyncBN", "GN", ""), the tower depths NUM_CLS_CONVS / NUM_BOX_CONVS /
FCOS3D.NUM_CONVS and FE.FPN.FUSE_TYPE ("sum", "avg").  oracle/dd3d_oracle.py's DD3DOracle follows these keys.

    python -m oracle.head_norm_oracle --golden   # tests/golden/golden_head_norms.npz + head_norms_inventory.json
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
from oracle.dd3d_oracle import DD3DOracle as HeadNormOracle  # noqa: E402,F401
from oracle.gen_golden import PRE_NMS_THRESH as _THRESH  # noqa: E402
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields, set_key  # noqa: E402

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (oracle/vovnet_oracle.py VOVNET_CASE)
HEAD_NORM_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))
# name -> (backbone, {cfg path: value}); PRE_NMS_THRESH is lowered where the synthetic weights give too few candidates
HEAD_NORM_CASES = {
    "dla34_gn": ("dla34", {"DD3D.FCOS2D.NORM": "GN", "DD3D.FCOS3D.NORM": "GN", "FE.FPN.NORM": "GN", _THRESH: 0.045}),
    "v2_99_gn_avg": ("v2_99", {"DD3D.FCOS2D.NORM": "GN", "DD3D.FCOS3D.NORM": "GN", "FE.FPN.NORM": "GN",
                               "FE.FPN.FUSE_TYPE": "avg", _THRESH: 0.025}),
    "dla34_none": ("dla34", {"DD3D.FCOS2D.NORM": "", "DD3D.FCOS3D.NORM": "", "FE.FPN.NORM": "", _THRESH: 0.03}),
    "dla34_syncbn_depth": ("dla34", {"DD3D.FCOS2D.NORM": "SyncBN", "DD3D.FCOS3D.NORM": "BN", "FE.FPN.NORM": "SyncBN",
                                     "DD3D.FCOS2D.NUM_CLS_CONVS": 2, "DD3D.FCOS2D.NUM_BOX_CONVS": 3,
                                     "DD3D.FCOS3D.NUM_CONVS": 1, _THRESH: 0.02}),
    "dla34_no_towers": ("dla34", {"DD3D.FCOS2D.NUM_CLS_CONVS": 0, "DD3D.FCOS2D.NUM_BOX_CONVS": 0, "DD3D.FCOS3D.NUM_CONVS": 0,
                                  "FE.FPN.FUSE_TYPE": "avg", _THRESH: 0.024}),
}


def case_cfg(case, **kw):
    backbone, keys = HEAD_NORM_CASES[case]
    cfg = get_cfg(backbone, HEAD_NORM_CASE[0], **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    return ragged_inputs(*HEAD_NORM_CASE[1:])


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_head_norms.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every case, fields
    "<case>/<field><image>" as in golden_vovnet.npz; head_norms_inventory.json: case -> inventory_digest of the reference's
    state_dict."""
    from oracle import ref_standin
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case in HEAD_NORM_CASES:
        cfg = case_cfg(case)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        blob.update(reference_fields(case, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_head_norms.npz"), **blob)
    with open(os.path.join(out_dir, "head_norms_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_head_norms.npz and head_norms_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
