"""TEST INFRASTRUCTURE ONLY -- the cases and reference fixtures for FE.BACKBONE.NORM ("FrozenBN", "BN", "SyncBN", "GN", "").

    python -m oracle.backbone_norm_oracle --golden   # tests/golden/golden_backbone_norms.npz + backbone_norms_inventory.json

BN / SyncBN differ from FrozenBN only by their num_batches_tracked keys, and DLA-34 "" (every backbone conv has a bias and no
norm: dla.py:33,44,154,230,277,337) is what DD3DOracle.conv does when the state_dict holds a bias and no BN.
DD3DOracle also builds the VoVNet "GN" backbone: GroupNorm(32, C) + ReLU after every stem, OSA 3x3, pointwise,
conv_reduction and concat conv (vovnet.py:100-159,286-287).  The storage emulation rounds where the engine stores: the raw
conv output in front of each GroupNorm, and its normalised output.
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
from oracle.dd3d_oracle import DD3DOracle as BackboneNormOracle  # noqa: E402,F401
from oracle.gen_golden import PRE_NMS_THRESH as _THRESH  # noqa: E402
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields, set_key  # noqa: E402

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (as oracle/vovnet_oracle.py VOVNET_CASE)
BACKBONE_NORM_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))
# name -> (backbone, {cfg path: value}); PRE_NMS_THRESH is lowered where the synthetic weights give too few candidates
BACKBONE_NORM_CASES = {
    "dla34_none": ("dla34", {"FE.BACKBONE.NORM": "", _THRESH: 0.02}),
    "dla34_bn": ("dla34", {"FE.BACKBONE.NORM": "BN", _THRESH: 0.03}),
    "dla34_none_syncbn_heads": ("dla34", {"FE.BACKBONE.NORM": "", "FE.FPN.NORM": "SyncBN", "DD3D.FCOS2D.NORM": "SyncBN",
                                _THRESH: 0.015}),
    "v2_39_syncbn": ("v2_39", {"FE.BACKBONE.NORM": "SyncBN"}),
    "v2_39_gn": ("v2_39", {"FE.BACKBONE.NORM": "GN", _THRESH: 0.03}),
    "v2_19_dw_gn": ("v2_19_dw", {"FE.BACKBONE.NORM": "GN", _THRESH: 0.012}),
    "v2_99_gn": ("v2_99", {"FE.BACKBONE.NORM": "GN"}),
}


def case_cfg(case, **kw):
    backbone, keys = BACKBONE_NORM_CASES[case]
    cfg = get_cfg(backbone, BACKBONE_NORM_CASE[0], **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    return ragged_inputs(*BACKBONE_NORM_CASE[1:])


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_backbone_norms.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every case,
    fields "<case>/<field><image>" as in golden_vovnet.npz; backbone_norms_inventory.json: case -> inventory_digest of the
    reference's state_dict."""
    from oracle import ref_standin
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case in BACKBONE_NORM_CASES:
        cfg = case_cfg(case)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        blob.update(reference_fields(case, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_backbone_norms.npz"), **blob)
    with open(os.path.join(out_dir, "backbone_norms_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true",
                    help="write tests/golden/golden_backbone_norms.npz and backbone_norms_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
