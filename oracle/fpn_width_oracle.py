"""TEST INFRASTRUCTURE ONLY -- the cases and reference fixtures for FE.FPN.OUT_CHANNELS, the width of the FPN and of every
FCOS head (the reference's FPN builders pass it to the laterals, the outputs and the top block, dla.py:546-557,
vovnet.py:438-450; FCOS2DHead / FCOS3DHead take their tower width from the backbone's output shape, fcos2d.py:43-45,
fcos3d.py:70-72), across backbones and head / FPN norms.  DD3DOracle reads every width from the state_dict.

    python -m oracle.fpn_width_oracle --golden   # tests/golden/golden_fpn_width.npz + fpn_width_inventory.json
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
from oracle.dd3d_oracle import DD3DOracle as FpnWidthOracle  # noqa: E402,F401
from oracle.gen_golden import PRE_NMS_THRESH as _THRESH  # noqa: E402
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields, set_key  # noqa: E402

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (as oracle/head_norm_oracle.py)
FPN_WIDTH_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))
_GN = {"DD3D.FCOS2D.NORM": "GN", "DD3D.FCOS3D.NORM": "GN", "FE.FPN.NORM": "GN"}
_BN = {"DD3D.FCOS2D.NORM": "BN", "DD3D.FCOS3D.NORM": "BN", "FE.FPN.NORM": "BN"}
_NONE = {"DD3D.FCOS2D.NORM": "", "DD3D.FCOS3D.NORM": "", "FE.FPN.NORM": ""}
# name -> (backbone, FE.FPN.OUT_CHANNELS, meta-architecture, {cfg path: value}); PRE_NMS_THRESH is lowered where the synthetic
# weights give too few candidates.  The widths cover the pair-tile widths (128, 384, 512) and the others (64, 192, 320), GN at
# 64 (cpg 2) and 320 (cpg 10).
FPN_WIDTH_CASES = {
    "dla34_gn_64": ("dla34", 64, "DD3D", dict(_GN, **{_THRESH: 0.04})),
    "v2_19_slim_192": ("v2_19_slim", 192, "DD3D", {_THRESH: 0.03}),
    "dla_x_46_c_128": ("dla_x_46_c", 128, "DD3D", {_THRESH: 0.03}),
    "v2_99_bn_384": ("v2_99", 384, "DD3D", dict(_BN, **{_THRESH: 0.03})),
    "dla34_none_512": ("dla34", 512, "DD3D", dict(_NONE, **{_THRESH: 0.02})),
    "nusc_dla34_gn_320": ("dla34", 320, "NuscenesDD3D", dict(_GN, **{_THRESH: 0.04})),
}


def case_cfg(case, **kw):
    backbone, width, meta_arch, keys = FPN_WIDTH_CASES[case]
    cfg = get_cfg(backbone, FPN_WIDTH_CASE[0], meta_arch=meta_arch, fpn_channels=width, **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    return ragged_inputs(*FPN_WIDTH_CASE[1:])


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_fpn_width.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every DD3D case,
    fields "<case>/<field><image>" as in golden_head_norms.npz; fpn_width_inventory.json: case -> inventory_digest of the
    reference's state_dict, for every case (NuscenesDD3D included: its forward needs the 6-camera sample aggregation, so its
    detections are checked against the emulating oracle instead)."""
    from oracle import ref_standin
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case, (_, _, meta_arch, _) in FPN_WIDTH_CASES.items():
        cfg = case_cfg(case)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        if meta_arch != "DD3D":
            continue
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        blob.update(reference_fields(case, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_fpn_width.npz"), **blob)
    with open(os.path.join(out_dir, "fpn_width_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_fpn_width.npz and fpn_width_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
