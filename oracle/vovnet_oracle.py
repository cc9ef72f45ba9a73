"""TEST INFRASTRUCTURE ONLY -- the case and reference fixtures for every VoVNetV2-eSE variant of the reference's _STAGE_SPECS
(tridet/modeling/feature_extractor/vovnet.py:19-97).  oracle/dd3d_oracle.py's DD3DOracle follows cfg.FE.BACKBONE.NAME
through its VOVNET table; oracle/calibrate_synthetic.py calibrates the synthetic weights of any variant.

    python -m oracle.vovnet_oracle --golden            # tests/golden/golden_vovnet.npz + vovnet_inventory.json
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
from oracle.dd3d_oracle import DD3DOracle as VoVNetOracle, VOVNET  # noqa: E402,F401
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields  # noqa: E402

# the variants other than V2-99 (golden_vovnet.npz, fields "<arch>/<field><image>"): the seeded ragged case, last image cropped
VOVNET_ARCHS = ("v2_19_slim_dw", "v2_19_dw", "v2_19_slim", "v2_19", "v2_39", "v2_57")
VOVNET_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))  # dataset, B, H, W, focal, crop (dh, dw) of the last image


def case_inputs(arch):
    """Inputs of the VoVNet fixture case (same seeds as oracle/gen_golden.py)."""
    return ragged_inputs(*VOVNET_CASE[1:])


def case_cfg(arch, **kw):
    return get_cfg(arch, VOVNET_CASE[0], **kw)


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_vovnet.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of each variant on the
    seeded case, in the fields of golden_<arch>.npz prefixed "<arch>/"; vovnet_inventory.json: arch -> inventory_digest of
    the reference's state_dict."""
    from oracle import ref_standin
    blob, inventory = {}, {}
    for arch in VOVNET_ARCHS:
        cfg = case_cfg(arch)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[arch] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(arch))
        blob.update(reference_fields(arch, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_vovnet.npz"), **blob)
    with open(os.path.join(out_dir, "vovnet_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_vovnet.npz and vovnet_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
