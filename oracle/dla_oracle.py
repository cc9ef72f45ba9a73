"""TEST INFRASTRUCTURE ONLY -- the case and reference fixtures for the DLA-X networks of the reference's DLA_NAME_TO_BUILDER
(tridet/modeling/feature_extractor/dla.py:104-441).  oracle/dd3d_oracle.py's DD3DOracle follows cfg.FE.BACKBONE.NAME through
its DLA table; oracle/calibrate_synthetic.py calibrates the synthetic weights of any network.

    python -m oracle.dla_oracle --golden               # tests/golden/golden_dla_x.npz + dla_x_inventory.json
"""
import json
import os
import sys
from unittest import mock

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.synthetic import make_state_dict  # noqa: E402
# DD3DOracle, by the name the code that imports the cases of this module uses for their oracle
from oracle.dd3d_oracle import DD3DOracle as DLAOracle, DLA  # noqa: E402,F401
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields  # noqa: E402

# the DLA-X networks (golden_dla_x.npz, fields "<arch>/<field><image>"): the DLA-34 golden case (ragged, last image cropped)
DLA_X_ARCHS = ("dla_x_46_c", "dla_x_60_c", "dla_x_60", "dla_x_102", "dla_x_102_64")
DLA_X_CASE = ("kitti_3d", 2, 192, 320, 721.5, (21, 34))  # dataset, B, H, W, focal, crop (dh, dw) of the last image


def case_inputs(arch):
    """Inputs of the DLA-X fixture case (the seeds of oracle/gen_golden.py's DLA-34 case)."""
    return ragged_inputs(*DLA_X_CASE[1:])


def case_cfg(arch, **kw):
    return get_cfg(arch, DLA_X_CASE[0], **kw)


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_dla_x.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of each DLA-X network on
    the seeded case, in the fields of golden_<arch>.npz prefixed "<arch>/"; dla_x_inventory.json: arch -> inventory_digest of
    the reference's state_dict.  dla102x2 sets BottleneckX.cardinality = 64 on the class for the rest of the process
    (dla.py:411), so every build starts from the class default of a fresh process (32)."""
    import inspect

    from oracle import ref_standin
    ref_standin.install()
    from tridet.modeling.feature_extractor import dla as ref_dla
    from_config = ref_dla.DLA.from_config

    def from_config_passing_extra(cls, *args, **kwargs):
        # detectron2's configurable (_get_args_from_config): keyword arguments from_config does not take (dla102x's
        # residual_root, dla.py:404-406) go to __init__ unchanged; the stand-in's configurable lacks that step
        names = inspect.signature(from_config).parameters
        extra = {k: kwargs.pop(k) for k in list(kwargs) if k not in names}
        return {**from_config(*args, **kwargs), **extra}

    blob, inventory = {}, {}
    for arch in DLA_X_ARCHS:
        cfg = case_cfg(arch)
        ref_dla.BottleneckX.cardinality = 32
        with mock.patch.object(ref_dla.DLA, "from_config", classmethod(from_config_passing_extra)):
            model = ref_standin.build_reference_model(cfg).eval()
        inventory[arch] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(arch))
        blob.update(reference_fields(arch, outs))
    np.savez_compressed(os.path.join(out_dir, "golden_dla_x.npz"), **blob)
    with open(os.path.join(out_dir, "dla_x_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_dla_x.npz and dla_x_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
