"""TEST INFRASTRUCTURE ONLY -- the cases and reference fixtures for FE.FPN.IN_FEATURES, the backbone outputs the FPN reads
(build_fcos_dla_fpn_backbone_p67, dla.py:537-561; build_fcos_vovnet_fpn_backbone_p6, vovnet.py:428-454; detectron2's FPN,
oracle/ref_standin.py FPN): one lateral / output conv pair per input, named by log2 of its stride, the top-down pass from the
last input, then the top block on p5.  The FPN outputs are p<log2 first stride> .. p5 and P6 (and P7 for a DLA);
DD3D.IN_FEATURES picks the head levels among them as before.

    python -m oracle.fpn_inputs_oracle --golden   # tests/golden/golden_fpn_inputs.npz + fpn_inputs_inventory.json
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
from oracle.dd3d_oracle import DD3DOracle as FpnInputsOracle  # noqa: E402,F401
from oracle.gen_golden import PRE_NMS_THRESH as _THRESH  # noqa: E402
from oracle.gen_golden import inventory_digest, ragged_inputs, reference_fields, set_key  # noqa: E402

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (as oracle/in_features_oracle.py)
FPN_INPUTS_CASE = ("kitti_3d", 2, 128, 192, 721.5, (21, 34))
# name -> (backbone, FE.FPN.IN_FEATURES, DD3D.IN_FEATURES or None, meta-architecture, {cfg path: value}); PRE_NMS_THRESH is
# lowered where the synthetic weights give too few candidates.  Small VoVNets keep the reference's CPU forward short; the -dw
# variant reads its 64-channel stem.
FPN_INPUTS_CASES = {
    "dla34_l2_l5": ("dla34", ["level2", "level3", "level4", "level5"], ["p2", "p3", "p4", "p5", "p6"], "DD3D", {}),
    "dla34_l4_l5": ("dla34", ["level4", "level5"], None, "DD3D", {_THRESH: 0.01}),
    "v2_19_slim_s3_s5": ("v2_19_slim", ["stage3", "stage4", "stage5"], None, "DD3D", {_THRESH: 0.03}),
    "v2_19_dw_stem_s3_s5": ("v2_19_dw", ["stem", "stage3", "stage4", "stage5"], None, "DD3D", {_THRESH: 0.03}),
    "v2_19_slim_s5": ("v2_19_slim", ["stage5"], None, "DD3D", {_THRESH: 0.005}),
    "nusc_v2_19_slim_stem": ("v2_19_slim", ["stem", "stage3", "stage4", "stage5"], None, "NuscenesDD3D", {_THRESH: 0.03}),
}

# lists the reference cannot build or run: (backbone, FE.BACKBONE.OUT_FEATURES, FE.FPN.IN_FEATURES); the fixture records the
# exception type and message the reference raises for each (construction, then one forward)
FPN_INPUTS_REFUSED = [
    ("dla34", ["level3", "level6"], ["level3"]),
    ("dla34", ["base_layer", "level3"], ["level3"]),
    ("v2_99", ["stage1", "stage5"], ["stage5"]),
    ("dla34", ["level4", "level5"], ["level3", "level4", "level5"]),
    ("v2_99", ["stem", "stage2", "stage3"], ["stem", "stage2", "stage3"]),
    ("dla34", ["level3", "level5"], ["level3", "level5"]),
    ("dla34", ["level5", "level4"], ["level5", "level4"]),
    ("v2_99", ["stage3"], ["stage3"]),
    ("dla34", ["level2"], ["level2"]),
    ("dla34", ["level3", "level4"], ["level3", "level4"]),
    ("v2_99", ["stage4"], ["stage4"]),
]


def refused_key(backbone, out, fpn_in):
    return f"{backbone}|{','.join(out)}|{','.join(fpn_in)}"


def refused_cfg(backbone, out, fpn_in):
    cfg = get_cfg(backbone)
    cfg.FE.BACKBONE.OUT_FEATURES, cfg.FE.FPN.IN_FEATURES = list(out), list(fpn_in)
    return cfg


def case_cfg(case, **kw):
    backbone, fpn_in, feats, meta_arch, keys = FPN_INPUTS_CASES[case]
    dataset = "nuscenes" if meta_arch == "NuscenesDD3D" else FPN_INPUTS_CASE[0]
    cfg = get_cfg(backbone, dataset, meta_arch=meta_arch, in_features=feats, fpn_in_features=fpn_in, **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    return ragged_inputs(*FPN_INPUTS_CASE[1:])


# ------------------------------------------------------------------------------------------------ fixtures
def assert_strides_are_log2_contiguous(strides):
    """detectron2.modeling.backbone.fpn._assert_strides_are_log2_contiguous, which the stand-in's FPN.__init__ leaves out."""
    for i, stride in enumerate(strides[1:], 1):
        assert stride == 2 * strides[i - 1], "Strides {} {} are not log2 contiguous".format(stride, strides[i - 1])


def build_reference(cfg):
    """The reference's own DD3D under oracle/ref_standin.py, with detectron2's FPN stride assertion."""
    from oracle import ref_standin
    model = ref_standin.build_reference_model(cfg)
    shapes = model.backbone.bottom_up.output_shape()
    assert_strides_are_log2_contiguous([shapes[f].stride for f in model.backbone.in_features])
    return model


def gen_goldens(out_dir):
    """golden_fpn_inputs.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every DD3D case,
    fields "<case>/<field><image>" as in golden_in_features.npz, plus "<case>/fpn_outputs" (backbone.output_shape() order);
    fpn_inputs_inventory.json: case -> inventory_digest of the reference's state_dict, for every case (NuscenesDD3D:
    inventory only, as in oracle/in_features_oracle.py), and under "refused" the reference's [exception type, message] for every
    list of FPN_INPUTS_REFUSED."""
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case, (_, _, _, meta_arch, _) in FPN_INPUTS_CASES.items():
        cfg = case_cfg(case)
        model = build_reference(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        if meta_arch != "DD3D":
            continue
        blob[f"{case}/fpn_outputs"] = np.array(list(model.backbone.output_shape()))
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        blob.update(reference_fields(case, outs))
    refused = {}
    for backbone, out, fpn_in in FPN_INPUTS_REFUSED:
        try:
            model = build_reference(refused_cfg(backbone, out, fpn_in)).eval()
            with torch.no_grad():
                model(case_inputs("dla34_l4_l5")[:1])
            raise RuntimeError(f"the reference ran {backbone} {fpn_in}")
        except (AssertionError, KeyError, ValueError, IndexError) as e:
            refused[refused_key(backbone, out, fpn_in)] = [type(e).__name__, str(e)]
    inventory["refused"] = refused
    np.savez_compressed(os.path.join(out_dir, "golden_fpn_inputs.npz"), **blob)
    with open(os.path.join(out_dir, "fpn_inputs_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_fpn_inputs.npz and fpn_inputs_inventory.json")
    args = ap.parse_args()
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
