"""TEST INFRASTRUCTURE ONLY -- the CPU oracle and reference fixtures for FE.BACKBONE.NORM ("FrozenBN", "BN", "SyncBN", "GN", ""),
on top of oracle/head_norm_oracle.py (FPN / head keys) and oracle/vovnet_oracle.py (every VoVNet variant).

    python -m oracle.backbone_norm_oracle --golden   # tests/golden/golden_backbone_norms.npz + backbone_norms_inventory.json

BN / SyncBN differ from FrozenBN only by their num_batches_tracked keys, and DLA-34 "" (every backbone conv has a bias and no
norm: dla.py:33,44,154,230,277,337) is what DD3DOracle.conv already does when the state_dict holds a bias and no BN.
``BackboneNormOracle`` adds the VoVNet "GN" backbone: GroupNorm(32, C) + ReLU after every stem, OSA 3x3, pointwise,
conv_reduction and concat conv (vovnet.py:100-159,286-287).  The storage emulation rounds where the engine stores: the raw
conv output in front of each GroupNorm, and its normalised output.
"""
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402
from oracle.head_norm_oracle import HeadNormOracle, set_key  # noqa: E402
from oracle.vovnet_oracle import VoVNetOracle  # noqa: E402

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (as oracle/vovnet_oracle.py VOVNET_CASE)
BACKBONE_NORM_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))
_THRESH = "DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH"
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
    _, B, H, W, focal, (dh, dw) = BACKBONE_NORM_CASE
    inputs = make_inputs(B, H, W, focal)
    inputs[-1]["image"] = inputs[-1]["image"][:, :H - dh, :W - dw].contiguous()
    return inputs


class BackboneNormOracle(HeadNormOracle, VoVNetOracle):
    """DD3DOracle following FE.BACKBONE.NAME / NORM, FE.FPN.* and the head NORM / depth keys."""

    def _bb_conv(self, x, conv, norm, stride=1):
        """VoVNet conv -> get_norm(FE.BACKBONE.NORM) -> ReLU; for GN the raw conv output is stored (rounded), then normalised."""
        if self.cfg.FE.BACKBONE.NORM != "GN":
            return self.conv(x, conv, stride=stride, relu=True, norm=norm)
        y = self.conv(x, conv, stride=stride, norm=norm + ".no_norm")
        return self._q(self._gn(y, norm, relu=True))

    def _vov_conv(self, x, p, name, stride=1):
        if not self.vov["dw"]:
            return self._bb_conv(x, f"{p}.{name}/conv", f"{p}.{name}/norm", stride)
        w = self.sd[f"{p}.{name}/dw_conv3x3.weight"]
        y = self._q(F.conv2d(x, self._q(w) if self.emu else w, None, stride, 1, 1, x.shape[1]))
        return self._bb_conv(y, f"{p}.{name}/pw_conv1x1", f"{p}.{name}/pw_norm")

    def _osa(self, x, p, name, identity):
        outs = [x]
        ident = x
        if self.vov["dw"] and x.shape[1] != self.vov["stage_ch"][int(name[3]) - 2]:
            r = f"{p}.conv_reduction.{name}_reduction_0"
            x = self._bb_conv(x, r + "/conv", r + "/norm")
        for i in range(self.vov["layers"]):
            x = self._vov_conv(x, f"{p}.layers.{i}", f"{name}_{i}")
            outs.append(x)
        xt = self._bb_conv(torch.cat(outs, 1), f"{p}.concat.{name}_concat/conv", f"{p}.concat.{name}_concat/norm")
        xt = self._ese(xt, p + ".ese")
        if identity:
            xt = xt + ident
        return self._q(xt)

    def v2_99(self, x):
        p = "backbone.bottom_up"
        x = self._bb_conv(x, f"{p}.stem.stem_1/conv", f"{p}.stem.stem_1/norm", 2)
        x = self._vov_conv(x, p + ".stem", "stem_2", 1)
        x = self._vov_conv(x, p + ".stem", "stem_3", 2)
        outs = {}
        for si, nblocks in zip((2, 3, 4, 5), self.vov["blocks"]):
            if si != 2:
                x = F.max_pool2d(x, kernel_size=3, stride=2, ceil_mode=True)
            for b in range(nblocks):
                name = f"OSA{si}_{b + 1}"
                x = self._osa(x, f"{p}.stage{si}.{name}", name, identity=b > 0)
            outs[f"stage{si}"] = x
        return outs


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_backbone_norms.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every case,
    fields "<case>/<field><image>" as in golden_vovnet.npz; backbone_norms_inventory.json: case -> inventory_digest of the
    reference's state_dict."""
    from oracle import ref_standin
    from oracle.gen_golden import inventory_digest
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case in BACKBONE_NORM_CASES:
        cfg = case_cfg(case)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[case] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(case))
        for b, o in enumerate(outs):
            inst = o["instances"]
            b3 = inst.pred_boxes3d
            blob.update({f"{case}/{k}": v for k, v in {
                f"boxes{b}": inst.pred_boxes.tensor.numpy(), f"scores{b}": inst.scores.numpy(),
                f"scores_3d{b}": inst.scores_3d.numpy(), f"classes{b}": inst.pred_classes.numpy(),
                f"levels{b}": inst.fpn_levels.numpy(), f"locations{b}": inst.locations.numpy(),
                f"quat{b}": b3.quat.numpy(), f"proj_ctr{b}": b3.proj_ctr.numpy(), f"depth{b}": b3.depth.numpy(),
                f"size{b}": b3.size.numpy(), f"tvec{b}": b3.tvec.numpy(), f"image_size{b}": np.array(inst.image_size),
            }.items()})
            print(case, "image", b, "detections", len(inst))
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
