"""TEST INFRASTRUCTURE ONLY -- the CPU oracle, synthetic-weight calibration and reference fixtures for every VoVNetV2-eSE
variant of the reference's _STAGE_SPECS (tridet/modeling/feature_extractor/vovnet.py:19-97), on top of oracle/dd3d_oracle.py
(whose VoVNet forward is the V-99 one).

    python -m oracle.vovnet_oracle --calibrate v2_39   # merge one arch's gains into dd3d_b200/data/synth_gains.json
    python -m oracle.vovnet_oracle --golden            # tests/golden/golden_vovnet.npz + vovnet_inventory.json

``VoVNetOracle(cfg, state_dict, ...)`` takes the same arguments as ``DD3DOracle`` and follows ``cfg.FE.BACKBONE.NAME``.
"""
import json
import os
import sys
from unittest import mock

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402
from oracle.dd3d_oracle import DD3DOracle  # noqa: E402

# vovnet.py:19-97 _STAGE_SPECS restated (the "eSE" flag is dead: _OSA_module always applies eSE, :216,233)
VOVNET = {
    name: dict(stem=stem, stage_ch=sc, out_ch=oc, layers=nl, blocks=nb, dw=dw)
    for name, stem, sc, oc, nl, nb, dw in (
        ("V-19-slim-dw-eSE", (64, 64, 64), (64, 80, 96, 112), (112, 256, 384, 512), 3, (1, 1, 1, 1), True),
        ("V-19-dw-eSE", (64, 64, 64), (128, 160, 192, 224), (256, 512, 768, 1024), 3, (1, 1, 1, 1), True),
        ("V-19-slim-eSE", (64, 64, 128), (64, 80, 96, 112), (112, 256, 384, 512), 3, (1, 1, 1, 1), False),
        ("V-19-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 3, (1, 1, 1, 1), False),
        ("V-39-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 5, (1, 1, 2, 2), False),
        ("V-57-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 5, (1, 1, 4, 3), False),
        ("V-99-eSE", (64, 64, 128), (128, 160, 192, 224), (256, 512, 768, 1024), 5, (1, 3, 9, 3), False),
    )
}

# the variants other than V2-99 (golden_vovnet.npz, fields "<arch>/<field><image>"): the seeded ragged case, last image cropped
VOVNET_ARCHS = ("v2_19_slim_dw", "v2_19_dw", "v2_19_slim", "v2_19", "v2_39", "v2_57")
VOVNET_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))  # dataset, B, H, W, focal, crop (dh, dw) of the last image


class VoVNetOracle(DD3DOracle):
    """DD3DOracle whose VoVNet backbone is the one cfg.FE.BACKBONE.NAME names (V-99 gives the parent's arithmetic)."""

    def __init__(self, cfg, state_dict, *a, **k):
        super().__init__(cfg, state_dict, *a, **k)
        self.vov = VOVNET[cfg.FE.BACKBONE.NAME] if self.arch != "dla34" else None

    def _vov_conv(self, x, p, name, stride=1):
        if not self.vov["dw"]:
            return super()._vov_conv(x, p, name, stride)
        # dw_conv3x3 (vovnet.py:100-121): depthwise 3x3 (groups = C, no bias, no norm) -> pointwise 1x1 -> pw_norm -> ReLU.
        # The depthwise output is a stored activation in the engine: rounded in the storage emulation.
        w = self.sd[f"{p}.{name}/dw_conv3x3.weight"]
        y = self._q(F.conv2d(x, self._q(w) if self.emu else w, None, stride, 1, 1, x.shape[1]))
        return self.conv(y, f"{p}.{name}/pw_conv1x1", relu=True, norm=f"{p}.{name}/pw_norm")

    def _osa(self, x, p, name, identity):
        """_OSA_module.forward (vovnet.py:218-236) with `layers` layers and the -dw conv_reduction."""
        outs = [x]
        ident = x
        if self.vov["dw"] and x.shape[1] != self.vov["stage_ch"][int(name[3]) - 2]:  # vovnet.py:200-205,221-222
            r = f"{p}.conv_reduction.{name}_reduction_0"
            x = self.conv(x, r + "/conv", relu=True, norm=r + "/norm")
        for i in range(self.vov["layers"]):
            x = self._vov_conv(x, f"{p}.layers.{i}", f"{name}_{i}")
            outs.append(x)
        xt = self.conv(torch.cat(outs, 1), f"{p}.concat.{name}_concat/conv", relu=True, norm=f"{p}.concat.{name}_concat/norm")
        xt = self._ese(xt, p + ".ese")
        if identity:
            xt = xt + ident
        return self._q(xt)

    def v2_99(self, x):  # the parent's backbone() calls this for every VoVNet
        p = "backbone.bottom_up"
        x = self.conv(x, f"{p}.stem.stem_1/conv", stride=2, relu=True, norm=f"{p}.stem.stem_1/norm")
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


def case_inputs(arch):
    """Inputs of the VoVNet fixture case (same seeds as oracle/gen_golden.py)."""
    _, B, H, W, focal, (dh, dw) = VOVNET_CASE
    inputs = make_inputs(B, H, W, focal)
    inputs[-1]["image"] = inputs[-1]["image"][:, :H - dh, :W - dw].contiguous()
    return inputs


def case_cfg(arch, **kw):
    return get_cfg(arch, VOVNET_CASE[0], **kw)


# ------------------------------------------------------------------------------------------------ calibration
def calibrate(arch):
    """oracle/calibrate_synthetic.calibrate (the V2-99 recipe) through the VoVNet oracle of `arch`."""
    from oracle import calibrate_synthetic as cs

    class CalibVoVNet(cs.CalibOracle, VoVNetOracle):
        pass

    with mock.patch.object(cs, "CalibOracle", CalibVoVNet):
        return cs.calibrate(arch, "nuscenes", 384, 640, 1266.4, target_frac=0.002)


def merge_gains(arch):
    """Calibrates `arch` and adds its entry to dd3d_b200/data/synth_gains.json; the other entries are written back unchanged
    (same json layout), so the file's diff holds only the added entry."""
    path = os.path.join(ROOT, "dd3d_b200", "data", "synth_gains.json")
    with open(path) as f:
        out = json.load(f)
    out[arch] = calibrate(arch)
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("wrote", os.path.abspath(path))


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_vovnet.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of each variant on the
    seeded case, in the fields of golden_<arch>.npz prefixed "<arch>/"; vovnet_inventory.json: arch -> inventory_digest of
    the reference's state_dict."""
    from oracle import ref_standin
    from oracle.gen_golden import inventory_digest
    blob, inventory = {}, {}
    for arch in VOVNET_ARCHS:
        cfg = case_cfg(arch)
        model = ref_standin.build_reference_model(cfg).eval()
        inventory[arch] = inventory_digest({k: tuple(v.shape) for k, v in model.state_dict().items()})
        model.load_state_dict(make_state_dict(cfg))
        with torch.no_grad():
            outs = model(case_inputs(arch))
        for b, o in enumerate(outs):
            inst = o["instances"]
            b3 = inst.pred_boxes3d
            blob.update({f"{arch}/{k}": v for k, v in {
                f"boxes{b}": inst.pred_boxes.tensor.numpy(), f"scores{b}": inst.scores.numpy(),
                f"scores_3d{b}": inst.scores_3d.numpy(), f"classes{b}": inst.pred_classes.numpy(),
                f"levels{b}": inst.fpn_levels.numpy(), f"locations{b}": inst.locations.numpy(),
                f"quat{b}": b3.quat.numpy(), f"proj_ctr{b}": b3.proj_ctr.numpy(), f"depth{b}": b3.depth.numpy(),
                f"size{b}": b3.size.numpy(), f"tvec{b}": b3.tvec.numpy(), f"image_size{b}": np.array(inst.image_size),
            }.items()})
            print(arch, "image", b, "detections", len(inst))
    np.savez_compressed(os.path.join(out_dir, "golden_vovnet.npz"), **blob)
    with open(os.path.join(out_dir, "vovnet_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--calibrate", metavar="ARCH", help="calibrate one VoVNet arch key and merge it into synth_gains.json")
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_vovnet.npz and vovnet_inventory.json")
    args = ap.parse_args()
    if args.calibrate:
        merge_gains(args.calibrate)
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
