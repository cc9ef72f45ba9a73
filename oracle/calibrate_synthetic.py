"""TEST/BENCH INFRASTRUCTURE -- one-off calibration of the synthetic-weight recipe (SURVEY.md 8c-3).

Runs the CPU oracle once per architecture on a small synthetic batch with unit gains, rescales each conv so its raw
(pre-BN) output has unit standard deviation on first use, then picks ``cls_logits`` gain/bias so that the fraction
of (pixel, class) scores above the 0.05 threshold is ~TARGET.  Every DLA takes the DLA-34 recipe and every VoVNet the
V2-99 one (RECIPES).  Merges each arch's entry (a few hundred scalars) into dd3d_b200/data/synth_gains.json.  Usage:

    python -m oracle.calibrate_synthetic                       # dla34 and v2_99
    python -m oracle.calibrate_synthetic --calibrate dla_x_60  # any arch key
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from dd3d_b200.arch import DLA_SPECS  # noqa: E402
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402
from oracle.dd3d_oracle import DD3DOracle  # noqa: E402


class CalibOracle(DD3DOracle):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.gains = {}

    def conv(self, x, prefix, stride=1, relu=False, norm=None, residual=None, quant_out=True, wkey=None):
        key = wkey or prefix
        if key not in self.gains:
            w = self.sd[key + ".weight"]
            y = F.conv2d(x, w, None, stride, (w.shape[-1] - 1) // 2, 1, x.shape[1] // w.shape[1])
            std = float(y.std())
            gain = 1.0 / std if std > 0 else 1.0
            self.gains[key] = gain
            self.sd[key + ".weight"] = w * gain
        if norm is not None and ".norm." in norm and norm not in self.gains:
            # per-level tower BN (ModuleListDial): record the level's raw-output statistics so the recipe can
            # centre the level's running stats on them (a trained BN would) -> every level yields candidates.
            w = self.sd[key + ".weight"]
            y = F.conv2d(x, w, None, stride, (w.shape[-1] - 1) // 2, 1, x.shape[1] // w.shape[1])
            m, v = float(y.mean()), float(y.var())
            self.gains[norm] = [m, v]
            self.sd[norm + ".running_mean"] = m + (v**0.5) * self.sd[norm + ".running_mean"]
            self.sd[norm + ".running_var"] = v * self.sd[norm + ".running_var"]
        return super().conv(x, prefix, stride, relu, norm, residual, quant_out, wkey)


# is a DLA -> (dataset, H, W, focal, target candidate fraction): the DLA-34 and V2-99 recipes
RECIPES = {True: ("kitti_3d", 384, 640, 721.5, 0.01), False: ("nuscenes", 384, 640, 1266.4, 0.002)}


def calibrate(arch):
    dataset, h, w, focal, target_frac = RECIPES[arch in DLA_SPECS]
    cfg = get_cfg(arch, dataset)
    sd = make_state_dict(cfg, seed=0, gains={})
    orc = CalibOracle(cfg, sd)
    inputs = make_inputs(2, h, w, focal)
    with torch.no_grad():
        batch, sizes, K = orc.preprocess(inputs)
        feats = orc.backbone(batch)
        maps = orc.heads(feats)
    # gains were applied on top of the recipe's role gains -> fold: final gain = role_gain * calib / role_gain
    gains = dict(orc.gains)
    from dd3d_b200.synthetic import _PRED
    for role_key, role in (("fcos2d_head.box2d_reg", "box2d_reg"), ("fcos2d_head.centerness", "centerness"),
                           ("fcos3d_head.box3d_quat.0", "quat"), ("fcos3d_head.box3d_ctr.0", "ctr"),
                           ("fcos3d_head.box3d_depth.0", "depth"), ("fcos3d_head.box3d_size.0", "size"),
                           ("fcos3d_head.box3d_conf.0", "conf")):
        # make_state_dict multiplies the stored gain by the role gain once more: store calib_gain * role_gain so
        # the generated layer has raw-output std == role gain.
        gains[role_key] = gains[role_key] * _PRED[role][0]
    # cls logits: unit-std logits (before bias); choose bias for the target candidate fraction
    bias0 = float(orc.sd["fcos2d_head.cls_logits.bias"][0])
    # equalise the per-level logit spread through the (positively homogeneous) last cls-tower BN affine
    for l, m in enumerate(maps["logits"]):
        std_l = float((m - bias0).std())
        k = 1.0 / std_l if std_l > 0 else 1.0
        gains[f"fcos2d_head.cls_tower.3.norm.{l}"] = list(gains[f"fcos2d_head.cls_tower.3.norm.{l}"]) + [k]
        maps["logits"][l] = (m - bias0) * k + bias0
    logit = torch.cat([m.permute(0, 2, 3, 1).reshape(-1) for m in maps["logits"]])
    ctr = torch.cat([
        m.permute(0, 2, 3, 1).reshape(-1, 1).expand(-1, cfg.DD3D.NUM_CLASSES).reshape(-1) for m in maps["centerness"]
    ])
    raw = logit - bias0
    lo, hi = -12.0, 4.0
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        frac = float(((raw + mid).sigmoid() * ctr.sigmoid() > 0.05).float().mean())
        if frac > target_frac:
            hi = mid
        else:
            lo = mid
    gains["cls_bias"] = round(0.5 * (lo + hi), 4)
    print(arch, "layers", len(gains), "cls_bias", gains["cls_bias"], "logit std", float(raw.std()))
    return {k: (round(v, 6) if isinstance(v, float) else [round(t, 6) for t in v]) for k, v in gains.items()}


def merge_gains(arch):
    """Calibrates `arch` and writes its entry into dd3d_b200/data/synth_gains.json; the other entries are written back
    unchanged (same json layout), so the file's diff holds only that entry."""
    path = os.path.join(os.path.dirname(__file__), "..", "dd3d_b200", "data", "synth_gains.json")
    with open(path) as f:
        out = json.load(f)
    out[arch] = calibrate(arch)
    with open(path, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    print("wrote", os.path.abspath(path))


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--calibrate", metavar="ARCH", nargs="+", default=["dla34", "v2_99"],
                    help="arch keys to calibrate and merge into synth_gains.json (default: dla34 v2_99)")
    for arch in ap.parse_args().calibrate:
        merge_gains(arch)


if __name__ == "__main__":
    main()
