"""TEST INFRASTRUCTURE ONLY -- the CPU oracle and reference fixtures for the FPN / FCOS head structure keys: DD3D.FCOS2D.NORM,
DD3D.FCOS3D.NORM, FE.FPN.NORM ("BN", "FrozenBN", "SyncBN", "GN", ""), the tower depths NUM_CLS_CONVS / NUM_BOX_CONVS /
FCOS3D.NUM_CONVS and FE.FPN.FUSE_TYPE ("sum", "avg"), on top of oracle/dd3d_oracle.py (whose FPN and towers are the shipped
layout).

    python -m oracle.head_norm_oracle --golden   # tests/golden/golden_head_norms.npz + head_norms_inventory.json

``HeadNormOracle(cfg, state_dict, ...)`` takes the same arguments as ``DD3DOracle``; for the default layout it reproduces it
bit for bit.
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
from oracle.dd3d_oracle import DD3DOracle  # noqa: E402

GN_GROUPS, GN_EPS = 32, 1e-5  # get_norm("GN") = nn.GroupNorm(32, C), eps 1e-5

# ragged fixture case: dataset, B, H, W, focal, crop (dh, dw) of the last image (oracle/vovnet_oracle.py VOVNET_CASE)
HEAD_NORM_CASE = ("nuscenes", 2, 128, 192, 1266.4, (21, 34))
# name -> (backbone, {cfg path: value}); PRE_NMS_THRESH is lowered where the synthetic weights give too few candidates
_THRESH = "DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH"
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


def set_key(cfg, path, value):
    node = cfg
    *parents, leaf = path.split(".")
    for p in parents:
        node = node[p]
    node[leaf] = value


def case_cfg(case, **kw):
    backbone, keys = HEAD_NORM_CASES[case]
    cfg = get_cfg(backbone, HEAD_NORM_CASE[0], **kw)
    for k, v in keys.items():
        set_key(cfg, k, v)
    return cfg


def case_inputs(case):
    _, B, H, W, focal, (dh, dw) = HEAD_NORM_CASE
    inputs = make_inputs(B, H, W, focal)
    inputs[-1]["image"] = inputs[-1]["image"][:, :H - dh, :W - dw].contiguous()
    return inputs


class HeadNormOracle(DD3DOracle):
    """DD3DOracle whose FPN and towers follow the NORM / depth / FUSE_TYPE keys.  Storage emulation rounds where the engine
    stores: the raw conv output in front of a GroupNorm, the lateral output in front of an avg add without GN, and the
    output of every norm / add pass."""

    def _conv_norm(self, x, prefix, norm, lvl=None, relu=False):
        """Conv2d(bias = no norm, norm = get_norm(norm)) -> optional ReLU; for GN the pre-norm output is rounded."""
        if norm in ("BN", "FrozenBN") and lvl is not None:  # ModuleListDial: level lvl uses norm lvl
            return self.conv(x, prefix, relu=relu, norm=f"{prefix}.norm.{lvl}")
        if norm == "GN":
            y = self.conv(x, prefix, norm=prefix + ".no_norm")  # raw conv (GN convs have no bias), stored
            return self._q(self._gn(y, prefix + ".norm", relu))
        {"BN": 0, "FrozenBN": 0, "SyncBN": 0, "": 0}[norm]  # KeyError like get_norm
        return self.conv(x, prefix, relu=relu)  # shared BN at <prefix>.norm, or the conv bias alone

    def _gn(self, y, prefix, relu=False, add=None, avg=False):
        y = F.group_norm(y, GN_GROUPS, self.sd[prefix + ".weight"], self.sd[prefix + ".bias"], GN_EPS)
        if add is not None:
            y = y + add
        if avg:
            y = y * 0.5
        return F.relu(y) if relu else y

    def _tower(self, x, p, lvl):
        f2, f3 = self.cfg.DD3D.FCOS2D, self.cfg.DD3D.FCOS3D
        depth, norm = {"fcos2d_head.cls_tower": (f2.NUM_CLS_CONVS, f2.NORM), "fcos2d_head.box2d_tower": (f2.NUM_BOX_CONVS, f2.NORM),
                       "fcos3d_head.box3d_tower": (f3.NUM_CONVS, f3.NORM)}[p]
        for i in range(depth):
            x = self._conv_norm(x, f"{p}.{i}", norm, lvl, relu=True)
        return x

    def fpn(self, feats):
        """detectron2 FPN.forward with norm and fuse_type (oracle/ref_standin.py FPN)."""
        p = "backbone"
        norm, avg = self.cfg.FE.FPN.NORM, self.cfg.FE.FPN.FUSE_TYPE == "avg"
        if self.arch == "dla34":
            names, stages = ["level3", "level4", "level5"], [3, 4, 5]
        else:
            names, stages = ["stage2", "stage3", "stage4", "stage5"], [2, 3, 4, 5]
        results = {}
        prev = None
        for name, st in zip(names[::-1], stages[::-1]):
            lat = f"{p}.fpn_lateral{st}"
            td = None if prev is None else F.interpolate(prev, scale_factor=2.0, mode="nearest")
            if norm == "GN":
                raw = self.conv(feats[name], lat, norm=lat + ".no_norm")
                prev = self._q(self._gn(raw, lat + ".norm", add=td, avg=avg and td is not None))
            elif td is not None and avg:
                prev = self._q((self._conv_norm(feats[name], lat, norm) + td) * 0.5)
            elif td is not None:
                prev = self.conv(feats[name], lat, residual=td)  # the add fused into the lateral conv, one rounding
            else:
                prev = self._conv_norm(feats[name], lat, norm)
            results[st] = self._conv_norm(prev, f"{p}.fpn_output{st}", norm)
        p6 = self.conv(results[stages[-1]], f"{p}.top_block.p6", stride=2)
        outs = [results[s] for s in stages] + [p6]
        if self.arch == "dla34":
            outs.append(self.conv(self._q(F.relu(p6)), f"{p}.top_block.p7", stride=2))
        return outs


# ------------------------------------------------------------------------------------------------ fixtures
def gen_goldens(out_dir):
    """golden_head_norms.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of every case, fields
    "<case>/<field><image>" as in golden_vovnet.npz; head_norms_inventory.json: case -> inventory_digest of the reference's
    state_dict."""
    from oracle import ref_standin
    from oracle.gen_golden import inventory_digest
    blob, inventory = {}, {}
    torch.set_num_threads(1)
    for case in HEAD_NORM_CASES:
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
