"""TEST INFRASTRUCTURE ONLY -- the CPU oracle, synthetic-weight calibration and reference fixtures for the DLA networks the
engine builds (DLA-34 and the DLA-X networks of the reference's DLA_NAME_TO_BUILDER, tridet/modeling/feature_extractor/
dla.py:104-441), on top of oracle/dd3d_oracle.py (whose DLA forward is the DLA-34 one).

    python -m oracle.dla_oracle --calibrate dla_x_60   # merge one arch's gains into dd3d_b200/data/synth_gains.json
    python -m oracle.dla_oracle --golden               # tests/golden/golden_dla_x.npz + dla_x_inventory.json

``DLAOracle(cfg, state_dict, ...)`` takes the same arguments as ``DD3DOracle`` and follows ``cfg.FE.BACKBONE.NAME``.
"""
import contextlib
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

# dla.py:358-441 restated: FE.BACKBONE.NAME -> (levels, channels, BottleneckX, residual_root, cardinality)
DLA = {
    name: dict(levels=lv, channels=ch, bottleneck_x=bx, root_residual=rr, cardinality=card)
    for name, lv, ch, bx, rr, card in (
        ("DLA-34", (1, 1, 1, 2, 2, 1), (16, 32, 64, 128, 256, 512), False, False, 0),
        ("DLA-X-46-C", (1, 1, 1, 2, 2, 1), (16, 32, 64, 64, 128, 256), True, False, 32),
        ("DLA-X-60-C", (1, 1, 1, 2, 3, 1), (16, 32, 64, 64, 128, 256), True, False, 32),
        ("DLA-X-60", (1, 1, 1, 2, 3, 1), (16, 32, 128, 256, 512, 1024), True, False, 32),
        ("DLA-X-102", (1, 1, 1, 3, 4, 1), (16, 32, 128, 256, 512, 1024), True, True, 32),
        ("DLA-X-102-64", (1, 1, 1, 3, 4, 1), (16, 32, 128, 256, 512, 1024), True, True, 64),
    )
}

# the DLA-X networks (golden_dla_x.npz, fields "<arch>/<field><image>"): the DLA-34 golden case (ragged, last image cropped)
DLA_X_ARCHS = ("dla_x_46_c", "dla_x_60_c", "dla_x_60", "dla_x_102", "dla_x_102_64")
DLA_X_CASE = ("kitti_3d", 2, 192, 320, 721.5, (21, 34))  # dataset, B, H, W, focal, crop (dh, dw) of the last image


@contextlib.contextmanager
def _grouped_conv2d(groups):
    """F.conv2d(x, w, b, stride, padding) -- the call DD3DOracle.conv makes -- with `groups` groups."""
    conv2d = F.conv2d

    def grouped(x, w, b=None, stride=1, padding=0, dilation=1, _groups=1):
        return conv2d(x, w, b, stride, padding, dilation, groups)

    with mock.patch.object(F, "conv2d", grouped):
        yield


class DLAOracle(DD3DOracle):
    """DD3DOracle whose DLA backbone is the one cfg.FE.BACKBONE.NAME names (DLA-34 gives the parent's arithmetic)."""

    def __init__(self, cfg, state_dict, *a, **k):
        super().__init__(cfg, state_dict, *a, **k)
        self.dla = DLA[cfg.FE.BACKBONE.NAME] if self.arch == "dla34" else None

    def conv(self, x, prefix, stride=1, relu=False, norm=None, residual=None, quant_out=True, wkey=None):
        """The parent's conv; a weight of C / groups input channels (BottleneckX conv2, dla.py:113-124) is a grouped conv.
        Its output is a stored activation like every other conv's: rounded in the storage emulation."""
        groups = x.shape[1] // self.sd[(wkey or prefix) + ".weight"].shape[1]
        if groups == 1:
            return super().conv(x, prefix, stride, relu, norm, residual, quant_out, wkey)
        with _grouped_conv2d(groups):
            return super().conv(x, prefix, stride, relu, norm, residual, quant_out, wkey)

    def _dla_block(self, x, p, stride, residual=None):
        if not self.dla["bottleneck_x"]:
            return super()._dla_block(x, p, stride, residual)
        # BottleneckX.forward (dla.py:128-143): the stride is on the grouped 3x3
        if residual is None:
            residual = x
        out = self.conv(x, p + ".conv1", relu=True)
        out = self.conv(out, p + ".conv2", stride=stride, relu=True)
        return self.conv(out, p + ".conv3", relu=True, residual=residual)

    def _dla_root(self, p, xs):
        # Root.forward (dla.py:160-167): + children[0] (= x2) before the ReLU when residual_root
        return self.conv(torch.cat(xs, 1), p + ".conv", relu=True, residual=xs[0] if self.dla["root_residual"] else None)

    def dla34(self, x):  # the parent's backbone() calls this for every DLA
        p = "backbone.bottom_up"
        ch, levels = self.dla["channels"], self.dla["levels"]
        x = self.conv(x, p + ".base_layer", relu=True)
        x = self.conv(x, p + ".level0.0", relu=True)
        x = self.conv(x, p + ".level1.0", stride=2, relu=True)
        outs = {}
        x = self._dla_tree(x, p + ".level2", levels[2], 2, False, ch[1], ch[2])
        for lvl in (3, 4, 5):
            x = self._dla_tree(x, p + f".level{lvl}", levels[lvl], 2, True, ch[lvl - 1], ch[lvl])
            outs[f"level{lvl}"] = x
        return outs


def case_inputs(arch):
    """Inputs of the DLA-X fixture case (the seeds of oracle/gen_golden.py's DLA-34 case)."""
    _, B, H, W, focal, (dh, dw) = DLA_X_CASE
    inputs = make_inputs(B, H, W, focal)
    inputs[-1]["image"] = inputs[-1]["image"][:, :H - dh, :W - dw].contiguous()
    return inputs


def case_cfg(arch, **kw):
    return get_cfg(arch, DLA_X_CASE[0], **kw)


# ------------------------------------------------------------------------------------------------ calibration
def calibrate(arch):
    """oracle/calibrate_synthetic.calibrate (the DLA-34 recipe) through the DLA oracle of `arch`."""
    from oracle import calibrate_synthetic as cs

    class CalibDLA(DLAOracle, cs.CalibOracle):  # DLAOracle.conv first: the calibration's own F.conv2d sees the groups
        pass

    with mock.patch.object(cs, "CalibOracle", CalibDLA):
        return cs.calibrate(arch, "kitti_3d", 384, 640, 721.5, target_frac=0.01)


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
    """golden_dla_x.npz: the reference's own DD3D.forward (fp32, CPU, under oracle/ref_standin.py) of each DLA-X network on
    the seeded case, in the fields of golden_<arch>.npz prefixed "<arch>/"; dla_x_inventory.json: arch -> inventory_digest of
    the reference's state_dict.  dla102x2 sets BottleneckX.cardinality = 64 on the class for the rest of the process
    (dla.py:411), so every build starts from the class default of a fresh process (32)."""
    import inspect

    from oracle import ref_standin
    from oracle.gen_golden import inventory_digest
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
    np.savez_compressed(os.path.join(out_dir, "golden_dla_x.npz"), **blob)
    with open(os.path.join(out_dir, "dla_x_inventory.json"), "w") as f:
        json.dump(inventory, f, indent=1, sort_keys=True)
        f.write("\n")


def main():
    import argparse
    ap = argparse.ArgumentParser()
    ap.add_argument("--calibrate", metavar="ARCH", help="calibrate one DLA arch key and merge it into synth_gains.json")
    ap.add_argument("--golden", action="store_true", help="write tests/golden/golden_dla_x.npz and dla_x_inventory.json")
    args = ap.parse_args()
    if args.calibrate:
        merge_gains(args.calibrate)
    if args.golden:
        gen_goldens(os.path.join(ROOT, "tests", "golden"))


if __name__ == "__main__":
    main()
