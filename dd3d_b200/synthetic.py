"""Deterministic synthetic weights and inputs for the DD3D inference path.

There is no network access for the published checkpoints (reference README.md:196-199), so benchmarks and parity
tests use random-init weights of the reference architecture.  Plain default init explodes through ~100 layers
(SURVEY.md 8c-3: all post-NMS boxes degenerate), so the recipe is *calibrated*: every conv gets a per-layer scalar
gain (dd3d_b200/data/synth_gains.json, produced once by oracle/calibrate_synthetic.py) that keeps raw conv outputs
at unit scale, BN statistics are randomised around identity so the BN fold is exercised, and predictor biases are
chosen so that a few hundred to a few thousand candidates per level survive the 0.05 threshold with
non-degenerate boxes.  Everything is generated from a seeded CPU generator -> identical tensors on every box.
"""
import json
import math
import os

import torch

from .arch import arch_of, level_strides, param_specs

_GAINS_PATH = os.path.join(os.path.dirname(__file__), "data", "synth_gains.json")

# predictor constants (role -> (weight gain, bias)); cls bias is per-arch (calibrated, see json "cls_bias")
_PRED = {
    "box2d_reg": (0.5, 2.0),
    "centerness": (0.5, 1.5),
    "quat": (1.0, 0.0),
    "ctr": (0.25, 0.0),
    "depth": (1.0, None),
    "size": (0.5, 0.0),
    "conf": (1.0, 0.0),
    "attr": (1.0, 0.0),
    "speed": (1.0, 0.5),
}


def load_gains(arch):
    if os.path.exists(_GAINS_PATH):
        with open(_GAINS_PATH) as f:
            return json.load(f).get(arch, {})
    return {}


def make_state_dict(cfg, seed=0, gains=None):
    """Reference-keyed state_dict (fp32 CPU tensors) for DD3D(cfg)."""
    arch = arch_of(cfg)
    if gains is None:
        gains = load_gains(arch)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    strides = level_strides(cfg)
    for name, (shape, kind) in param_specs(cfg).items():
        base = kind.split(":")[0]
        role = kind.split(":")[1] if ":" in kind else ""
        layer = name.rsplit(".", 1)[0]
        if base == "conv":
            fan_in = shape[1] * shape[2] * shape[3]  # role "dw" (depthwise [C, 1, 3, 3]): fan-in 9
            gain = gains.get(layer, 1.0)
            if role == "cls_logits":
                gain = gains.get(layer, 1.0)
            elif role in _PRED:
                gain = gain * _PRED[role][0]
            elif role == "ese":
                gain = 0.5
            w = torch.randn(shape, generator=g) * (gain / math.sqrt(fan_in))
            sd[name] = w
        elif base == "bias":
            if role == "cls_logits":
                sd[name] = torch.full(shape, float(gains.get("cls_bias", -4.0)))
            elif role in _PRED:
                b0 = _PRED[role][1]
                if b0 is None:  # box3d_depth has a bias only when FCOS3D.USE_SCALE is off (fcos3d.py:116): a plausible depth
                    b0 = 20.0
                sd[name] = torch.full(shape, float(b0)) + 0.1 * torch.randn(shape, generator=g)
            elif role == "ese":
                sd[name] = torch.randn(shape, generator=g)
            else:  # top_block p6/p7
                sd[name] = 0.1 * torch.randn(shape, generator=g)
        elif base in ("bn_w", "gn_w"):
            sd[name] = 0.7 + 0.6 * torch.rand(shape, generator=g)
            if layer in gains and len(gains[layer]) > 2:  # per-level output equalisation (see calibrate_synthetic)
                sd[name] = sd[name] * gains[layer][2]
        elif base in ("bn_b", "gn_b"):
            sd[name] = 0.1 * torch.randn(shape, generator=g)
            if layer in gains and len(gains[layer]) > 2:
                sd[name] = sd[name] * gains[layer][2]
        elif base == "bn_mean":
            sd[name] = 0.1 * torch.randn(shape, generator=g)
            if layer in gains:  # per-level tower BN: centre on the calibrated level statistics
                m, v = gains[layer][:2]
                sd[name] = m + math.sqrt(v) * sd[name]
        elif base == "bn_var":
            sd[name] = 0.7 + 0.6 * torch.rand(shape, generator=g)
            if layer in gains:
                sd[name] = gains[layer][1] * sd[name]
        elif base == "nbt":
            sd[name] = torch.tensor(0, dtype=torch.long)
        elif base == "scalar":
            lvl = int(name.split(".")[-2])
            if role == "box2d":
                v = strides[lvl] * cfg.DD3D.FCOS2D.BOX2D_SCALE_INIT_FACTOR
            elif role == "ctr":
                v = strides[lvl] * cfg.DD3D.FCOS3D.PROJ_CTR_SCALE_INIT_FACTOR
            elif role == "depth":
                v = cfg.DD3D.FCOS3D.STD_DEPTH_PER_LEVEL[lvl] * cfg.DD3D.FCOS3D.DEPTH_SCALE_INIT_FACTOR
            elif role == "depth_offset":
                v = cfg.DD3D.FCOS3D.MEAN_DEPTH_PER_LEVEL[lvl]
            else:
                v = 1.0
            # perturb away from the init value so per-level folding bugs cannot hide
            sd[name] = torch.tensor([v * (1.0 + 0.05 * (lvl - 2))], dtype=torch.float32)
        elif base == "buffer":
            if name == "pixel_mean":
                sd[name] = torch.tensor(cfg.MODEL.PIXEL_MEAN, dtype=torch.float32).view(3, 1, 1)
            elif name == "pixel_std":
                sd[name] = torch.tensor(cfg.MODEL.PIXEL_STD, dtype=torch.float32).view(3, 1, 1)
            elif name.endswith("mean_depth_per_level"):
                sd[name] = torch.tensor(cfg.DD3D.FCOS3D.MEAN_DEPTH_PER_LEVEL, dtype=torch.float32)
            else:
                sd[name] = torch.tensor(cfg.DD3D.FCOS3D.STD_DEPTH_PER_LEVEL, dtype=torch.float32)
        else:
            raise ValueError(kind)
    return sd


def make_inputs(batch, height, width, focal, seed_base=1, with_size=False, dtype=torch.uint8):
    """BASELINE.md 3: uint8-valued BGR noise images (generator seed = seed_base + index) and a pinhole K with
    principal point at the image centre."""
    inputs = []
    for i in range(batch):
        g = torch.Generator().manual_seed(seed_base + i)
        img = torch.randint(0, 256, (3, height, width), generator=g, dtype=torch.uint8)
        # low-frequency structure so feature maps are not pure noise
        yy = torch.linspace(0, 1, height).view(1, height, 1)
        xx = torch.linspace(0, 1, width).view(1, 1, width)
        phase = torch.rand(3, 1, 1, generator=g) * 6.28318
        wave = 0.5 + 0.5 * torch.sin(6.28318 * (2 * xx + 3 * yy) + phase)
        img = (0.5 * img.float() + 0.5 * 255.0 * wave).round().clamp(0, 255).to(torch.uint8)
        K = torch.tensor([[focal, 0.0, width / 2.0], [0.0, focal, height / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float32)
        d = {"image": img.to(dtype), "intrinsics": K}
        if with_size:
            d["height"], d["width"] = height, width
        inputs.append(d)
    return inputs


# camera yaw (degrees, about the ego z axis) of the 6 synthetic cameras of a sample: two triplets of nearly parallel
# cameras so that the cross-camera BEV NMS of NuscenesDD3D has overlapping boxes to suppress, plus one isolated view
NUSC_CAMERA_YAWS = (0.0, 4.0, -4.0, 180.0, 176.0, -70.0)


def make_nusc_inputs(num_samples, height, width, focal, seed_base=1, with_size=False):
    """NuscenesDD3D batches (nuscenes_dd3d.py:337-469): 6 images per sample, each with "sample_token" and a global
    camera "pose" given as a (quaternion wxyz, translation) pair (camera frame: x right, y down, z forward)."""
    from .structures import matrix_to_quaternion_wxyz
    inputs = make_inputs(6 * num_samples, height, width, focal, seed_base=seed_base, with_size=with_size)
    cam_to_ego = torch.tensor([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]], dtype=torch.float64)

    def rot_z(deg):
        a = math.radians(deg)
        return torch.tensor([[math.cos(a), -math.sin(a), 0.0], [math.sin(a), math.cos(a), 0.0], [0.0, 0.0, 1.0]],
                            dtype=torch.float64)

    for s in range(num_samples):
        ego_R = rot_z(30.0 + 17.0 * s)
        ego_t = torch.tensor([100.0 + 35.0 * s, 50.0 - 20.0 * s, 0.0], dtype=torch.float64)
        for c, yaw in enumerate(NUSC_CAMERA_YAWS):
            R = ego_R @ rot_z(yaw) @ cam_to_ego
            t = ego_t + ego_R @ torch.tensor([0.5 * math.cos(math.radians(yaw)), 0.5 * math.sin(math.radians(yaw)), 1.5],
                                             dtype=torch.float64)
            x = inputs[6 * s + c]
            x["sample_token"] = f"sample{s:04d}"
            x["pose"] = (matrix_to_quaternion_wxyz(R), [float(v) for v in t])
    return inputs
