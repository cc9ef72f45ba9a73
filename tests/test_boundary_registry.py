"""The boundary a reference deployment uses, without the reference: DD3DB200 / NuscenesDD3DB200 register themselves in
detectron2's META_ARCH_REGISTRY (here the repository's stand-in registry, oracle/ref_standin.py) and are built from the
config string MODEL.META_ARCHITECTURE the way the reference's build_model does (scripts/train.py:48); and DD3DB200._wrap
turns the packed C-ABI detection buffer back into the reference's own detections (tests/golden/golden_dla34.npz, the
reference DD3D.forward on the dla34 golden case)."""
import os
import subprocess
import sys

import numpy as np
import torch

from conftest import GOLDEN_DIR
from util import quat_dist

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")

PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
from oracle import ref_standin
for name in ("detectron2", "detectron2.modeling", "detectron2.modeling.meta_arch"):
    ref_standin._mod(name)
ref_standin._mod("detectron2.modeling.meta_arch.build", META_ARCH_REGISTRY=ref_standin.META_ARCH_REGISTRY)
import dd3d_b200.meta_arch as M
from dd3d_b200.config import get_cfg
from detectron2.modeling.meta_arch.build import META_ARCH_REGISTRY
assert META_ARCH_REGISTRY.get("DD3DB200") is M.DD3DB200
assert META_ARCH_REGISTRY.get("NuscenesDD3DB200") is M.NuscenesDD3DB200
for backbone, dataset, meta in (("dla34", "kitti_3d", "DD3D"), ("v2_99", "nuscenes", "NuscenesDD3D")):
    cfg = get_cfg(backbone, dataset, meta_arch=meta)
    cfg.MODEL.META_ARCHITECTURE = meta + "B200"  # the one line a deployment changes (INTEGRATION.md)
    model = META_ARCH_REGISTRY.get(cfg.MODEL.META_ARCHITECTURE)(cfg)
    assert type(model).__name__ == cfg.MODEL.META_ARCHITECTURE, type(model)
print("registry ok")
"""


def test_registry_builds_the_mirror_from_the_config_string():
    res = subprocess.run([sys.executable, "-c", PROBE, os.path.abspath(ROOT)], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0 and "registry ok" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def test_wrap_returns_the_reference_detections():
    """Pack the reference's detections into the C ABI's [B][cap][24] words (include/dd3d_b200.h dd3d_det) and read them back
    through DD3DB200._wrap: every Instances field, including the 3-D boxes rebuilt from (quat, proj_ctr, depth, size, K)."""
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from oracle.gen_golden import case_inputs
    g = np.load(os.path.join(GOLDEN_DIR, "golden_dla34.npz"))
    inputs = case_inputs("dla34")
    B = len(inputs)
    cap = max(int(g[f"boxes{b}"].shape[0]) for b in range(B)) + 3
    out = torch.zeros(B, cap, 24, dtype=torch.float32)
    ints = out.view(torch.int32)
    counts = torch.zeros(B, dtype=torch.int32)
    sizes = torch.zeros(B, 4, dtype=torch.int32)
    K = torch.stack([torch.as_tensor(x["intrinsics"], dtype=torch.float32).reshape(3, 3) for x in inputs])
    for b, x in enumerate(inputs):
        n = g[f"boxes{b}"].shape[0]
        counts[b] = n
        h, w = x["image"].shape[-2:]
        sizes[b] = torch.tensor([h, w, *[int(v) for v in g[f"image_size{b}"]]])
        out[b, :n, 0:4] = torch.as_tensor(g[f"boxes{b}"])
        out[b, :n, 4] = torch.as_tensor(g[f"scores{b}"])
        out[b, :n, 5] = torch.as_tensor(g[f"scores_3d{b}"])
        ints[b, :n, 6] = torch.as_tensor(g[f"classes{b}"], dtype=torch.int32)
        ints[b, :n, 7] = torch.as_tensor(g[f"levels{b}"], dtype=torch.int32)
        out[b, :n, 8:12] = torch.as_tensor(g[f"quat{b}"])
        out[b, :n, 12:14] = torch.as_tensor(g[f"proj_ctr{b}"])
        out[b, :n, 14] = torch.as_tensor(g[f"depth{b}"]).reshape(-1)
        out[b, :n, 15:18] = torch.as_tensor(g[f"size{b}"])
        out[b, :n, 18:20] = torch.as_tensor(g[f"locations{b}"])
    model = DD3DB200(get_cfg("dla34", "kitti_3d"))
    res = model._wrap(out, counts, K, sizes, torch.device("cpu"))
    assert len(res) == B
    for b, r in enumerate(res):
        inst = r["instances"]
        assert tuple(inst.image_size) == tuple(int(v) for v in g[f"image_size{b}"])
        assert len(inst) == g[f"boxes{b}"].shape[0]
        np.testing.assert_array_equal(inst.pred_boxes.tensor.numpy(), g[f"boxes{b}"])
        np.testing.assert_array_equal(inst.scores.numpy(), g[f"scores{b}"])
        np.testing.assert_array_equal(inst.scores_3d.numpy(), g[f"scores_3d{b}"])
        np.testing.assert_array_equal(inst.pred_classes.numpy(), g[f"classes{b}"])
        np.testing.assert_array_equal(inst.fpn_levels.numpy(), g[f"levels{b}"])
        np.testing.assert_array_equal(inst.locations.numpy(), g[f"locations{b}"])
        b3 = inst.pred_boxes3d
        assert quat_dist(b3.quat, torch.as_tensor(g[f"quat{b}"])).max() < 1e-6
        np.testing.assert_allclose(b3.tvec.numpy(), g[f"tvec{b}"], rtol=1e-4, atol=1e-4)
        np.testing.assert_allclose(b3.size.numpy(), g[f"size{b}"], rtol=1e-6)
