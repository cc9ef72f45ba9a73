"""GPU suite (-m gpu) for the self-contained model file: the engine dd3d_create_from_file builds from
DD3DB200.save_model_file's output returns the detections of the engine built from the state_dict bit for bit, with the same
op list, launches and conv kernels; examples/dd3d_infer.c, compiled with the host C compiler against the built library,
prints the same detections as the Python model; and errors after validation come back unchanged without a handle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict
from oracle import dla_oracle, gen_golden

pytestmark = pytest.mark.gpu

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_ERR_INVALID, DD3D_ERR_MISSING = -1, -4


def _nusc_bev_cfg():
    cfg = get_cfg("dla34", "nuscenes", meta_arch="NuscenesDD3D")
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.01  # enough candidates for the BEV NMS and the aggregation to act on
    return cfg


CASES = {
    "dla34": (lambda: get_cfg("dla34", "kitti_3d"), lambda: gen_golden.case_inputs("dla34")),
    "v2_99": (lambda: get_cfg("v2_99", "nuscenes"), lambda: gen_golden.case_inputs("v2_99")),
    "nusc_dla34_bev_nms": (_nusc_bev_cfg, lambda: make_nusc_inputs(1, 128, 192, 1266.4)),
    "dla_x_46_c": (lambda: dla_oracle.case_cfg("dla_x_46_c"), lambda: dla_oracle.case_inputs("dla_x_46_c")),
}


def _cls(cfg):
    return NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200


def _from_file(cfg, path):
    """A model whose engine comes from the file instead of a state_dict; the Python side only drives it."""
    L = lib.load()
    m = _cls(cfg)(cfg).to("cuda")
    h = C.c_void_p()
    with torch.cuda.device(m.device):
        lib.check(L.dd3d_create_from_file(str(path).encode(), C.byref(h)))
    m._handle = h
    m._desc.out_cap = L.dd3d_out_cap(h)
    return m


def _fields(out):
    """Every detection field of the outputs as int32 bits."""
    rows = []
    for o in out:
        inst = o["instances"]
        cols = [inst.pred_boxes.tensor, inst.scores[:, None], inst.pred_classes[:, None].float(), inst.locations,
                inst.fpn_levels[:, None].float(), inst.scores_3d[:, None], inst.pred_boxes3d.quat,
                inst.pred_boxes3d.proj_ctr, inst.pred_boxes3d.depth, inst.pred_boxes3d.size]
        if inst.has("pred_attributes"):
            cols += [inst.pred_attributes[:, None].float(), inst.pred_speeds[:, None]]
        if inst.has("pred_boxes3d_global"):
            g = inst.pred_boxes3d_global
            cols += [g.quat, g.tvec, g.size]
        rows.append(torch.cat([c.reshape(len(inst), -1).float().cpu() for c in cols], 1).contiguous().view(torch.int32))
    return rows


@pytest.mark.parametrize("case", list(CASES))
def test_engine_from_file_matches_state_dict_engine(case, tmp_path):
    make_cfg, make_case_inputs = CASES[case]
    cfg = make_cfg()
    ref_model = _cls(cfg)(cfg).to("cuda")
    ref_model.load_state_dict(make_state_dict(cfg))
    path = tmp_path / "model.dd3d"
    ref_model.save_model_file(str(path))
    inputs = make_case_inputs()
    ref = ref_model(inputs)
    model = _from_file(cfg, path)
    out = model(inputs)
    torch.cuda.synchronize()
    assert ref_model.overflow_flags() == 0 and model.overflow_flags() == 0
    a, b = _fields(ref), _fields(out)
    assert sum(len(x) for x in a) > 0
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and torch.equal(x, y), (case, i)
    if case == "nusc_dla34_bev_nms":
        assert all(o["instances"].has("pred_boxes3d_global") for o in out)
    L = lib.load()
    assert L.dd3d_num_ops(model._handle) == L.dd3d_num_ops(ref_model._handle) > 0
    assert model.launches_per_forward() == ref_model.launches_per_forward() > 0
    assert model.get_conv_info() == ref_model.get_conv_info()


def test_c_example_prints_the_python_detections(tmp_path):
    cfg = get_cfg("dla34", "kitti_3d")
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    path = tmp_path / "dla34.dd3d"
    model.save_model_file(str(path))
    x = make_inputs(1, 192, 320, 721.5)[0]
    image = tmp_path / "image.bgr"
    image.write_bytes(x["image"].contiguous().numpy().tobytes())
    inst = model([x])[0]["instances"]

    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "examples"), f"OUT={tmp_path}"], check=True)
    K = ["%.9g" % float(v) for v in x["intrinsics"].reshape(-1)]
    res = subprocess.run([str(tmp_path / "dd3d_infer"), str(path), str(image), "192", "320", *K], capture_output=True,
                         text=True, timeout=600)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.splitlines()
    assert lines[0] == f"{len(inst)} detections" and len(lines) == len(inst) + 1 and len(inst) > 0
    printed = np.array([[np.float32(v) for v in line.split()] for line in lines[1:]], dtype=np.float32).reshape(len(inst), -1)
    b3 = inst.pred_boxes3d
    cols = [inst.pred_classes[:, None].float(), inst.scores[:, None], inst.scores_3d[:, None], inst.pred_boxes.tensor,
            b3.quat, b3.proj_ctr, b3.depth.reshape(-1, 1), b3.size, inst.locations, inst.fpn_levels[:, None].float()]
    expected = torch.cat([c.cpu() for c in cols] + [torch.zeros(len(inst), 2)], 1).numpy()  # attr, speed: 0 for DD3D
    assert printed.shape == expected.shape
    assert np.array_equal(printed.view(np.int32), expected.view(np.int32))


def test_errors_after_validation_pass_through_without_a_handle(tmp_path):
    """A well-formed file whose contents the engine refuses: the inner call's status, its text prefixed with the call."""
    L = lib.load()
    cfg = get_cfg("dla34", "kitti_3d")

    def spec(fpn_channels, tensors):
        return lib.EngineSpec(lib.desc_from_cfg(cfg), lib.layout_from_cfg(cfg), lib.NORM_BN_SHARED, fpn_channels, None,
                              None, None, lambda: tensors)

    path = tmp_path / "m.dd3d"
    for fpn_channels, tensors, status, prefix in ((256, [("x", torch.ones(2))], DD3D_ERR_MISSING, "dd3d_finalize: missing"),
                                                  (100, [], DD3D_ERR_INVALID, "dd3d_set_fpn_channels: ")):
        lib.write_model_file(str(path), spec(fpn_channels, tensors))
        h = C.c_void_p(1)
        assert L.dd3d_create_from_file(str(path).encode(), C.byref(h)) == status
        assert h.value is None
        assert L.dd3d_last_error(None).decode().startswith(prefix), L.dd3d_last_error(None)
