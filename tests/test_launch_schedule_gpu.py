"""Launch schedule (-m gpu): a forward launches what the plan's step list says.  For each configuration below, the kernels one
forward enqueues (counted with torch.profiler: every engine kernel lives in namespace dd3d, torch's own copies and fills do
not) equal dd3d_launches_per_forward and the launches of dd3d_get_profile; every dd3d_get_op_times entry that names an engine
op has that op's category, the ops appear once each and in order; and the FLOPs of the op-times entries add up to the FLOPs
dd3d_get_profile books."""
import pytest
import torch

from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_inputs, make_state_dict
from oracle.gen_golden import case_inputs, set_key
from oracle import num_classes_oracle

pytestmark = pytest.mark.gpu


def _plain(backbone, dataset="kitti_3d", keys=None):
    cfg = get_cfg(backbone, dataset)
    for k, v in (keys or {}).items():
        set_key(cfg, k, v)
    return cfg


def _bev(config, bev=True):
    from test_bev_nms_large_gpu import _inputs, _model
    return _model(config, bev=bev), _inputs()


_GN_AVG = {"FE.BACKBONE.NORM": "GN", "FE.FPN.NORM": "GN", "DD3D.FCOS2D.NORM": "GN", "DD3D.FCOS3D.NORM": "GN",
           "FE.FPN.FUSE_TYPE": "avg"}

# name -> (cfg or (model, inputs) factory, inputs factory, engine options, tile-list steps the plan must have)
CONFIGS = {
    "dla34": (lambda: _plain("dla34"), lambda: case_inputs("dla34"), {}, 0),
    # the V2-99 benchmark config at one image: sparse predictor, sparse box2d and box3d towers
    "v2_99_900x1600": (lambda: _plain("v2_99", "nuscenes"), lambda: make_inputs(1, 900, 1600, 1266.4), {}, 2),
    "v2_99_900x1600_dense_box3d": (lambda: _plain("v2_99", "nuscenes"), lambda: make_inputs(1, 900, 1600, 1266.4),
                                   {"sparse_box3d": 0}, 0),
    "v2_39_gn_avg": (lambda: _plain("v2_39", "nuscenes", _GN_AVG), lambda: make_inputs(2, 128, 192, 1266.4), {}, 0),
    "c128_gathered": (lambda: num_classes_oracle.case_cfg("v2_19_slim_c128"),
                      lambda: num_classes_oracle.case_inputs("v2_19_slim_c128"), {"sparse_box3d": 1}, 0),
    "bev_one_cta": (lambda: _bev("default"), None, {}, 0),
    "bev_multi_cta": (lambda: _bev("no_nms"), None, {}, 0),
    "no_nms": (lambda: _bev("no_nms", bev=False), None, {}, 0),
    "nms_single_cta": (lambda: _plain("dla34"), lambda: case_inputs("dla34"), {}, 0),
}


def _engine_kernels(model, inputs):
    """Kernels of one _forward_device of a planned model."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        model._forward_device(inputs)
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "dd3d::" in e.name)


@pytest.fixture(scope="module", params=list(CONFIGS))
def run(request):
    name = request.param
    make, make_inputs_, opts, tiles = CONFIGS[name]
    L = lib.load()
    if name == "nms_single_cta":
        assert L.dd3d_set_conv_policy(b"nms_class_parallel", 0) == 0
    try:
        if make_inputs_ is None:
            model, inputs = make()
        else:
            cfg = make()
            model = DD3DB200(cfg).to("cuda")
            model.load_state_dict(make_state_dict(cfg))
            inputs = make_inputs_()
        for k, v in opts.items():
            model.set_engine_option(k, v)
        model.set_profile(True)
        model(inputs)  # plans
        torch.cuda.synchronize()
        kernels = _engine_kernels(model, inputs)
        res = dict(name=name, tiles=tiles, kernels=kernels, launches=model.launches_per_forward(),
                   profile=model.get_profile(), times=model.get_op_times(with_op=True), conv_info=model.get_conv_info(),
                   num_ops=L.dd3d_num_ops(model._handle))
        model._release()
    finally:
        L.dd3d_set_conv_policy(b"nms_class_parallel", -1)
    yield res
    torch.cuda.empty_cache()


def test_kernels_launched_equal_the_counts(run):
    profile_launches = sum(v["launches"] for v in run["profile"].values())
    assert run["kernels"] == run["launches"] == profile_launches
    if run["name"] == "nms_single_cta":
        assert run["profile"]["nms"]["launches"] == 1


def test_op_times_name_their_ops(run):
    ops = [e[3] for e in run["times"]]
    assert [op for op in ops if op >= 0] == list(range(run["num_ops"]))
    assert ops.count(-1) == 3 + run["tiles"]  # preprocess, detect, NMS and the tile lists of the sparse towers
    for cat, _, _, op in run["times"]:
        if op >= 0:  # the implicit-GEMM convs are the ops with a conv kernel choice
            assert (cat == "conv_igemm") == (run["conv_info"][op] is not None), (op, cat)


def test_op_times_flops_sum_to_the_profile(run):
    total = sum(v["flops"] for v in run["profile"].values())
    assert total > 0
    assert sum(e[2] for e in run["times"]) == pytest.approx(total, rel=1e-12)
