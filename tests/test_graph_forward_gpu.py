"""GPU suite (-m gpu) for the CUDA-graph forward (dd3d_graph_create / dd3d_graph_launch, DD3DB200.capture_forward): a
replay returns dd3d_forward's detections, counts, flags (and NuscenesDD3D global rows) bit for bit on every config family,
reads the bound input buffers at every launch, holds dd3d_launches_per_forward kernel nodes with the PDL launches as
programmatic edges, refuses to launch once stale, refuses capture with profiling on or before a plan, never leaves a
stream capturing, runs on any stream; examples/dd3d_infer -g prints what dd3d_infer prints."""
import ctypes as C
import os
import subprocess

import pytest
import torch

from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict
from oracle import dla_oracle, in_features_oracle, num_classes_oracle
from oracle.gen_golden import PRE_NMS_THRESH, case_inputs, ragged_inputs, set_key

pytestmark = pytest.mark.gpu

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
DD3D_ERR_STATE = -2
SENTINEL = 0x7FC0DEAD  # a NaN pattern no forward writes
_SPARSE_ON = dict(sparse_box3d=1, sparse_tower=1, sparse_box2d_tower=1)
_SPARSE_OFF = dict(sparse_box3d=0, sparse_tower=0, sparse_box2d_tower=0)
_GN_AVG = {"FE.BACKBONE.NORM": "GN", "FE.FPN.NORM": "GN", "DD3D.FCOS2D.NORM": "GN", "DD3D.FCOS3D.NORM": "GN",
           "FE.FPN.FUSE_TYPE": "avg"}


def _cfg(backbone, dataset="kitti_3d", keys=None, **kw):
    cfg = get_cfg(backbone, dataset, **kw)
    for k, v in (keys or {}).items():
        set_key(cfg, k, v)
    return cfg


def _nusc_v2_99():
    return _cfg("v2_99", "nuscenes", {"DD3D.INFERENCE.DO_BEV_NMS": True, PRE_NMS_THRESH: 0.01}, meta_arch="NuscenesDD3D")


def _num_classes_cfg():
    cfg = num_classes_oracle.num_classes_cfg("dla34", 26)  # 11 x 26 box3d outputs: the class-gathered predictor
    set_key(cfg, PRE_NMS_THRESH, 0.02)
    return cfg


# name -> (cfg factory, inputs factory, engine options)
CASES = {
    "dla34_sparse_towers": (lambda: _cfg("dla34"), lambda: case_inputs("dla34"), _SPARSE_ON),
    "nusc_v2_99_bev_aggregate": (_nusc_v2_99, lambda: make_nusc_inputs(1, 128, 192, 1266.4), {}),
    "dla_x_46_c": (lambda: dla_oracle.case_cfg("dla_x_46_c"), lambda: dla_oracle.case_inputs("dla_x_46_c"), {}),
    "v2_39_gn_avg": (lambda: _cfg("v2_39", "nuscenes", dict(_GN_AVG, **{PRE_NMS_THRESH: 0.02})),
                     lambda: make_inputs(2, 128, 192, 1266.4), {}),
    "in_features_p3_p6": (lambda: in_features_oracle.case_cfg("dla34_p3_p6"),
                          lambda: in_features_oracle.case_inputs("dla34_p3_p6"), {}),
    "num_classes_26_gathered": (lambda: _num_classes_cfg(), lambda: ragged_inputs(*num_classes_oracle.NUM_CLASSES_CASE),
                                dict(sparse_box3d=1)),
    "dla34_fp16": (lambda: _cfg("dla34", act_dtype="fp16"), lambda: case_inputs("dla34"), {}),
    "dla34_dense_towers": (lambda: _cfg("dla34"), lambda: case_inputs("dla34"), _SPARSE_OFF),
}


def _model(cfg, options):
    cls = NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200
    m = cls(cfg).to("cuda")
    m.load_state_dict(make_state_dict(cfg))
    for k, v in options.items():
        m.set_engine_option(k, v)
    return m


def _bound(model, inputs):
    """The device buffers a deployment keeps: images, intrinsics, sizes (+ poses and groups), from batched inputs."""
    batch, K, sizes, _, _ = model._gather_inputs(inputs, model.device)
    d = dict(images=batch.cuda().contiguous(), intrinsics=K.cuda().contiguous(), sizes=sizes.cuda().contiguous())
    if model.do_bev_nms or isinstance(model, NuscenesDD3DB200):
        d["poses"] = model._gather_poses(inputs).cuda()
    if isinstance(model, NuscenesDD3DB200) and model._groups is not None:
        d["groups"] = list(model._groups)
    return d


def _capture(model, bound):
    return model.capture_forward(bound["images"], bound["intrinsics"], bound["sizes"], poses=bound.get("poses"),
                                 groups=bound.get("groups"))


def _eager(model, graph):
    """dd3d_forward through the same handle on the graph's bound buffers, into fresh output buffers: (dets, counts, flags,
    global rows) on the host, only the valid rows of each image."""
    L, h = lib.load(), model._handle
    b = graph._buffers
    B = b["images"].shape[0]
    cap = model._desc.out_cap
    out = torch.empty((B, cap, lib.DET_WORDS), dtype=torch.float32, device="cuda")
    counts = torch.zeros(B + 1, dtype=torch.int32, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    lib.check(L.dd3d_forward(h, C.c_void_p(b["images"].data_ptr()),
                             lib.IMG_U8 if b["images"].dtype == torch.uint8 else lib.IMG_F32,
                             C.c_void_p(b["intrinsics"].data_ptr()), C.c_void_p(b["sizes"].data_ptr()),
                             C.c_void_p(out.data_ptr()), C.c_void_p(counts.data_ptr()), stream), h)
    lib.check(L.dd3d_copy_flags(h, C.c_void_p(counts[B:].data_ptr()), stream), h)
    return _host(out, counts[:B], counts[B:], graph.global_rows)


def _host(out, counts, flags, glob):
    torch.cuda.synchronize()
    c = counts.cpu()
    dets = [out[b, :n].cpu().view(torch.int32).clone() for b, n in enumerate(c.tolist())]
    rows = None if glob is None else [glob[b, :n].cpu().view(torch.int32).clone() for b, n in enumerate(c.tolist())]
    return dets, c.clone(), flags.cpu().clone(), rows


def _replay(graph, stream=None):
    graph.launch(stream)
    return _host(*graph.outputs(), graph.global_rows)


def _same(a, b):
    dets_a, counts_a, flags_a, rows_a = a
    dets_b, counts_b, flags_b, rows_b = b
    assert torch.equal(counts_a, counts_b) and torch.equal(flags_a, flags_b), (counts_a, counts_b, flags_a, flags_b)
    for x, y in zip(dets_a, dets_b):
        assert torch.equal(x, y)
    assert (rows_a is None) == (rows_b is None)
    for x, y in zip(rows_a or [], rows_b or []):
        assert torch.equal(x, y)


def _fill_sentinel(graph):
    out, counts, flags = graph.outputs()
    for t in (out, counts, flags) + (() if graph.global_rows is None else (graph.global_rows, )):
        t.view(torch.int32).fill_(SENTINEL)
    torch.cuda.synchronize()


def _is_sentinel(graph):
    torch.cuda.synchronize()
    out, counts, flags = graph.outputs()
    return bool((out.view(torch.int32) == SENTINEL).all() and (counts == SENTINEL).all() and (flags == SENTINEL).all())


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    make_cfg, make_case_inputs, options = CASES[request.param]
    cfg = make_cfg()
    model = _model(cfg, options)
    inputs = make_case_inputs()
    bound = _bound(model, inputs)
    graph = _capture(model, bound)
    yield request.param, model, bound, graph
    graph.close()
    model._release()


def test_replay_matches_eager_bit_for_bit(case):
    name, model, _, graph = case
    ref = _eager(model, graph)
    _fill_sentinel(graph)
    got = _replay(graph)
    _same(ref, got)
    assert int(got[1].sum()) > 0, name  # the case exercises the decode and the NMS
    assert int(got[2][0]) == 0
    if name == "nusc_v2_99_bev_aggregate":
        assert got[3] is not None and sum(len(r) for r in got[3]) > 0
    _same(ref, _replay(graph))  # and again: the tickets and the flags word start every replay as the first one


def test_graph_holds_the_forward_launches_with_programmatic_edges(case):
    _, model, _, graph = case
    n = model.launches_per_forward()
    assert graph.kernel_nodes == n > 0
    # every launch behind the first one of the forward is a PDL launch except the BEV NMS / sample aggregation kernels
    if os.environ.get("DD3D_NO_PDL", "0") in ("", "0"):
        assert 0 < graph.programmatic_edges <= n - 1
    else:
        assert graph.programmatic_edges == 0


def test_replay_reads_the_bound_buffers_at_every_launch(case):
    _, model, bound, graph = case
    images = bound["images"]
    original = images.clone()
    try:
        for frame in (original.flip(-1), original.roll(37, dims=-1), 255 - original if images.dtype == torch.uint8
                      else 255.0 - original):
            images.copy_(frame)
            torch.cuda.synchronize()
            got = _replay(graph)
            _same(_eager(model, graph), got)
    finally:
        images.copy_(original)
        torch.cuda.synchronize()


def _dla34():
    cfg = _cfg("dla34")
    model = _model(cfg, {})
    return model, _bound(model, case_inputs("dla34"))


def test_stale_graphs_launch_nothing_and_a_new_capture_matches_again():
    model, bound = _dla34()
    L = lib.load()
    B, _, H, W = bound["images"].shape
    graph = _capture(model, bound)
    h = model._handle

    def replan_other_shape():
        lib.check(L.dd3d_plan(h, B, H, W + 64, None, 0), h)
        lib.check(L.dd3d_plan(h, B, H, W, None, 0), h)  # back to the captured shape: still stale

    actions = {"dd3d_plan": replan_other_shape,
               "dd3d_set_bev_nms": lambda: lib.check(L.dd3d_set_bev_nms(h, 0, C.c_float(0.1)), h),
               "do_postprocess": lambda: lib.check(L.dd3d_set_option(h, b"do_postprocess", 1), h)}
    for what, act in actions.items():
        act()
        _fill_sentinel(graph)
        assert L.dd3d_graph_launch(graph._graph, None) == DD3D_ERR_STATE, what
        assert b"stale" in L.dd3d_last_error(None) and b"stale" in L.dd3d_last_error(h)
        with pytest.raises(RuntimeError, match="stale"):
            graph.launch()
        assert _is_sentinel(graph), what
        graph.close()
        graph = _capture(model, bound)
        _same(_eager(model, graph), _replay(graph))
    graph.close()
    model._release()


def test_refusals_leave_no_capturing_stream():
    L = lib.load()
    model, bound = _dla34()
    s = torch.cuda.Stream()
    args = [C.c_void_p(bound[k].data_ptr()) for k in ("images", "intrinsics", "sizes")]
    out = torch.empty((1, model._desc.out_cap, lib.DET_WORDS), device="cuda")
    counts = torch.zeros(2, dtype=torch.int32, device="cuda")
    g = C.c_void_p(1)

    def create(h):
        return L.dd3d_graph_create(h, args[0], lib.IMG_U8, args[1], args[2], C.c_void_p(out.data_ptr()),
                                   C.c_void_p(counts.data_ptr()), C.c_void_p(s.cuda_stream), C.byref(g))

    with torch.cuda.stream(s):
        # before dd3d_plan
        h = model._engine()
        assert create(h) == DD3D_ERR_STATE and g.value is None
        assert b"plan" in L.dd3d_last_error(h)
        assert not torch.cuda.is_current_stream_capturing()
        # with profiling on
        model.set_profile(True)
        with pytest.raises(RuntimeError, match="profile"):
            _capture(model, bound)
        assert not torch.cuda.is_current_stream_capturing()
        model.set_profile(False)
        # a forward that fails inside the capture (BEV NMS on, no poses): the capture is ended and discarded
        lib.check(L.dd3d_set_bev_nms(h, 1, C.c_float(0.1)), h)
        lib.check(L.dd3d_set_poses(h, None), h)
        lib.check(L.dd3d_plan(h, *bound["images"].shape[:1], *bound["images"].shape[2:], None, 0), h)
        assert create(h) == DD3D_ERR_STATE and g.value is None
        assert b"graph capture" in L.dd3d_last_error(h) and b"poses" in L.dd3d_last_error(h)
        assert not torch.cuda.is_current_stream_capturing()
        lib.check(L.dd3d_set_bev_nms(h, 0, C.c_float(0.1)), h)
    # the engine still runs eagerly and captures afterwards
    model._plan_key = None
    graph = _capture(model, bound)
    _same(_eager(model, graph), _replay(graph))
    # destroying the handle makes its graphs stale; the graph is still freed by close()
    _fill_sentinel(graph)
    model._release()
    assert L.dd3d_graph_launch(graph._graph, None) == DD3D_ERR_STATE
    assert b"handle was destroyed" in L.dd3d_last_error(None)
    assert _is_sentinel(graph)
    graph.close()


def test_two_graphs_and_another_stream():
    model, bound = _dla34()
    g1 = _capture(model, bound)
    g2 = _capture(model, bound)
    ref = _eager(model, g1)
    _fill_sentinel(g1)
    _fill_sentinel(g2)
    g1.launch()
    g2.launch()  # back to back on one stream
    _same(ref, _host(*g1.outputs(), None))
    _same(ref, _host(*g2.outputs(), None))
    other = torch.cuda.Stream()
    with torch.cuda.stream(other):
        g3 = _capture(model, bound)  # captured on `other` ...
    _fill_sentinel(g3)
    g3.launch(torch.cuda.current_stream())  # ... launched on the default stream
    _same(ref, _host(*g3.outputs(), None))
    side = torch.cuda.Stream()
    _fill_sentinel(g1)
    side.wait_stream(torch.cuda.current_stream())
    g1.launch(side)  # captured on the default stream, launched on a side stream
    side.synchronize()
    _same(ref, _host(*g1.outputs(), None))
    for g in (g1, g2, g3):
        g.close()
    model._release()


def test_c_example_graph_flag_prints_the_same_lines(tmp_path):
    cfg = get_cfg("dla34", "kitti_3d")
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    path = tmp_path / "dla34.dd3d"
    model.save_model_file(str(path))
    x = make_inputs(1, 192, 320, 721.5)[0]
    image = tmp_path / "image.bgr"
    image.write_bytes(x["image"].contiguous().numpy().tobytes())
    subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "examples"), f"OUT={tmp_path}"], check=True)
    K = ["%.9g" % float(v) for v in x["intrinsics"].reshape(-1)]
    runs = [subprocess.run([str(tmp_path / "dd3d_infer"), *flag, str(path), str(image), "192", "320", *K],
                           capture_output=True, text=True, timeout=600) for flag in ([], ["-g"])]
    for r in runs:
        assert r.returncode == 0, r.stderr
    assert runs[0].stdout == runs[1].stdout
    assert int(runs[0].stdout.splitlines()[0].split()[0]) > 0
