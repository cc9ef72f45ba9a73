"""NuscenesDD3D sample aggregation as the engine's last step (dd3d_set_sample_aggregate): bit-identical to the forward
followed by dd3d_op_sample_aggregate on the default config, the same results on every forward path, the blocked path on
sets beyond the one-CTA kernel against the CPU oracle, the launch / op / workspace accounting, workspace poisoning and
batch independence."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import bev_nms_oracle as BO
from util import det_key, quat_dist

pytestmark = pytest.mark.gpu

H, W, FOCAL = 128, 192, 1266.4
TOKENS_18 = ["a", "a", "a", "b", "b", "b", "c", "c", "c", "a", "a", "a", "b", "b", "b", "c", "c", "c"]


def _cfg(**inf):
    from dd3d_b200.config import get_cfg
    cfg = get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D")
    cfg.INPUT.AUG_ENABLED = False  # forward_raw without a resize: the raw images are the mapped ones
    for k, v in inf.items():
        if k == "DO_NMS":
            cfg.DD3D.INFERENCE.DO_NMS = v
        else:
            setattr(cfg.DD3D.FCOS2D.INFERENCE, k, v)
    return cfg


_SD = {}


def _model(cfg):
    from dd3d_b200.meta_arch import NuscenesDD3DB200
    from dd3d_b200.synthetic import make_state_dict
    if "sd" not in _SD:
        _SD["sd"] = make_state_dict(cfg)
    m = NuscenesDD3DB200(cfg).to("cuda")
    m.load_state_dict(_SD["sd"])
    return m


@pytest.fixture(scope="module")
def model():
    return _model(_cfg())


def _inputs(num_samples, tokens=None, seed=1):
    """num_samples 6-camera samples; tokens (optional) interleave the samples' images across the call."""
    from dd3d_b200.synthetic import make_nusc_inputs
    inputs = make_nusc_inputs(num_samples, H, W, FOCAL, seed_base=seed)
    for x in inputs:
        x["height"], x["width"] = H, W
    if tokens is not None:
        for x, t in zip(inputs, tokens):
            x["sample_token"] = t
    return inputs


def _groups(inputs):
    from dd3d_b200.meta_arch import group_indices
    return group_indices([x["sample_token"] for x in inputs], 6)


def _parent_route(model, inputs):
    """The route before the step existed: dd3d_forward (aggregation off) then dd3d_op_sample_aggregate on its output."""
    from dd3d_b200 import lib
    L = lib.load()
    model.sample_aggregate_in_inference = False
    try:
        r = model._forward_device(inputs)
    finally:
        model.sample_aggregate_in_inference = True
    B, cap = r["B"], r["cap"]
    groups = _groups(inputs)
    d_poses = model._gather_poses(inputs).cuda()
    d_group = torch.tensor(groups, dtype=torch.int32).cuda()
    glob = torch.zeros((B, cap, 10), dtype=torch.float32, device="cuda")
    scratch = torch.empty(int(L.dd3d_op_sample_aggregate_scratch_bytes(B, cap)), dtype=torch.uint8, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    lib.check(L.dd3d_op_sample_aggregate(C.c_void_p(r["out"].data_ptr()), C.c_void_p(r["counts"].data_ptr()),
                                         C.c_void_p(r["d_K"].data_ptr()), C.c_void_p(d_poses.data_ptr()),
                                         C.c_void_p(d_group.data_ptr()), max(groups) + 1, C.c_void_p(glob.data_ptr()),
                                         C.c_void_p(scratch.data_ptr()), C.c_void_p(flags.data_ptr()), B, cap,
                                         float(model.bev_nms_iou_thresh), int(model.max_num_dets_per_sample or 0),
                                         C.c_void_p(r["stream"])))
    torch.cuda.synchronize()
    assert int(flags.item()) == 0 and int(r["counts"][B].item()) == 0
    return r["out"].cpu(), r["counts"][:B].cpu(), glob.cpu()


def _step_route(model, inputs):
    r = model._forward_device(inputs)
    torch.cuda.synchronize()
    B = r["B"]
    assert int(r["counts"][B].item()) == 0
    return r["out"].cpu(), r["counts"][:B].cpu(), r["d_poses"].glob.cpu()


def _assert_same_rows(a, b):
    (oa, ca, ga), (ob, cb, gb) = a, b
    assert torch.equal(ca, cb)
    for i, n in enumerate(ca.tolist()):
        assert torch.equal(oa[i, :n].view(torch.int32), ob[i, :n].view(torch.int32)), i
        assert torch.equal(ga[i, :n].view(torch.int32), gb[i, :n].view(torch.int32)), i


def _vec(inst):
    b3 = inst.pred_boxes3d  # the stored fields (tvec is derived with the inverse intrinsics on the result's device)
    return torch.cat([inst.pred_boxes.tensor, inst.scores[:, None], inst.scores_3d[:, None],
                      inst.pred_classes[:, None].float(), inst.locations, b3.quat, b3.proj_ctr, b3.depth.reshape(-1, 1),
                      b3.size,
                      inst.pred_attributes[:, None].float(), inst.pred_speeds[:, None],
                      inst.pred_boxes3d_global.vectorize()], 1).cpu()


def _rows_in_key_order(v):
    return v[sorted(range(v.shape[0]), key=lambda i: tuple(v[i].tolist()))] if v.shape[0] else v


def _assert_same_instances(a, b, ordered=True):
    """Bit-identical instances; ordered=False: as sets of rows (without the 2-D NMS the per-image candidate order is the
    decode's unsorted top-k, which differs from forward to forward, and the aggregation keeps the order it receives)."""
    assert len(a) == len(b)
    for x, y in zip(a, b):
        ix, iy = x["instances"], y["instances"]
        assert tuple(ix.image_size) == tuple(iy.image_size)
        vx, vy = _vec(ix), _vec(iy)
        if not ordered:
            vx, vy = _rows_in_key_order(vx), _rows_in_key_order(vy)
        assert torch.equal(vx, vy)


@pytest.mark.parametrize("n", [6, 18])
def test_parity_with_forward_then_operator(model, n):
    from dd3d_b200 import lib
    assert lib.load().dd3d_sample_aggregate_path(model._desc) == lib.AGG_PATH_ONE_CTA
    inputs = _inputs(n // 6, TOKENS_18[:n] if n == 18 else None)
    ref = _parent_route(model, inputs)
    got = _step_route(model, inputs)
    assert int(got[1].sum()) > 0
    _assert_same_rows(got, ref)


def test_every_forward_path_agrees(model):
    inputs = _inputs(3, TOKENS_18)
    dev = model(inputs)
    assert model.overflow_flags() == 0
    assert all(x["instances"].has("pred_boxes3d_global") for x in dev)
    assert sum(len(x["instances"]) for x in dev) > 0
    _assert_same_instances(model.forward_host(inputs), dev)
    model.submit_host(inputs, 0)
    model.submit_host(inputs, 1)
    s0, s1 = model.wait_host(0), model.wait_host(1)
    _assert_same_instances(s0, dev)
    _assert_same_instances(s1, dev)
    raws = [dict(image_hwc=x["image"].permute(1, 2, 0).contiguous().numpy(), intrinsics=x["intrinsics"],
                 sample_token=x["sample_token"], pose=x["pose"]) for x in inputs]
    _assert_same_instances(model.forward_raw(raws), dev)
    # the test hook switches the step off on every path: per-image detections, no global rows
    model.sample_aggregate_in_inference = False
    try:
        pre_dev, pre_host = model(inputs), model.forward_host(inputs)
        assert not any(x["instances"].has("pred_boxes3d_global") for x in pre_dev + pre_host)
        assert sum(len(x["instances"]) for x in pre_dev) > sum(len(x["instances"]) for x in dev)
    finally:
        model.sample_aggregate_in_inference = True


def _blocked_launches(B):
    key_bits = 32 + (B * 128).bit_length()
    return 2 + 3 * ((key_bits + 7) // 8) + 4


def test_launches_ops_workspace(model):
    from dd3d_b200 import lib
    L = lib.load()
    inputs = _inputs(1)
    model(inputs)
    h = model._handle
    on = (L.dd3d_num_ops(h), L.dd3d_launches_per_forward(h), L.dd3d_workspace_bytes(h, 6, H, W))
    model.sample_aggregate_in_inference = False
    try:
        model(inputs)
        off = (L.dd3d_num_ops(h), L.dd3d_launches_per_forward(h), L.dd3d_workspace_bytes(h, 6, H, W))
    finally:
        model.sample_aggregate_in_inference = True
    assert on[0] == off[0] and on[1] == off[1] + 2 and on[2] > off[2]
    # off equals an engine that never heard of the step
    fresh = _model(_cfg())
    fresh.sample_aggregate_in_inference = False
    fresh(inputs)
    hf = fresh._handle
    assert (L.dd3d_num_ops(hf), L.dd3d_launches_per_forward(hf), L.dd3d_workspace_bytes(hf, 6, H, W)) == off
    # the profile books the step under category 7
    model.set_profile(True)
    model(inputs)
    prof = model.get_profile()
    model.set_profile(False)
    model.sample_aggregate_in_inference = False
    model.set_profile(True)
    model(inputs)
    prof_off = model.get_profile()
    model.set_profile(False)
    model.sample_aggregate_in_inference = True
    assert prof["nms"]["launches"] == prof_off["nms"]["launches"] + 2
    # DD3D: the switch off leaves ops, launches and workspace as they were
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_inputs, make_state_dict
    dcfg = get_cfg("dla34", "kitti_3d")
    dm = DD3DB200(dcfg).to("cuda")
    dm.load_state_dict(make_state_dict(dcfg))
    dm(make_inputs(2, 96, 320, 721.5))
    hd = dm._handle
    before = (L.dd3d_num_ops(hd), L.dd3d_launches_per_forward(hd), L.dd3d_workspace_bytes(hd, 2, 96, 320))
    lib.check(L.dd3d_set_sample_aggregate(hd, 0, 0.3, 0), hd)
    assert L.dd3d_num_ops(hd) == before[0]  # the plan survives a no-op switch
    lib.check(L.dd3d_set_sample_aggregate(hd, 1, 0.3, 0), hd)
    assert L.dd3d_num_ops(hd) < 0  # turning it on drops the plans
    lib.check(L.dd3d_plan(hd, 2, 96, 320, None, 0), hd)
    assert L.dd3d_launches_per_forward(hd) == before[1] + 2  # DLA-34 kitti config: one-CTA path
    lib.check(L.dd3d_set_sample_aggregate(hd, 0, 0.3, 0), hd)
    lib.check(L.dd3d_plan(hd, 2, 96, 320, None, 0), hd)
    assert (L.dd3d_num_ops(hd), L.dd3d_launches_per_forward(hd), L.dd3d_workspace_bytes(hd, 2, 96, 320)) == before


def test_state_errors(model):
    """A forward with the step on but without poses, groups or global rows returns DD3D_ERR_STATE."""
    from dd3d_b200 import lib
    L = lib.load()
    inputs = _inputs(1)
    model(inputs)  # step on, plan made
    h = model._handle
    r = model._forward_device(inputs)  # operands registered: fine
    torch.cuda.synchronize()
    agg = r["d_poses"]
    B, cap = 6, model._desc.out_cap
    out = torch.empty((B, cap, 24), device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    d_img = torch.zeros((B, 3, H, W), dtype=torch.uint8, device="cuda")
    d_sizes = torch.tensor([[H, W, H, W]] * B, dtype=torch.int32, device="cuda")
    stream = C.c_void_p(r["stream"])

    def fwd():
        return L.dd3d_forward(h, C.c_void_p(d_img.data_ptr()), lib.IMG_U8, C.c_void_p(r["d_K"].data_ptr()),
                              C.c_void_p(d_sizes.data_ptr()), C.c_void_p(out.data_ptr()), C.c_void_p(cnt.data_ptr()), stream)

    lib.check(L.dd3d_set_groups(h, None, 0), h)
    assert fwd() == -2
    lib.check(L.dd3d_set_groups(h, C.c_void_p(agg.group.data_ptr()), 1), h)
    lib.check(L.dd3d_set_global_out(h, None), h)
    assert fwd() == -2
    lib.check(L.dd3d_set_global_out(h, C.c_void_p(agg.glob.data_ptr())), h)
    lib.check(L.dd3d_set_poses(h, None), h)
    assert fwd() == -2
    lib.check(L.dd3d_set_poses(h, C.c_void_p(agg.poses.data_ptr())), h)
    assert L.dd3d_set_groups(h, C.c_void_p(agg.group.data_ptr()), 0) == -1
    lib.check(fwd(), h)
    torch.cuda.synchronize()
    # host path of a new engine: slot 0 never received its group indices / global-row buffer
    model._release()
    model(inputs)
    h = model._handle
    h_img = torch.zeros((B, 3, H, W), dtype=torch.uint8).pin_memory()
    h_K = torch.eye(3).repeat(B, 1, 1).reshape(B, 9).contiguous()
    h_sizes = d_sizes.cpu()
    h_out = torch.empty((B, cap, 24)).pin_memory()
    h_cnt = torch.zeros(B, dtype=torch.int32).pin_memory()
    st = L.dd3d_forward_host(h, C.c_void_p(h_img.data_ptr()), lib.IMG_U8, C.c_void_p(h_K.data_ptr()),
                             C.c_void_p(h_sizes.data_ptr()), C.c_void_p(h_out.data_ptr()), C.c_void_p(h_cnt.data_ptr()),
                             stream)
    assert st == -2


def test_poison_and_batch_independence(model):
    inputs = _inputs(3, TOKENS_18, seed=5)
    model.max_num_dets_per_sample = 0  # no cap: a sample's survivors cannot depend on the other samples
    try:
        ref = _step_route(model, inputs)
        model.set_engine_option("workspace_fill", 255)
        poisoned = _step_route(model, inputs)
        model.set_engine_option("workspace_fill", -1)
        _assert_same_rows(poisoned, ref)
        out, cnt, glob = ref
        for tok in "abc":
            idx = [i for i, t in enumerate(TOKENS_18) if t == tok]
            o, c, g = _step_route(model, [inputs[i] for i in idx])
            _assert_same_rows((o, c, g), (out[idx], cnt[idx], glob[idx]))
    finally:
        model.max_num_dets_per_sample = 500
        model.set_engine_option("workspace_fill", -1)


def _pre_dicts(out):
    res = []
    for o in out:
        inst = o["instances"]
        b3 = inst.pred_boxes3d
        res.append(dict(score3d=inst.scores_3d.cpu(), cls=inst.pred_classes.cpu(), loc=inst.locations.cpu(),
                        level=inst.fpn_levels.cpu(), quat=b3.quat.cpu(), tvec=b3.tvec.cpu(), size=b3.size.cpu()))
    return res


LARGE = {
    "nonms": dict(DO_NMS=False, PRE_NMS_TOPK=40, PRE_NMS_THRESH=0.01),
    "post300": dict(POST_NMS_TOPK=300, PRE_NMS_TOPK=60, PRE_NMS_THRESH=0.01),
    "post1000": dict(POST_NMS_TOPK=1000, PRE_NMS_TOPK=60, PRE_NMS_THRESH=0.01),
}


@pytest.mark.parametrize("case", list(LARGE))
def test_blocked_path_vs_oracle(case):
    from dd3d_b200 import lib
    from oracle.dd3d_oracle import pose_of
    L = lib.load()
    cfg = _cfg(**LARGE[case])
    model = _model(cfg)
    assert L.dd3d_sample_aggregate_path(model._desc) == lib.AGG_PATH_BLOCKED
    sorted_input = cfg.DD3D.INFERENCE.DO_NMS  # the 2-D NMS output is in scores_3d order, the decode's top-k is not
    inputs = _inputs(1, seed=3)
    model.sample_aggregate_in_inference = False
    pre = _pre_dicts(model(inputs))
    model.sample_aggregate_in_inference = True
    n_pre = sum(p["score3d"].shape[0] for p in pre)
    print(f"{case}: {n_pre} boxes enter the aggregation of the sample")
    assert n_pre > 768  # beyond the one-CTA kernel's group
    thr = cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH
    poses = [pose_of(x) for x in inputs]
    full = BO.sample_aggregate(pre, [0] * 6, poses, thr, None)
    n_surv = sum(r["score3d"].shape[0] for r in full)
    for max_dets in (500, 7, 0):
        model.max_num_dets_per_sample = max_dets
        got = model(inputs)
        assert model.overflow_flags() == 0
        ref = BO.sample_aggregate(pre, [0] * 6, poses, thr, max_dets) if max_dets and max_dets < n_surv else full
        total = 0
        for o, r in zip(got, ref):
            inst = o["instances"]
            m = len(inst)
            total += m
            assert m == r["score3d"].shape[0]
            g = inst.pred_boxes3d_global
            got_rows = dict(key=[det_key(*k) for k in zip(inst.fpn_levels.cpu(), inst.locations.cpu(), inst.pred_classes.cpu())],
                            score3d=inst.scores_3d.cpu(), quat=g.quat.cpu(), tvec=g.tvec.cpu(), size=g.size.cpu())
            ref_rows = dict(key=[det_key(*k) for k in zip(r["level"], r["loc"], r["cls"])], score3d=r["score3d"],
                            quat=r["quat_global"], tvec=r["tvec_global"], size=r["size"])
            if not sorted_input:  # the same survivors; their order is the (unsorted) order the step received
                at = {k: i for i, k in enumerate(ref_rows["key"])}
                assert sorted(got_rows["key"]) == sorted(ref_rows["key"])
                perm = torch.tensor([at[k] for k in got_rows["key"]], dtype=torch.long)
                ref_rows = {k: ([v[i] for i in perm.tolist()] if k == "key" else v[perm]) for k, v in ref_rows.items()}
            assert got_rows["key"] == ref_rows["key"]  # the same survivors in the same order
            assert torch.equal(got_rows["score3d"], ref_rows["score3d"])
            if m:
                assert quat_dist(got_rows["quat"], ref_rows["quat"]).max().item() < 1e-5
                np.testing.assert_allclose(got_rows["tvec"].numpy(), ref_rows["tvec"].numpy(), rtol=1e-5, atol=1e-4)
                np.testing.assert_allclose(got_rows["size"].numpy(), ref_rows["size"].numpy(), rtol=0, atol=0)
        assert total == (min(max_dets, n_surv) if max_dets else n_surv)
    # every forward path runs the blocked step too
    dev = model(inputs)
    _assert_same_instances(model.forward_host(inputs), dev, ordered=sorted_input)
    launches = L.dd3d_launches_per_forward(model._handle)
    model.sample_aggregate_in_inference = False
    model(inputs)
    assert launches == L.dd3d_launches_per_forward(model._handle) + _blocked_launches(6)
