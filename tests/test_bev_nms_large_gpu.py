"""GPU: the BEV NMS of DD3D.forward on thousands of boxes per image.  The multi-CTA kernels (dd3d_op_bev_nms_large)
against the oracle on constructed scenes, and the BEV NMS as the engine's last op: against the oracle applied to the same
engine's pre-BEV detections, identical on every forward path, and absent from the default op list."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import bev_nms_oracle as B
from oracle import input_oracle as IO
from oracle.dd3d_oracle import DD3DOracle
from test_bev_geom_gpu import _assert_clear_of_threshold, _objects, _record
from test_group_bev_nms import _rig_pose, pack

pytestmark = pytest.mark.gpu

BEV_THR = 0.05
POSES = [([1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0]), ([0.9238795, 0.0, 0.3826834, 0.0], [3.0, -1.0, 2.0])]


def tiled_image(seed, n, thr):
    """n camera-frame detections of one image: tiles of the scene objects of test_bev_geom_gpu (rows of parked cars that
    share long edges, near-duplicate pairs with IoU on both sides of thr, tied scores_3d), 70 m x 50 m apart so that no
    two tiles interact, in a random order (the kernel sorts).  Returns (detections, tile of each, camera pose)."""
    rs = np.random.RandomState(seed)
    q, t = _rig_pose(rs, 0)
    R = B.quaternion_to_matrix(torch.tensor(q, dtype=torch.float32)[None])[0].double().numpy()
    tw = np.array(t)
    fwd = R[:2, 2] / np.linalg.norm(R[:2, 2])
    left = np.array([-fwd[1], fwd[0]])
    rows, tiles, k = [], [], 0
    while len(rows) < n:
        i, j = divmod(k, 16)
        for o in _objects(rs, thr, tw[:2] + fwd * 70.0 * i + left * 50.0 * (j - 8), fwd, False):
            rows.append(_record(o, R, tw))
            tiles.append(k)
        k += 1
    perm = rs.permutation(n)
    rows = [rows[p] for p in perm]
    quat, tvec, size, cls, score = zip(*rows)
    det = dict(quat=torch.stack(quat), tvec=torch.stack(tvec), size=torch.stack(size), cls=torch.tensor(cls),
               score3d=torch.tensor(score, dtype=torch.float32), view=torch.zeros(n, dtype=torch.long))
    return det, torch.tensor(tiles)[torch.as_tensor(perm)], (q, t)


def oracle_keep(det, tile, pose, thr, check=False):
    """bev_nms_image tile by tile (tiles never interact, so the greedy keep set is the union of theirs), in slot order."""
    qg, tg = B.to_global(det["quat"], det["tvec"], *pose)
    rects = B.boxes3d_to_rotated_boxes(qg, tg, det["size"])
    keep = []
    for k in torch.unique(tile).tolist():
        idx = torch.nonzero(tile == k).flatten()
        if check:
            _assert_clear_of_threshold(rects[idx], det["cls"][idx], thr)
        keep.append(idx[B.nms_rotated(rects[idx], det["score3d"][idx], det["cls"][idx], thr)])
    return torch.sort(torch.cat(keep)).values


def run_large(buf, counts, Ks, poses, sizes, thr, post):
    from dd3d_b200 import lib
    L = lib.load()
    Bn, cap = buf.shape[0], buf.shape[1]
    d_d, d_c = buf.cuda(), counts.cuda()
    d_K = Ks.reshape(Bn, 9).contiguous().cuda()
    d_p = torch.tensor([list(q) + list(t) for q, t in poses], dtype=torch.float32).cuda()
    scratch = torch.empty(int(L.dd3d_op_bev_nms_large_scratch_bytes(Bn, cap)), dtype=torch.uint8, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = L.dd3d_op_bev_nms_large(C.c_void_p(d_d.data_ptr()), C.c_void_p(d_c.data_ptr()), C.c_void_p(d_K.data_ptr()),
                                 C.c_void_p(d_p.data_ptr()), C.c_void_p(sizes.cuda().data_ptr()), C.c_void_p(scratch.data_ptr()),
                                 C.c_void_p(flags.data_ptr()), Bn, cap, thr, post,
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return d_d.cpu(), d_c.cpu(), int(flags.item())


@pytest.mark.parametrize("n,thr", [(257, 0.3), (1000, 0.05), (1000, 0.3), (5750, 0.05)])
@pytest.mark.parametrize("post", [0, 1])
def test_large_path_vs_oracle(n, thr, post):
    dets, tiles, poses = [], [], []
    for b in range(2):
        det, tile, pose = tiled_image(10 * n + b, n - 3 * b, thr)
        dets.append(det)
        tiles.append(tile)
        poses.append(pose)
    Ks = torch.tensor([[[1260.0, 0.0, 800.0], [0.0, 1260.0, 450.0], [0.0, 0.0, 1.0]]]).repeat(2, 1, 1)
    buf, counts, packed = pack(dets, Ks[:, None], n)
    buf[:, :, 0:4] = torch.tensor([10.0, 20.0, 200.0, 220.0])  # inside the image: the postprocess only rescales
    sizes = torch.tensor([[900, 1600, 900, 1600], [900, 1600, 1800, 3200]], dtype=torch.int32)
    out, cnt, flags = run_large(buf, counts, Ks, poses, sizes, thr, post)
    assert flags == 0
    for b in range(2):
        keep = oracle_keep(packed[b], tiles[b], poses[b], thr, check=n < 5000)
        assert 0 < len(keep) < counts[b]
        m = int(cnt[b])
        assert m == len(keep)
        assert torch.equal(out.view(torch.int32)[b, :m, 20].long(), keep)  # the same set, in slot order
        assert torch.equal(out[b, :m, 5], packed[b]["score3d"][keep])
        scale = 2.0 if (post and b == 1) else 1.0
        assert torch.equal(out[b, :m, 0:4], torch.tensor([10.0, 20.0, 200.0, 220.0]).expand(m, 4) * scale)


def test_large_path_capacity_flag():
    """A count above cap is reported (bit 6) instead of read past the image's slots."""
    det, tile, pose = tiled_image(3, 300, 0.3)
    Ks = torch.tensor([[[1260.0, 0.0, 800.0], [0.0, 1260.0, 450.0], [0.0, 0.0, 1.0]]])
    buf, counts, _ = pack([det], Ks[:, None], 300)
    counts[0] = 301
    _, _, flags = run_large(buf, counts, Ks, [pose], torch.tensor([[900, 1600, 900, 1600]], dtype=torch.int32), 0.3, 0)
    assert flags == 64


# ------------------------------------------------------------------------------------------------ engine op
CONFIGS = {"no_nms": dict(DO_NMS=False), "post_topk0": dict(POST_NMS_TOPK=0)}


def _model(config, dtype="bf16", bev=True):
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_state_dict
    cfg = get_cfg("dla34", "kitti_3d", act_dtype=dtype)
    for k, v in CONFIGS.get(config, {}).items():
        if k == "DO_NMS":
            cfg.DD3D.INFERENCE.DO_NMS = v
        else:
            setattr(cfg.DD3D.FCOS2D.INFERENCE, k, v)
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.02  # more than 256 boxes per image enter the BEV NMS
    cfg.DD3D.INFERENCE.DO_BEV_NMS = bev
    cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH = BEV_THR
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    return model


def _inputs(seed_base=1, poses=POSES):
    from oracle.gen_golden import case_inputs
    from dd3d_b200.synthetic import make_inputs
    inputs = case_inputs("dla34") if seed_base == 1 else make_inputs(2, 192, 320, 721.5, seed_base=seed_base)
    for x, p in zip(inputs, poses):
        x["pose"] = p
    return inputs


def _canonical(inst):
    """Row order by (level, location, class): with DO_NMS off the order of the candidates inside a level is not fixed
    (the decode appends them with atomics; the reference's topk(sorted=False) fixes none either), and the BEV NMS keeps
    its input order."""
    key = (inst.fpn_levels.cpu().double() * 1e12 + inst.locations[:, 1].cpu().double() * 1e6 +
           inst.locations[:, 0].cpu().double() * 16 + inst.pred_classes.cpu().double())
    return torch.argsort(key)


def _same(a, b, ordered=True):
    for oa, ob in zip(a, b):
        ia, ib = oa["instances"], ob["instances"]
        assert tuple(ia.image_size) == tuple(ib.image_size)
        assert len(ia) == len(ib)
        pa, pb = (slice(None), slice(None)) if ordered else (_canonical(ia), _canonical(ib))
        for f in ("scores", "scores_3d", "pred_classes", "fpn_levels", "locations"):
            assert torch.equal(ia.get(f).cpu()[pa], ib.get(f).cpu()[pb]), f
        assert torch.equal(ia.pred_boxes.tensor.cpu()[pa], ib.pred_boxes.tensor.cpu()[pb])
        assert torch.equal(ia.pred_boxes3d.vectorize().cpu()[pa], ib.pred_boxes3d.vectorize().cpu()[pb])


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_forward_with_large_bev_nms_vs_oracle(config, dtype):
    """DO_BEV_NMS forward == the oracle BEV NMS on the same engine's pre-BEV detections, then detector_postprocess."""
    from dd3d_b200 import lib
    model = _model(config, dtype)
    assert lib.load().dd3d_bev_nms_path(C.byref(model._desc)) == 2
    inputs = _inputs()
    out = model(inputs)
    assert model.last_overflow_flags == 0
    model.do_bev_nms = False
    model.postprocess_in_inference = False
    pre = model(inputs)
    entering, removed = [], 0
    for b, (o, q) in enumerate(zip(out, pre)):
        pi = q["instances"]
        entering.append(len(pi))
        det = dict(quat=pi.pred_boxes3d.quat.cpu(), tvec=pi.pred_boxes3d.tvec.cpu(), size=pi.pred_boxes3d.size.cpu(),
                   score3d=pi.scores_3d.cpu(), cls=pi.pred_classes.cpu(), box2d=pi.pred_boxes.tensor.cpu())
        keep = B.bev_nms_image(det, POSES[b][0], POSES[b][1], BEV_THR)
        removed += len(pi) - len(keep)
        h, w = pi.image_size
        oh, ow = inputs[b].get("height", h), inputs[b].get("width", w)
        ref = DD3DOracle.postprocess({k: v[keep] for k, v in det.items()}, (h, w), (oh, ow))
        inst = o["instances"]
        assert tuple(inst.image_size) == (oh, ow)
        assert len(inst) == ref["box2d"].shape[0]
        # the two forwards may order the candidates of a level differently (DO_NMS off): compare the sets, ordered by
        # scores_3d and class (the BEV NMS keeps its input order either way)
        ka = np.lexsort((inst.pred_classes.cpu().numpy(), inst.scores_3d.cpu().numpy()))
        kb = np.lexsort((ref["cls"].numpy(), ref["score3d"].numpy()))
        assert torch.equal(inst.scores_3d.cpu()[ka], ref["score3d"][kb])
        assert torch.equal(inst.pred_classes.cpu()[ka], ref["cls"][kb])
        np.testing.assert_allclose(inst.pred_boxes.tensor.cpu().numpy()[ka], ref["box2d"].numpy()[kb], rtol=1e-6, atol=1e-4)
    assert max(entering) > 256, entering
    assert removed > 0


@pytest.mark.parametrize("config", ["default"] + list(CONFIGS))
def test_every_entry_point_same_detections(config):
    """forward, forward_host, submit_host / wait_host on alternating slots and forward_raw (against the mapper, then
    forward) return identical Instances under DO_BEV_NMS; two runs are bit-identical."""
    model = _model(config)
    ordered = model.do_nms  # see _canonical
    batches = [_inputs(seed_base=1 + 7 * i, poses=POSES[::1 - 2 * (i % 2)]) for i in range(3)]
    ref = [model(b) for b in batches]
    _same(ref[0], model(batches[0]), ordered)
    for b, r in zip(batches, ref):
        _same(r, model.forward_host(b), ordered)
    got = []
    model.submit_host(batches[0], 0)
    for k in range(3):
        if k + 1 < 3:
            model.submit_host(batches[k + 1], (k + 1) & 1)
        got.append(model.wait_host(k & 1))
    for r, g in zip(ref, got):
        _same(r, g, ordered)
    raws = []
    for x in batches[1]:
        raws.append({"image_hwc": x["image"].permute(1, 2, 0).contiguous().numpy(), "intrinsics": x["intrinsics"],
                     "pose": x["pose"]})
    rs = model.cfg.INPUT.RESIZE
    mapped = [IO.map_input(r, rs.MIN_SIZE_TEST, rs.MAX_SIZE_TEST) for r in raws]
    for m, r in zip(mapped, raws):
        m["pose"] = r["pose"]
    _same(model(mapped), model.forward_raw(raws), ordered)
    assert sum(len(o["instances"]) for o in ref[0]) > 0


def test_bev_off_leaves_the_default_path():
    """Turning the BEV NMS on and off again gives back the default op list, launches and detections, bit for bit."""
    from dd3d_b200 import lib
    L = lib.load()
    model = _model("default", bev=False)
    inputs = _inputs()
    base = model(inputs)
    ops, launches = L.dd3d_num_ops(model._handle), model.launches_per_forward()
    model.do_bev_nms = True
    on = model(inputs)
    assert model.launches_per_forward() == launches + 1  # the one-CTA kernel
    assert sum(len(o["instances"]) for o in on) < sum(len(o["instances"]) for o in base)
    model.do_bev_nms = False
    _same(base, model(inputs))
    assert (L.dd3d_num_ops(model._handle), model.launches_per_forward()) == (ops, launches)
