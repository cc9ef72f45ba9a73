"""The 3-D box decode (decode_one, csrc/decode.cu) against the float64 reference of tests/box3d_cases.py (-m gpu).

dd3d_op_detect_flags runs on the constructed head maps of every configuration: the 16 combinations of
FEATURE_LOCATIONS_OFFSET half, PREDICT_DISTANCE, PREDICT_ALLOCENTRIC_ROT and SCALE_DEPTH_BY_FOCAL_LENGTHS, class-agnostic
3-D maps, NuscenesDD3D attribute / speed channels and BOX3D_ON = 0.  The pre-NMS records, matched to the reference by
their `index` word, must meet the bounds of box3d_cases.compare:
  bit-exact  box, proj_ctr, loc, score, cls, level, index, attr, speed, and depth where the reference clamps;
  depth      relative error <= 1e-6;
  score3d    <= 4 ulps (the device sigmoid uses expf);
  size       |delta| <= 2^-21 * canonical size (tanh + 1 cancels for negative logits, in any float32 decode);
  quat       norm within 1e-6 of 1; rotation distance min(|q - r|, |q + r|) <= 4e-6 except on rays 60-80 degrees off
             axis (reported: the float32 Gram-Schmidt step loses accuracy there); and where the float64
             matrix_to_quaternion candidates are more than 1e-3 from a tie, pytorch3d's sign (q . r > 0).
Every record the NMS writes carries the 3-D fields of its pre-NMS record bit for bit, through both NMS paths, and the two
paths write the same detections.  Each configuration prints one `box3d-worst` JSON line: the worst error per family and
field."""
import ctypes as C
import json

import numpy as np
import pytest
import torch

import box3d_cases as B3
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg

pytestmark = pytest.mark.gpu


def _desc(case):
    cfg = case.cfg
    d = lib.desc_from_cfg(get_cfg("dla34", "kitti_3d"))
    d.num_classes = case.C
    d.pre_nms_topk = case.topk
    d.pre_nms_thresh = case.thresh
    d.thresh_with_ctr = 1
    d.nms_thresh = case.nms_thresh
    d.post_nms_topk = case.post_topk
    d.out_cap = case.out_cap
    d.do_nms = 1
    d.box3d_on = int(cfg["box3d_on"])
    d.class_agnostic_box3d = int(case.C3 == 1)
    d.feature_locations_offset_half = int(cfg["half"])
    d.predict_distance = int(cfg["distance"])
    d.predict_allocentric_rot = int(cfg["allocentric"])
    d.scale_depth_by_focal_lengths = int(cfg["scale_depth"])
    d.scale_depth_by_focal_lengths_factor = float(B3.DEPTH_FACTOR)
    d.min_depth, d.max_depth = float(B3.MIN_DEPTH), float(B3.MAX_DEPTH)
    for c in range(case.C):
        for k in range(3):
            d.canonical_box3d_sizes[c * 3 + k] = float(case.canon[c, k])
    d.nuscenes_heads = int(cfg["nuscenes"])
    return d


def run(case, parallel):
    """dd3d_op_detect_flags on the case's maps; host (pre [B, 5 * topk, 24], pre_n [B, 5], out [B, out_cap, 24], cnt)."""
    L = lib.load()
    B = case.B
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    cls, box, b3d = [dev(a) for a in case.cls], [dev(a) for a in case.box], [dev(a) for a in case.b3d]
    arr = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    scratch = torch.empty(L.dd3d_op_detect_scratch_bytes(B, case.topk), dtype=torch.uint8, device="cuda")
    pre = torch.zeros(B, 5 * case.topk, 24, dtype=torch.float32, device="cuda")
    pre_n = torch.zeros(B, 5, dtype=torch.int32, device="cuda")
    out = torch.full((B, case.out_cap, 24), -7.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    flags = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    hw = (C.c_int32 * 10)(*[v for q in case.level_hw for v in q])
    st = (C.c_int32 * 5)(*case.strides)
    K = dev(case.K)
    sizes = dev(case.sizes)
    desc = _desc(case)
    try:
        assert L.dd3d_set_conv_policy(b"nms_class_parallel", parallel) == 0
        r = L.dd3d_op_detect_flags(C.byref(desc), B, hw, st, arr(cls), arr(box), arr(b3d), case.cls_pitch,
                                   case.b3d_pitch, p(K), p(sizes), p(scratch), p(pre), p(pre_n), p(out), p(cnt),
                                   p(flags), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert r == 0
        torch.cuda.synchronize()
    finally:
        L.dd3d_set_conv_policy(b"nms_class_parallel", -1)
    assert int(flags) == 0
    return pre.cpu().numpy(), pre_n.cpu().numpy(), out.cpu().numpy(), cnt.cpu().numpy()


def pre_records(case, pre, pre_n):
    """The pre-NMS records in the reference's record order (matched by index); the candidate sets must be equal."""
    r = case.rec
    got = np.empty((len(r["b"]), 24), np.float32)
    for b in range(case.B):
        for l in range(5):
            n = int(pre_n[b, l])
            rows = pre[b, l * case.topk:l * case.topk + n]
            idx = rows.view(np.int32)[:, 20]
            m = (r["b"] == b) & (r["l"] == l)
            assert np.array_equal(np.sort(idx), r["index"][m]), f"image {b} level {l}: candidate set"
            got[m] = rows[np.argsort(idx)]
    return got


@pytest.mark.parametrize("name", list(B3.CONFIGS))
def test_decode_meets_the_float64_bounds(name):
    case = B3.build(B3.CONFIGS[name])
    ref = B3.box3d_ref64(case)
    runs = [run(case, 1), run(case, 0)]
    got = pre_records(case, runs[0][0], runs[0][1])
    worst, fails = B3.compare(got, ref, case.cfg["box3d_on"])
    print("box3d-worst", json.dumps(dict(config=name, worst={f"{k[0]}/{k[1]}": v for k, v in worst.items()})))
    assert not fails, fails

    # NMS: every written record carries its pre-NMS record; boxes only clipped to the (unscaled) output size
    r = case.rec
    pos = {(int(b), int(l), int(i)): k for k, (b, l, i) in enumerate(zip(r["b"], r["l"], r["index"]))}
    gw = got.view(np.uint32)
    for pre, pre_n, out, cnt in runs:
        assert np.array_equal(pre_records(case, pre, pre_n).view(np.uint32), gw)
        for b in range(case.B):
            n = int(cnt[b])
            assert 0 < n <= case.out_cap
            w = out[b, :n]
            wi = w.view(np.int32)
            k = np.array([pos[(b, int(l), int(i))] for l, i in zip(wi[:, 7], wi[:, 20])])
            assert np.array_equal(w.view(np.uint32)[:, 4:24], gw[k, 4:24]), f"image {b}: 3-D fields changed by the NMS"
            h, wd = (np.float32(v) for v in case.sizes[b, 2:4])
            clip = got[k, 0:4].copy()
            clip[:, 0::2] = np.minimum(np.maximum(clip[:, 0::2], np.float32(0)), wd)
            clip[:, 1::2] = np.minimum(np.maximum(clip[:, 1::2], np.float32(0)), h)
            assert np.array_equal(w[:, 0:4], clip), f"image {b}: boxes"
    a, b = runs
    assert np.array_equal(a[3], b[3]), "NMS paths keep different counts"
    assert np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32)), "NMS paths write different detections"
