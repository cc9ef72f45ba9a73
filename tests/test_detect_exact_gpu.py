"""The detection top-k and NMS kernels (csrc/decode.cu, csrc/nms.cu) against the exact host reference of
tests/detect_cases.py, on constructed head maps (-m gpu): ties, saturated scores, a score on the threshold, levels with
PRE_NMS_TOPK +- 1 candidates, more than the boundary buffer's 4096 candidates in the k-th score's histogram bin, IoUs on
NMS_THRESH, the segment / word edges of the multi-CTA NMS, post-NMS ties past out_cap.  Every integer or choice field --
candidate counts and sets, kept detections, their order, classes, levels, the flags word -- must be equal; both NMS paths
must give bit-identical outputs."""
import ctypes as C

import numpy as np
import pytest
import torch

import detect_cases as D
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg

pytestmark = pytest.mark.gpu


def _desc(case):
    d = lib.desc_from_cfg(get_cfg("dla34", "kitti_3d"))
    d.num_classes = case.C
    d.pre_nms_topk = case.topk
    d.pre_nms_thresh = case.thresh
    d.thresh_with_ctr = int(case.with_ctr)
    d.nms_thresh = case.nms_thresh
    d.post_nms_topk = case.post_topk
    d.out_cap = case.out_cap
    d.do_nms = 1
    d.box3d_on = 1
    d.class_agnostic_box3d = int(case.C3 == 1)
    d.feature_locations_offset_half = 0
    return d


def run(case, parallel, images=None, pad=64, plain=False):
    """dd3d_op_detect_flags on the case's maps (images: a subset of the batch); returns host (pre, pre_n, out, cnt, flags).
    `pad` sentinel records follow the B * out_cap output records and must stay untouched.  plain: through dd3d_op_detect,
    which reports no flags (returned as -1)."""
    L = lib.load()
    sel = list(range(case.B)) if images is None else list(images)
    B = len(sel)
    desc = _desc(case)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a[sel])).cuda()  # noqa: E731
    cls, box, b3d = [dev(a) for a in case.cls], [dev(a) for a in case.box], [dev(a) for a in case.b3d]
    arr = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    scratch = torch.empty(L.dd3d_op_detect_scratch_bytes(B, case.topk), dtype=torch.uint8, device="cuda")
    pre = torch.zeros(B, 5 * case.topk, 24, dtype=torch.float32, device="cuda")
    pre_n = torch.zeros(B, 5, dtype=torch.int32, device="cuda")
    out = torch.full((B * case.out_cap + pad, 24), -7.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((B,), -1, dtype=torch.int32, device="cuda")
    flags = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    hw = (C.c_int32 * 10)(*[v for q in case.level_hw for v in q])
    st = (C.c_int32 * 5)(*case.strides)
    K = torch.tensor([[700.0, 0, 320.0, 0, 700.0, 240.0, 0, 0, 1]]).repeat(B, 1).cuda()
    sizes = torch.from_numpy(case.sizes[sel]).cuda()
    try:
        assert L.dd3d_set_conv_policy(b"nms_class_parallel", parallel) == 0
        args = (C.byref(desc), B, hw, st, arr(cls), arr(box), arr(b3d), case.cls_pitch, case.b3d_pitch, p(K), p(sizes),
                p(scratch), p(pre), p(pre_n), p(out), p(cnt))
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        r = L.dd3d_op_detect(*args, stream) if plain else L.dd3d_op_detect_flags(*args, p(flags), stream)
        assert r == 0
        torch.cuda.synchronize()
    finally:
        L.dd3d_set_conv_policy(b"nms_class_parallel", -1)
    out = out.cpu()
    assert (out[B * case.out_cap:] == -7.0).all(), "records written past B * out_cap"
    return pre.cpu(), pre_n.cpu(), out[:B * case.out_cap].reshape(B, case.out_cap, 24), cnt.cpu(), int(flags)


def check(case, got, images=None):
    pre, pre_n, out, cnt, flags = got
    sel = list(range(case.B)) if images is None else list(images)
    overflow = False
    for j, b in enumerate(sel):
        ref = D.reference(case, b)
        overflow |= ref["flag_overflow"]
        for l in range(5):
            n = int(pre_n[j, l])
            assert n == len(ref["pre"][l]), f"image {b} level {l}: {n} candidates, reference {len(ref['pre'][l])}"
            gi = pre[j, l * case.topk:l * case.topk + n].view(torch.int32)
            idx = np.sort(gi[:, 20].numpy())
            assert np.array_equal(idx, np.sort(ref["pre"][l])), f"image {b} level {l}: candidate set"
            assert (gi[:, 7] == l).all()
        n = int(cnt[j])
        assert n == ref["n_written"], f"image {b}: {n} detections, reference {ref['n_written']}"
        w = out[j, :n]
        wi = w.view(torch.int32)
        assert np.array_equal(wi[:, 7].numpy(), ref["level"]), f"image {b}: levels / order"
        assert np.array_equal(wi[:, 20].numpy(), ref["index"]), f"image {b}: indices / order"
        assert np.array_equal(wi[:, 6].numpy(), ref["cls"])
        assert np.array_equal(w[:, 0:4].numpy(), ref["box"]), f"image {b}: boxes"  # integer arithmetic: exact
        np.testing.assert_allclose(w[:, 4].numpy(), ref["score"], rtol=1e-5)
        np.testing.assert_allclose(w[:, 5].numpy(), ref["score"], rtol=1e-5)
    assert flags == (2 if overflow else 0), f"flags {flags}"


def both_paths(case):
    D.check_unambiguous(case)
    a, b = run(case, 1), run(case, 0)
    check(case, a)
    for x, y in zip((a[2], a[3]), (b[2], b[3])):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "NMS paths differ"
    assert a[4] == b[4]
    return a


@pytest.mark.parametrize("with_ctr,distinct,copies", [(True, 50, 100), (True, 1, 5000), (False, 1100, 4),
                                                      (False, 1, 5000)], ids=["clustered", "tied", "clustered-cls", "tied-cls"])
def test_more_than_the_boundary_buffer_in_one_bin(with_ctr, distinct, copies):
    """> 4096 candidates share the k-th score's histogram bin: exact top-k, no flag (it used to set bit 0 / come short)."""
    both_paths(D.clustered(with_ctr, distinct, copies))


@pytest.mark.parametrize("with_ctr", [True, False])
@pytest.mark.parametrize("topk", [16, 1000, 1150])
def test_whole_levels_of_one_score(with_ctr, topk):
    both_paths(D.all_tied(with_ctr, topk))


def test_plain_entry_point_gives_the_same_detections():
    """dd3d_op_detect (no flags word) runs the same kernels as dd3d_op_detect_flags: bit-identical outputs."""
    case = D.clustered(True, 1, 5000)
    a, b = run(case, 1), run(case, 1, plain=True)
    assert b[4] == -1
    for x, y in zip(a[1:4], b[1:4]):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_topk_beyond_the_nms_capacity_is_refused():
    """PRE_NMS_TOPK 1150 is the largest whose 5 levels of candidates fit the NMS's shared memory; 1151 is refused before
    any launch (it used to be accepted up to 1638 and fail with a CUDA error in the NMS)."""
    case = D.passing_count(10, 1151)
    with pytest.raises(AssertionError, match="-1 == 0"):
        run(case, 1)


@pytest.mark.parametrize("n_off", [-1, 0, 1, None])
@pytest.mark.parametrize("topk", [16, 64, 1000, 1150])
def test_passing_count_around_topk(topk, n_off):
    both_paths(D.passing_count(0 if n_off is None else topk + n_off, topk))


@pytest.mark.parametrize("with_ctr", [True, False])
def test_value_on_the_threshold_is_excluded(with_ctr):
    both_paths(D.at_threshold(with_ctr))


@pytest.mark.parametrize("topk", [16, 64])
def test_saturated_scores_across_classes(topk):
    both_paths(D.saturated(topk))


@pytest.mark.parametrize("topk,seed", [(16, 1), (64, 2), (1000, 3), (1150, 4)])
def test_flooded_levels_with_ties(topk, seed):
    both_paths(D.random_level(topk, seed))


@pytest.mark.parametrize("nms_thresh", [0.5, 0.75])
def test_iou_on_the_threshold_and_degenerate_boxes(nms_thresh):
    both_paths(D.iou_edges(nms_thresh))


def test_class_segments_and_chains_across_blocks():
    both_paths(D.class_sizes())


@pytest.mark.parametrize("n_tied", [20, 60])
def test_post_nms_ties(n_tied):
    """Ties at the 100th 2-D score keep more than 100; past out_cap bit 1 is set and nothing is written beyond it."""
    both_paths(D.post_ties(n_tied))


def test_score3d_ties_across_levels():
    both_paths(D.level_ties())


def test_batch_of_32_at_v2_99_shapes():
    """B = 32 at the V2-99 900x1600 level shapes, a different distribution per image; each image equals its own B = 1
    run bit for bit and the reference."""
    case = D.big_batch(32)
    D.check_unambiguous(case)
    full = run(case, 1)
    check(case, full)
    for b in range(case.B):
        one = run(case, 1, images=[b])
        assert int(one[3][0]) == int(full[3][b])
        n = int(full[3][b])
        assert torch.equal(one[2][0, :n].view(torch.int32), full[2][b, :n].view(torch.int32)), f"image {b}"
        assert torch.equal(one[1][0], full[1][b])


def test_engine_with_constant_heads():
    """DLA-34 DD3DB200 whose cls and centerness predictors have zero weights: every pixel of every level passes with the
    same score (24 x 40 x 5 = 4800 tied candidates at level 0 of a 192x320 image, more than the boundary buffer).  The
    forward returns (it used to raise on bit 0) and its detections equal dd3d_op_detect_flags' on the engine's own head maps."""
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from oracle.gen_golden import case_cfg, case_inputs

    cfg = case_cfg("dla34")
    sd = make_state_dict(cfg)
    # box2d_reg too: every box spans +-1e4 pixels, so the NMS keeps one box per class and out_cap is not reached
    for name, bias in (("cls_logits", 2.0), ("centerness", 1.0), ("box2d_reg", 1e4)):
        sd[f"fcos2d_head.{name}.weight"].zero_()
        sd[f"fcos2d_head.{name}.bias"].fill_(bias)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    L = lib.load()
    h = model._engine()
    for opt in (b"sparse_box3d", b"sparse_tower", b"sparse_box2d_tower"):
        lib.check(L.dd3d_set_option(h, opt, 0), h)
    inputs = case_inputs("dla34")
    r = model._forward_device(inputs)
    torch.cuda.synchronize()
    B = r["B"]
    counts = r["counts"].cpu()
    assert int(counts[B]) == 0, f"engine flags {int(counts[B])}"
    eng = r["out"].reshape(B, -1, 24)[:, :model._desc.out_cap].cpu()
    maps = {n: [model.get_tensor(f"{n}{l}") for l in range(5)] for n in ("cls", "box", "b3d")}
    assert all((m[0, ..., :cfg.DD3D.NUM_CLASSES] == 2.0).all() for m in maps["cls"])
    desc = model._desc
    topk = desc.pre_nms_topk
    arr = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    scratch = torch.empty(L.dd3d_op_detect_scratch_bytes(B, topk), dtype=torch.uint8, device="cuda")
    pre = torch.zeros(B, 5 * topk, 24, dtype=torch.float32, device="cuda")
    pre_n = torch.zeros(B, 5, dtype=torch.int32, device="cuda")
    out = torch.zeros(B, desc.out_cap, 24, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    flags = torch.full((1,), -1, dtype=torch.int32, device="cuda")
    hw = (C.c_int32 * 10)(*[v for m in maps["cls"] for v in m.shape[1:3]])
    st = (C.c_int32 * 5)(8, 16, 32, 64, 128)
    r2 = L.dd3d_op_detect_flags(C.byref(desc), B, hw, st, arr(maps["cls"]), arr(maps["box"]), arr(maps["b3d"]),
                                maps["cls"][0].stride(2), maps["b3d"][0].stride(2), p(r["d_K"]),
                                p(r["sizes"].to("cuda", torch.int32).contiguous()), p(scratch), p(pre), p(pre_n), p(out),
                                p(cnt), p(flags), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert r2 == 0
    torch.cuda.synchronize()
    assert int(flags) == 0
    want = [min(topk, m.shape[1] * m.shape[2] * cfg.DD3D.NUM_CLASSES) for m in maps["cls"]]
    assert (pre_n.cpu() == torch.tensor(want)).all(), (pre_n, want)
    for b in range(B):
        n = int(cnt[b])
        assert n == int(counts[b]) and n > 0
        assert torch.equal(out[b, :n].cpu().view(torch.int32), eng[b, :n].view(torch.int32)), f"image {b}"
