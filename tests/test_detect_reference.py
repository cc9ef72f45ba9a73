"""CPU checks of the constructed detection cases and the host reference of tests/detect_cases.py: every case keeps its
rankings unambiguous, hits the capacity edge it is built for, and the reference's output changes under each wrong rule
(`>=` at the threshold, index-descending ties, a boundary bin truncated to 4096 entries, `>` after the NMS, `>=` IoU) -- a
negative control showing that tests/test_detect_exact_gpu.py can tell those kernels apart, with no GPU."""
import numpy as np
import pytest

import detect_cases as D


def _differs(case, variant):
    for b in range(case.B):
        r, w = D.reference(case, b), D.reference(case, b, variant)
        if any(len(x) != len(y) or set(x.tolist()) != set(y.tolist()) for x, y in zip(r["pre"], w["pre"])):
            return True
        if r["n_written"] != w["n_written"] or not np.array_equal(r["index"], w["index"]) or \
                not np.array_equal(r["level"], w["level"]):
            return True
    return False


# (case, the wrong rules it must catch)
CONTROLS = {
    "clustered_ctr": (lambda: D.clustered(True, 50, 100), ("boundary_trunc", "index_desc")),
    "tied_ctr": (lambda: D.clustered(True, 1, 5000), ("boundary_trunc", "index_desc")),
    "clustered_cls": (lambda: D.clustered(False, 1100, 4), ("boundary_trunc", "index_desc")),
    "all_tied": (lambda: D.all_tied(True), ("boundary_trunc", "index_desc")),
    "at_threshold_ctr": (lambda: D.at_threshold(True), ("thresh_ge", )),
    "at_threshold_cls": (lambda: D.at_threshold(False), ("thresh_ge", )),
    "saturated": (lambda: D.saturated(64), ("index_desc", )),
    "post_ties": (lambda: D.post_ties(20), ("post_gt", )),
    "iou_half": (lambda: D.iou_edges(0.5), ("iou_ge", )),
    "iou_three_quarters": (lambda: D.iou_edges(0.75), ("iou_ge", )),
}


@pytest.mark.parametrize("name", sorted(CONTROLS))
def test_wrong_rule_changes_the_reference(name):
    build, variants = CONTROLS[name]
    case = build()
    D.check_unambiguous(case)
    for v in variants:
        assert _differs(case, v), f"{name}: the reference does not see the wrong rule {v}"


@pytest.mark.parametrize("with_ctr,distinct,copies", [(True, 50, 100), (True, 1, 5000), (False, 1100, 4),
                                                      (False, 1, 5000)])
def test_clusters_exceed_the_boundary_buffer_in_one_bin(with_ctr, distinct, copies):
    """The k-th score's histogram bin holds more than 4096 candidates: the case reaches the boundary buffer's limit."""
    case = D.clustered(with_ctr, distinct, copies)
    D.check_unambiguous(case)
    tb, shift = D.hist_params(case.thresh, case.with_ctr)
    s, t = case.level_scores(0, 0)
    sv = s[t > case.thresh].astype(np.float32)
    bins = (sv.view(np.uint32).astype(np.int64) - tb) >> shift
    kth = np.sort(sv)[::-1][case.topk - 1]
    T = (int(kth.view(np.uint32)) - tb) >> shift
    assert (bins == T).sum() > D.BOUNDARY_CAP
    assert len(D.reference(case, 0)["pre"][0]) == case.topk


@pytest.mark.parametrize("n_off", [-1, 0, 1])
@pytest.mark.parametrize("topk", [16, 1000])
def test_passing_count_edges(topk, n_off):
    case = D.passing_count(topk + n_off, topk)
    D.check_unambiguous(case)
    assert len(D.reference(case, 0)["pre"][1]) == min(topk, topk + n_off)
    assert len(D.reference(D.passing_count(0, topk), 0)["pre"][1]) == 0


def test_iou_cases_sit_exactly_on_the_threshold():
    """fp32 IoU of the constructed boxes: exactly 0.5 and 0.75 against box A, NaN for the inverted and zero-area pairs."""
    case = D.iou_edges(0.5)
    bx = case.box[0][0, :11, 0:4]
    lx = (np.arange(11) * case.strides[0]).astype(np.float32)
    boxes = np.stack([lx - bx[:, 0], -bx[:, 1], lx + bx[:, 2], bx[:, 3]], 1).astype(np.float32)
    iou = D.iou_f32(boxes[0], boxes[1:5])
    assert iou.tolist() == [0.5, 0.75, 0.5625, 0.8125]
    assert np.isnan(D.iou_f32(boxes[7], boxes[8:9]))[0] and np.isnan(D.iou_f32(boxes[9], boxes[10:11]))[0]
    assert D.iou_f32(boxes[5], boxes[6:7])[0] == 0.0


def test_post_nms_ties_and_out_cap():
    r = D.reference(D.post_ties(20), 0)
    assert r["n_written"] == 110 and not r["flag_overflow"]
    r = D.reference(D.post_ties(60), 0)
    assert r["n_written"] == 128 and r["flag_overflow"]


def test_class_chain_keeps_every_second_box():
    case = D.class_sizes()
    r = D.reference(case, 0)
    for c, n in enumerate((1, 63, 64, 65, 129)):
        assert (r["cls"] == c).sum() == (n + 1) // 2
