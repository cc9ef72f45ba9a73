"""End-to-end parity at the BASELINE.json shapes (-m gpu; VERDICT r1 weak #1-2): one 900x1600 V2-99 image and one
384x1280 DLA-34 image through DD3DB200.forward and through the CPU oracle (emulating the engine's storage type on ONE
thread, and pure fp32 = the reference's arithmetic), for both storage types.  What is compared and how is described in
tests/parity_lib.py; tools/parity_report.py writes the measured numbers of the same code, and the thresholds below are
those numbers plus margin.

Exactness claims (no tolerance): the preprocessed input, the candidate SETS of the decode kernels and the kept set + order
of the NMS kernel, given the engine's own head maps.  Everything else is bounded by the storage precision of the conv
stack (bf16: 8 mantissa bits, fp16: 11), which the tables make visible: fp16 sits ~8x closer to the fp32 reference."""
import pytest

from parity_lib import measure_case

pytestmark = pytest.mark.gpu

# thresholds = measured parity (tools/parity_report.py) x ~2, per storage type:
#   maps_emu / maps_fp32 : worst relative L2 error over all FPN + head maps vs the emulating / fp32 oracle
#   pre_rate             : matched fraction of the oracle's pre-NMS candidates (emulating oracle)
#   hard                 : unmatched candidates OUTSIDE the threshold / top-k margins, as a fraction of all candidates
#   p99 / max            : error bounds over matched pre-NMS candidates vs the emulating oracle (field -> bound)
#   post_rate_emu / post_rate_golden : matched fraction of the final detections vs emulating oracle / reference goldens
LIMITS = {
    # measured parity of the original build (cases dla34_full / v2_99_full):
    #   bf16: maps 1.22e-2 / 9.2e-3 (emu) 1.42e-2 / 8.8e-3 (fp32); pre-NMS match 0.979 / 0.966, 0 outside the margins;
    #         p99 box 8.0e-3 score 3.5e-3 score3d 1.9e-3 quat 1.9e-2 depth 6.4e-3 size 2.1e-2; post-NMS 0.94 / 0.95 (emu),
    #         0.90 / 0.95 (reference goldens)
    #   fp16: maps 1.67e-3 / 1.17e-3 (emu) 1.74e-3 / 1.17e-3 (fp32); pre-NMS match 0.995 / 0.991, 0 outside the margins;
    #         p99 box 9.4e-4 score 4.7e-4 score3d 1.9e-4 quat 2.3e-3 depth 8.0e-4 size 2.4e-3; post-NMS 0.99 / 1.00, 0.99 / 1.00
    "bf16": dict(maps_emu=2e-2, maps_fp32=2.5e-2, pre_rate=0.94, hard=0.005, post_rate_emu=0.88, post_rate_golden=0.85,
                 p99=dict(box=1.5e-2, score=7e-3, score3d=4e-3, quat=4e-2, depth=1.2e-2, size=4e-2)),
    "fp16": dict(maps_emu=3e-3, maps_fp32=3e-3, pre_rate=0.985, hard=0.003, post_rate_emu=0.97, post_rate_golden=0.97,
                 p99=dict(box=2e-3, score=1e-3, score3d=5e-4, quat=5e-3, depth=1.6e-3, size=5e-3)),
}


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("case", ["dla34_full", "v2_99_full"])
def test_parity_at_baseline_shape(case, dtype):
    rep = measure_case(case, dtype)
    lim = LIMITS[dtype]
    assert rep["input_bit_exact"]
    # decode + NMS kernels vs the oracle on identical (engine) head maps: exact sets / order, fp32-rounding field errors
    hyb = rep["hybrid"]
    assert hyb["candidate_sets_equal"] and hyb["kept_order_equal"] and hyb["forward_equals_operator"], hyb
    # the default (sparse) box3d predictor reproduces the dense one: same detections, same order, 2-D fields bit-equal,
    # 3-D fields within the fp32 summation-order noise of a K = 2304 dot product
    sv = rep["sparse_vs_dense_box3d"]
    assert sv["same_keys_and_order"] and sv["n"] > 0, sv
    assert sv["max_err"]["box"] == 0.0 and sv["max_err"]["score"] == 0.0, sv
    for f in ("score3d", "quat", "proj_ctr", "depth", "size", "tvec"):
        assert sv["max_err"][f] < 2e-5, (f, sv)
    assert hyb["candidates"] > 500 and hyb["kept"] >= 50
    for f, e in hyb["max_err"].items():
        assert e < 1e-5, (f, e)  # measured <= 4e-7: fp32 rounding only
    # conv stack: storage-precision bound
    assert rep["maps"]["emu"]["worst_rel_l2"] < lim["maps_emu"], rep["maps"]["emu"]
    assert rep["maps"]["fp32"]["worst_rel_l2"] < lim["maps_fp32"], rep["maps"]["fp32"]
    pre = rep["pre_nms"]["emu"]
    n = max(pre["sets"]["n_ref"], 1)
    assert pre["sets"]["match_rate"] > lim["pre_rate"], pre["sets"]
    assert (pre["sets"]["missing_outside_margin"] + pre["sets"]["extra_outside_margin"]) / n < lim["hard"], pre["sets"]
    for f, bound in lim["p99"].items():
        assert pre["errors"][f]["p99"] < bound, (f, pre["errors"][f])
    assert rep["post_nms"]["emu"]["sets"]["match_rate"] > lim["post_rate_emu"], rep["post_nms"]["emu"]["sets"]
    assert rep["post_nms"]["reference_golden"]["sets"]["match_rate"] > lim["post_rate_golden"], \
        rep["post_nms"]["reference_golden"]["sets"]
