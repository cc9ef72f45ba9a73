"""The consumer-warpgroup skew of the conv kernel (policy "stagger": 0 = both warpgroups start together, -1 = the default
rule, n = n k-blocks) changes only when each warpgroup runs, never what it computes: on the exact operands of
tests/exact_ops.py every conv variant must equal RN_storage(float64 reference) at every skew, and a whole V2-99 forward
(eSE pool partials handed between the warpgroups, pair tile, work-list towers) must give bit-identical outputs at skew 0
and at the default skew."""
import pytest
import torch

import gpu_ops
from dd3d_b200 import lib
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_inputs, make_state_dict
from test_exact_kernels_gpu import _conv_exact

pytestmark = pytest.mark.gpu

SKEWS = [{"stagger": 0}, {}, {"stagger": 1}, {"stagger": 6}]

# cin, cout, k, stride, B, H, W, relu, residual, fp32 out, channel slices, extra policy -- the layer classes of the V2-99
# benchmark step at reduced maps: generic 1x1 concat (N 256, K 1056), halo OSA 3x3 (N 160 / 192 / 224, K tail), the pair
# tile (tower 256 -> 256, with residual), weight-stationary 64 -> 64, stride 2, the 1 x 128 tile, fp32 predictor output.
CASES = [
    (1056, 512, 1, 1, 2, 29, 50, True, 0, False, False, {}),
    (768, 256, 1, 1, 1, 57, 100, True, 1, False, True, {}),
    (160, 160, 3, 1, 2, 57, 100, True, 0, False, False, {"pair_tile": 0}),
    (192, 192, 3, 1, 1, 29, 50, True, 1, False, False, {}),
    (224, 224, 3, 1, 1, 15, 25, True, 0, False, False, {}),
    (256, 256, 3, 1, 2, 57, 100, True, 1, False, False, {"pair_tile": 1}),
    (64, 64, 3, 1, 2, 96, 160, True, 0, False, False, {"wstat": 1}),
    (64, 128, 3, 2, 2, 96, 160, True, 0, False, False, {}),
    (256, 256, 1, 1, 1, 1, 300, False, 2, False, False, {}),
    (256, 110, 3, 1, 2, 30, 50, False, 0, True, False, {}),
]


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


@pytest.mark.parametrize("case", CASES, ids=lambda c: "-".join(str(int(v)) for v in c[:11]))
def test_conv_stagger_exact(case, act):
    *shape, extra = case
    _conv_exact(*shape, mode="round", seed=shape[0] + 3 * shape[1], policies=[dict(extra, **s) for s in SKEWS])


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
def test_forward_stagger_bit_identical(dtype):
    L = lib.load()
    cfg = get_cfg("v2_99", "nuscenes", act_dtype=dtype)
    sd = make_state_dict(cfg)
    inp = make_inputs(4, 450, 800, 1266.4)
    outs = []
    try:
        for skew in (0, -1):
            assert L.dd3d_set_conv_policy(b"stagger", skew) == 0
            m = DD3DB200(cfg).to("cuda")
            m.load_state_dict(sd)
            out = m(inp)
            torch.cuda.synchronize()
            outs.append(out)
    finally:
        L.dd3d_set_conv_policy(b"stagger", -1)
    a, b = outs
    assert len(a) == len(b)
    for ia, ib in zip(a, b):
        x, y = ia["instances"], ib["instances"]
        assert len(x) > 0 and len(x) == len(y)
        assert torch.equal(x.pred_boxes.tensor, y.pred_boxes.tensor)
        assert torch.equal(x.pred_boxes3d.vectorize(), y.pred_boxes3d.vectorize())
        assert torch.equal(x.scores, y.scores) and torch.equal(x.scores_3d, y.scores_3d)
