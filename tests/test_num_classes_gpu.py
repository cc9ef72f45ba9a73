"""GPU suite (-m gpu) for DD3D.NUM_CLASSES up to 128: the class-gathered box3d predictor exact against a float64 reference and
bit-identical to the sparse predictor's columns, every case of oracle/num_classes_oracle.py end to end against the emulating
oracle and the reference's own forward, the predictor and sparse-tower modes, class ids 64..127 through the group BEV NMS
and both engine DO_BEV_NMS paths, dd3d_op_detect_c on the exact detect fixtures at 17 and 128 classes, the TTA wrapper at 26
classes, the canonical-size setter's call order and the poisoned-workspace test at 128 classes."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import exact_ops as X
import gpu_ops
import parity_lib as PL
from conftest import GOLDEN_DIR
from dd3d_b200 import lib
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict
from oracle.dd3d_oracle import DD3DOracle
from oracle.num_classes_oracle import NUM_CLASSES_CASES, case_cfg, case_inputs, num_classes_cfg
from util import quat_dist

pytestmark = pytest.mark.gpu

_LEVELS = [(23, 40), (12, 20), (6, 10), (1, 5), (1, 1)]
_TOPK = 300


@pytest.fixture(params=["bf16", "fp16"])
def act(request):
    gpu_ops.set_act_dtype(request.param)
    yield request.param
    gpu_ops.set_act_dtype("bf16")


def _candidates(B, C_, counts, g):
    """fin [B][5][topk] (score bits, pixel * C + class) and the (pixel, class) lists: the corners and border midpoints of
    every level first, one pixel with several classes, then random pixels and classes (the top class included)."""
    fin = torch.zeros(B, 5, _TOPK, 2, dtype=torch.int64)
    cand = [[None] * 5 for _ in range(B)]
    for b in range(B):
        for l, (H, W) in enumerate(_LEVELS):
            edge = [0, W - 1, (H - 1) * W, H * W - 1, W // 2, (H - 1) * W + W // 2, (H // 2) * W, (H // 2) * W + W - 1]
            rnd = torch.randint(0, H * W, (_TOPK, ), generator=g).tolist()
            p = (edge + [rnd[0]] * 4 + rnd)[:_TOPK]
            cls = torch.randint(0, C_, (_TOPK, ), generator=g)
            cls[0] = C_ - 1
            n = min(counts[b][l], _TOPK)
            fin[b, l, :, 0] = torch.randint(0, 2**31, (_TOPK, ), generator=g)
            fin[b, l, :, 1] = torch.tensor(p) * C_ + cls
            cand[b][l] = (p[:n], cls[:n].tolist())
    return cand, fin.to(torch.int32)


def _gather(levels, pitches, cin, ws, sb, fin, counts, B, C_):
    L = lib.load()
    d_w = [gpu_ops.pack_conv_weight(w).cuda() for w in ws]
    d_sc, d_bi = [s.cuda() for s, _ in sb], [b.cuda() for _, b in sb]
    d_fin, d_cnt = fin.cuda(), torch.tensor(counts, dtype=torch.int32).cuda()
    rows = torch.full((B, 5, _TOPK, 16), float("nan"), device="cuda")
    scratch = torch.full((L.dd3d_op_b3d_gather_scratch_bytes(B, C_, _TOPK), ), 255, dtype=torch.uint8, device="cuda")
    ptrs = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    hw = (C.c_int32 * 10)(*[v for p in _LEVELS for v in p])
    st = L.dd3d_op_b3d_gather(ptrs(levels), hw, (C.c_int32 * 5)(*pitches), ptrs(d_w), ptrs(d_sc), ptrs(d_bi),
                              gpu_ops._p(d_fin), gpu_ops._p(d_cnt), B, C_, _TOPK, cin, gpu_ops._p(rows), gpu_ops._p(scratch),
                              gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    return rows


def _ref64(levels, cin, ws, sb, cand, B, C_):
    """float64: for each candidate (pixel p, class c) of (b, l), channel q * C + c of the 3x3 conv at p (zero padding) times
    scale plus bias, q < 11."""
    out = {}
    for b in range(B):
        for l, (H, W) in enumerate(_LEVELS):
            pix, cls = cand[b][l]
            if not pix:
                out[b, l] = torch.zeros(0, 11, dtype=torch.float64)
                continue
            x = torch.nn.functional.pad(levels[l][b, :, :, :cin].double().cpu(), (0, 0, 1, 1, 1, 1))  # [H+2][W+2][cin]
            p = torch.tensor(pix)
            y, xx = p // W, p % W
            patch = torch.stack([x[y + ky, xx + kx] for ky in range(3) for kx in range(3)], 1)  # [n][9][cin]
            ch = torch.tensor([[q * C_ + c for q in range(11)] for c in cls])  # [n][11]
            w = ws[l].double().permute(0, 2, 3, 1).reshape(ws[l].shape[0], 9, cin)[ch]  # [n][11][9][cin]
            acc = torch.einsum("ntc,nqtc->nq", patch, w)
            s, bb = sb[l]
            out[b, l] = acc * s.double()[ch] + bb.double()[ch]
    return out


@pytest.mark.parametrize("cin", [64, 256, 512])
@pytest.mark.parametrize("C_", [17, 26, 128])
def test_b3d_gather_exact(C_, cin, act):
    """dd3d_op_b3d_gather: exact fp32 rows (integer operands) with per-level weights, on every border and corner, counts 0, 1,
    127, 128, 129, topk and topk + 7, the top class; rows past the count and columns 11..15 keep their NaN sentinel."""
    g = X._gen(C_ * 1000 + cin)
    B, n = 2, 11 * C_
    counts = [[_TOPK + 7, 129, 128, 1, 127], [127, 0, _TOPK, 129, 1]]
    cand, fin = _candidates(B, C_, counts, g)
    pitches = [cin + 8 * (l % 2) for l in range(5)]
    K = 9 * cin
    levels = [X.operand((B, H, W, pitches[l]), "round", K, g).to(gpu_ops.ACT).cuda() for l, (H, W) in enumerate(_LEVELS)]
    ws = [X.operand((n, cin, 3, 3), "round", K, g) for _ in range(5)]
    sb = [X.epilogue(n, "round", K, g) for _ in range(5)]
    rows = _gather(levels, pitches, cin, ws, sb, fin, counts, B, C_)
    ref = _ref64(levels, cin, ws, sb, cand, B, C_)
    for b in range(B):
        for l in range(5):
            m = min(counts[b][l], _TOPK)
            X.assert_exact(rows[b, l, :m, :11], ref[b, l].cuda(), f"C {C_} cin {cin} image {b} level {l}")
            assert torch.isnan(rows[b, l, m:]).all()
    assert torch.isnan(rows[..., 11:]).all()


@pytest.mark.parametrize("cin", [128, 256])
@pytest.mark.parametrize("C_", [1, 5, 10])
def test_b3d_gather_is_bit_identical_to_the_sparse_predictor(C_, cin, act):
    """Non-integer operands: the gathered rows equal columns {q * C + c} of dd3d_op_b3d_sparse_c's rows bit for bit."""
    g = torch.Generator().manual_seed(C_ * 7 + cin)
    B, n_pad = 2, (11 * C_ + 15) // 16 * 16
    counts = [[_TOPK, 129, 128, 1, 127], [127, 0, _TOPK + 7, 129, 128]]
    cand, fin = _candidates(B, C_, counts, g)
    pitches = [cin + 8 * (l % 2) for l in range(5)]
    levels = [torch.randn(B, H, W, pitches[l], generator=g).to(gpu_ops.ACT).cuda() for l, (H, W) in enumerate(_LEVELS)]
    ws = [torch.randn(n_pad, cin, 3, 3, generator=g) / 48.0 for _ in range(5)]
    sb = [(torch.rand(n_pad, generator=g) + 0.5, torch.randn(n_pad, generator=g)) for _ in range(5)]
    a = _gather(levels, pitches, cin, ws, sb, fin, counts, B, C_)
    L = lib.load()
    d_w = [gpu_ops.pack_conv_weight(w).cuda() for w in ws]
    d_sc, d_bi = [s.cuda() for s, _ in sb], [b.cuda() for _, b in sb]
    rows = torch.full((B, 5, _TOPK, n_pad), float("nan"), device="cuda")
    d_fin, d_cnt = fin.cuda(), torch.tensor(counts, dtype=torch.int32).cuda()  # kept alive until the kernel has run
    ptrs = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    hw = (C.c_int32 * 10)(*[v for p in _LEVELS for v in p])
    st = L.dd3d_op_b3d_sparse_c(ptrs(levels), hw, (C.c_int32 * 5)(*pitches), ptrs(d_w), ptrs(d_sc), ptrs(d_bi),
                                gpu_ops._p(d_fin), gpu_ops._p(d_cnt), B, C_, _TOPK,
                                n_pad, gpu_ops._p(rows), n_pad, cin, gpu_ops._stream())
    assert st == 0
    torch.cuda.synchronize()
    for b in range(B):
        for l in range(5):
            pix, cls = cand[b][l]
            if not pix:
                continue
            ch = torch.tensor([[q * C_ + c for q in range(11)] for c in cls], device="cuda")
            want = torch.gather(rows[b, l, :len(pix)], 1, ch)
            got = a[b, l, :len(pix), :11]
            assert torch.equal(got.contiguous().view(torch.int32), want.contiguous().view(torch.int32)), (C_, cin, b, l)


def test_b3d_gather_refuses_bad_arguments():
    L = lib.load()
    x = torch.zeros(1, 2, 2, 576, dtype=gpu_ops.ACT, device="cuda")
    w = torch.zeros(11 * 128, 9, 576, dtype=gpu_ops.ACT, device="cuda")
    sb = torch.zeros(11 * 128, device="cuda")
    fin = torch.zeros(1, 5, 4, 2, dtype=torch.int32, device="cuda")
    cnt = torch.zeros(1, 5, dtype=torch.int32, device="cuda")
    rows = torch.zeros(1, 5, 4, 16, device="cuda")
    scratch = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    five = lambda t: (C.c_void_p * 5)(*([t.data_ptr()] * 5))  # noqa: E731
    hw = (C.c_int32 * 10)(*([2] * 10))
    for C_, cin, pitch in ((17, 96, 96), (17, 0, 64), (17, 576, 576), (17, 128, 64), (0, 64, 64), (129, 64, 64)):
        st = L.dd3d_op_b3d_gather(five(x), hw, (C.c_int32 * 5)(*([pitch] * 5)), five(w), five(sb), five(sb), gpu_ops._p(fin),
                                  gpu_ops._p(cnt), 1, C_, 4, cin, gpu_ops._p(rows), gpu_ops._p(scratch), gpu_ops._stream())
        assert st == -1, (C_, cin, pitch, st)


# ------------------------------------------------------------------------------------------------ end to end
# The bounds of tests/test_fpn_width_gpu.py (BN heads).
_BOUNDS = {"box": 1.3e-2, "size": 2.6e-2, "depth": 8e-3, "score": 8e-3, "score3d": 8e-3}
# DLA-X-46-C at 64 classes, bf16: the 2-D score error was 8.4e-3 in each of three H100 runs (deterministic kernels: the same
# value every run), with either box3d predictor -- the score comes from the cls map alone, and 64 classes put ~2x more
# candidates per image in the NMS than the 10-class fixtures, so the largest matched error grows.  Its bound is 1.2e-2.
_SCORE_BF16 = {"dla_x_46_c_c64_agnostic": 1.2e-2}


def _model(cfg, **opts):
    nusc = cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D"
    m = (NuscenesDD3DB200 if nusc else DD3DB200)(cfg).to("cuda")
    m.load_state_dict(make_state_dict(cfg))
    if nusc:
        m.sample_aggregate_in_inference = False  # per-image detections, as the oracle returns them
    for k, v in opts.items():
        m.set_engine_option(k, v)
    return m


def _inputs(case):
    if NUM_CLASSES_CASES[case][2] == "NuscenesDD3D":
        return make_nusc_inputs(1, 128, 192, 1266.4)
    return case_inputs(case)


@pytest.mark.parametrize("sparse", [1, 0], ids=["gathered", "dense"])
@pytest.mark.parametrize("act_dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("case", list(NUM_CLASSES_CASES))
def test_forward_vs_emulating_oracle(case, act_dtype, sparse):
    cfg = case_cfg(case, act_dtype=act_dtype)
    model = _model(cfg, sparse_box3d=sparse)
    inputs = _inputs(case)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    ref = DD3DOracle(cfg, make_state_dict(cfg), emulate=act_dtype, threads=1).forward(inputs)
    worst = {f: 0.0 for f in _BOUNDS}
    n = 0
    for b, (o, r) in enumerate(zip(out, ref)):
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_oracle(r)
        rep, ia, ib = PL.compare_sets(a, e)
        n += rep["n_ref"]
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        for f in _BOUNDS:
            if len(errs[f]):
                worst[f] = max(worst[f], float(errs[f].max()))
        if len(ia):
            assert quat_dist(a["quat"][ia], e["quat"][ib]).max() < 1e-1
    print(f"\n{case} {act_dtype} sparse_box3d={sparse}: {n} detections, worst {worst}")
    assert n > 0
    bounds = dict(_BOUNDS, score=_SCORE_BF16.get(case, _BOUNDS["score"]) if act_dtype == "bf16" else _BOUNDS["score"])
    for f, bound in bounds.items():
        assert worst[f] < bound, f"{f}: {worst[f]} >= {bound}"


@pytest.mark.parametrize("case", [c for c, v in NUM_CLASSES_CASES.items() if v[2] == "DD3D"])
def test_forward_vs_reference_golden(case):
    g = np.load(os.path.join(GOLDEN_DIR, "golden_num_classes.npz"))
    g = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(case + "/")}
    cfg = case_cfg(case)
    out = _model(cfg, sparse_box3d=1)(case_inputs(case))
    for b, o in enumerate(out):
        a, e = PL.dets_from_instances(o["instances"]), PL.dets_from_golden(g, b)
        assert tuple(o["instances"].image_size) == tuple(g[f"image_size{b}"].tolist())
        rep, ia, ib = PL.compare_sets(a, e)
        assert rep["matched"] >= 0.9 * rep["n_ref"] - 1, f"image {b}: {rep}"
        errs = PL.field_errors(a, e, ia, ib)
        if len(ia):
            print(f"\n{case} image {b}: box {errs['box'].max():.3e} size {errs['size'].max():.3e}")
            assert errs["box"].max() < 1.6e-2
            assert errs["size"].max() < 2.6e-2


# ------------------------------------------------------------------------------------------------ predictor / tower modes
def _dets(out):
    res = []
    for o in out:
        inst = o["instances"]
        b3 = inst.pred_boxes3d
        two = torch.cat([inst.pred_boxes.tensor, inst.scores[:, None]], 1).contiguous().view(torch.int32).cpu()
        three = torch.cat([inst.scores_3d[:, None], b3.quat, b3.size, b3.tvec], 1).cpu()
        res.append((two, inst.pred_classes.cpu().clone(), inst.fpn_levels.cpu().clone(), three))
    return res


def _run_opts(cfg, inputs, **opts):
    model = _model(cfg, **opts)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    n = model.launches_per_forward()
    del model
    return _dets(out), n


@pytest.mark.parametrize("n", [26, 128])
def test_predictor_and_tower_modes(n):
    """DLA-34 at 26 / 128 classes: the sparse box2d / box3d towers are bit-identical to the dense towers; the gathered
    predictor (two launches: class grouping + predictor) matches the dense predictor to the fp32 summation order."""
    lib.load().dd3d_set_conv_policy(b"pair_tile", 1)
    try:
        cfg = num_classes_cfg("dla34", n)
        cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.02
        inputs = make_inputs(2, 192, 320, 721.5)
        off = dict(sparse_box3d=0, sparse_tower=0, sparse_box2d_tower=0)
        dense, n_dense = _run_opts(cfg, inputs, **off)
        assert sum(len(d[0]) for d in dense) > 0
        box2d, n_box2d = _run_opts(cfg, inputs, **dict(off, sparse_box2d_tower=1))
        assert n_box2d == n_dense + 2
        sp3, n_sp3 = _run_opts(cfg, inputs, **dict(off, sparse_box3d=1))
        assert n_sp3 == n_dense - 1 + 2  # the dense predictor conv -> class grouping + gathered predictor
        tower, n_tower = _run_opts(cfg, inputs, **dict(off, sparse_box3d=1, sparse_tower=1))
        assert n_tower == n_sp3 + 1
        for i, (d, b, s, t) in enumerate(zip(dense, box2d, sp3, tower)):
            for k in range(4):
                assert torch.equal(d[k], b[k]), f"{n} classes image {i}: sparse box2d tower differs"
                assert torch.equal(s[k], t[k]), f"{n} classes image {i}: sparse box3d tower differs"
            kd = [(int(l), int(c), *d[0][j, :4].tolist()) for j, (c, l) in enumerate(zip(d[1], d[2]))]
            ks = {(int(l), int(c), *s[0][j, :4].tolist()): j for j, (c, l) in enumerate(zip(s[1], s[2]))}
            ia = [j for j, k in enumerate(kd) if k in ks]
            assert len(ia) >= len(kd) - 2 and abs(len(ks) - len(kd)) <= 2, f"{n} classes image {i}: {len(ia)} of {len(kd)}"
            ib = [ks[kd[j]] for j in ia]
            assert torch.allclose(d[3][ia], s[3][ib], rtol=1e-4, atol=1e-4), f"{n} classes image {i}: 3-D fields"
    finally:
        lib.load().dd3d_set_conv_policy(b"pair_tile", -1)


def test_set_canonical_sizes_call_order():
    cfg = num_classes_cfg("dla34", 26)
    m = _model(cfg)
    h = m._engine()  # finalized
    L = lib.load()
    sizes = (C.c_float * 78)(*([1.0] * 78))
    assert L.dd3d_set_canonical_sizes(h, 26, sizes) == -2  # DD3D_ERR_STATE after finalize
    # without the sizes an engine above 16 classes does not finalize
    d = lib.desc_from_cfg(cfg)
    h2 = C.c_void_p()
    assert L.dd3d_create(C.byref(d), C.byref(h2)) == 0
    try:
        assert L.dd3d_set_canonical_sizes(h2, 25, sizes) == -1  # the desc's class count only
        assert L.dd3d_finalize(h2) == -2
        assert b"dd3d_set_canonical_sizes" in L.dd3d_last_error(h2)
    finally:
        L.dd3d_destroy(h2)


# ------------------------------------------------------------------------------------------------ BEV NMS class ids
def test_group_bev_nms_takes_class_ids_up_to_127():
    """Class ids only key the per-class segments: a set with ids 64..127 gives exactly the result of the same set with ids
    shifted to 0..63, and no flag."""
    L = lib.load()
    g = torch.Generator().manual_seed(127)
    B, cap = 2, 256
    dets = torch.zeros(B, cap, lib.DET_WORDS, dtype=torch.float32)
    n = torch.tensor([200, 137], dtype=torch.int32)
    for b in range(B):
        m = int(n[b])
        d = dets[b, :m]
        d[:, 5] = torch.rand(m, generator=g)                                   # score_3d (cls, word 6, set by run())
        d[:, 4] = d[:, 5]
        ctr = torch.rand(m, 2, generator=g) * torch.tensor([60.0, 20.0]) + 380  # clustered centres: overlaps
        d[:, 12:14] = ctr
        d[:, 14] = 20 + torch.rand(m, generator=g) * 2                          # depth
        d[:, 15:18] = 1 + torch.rand(m, 3, generator=g) * 3                    # size
        q = torch.randn(m, 4, generator=g)
        d[:, 8:12] = q / q.norm(dim=1, keepdim=True)
    cls = torch.randint(0, 64, (B, cap), generator=g, dtype=torch.int32)
    K = torch.tensor([[700.0, 0, 400], [0, 700, 200], [0, 0, 1]]).repeat(B, 1, 1)
    poses = torch.tensor([[1.0, 0, 0, 0, 0, 0, 0], [0.9, 0.1, 0.3, 0.3, 1, 2, 3]])
    group = torch.tensor([0, 0], dtype=torch.int32)

    def run(offset):
        d = dets.clone()
        d.view(torch.int32)[:, :, 6] = cls + offset
        d = d.cuda()
        cnt = n.clone().cuda()
        d_K, d_poses, d_group = K.contiguous().cuda(), poses.cuda(), group.cuda()
        flags = torch.zeros(1, dtype=torch.int32, device="cuda")
        scratch = torch.zeros(L.dd3d_op_group_bev_nms_scratch_bytes(B, cap, 2), dtype=torch.uint8, device="cuda")
        glob = torch.zeros(B, cap, 10, device="cuda")
        st = L.dd3d_op_group_bev_nms(gpu_ops._p(d), gpu_ops._p(cnt), gpu_ops._p(d_K), 1, gpu_ops._p(d_poses),
                                     lib.POSE_GLOBAL, gpu_ops._p(d_group), 1, 2, gpu_ops._p(glob), gpu_ops._p(scratch),
                                     gpu_ops._p(flags), B, cap, 0.1, 0, gpu_ops._stream())
        assert st == 0
        torch.cuda.synchronize()
        return d.cpu(), cnt.cpu(), int(flags.item())

    d0, c0, f0 = run(0)
    d1, c1, f1 = run(64)
    assert f0 == 0 and f1 == 0, (f0, f1)
    assert torch.equal(c0, c1) and 0 < int(c0.sum()) < int(n.sum())  # something was suppressed
    for b in range(B):
        m = int(c0[b])
        a, e = d1[b, :m].clone(), d0[b, :m].clone()
        assert torch.equal(a.view(torch.int32)[:, 6], e.view(torch.int32)[:, 6] + 64)
        a.view(torch.int32)[:, 6] = 0
        e.view(torch.int32)[:, 6] = 0
        assert torch.equal(a.view(torch.int32), e.view(torch.int32))


# ------------------------------------------------------------------------------------------------ determinism
def test_poisoned_workspace_changes_nothing_at_128_classes():
    cfg = case_cfg("v2_19_slim_c128")
    snaps = []
    for fill in (0x00, 0xFF):
        m = _model(cfg, workspace_fill=fill, sparse_box3d=1)
        out = m(case_inputs("v2_19_slim_c128"))
        torch.cuda.synchronize()
        assert m.overflow_flags() == 0
        snaps.append([torch.cat([o["instances"].pred_boxes.tensor, o["instances"].scores_3d[:, None],
                                 o["instances"].pred_boxes3d.quat, o["instances"].pred_boxes3d.size], 1).contiguous()
                      .view(torch.int32).cpu() for o in out])
        del m
    assert sum(len(s) for s in snaps[0]) > 0
    for a, b in zip(*snaps):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ dd3d_op_detect_c
def _run_detect_c(case, parallel, canon):
    """dd3d_op_detect_c on the case's maps, with a 0xFF-poisoned scratch; returns what test_detect_exact_gpu.run returns."""
    from test_detect_exact_gpu import _desc
    L = lib.load()
    B = case.B
    desc = _desc(case)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    cls, box, b3d = [dev(a) for a in case.cls], [dev(a) for a in case.box], [dev(a) for a in case.b3d]
    arr = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    nbytes = L.dd3d_op_detect_c_scratch_bytes(B, case.topk, case.C)
    assert nbytes > 0
    scratch = torch.full((nbytes + 4096, ), 255, dtype=torch.uint8, device="cuda")
    pre = torch.zeros(B, 5 * case.topk, 24, dtype=torch.float32, device="cuda")
    pre_n = torch.zeros(B, 5, dtype=torch.int32, device="cuda")
    out = torch.full((B * case.out_cap + 64, 24), -7.0, dtype=torch.float32, device="cuda")
    cnt = torch.full((B, ), -1, dtype=torch.int32, device="cuda")
    flags = torch.full((1, ), -1, dtype=torch.int32, device="cuda")
    hw = (C.c_int32 * 10)(*[v for q in case.level_hw for v in q])
    st = (C.c_int32 * 5)(*case.strides)
    K = torch.tensor([[700.0, 0, 320.0, 0, 700.0, 240.0, 0, 0, 1]]).repeat(B, 1).cuda()
    sizes = torch.from_numpy(case.sizes).cuda()
    h_canon = (C.c_float * (3 * case.C))(*canon.reshape(-1).tolist())
    try:
        assert L.dd3d_set_conv_policy(b"nms_class_parallel", parallel) == 0
        r = L.dd3d_op_detect_c(C.byref(desc), h_canon, B, hw, st, arr(cls), arr(box), arr(b3d), case.cls_pitch, case.b3d_pitch,
                               p(K), p(sizes), p(scratch), p(pre), p(pre_n), p(out), p(cnt), p(flags),
                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert r == 0
        torch.cuda.synchronize()
    finally:
        L.dd3d_set_conv_policy(b"nms_class_parallel", -1)
    assert bool((scratch[nbytes:] == 255).all()), "scratch written past dd3d_op_detect_c_scratch_bytes"
    out = out.cpu()
    assert (out[B * case.out_cap:] == -7.0).all(), "records written past B * out_cap"
    return pre.cpu(), pre_n.cpu(), out[:B * case.out_cap].reshape(B, case.out_cap, 24), cnt.cpu(), int(flags)


def _mirrored(case):
    """The case with class c's logits moved to class C - 1 - c: the fixtures put their tied / clustered candidates in the
    low classes, and these must reach the size rows and class ids past 64."""
    for a in case.cls:
        a[..., :case.C] = a[..., :case.C][..., ::-1].copy()
    return case


def _detect_c_cases():
    import detect_cases as D
    return {"clustered-128": lambda: D.clustered(True, 50, 100, C=128),
            "tied-128": lambda: D.clustered(True, 1, 5000, C=128),
            "clustered-cls-128": lambda: D.clustered(False, 1100, 4, C=128),
            "flooded-128": lambda: D.random_level(1000, 3, C=128),
            "flooded-17": lambda: D.random_level(1150, 4, C=17)}


@pytest.mark.parametrize("name", list(_detect_c_cases()))
def test_detect_c_exact_at_many_classes(name):
    """dd3d_op_detect_c above 16 classes on tests/detect_cases.py operands (tied and clustered scores, flooded levels): the
    exact reference of tests/test_detect_exact_gpu.py on both NMS paths, which agree bit for bit; every detection's size is
    its class's own canonical row (the 3-D maps are zero: size = (tanh(0) + 1) * canon[c])."""
    import detect_cases as D
    from test_detect_exact_gpu import check
    case = _mirrored(_detect_c_cases()[name]())
    D.check_unambiguous(case)
    canon = torch.tensor(canonical_sizes_np(case.C))
    a, b = _run_detect_c(case, 1, canon), _run_detect_c(case, 0, canon)
    check(case, a)
    for x, y in zip((a[2], a[3]), (b[2], b[3])):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "NMS paths differ"
    seen = set()
    for j in range(case.B):
        n = int(a[3][j])
        w = a[2][j, :n]
        cls = w.view(torch.int32)[:, 6].long()
        seen |= set(cls.tolist())
        assert torch.equal(w[:, 15:18], canon[cls]), "canonical size rows"
    assert max(seen) >= (64 if case.C == 128 else 16)


def canonical_sizes_np(n):
    from oracle.num_classes_oracle import canonical_sizes
    return np.array(canonical_sizes(n), dtype=np.float32)


def test_detect_c_at_16_classes_is_detect_flags():
    """At 16 classes or fewer dd3d_op_detect_c with the desc's rows is dd3d_op_detect_flags, bit for bit: candidate counts,
    detections, counts and flags (the pre-NMS records are in atomic-append order and are compared as sets by check())."""
    import detect_cases as D
    from test_detect_exact_gpu import _desc, check, run
    case = D.random_level(1000, 3, C=10)
    d = _desc(case)
    canon = torch.tensor([d.canonical_box3d_sizes[i] for i in range(30)]).reshape(10, 3)
    a, b = run(case, 1), _run_detect_c(case, 1, canon)
    for x, y in zip(a[1:4], b[1:4]):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert a[4] == b[4]
    check(case, b)
    assert lib.load().dd3d_op_detect_c_scratch_bytes(1, 1000, 16) <= lib.load().dd3d_op_detect_scratch_bytes(1, 1000) + 255


# ------------------------------------------------------------------------------------------------ engine DO_BEV_NMS
@pytest.mark.parametrize("path", [1, 2], ids=["one_cta", "multi_cta"])
def test_engine_bev_nms_with_classes_above_64(path):
    """DO_BEV_NMS at 128 classes on both engine paths: the BEV NMS op equals the reference BEV NMS
    (oracle/bev_nms_oracle.py) on the same engine's pre-BEV detections, with predicted classes 64..127 among them."""
    from oracle import bev_nms_oracle as BO
    from oracle.dd3d_oracle import DD3DOracle
    from test_bev_nms_large_gpu import BEV_THR, _inputs, POSES
    cfg = num_classes_cfg("dla34", 128)
    cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH = 0.02
    if path == 2:
        cfg.DD3D.INFERENCE.DO_NMS = False
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH = BEV_THR
    model = _model(cfg)
    assert lib.load().dd3d_bev_nms_path(C.byref(model._desc)) == path
    inputs = _inputs()
    out = model(inputs)
    assert model.last_overflow_flags == 0
    model.do_bev_nms = False
    model.postprocess_in_inference = False
    pre = model(inputs)
    removed, high = 0, 0
    for b, (o, q) in enumerate(zip(out, pre)):
        pi = q["instances"]
        high += int((pi.pred_classes >= 64).sum())
        det = dict(quat=pi.pred_boxes3d.quat.cpu(), tvec=pi.pred_boxes3d.tvec.cpu(), size=pi.pred_boxes3d.size.cpu(),
                   score3d=pi.scores_3d.cpu(), cls=pi.pred_classes.cpu(), box2d=pi.pred_boxes.tensor.cpu())
        keep = BO.bev_nms_image(det, POSES[b][0], POSES[b][1], BEV_THR)
        removed += len(pi) - len(keep)
        h, w = pi.image_size
        oh, ow = inputs[b].get("height", h), inputs[b].get("width", w)
        ref = DD3DOracle.postprocess({k: v[keep] for k, v in det.items()}, (h, w), (oh, ow))
        inst = o["instances"]
        assert len(inst) == ref["box2d"].shape[0]
        ka = np.lexsort((inst.pred_classes.cpu().numpy(), inst.scores_3d.cpu().numpy()))
        kb = np.lexsort((ref["cls"].numpy(), ref["score3d"].numpy()))
        assert torch.equal(inst.scores_3d.cpu()[ka], ref["score3d"][kb])
        assert torch.equal(inst.pred_classes.cpu()[ka], ref["cls"][kb])
        np.testing.assert_allclose(inst.pred_boxes.tensor.cpu().numpy()[ka], ref["box2d"].numpy()[kb], rtol=1e-6, atol=1e-4)
    assert high > 0, "no predicted class >= 64 entered the BEV NMS"
    assert removed > 0


# ------------------------------------------------------------------------------------------------ TTA
def test_tta_at_26_classes_vs_emulating_oracle():
    """DD3DB200WithTTA at 26 classes (the class-gathered predictor is forced on) against the bf16-emulating oracle's TTA,
    with tests/test_tta.py's matching rule and bounds."""
    from dd3d_b200.tta import DD3DB200WithTTA
    from oracle import tta_oracle as T
    from oracle.dd3d_oracle import DD3DOracle
    from oracle.gen_golden import tta_case
    from oracle.num_classes_oracle import canonical_sizes
    from util import rel_err
    cfg, x = tta_case()
    cfg.DD3D.NUM_CLASSES = 26
    cfg.DD3D.FCOS3D.CANONICAL_BOX3D_SIZES = canonical_sizes(26)
    sd = make_state_dict(cfg)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    model.set_engine_option("sparse_box3d", 1)
    tta = DD3DB200WithTTA(cfg, model)
    inst = tta([x])[0]["instances"]
    assert tta.overflow_flags() == 0
    assert tuple(inst.image_size) == (x["height"], x["width"])
    emu = T.tta_forward(DD3DOracle(cfg, sd, emulate_bf16=True), x, cfg.TEST.AUG.MIN_SIZES, cfg.TEST.AUG.MAX_SIZE,
                        cfg.TEST.AUG.FLIP, cfg.TEST.IMS_PER_BATCH, cfg.DD3D.FCOS2D.INFERENCE.NMS_THRESH)
    n, m = len(inst), emu["score3d"].shape[0]
    assert m > 0 and abs(n - m) <= 0.1 * m

    def keys(box, cls):
        return [(int(c), ) + tuple(int(round(float(v) / 2.0)) for v in b) for b, c in zip(box, cls)]
    ka, kb = keys(inst.pred_boxes.tensor.cpu(), inst.pred_classes.cpu()), keys(emu["box2d"], emu["cls"])
    pos = {k: i for i, k in enumerate(kb)}
    pairs = [(i, pos[k]) for i, k in enumerate(ka) if k in pos]
    assert len(pairs) >= 0.7 * m
    ia, ib = (torch.tensor(p) for p in zip(*pairs))
    assert rel_err(inst.pred_boxes.tensor.cpu()[ia], emu["box2d"][ib], floor=16.0) < 0.1
    assert rel_err(inst.scores_3d.cpu()[ia], emu["score3d"][ib], floor=0.05) < 0.2
    assert rel_err(inst.pred_boxes3d.depth.cpu()[ia].reshape(-1), emu["depth"][ib], floor=1.0) < 0.05
    assert quat_dist(inst.pred_boxes3d.quat.cpu()[ia], emu["quat"][ib]).median().item() < 0.05
    assert int(inst.pred_classes.max()) >= 16  # the size rows past the desc's 16 are read

