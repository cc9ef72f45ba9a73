"""Large-set test-time augmentation on the GPU (csrc/tta_large.cu): bit-identical agreement with the one-CTA merge and the
grouped BEV NMS on sets they hold, exact results on 5 k - 92 k boxes built from disjoint clusters, a dense cluster against
the CPU oracle, scratch independence, capacity flags, and the TTA wrappers on the configs that need the large path."""
import ctypes as C
import math

import pytest
import torch

import nusc_tta_oracle as NT
from test_group_bev_nms import GLOBAL_CASES, make_case, pack, run_kernel

pytestmark = pytest.mark.gpu


def _L():
    from dd3d_b200 import lib
    return lib, lib.load()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


# ------------------------------------------------------------------------------------------------ merge
def _identity_views(A, K=((700.0, 0.0, 320.0), (0.0, 690.0, 180.0), (0.0, 0.0, 1.0)), scales=None, flips=None):
    lib, _ = _L()
    views = []
    for a in range(A):
        v = lib.TtaView()
        v.flip = int(flips[a]) if flips else 0
        v.view_w = 640.0
        sx, sy = scales[a] if scales else (1.0, 1.0)
        v.inv_sx[0], v.inv_sy[0], v.inv_sx[1], v.inv_sy[1] = sx, sy, 1.0, 1.0
        for i in range(9):
            v.K_view[i] = float(K[i // 3][i % 3])
            v.K_orig[i] = float(K[i // 3][i % 3])
        views.append(v)
    return views


def _view_dets(seed, A, cap, counts, num_classes=3, levels=None, dup=0.3, spread=600.0):
    """[A][cap][24] records: boxes over a wide field with near-duplicate copies, scores quantized to `levels` values
    (tie runs), unique Det::index per view (view * 100000 + slot)."""
    g = torch.Generator().manual_seed(seed)
    buf = torch.zeros(A, cap, 24)
    for a in range(A):
        n = counts[a]
        xy = torch.rand(n, 2, generator=g) * spread
        wh = torch.rand(n, 2, generator=g) * 40 + 4
        m = int(n * dup)
        if m and n > m:
            src = torch.randint(0, n - m, (m, ), generator=g)
            xy[n - m:] = xy[src] + torch.randn(m, 2, generator=g) * 2.0
            wh[n - m:] = wh[src]
        s = torch.rand(n, generator=g)
        if levels:
            s = torch.floor(s * levels) / levels + 0.01
        buf[a, :n, 0:2], buf[a, :n, 2:4] = xy, xy + wh
        buf[a, :n, 4], buf[a, :n, 5] = s.sqrt(), s
        q = torch.randn(n, 4, generator=g)
        buf[a, :n, 8:12] = q / q.norm(dim=1, keepdim=True)
        buf[a, :n, 12:14] = torch.rand(n, 2, generator=g) * torch.tensor([640.0, 360.0])
        buf[a, :n, 14] = torch.rand(n, generator=g) * 40 + 3
        buf[a, :n, 15:18] = torch.rand(n, 3, generator=g) + 1
        buf.view(torch.int32)[a, :n, 6] = torch.randint(0, num_classes, (n, ), generator=g).to(torch.int32)
        buf.view(torch.int32)[a, :n, 20] = torch.arange(n, dtype=torch.int32) + 100000 * a
    return buf


def run_merge(buf, counts, views, thr, do_nms, large, poison=None):
    lib, L = _L()
    A, cap = buf.shape[0], buf.shape[1]
    d, c = buf.cuda(), torch.tensor(counts, dtype=torch.int32).cuda()
    if large:
        mcap, nbytes, op = L.dd3d_op_tta_merged_cap_large(A, cap), L.dd3d_op_tta_merge_large_scratch_bytes(A, cap), \
            L.dd3d_op_tta_merge_large
    else:
        mcap, nbytes, op = L.dd3d_op_tta_merged_cap(A, cap), L.dd3d_op_tta_merge_scratch_bytes(A, cap), L.dd3d_op_tta_merge
    assert mcap > 0 and nbytes > 0
    out = torch.full((mcap, 24), float("nan"), device="cuda")
    n_out = torch.zeros(1, dtype=torch.int32, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(nbytes), dtype=torch.uint8, device="cuda")
    if poison is not None:
        scratch.fill_(poison)
    varr = (lib.TtaView * A)(*views)
    st = op(_p(d), _p(c), varr, A, cap, thr, do_nms, _p(scratch), _p(out), _p(n_out), _p(flags), _stream())
    torch.cuda.synchronize()
    assert st == 0
    n = int(n_out.item())
    return out[:n].cpu(), int(flags.item())


MERGE_CASES = {
    # name: (seed, A, cap, counts, classes, score levels)
    "random": (1, 8, 128, [128, 97, 0, 128, 64, 128, 1, 128], 3, None),
    "ties": (2, 8, 128, [128] * 8, 3, 6),
    "one_class_ties": (3, 10, 100, [100] * 10, 1, 3),
    "many_classes": (4, 6, 160, [160, 150, 140, 130, 120, 30], 128, 20),
}


@pytest.mark.parametrize("name", sorted(MERGE_CASES))
@pytest.mark.parametrize("do_nms,thr", [(1, 0.5), (1, 0.0), (0, 0.5)])
def test_merge_large_equals_one_cta_merge(name, do_nms, thr):
    seed, A, cap, counts, ncls, levels = MERGE_CASES[name]
    assert sum(counts) <= 1024
    buf = _view_dets(seed, A, cap, counts, ncls, levels)
    views = _identity_views(A, scales=[(1.0 + 0.1 * a, 1.0 + 0.05 * a) for a in range(A)], flips=[a % 2 for a in range(A)])
    ref, f0 = run_merge(buf, counts, views, thr, do_nms, large=False)
    out, f1 = run_merge(buf, counts, views, thr, do_nms, large=True)
    assert f0 == 0 and f1 == 0
    assert out.shape == ref.shape
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))
    if do_nms and thr > 0:
        assert out.shape[0] < sum(counts)


def _cluster_boxes(seed, n_clusters, per, num_classes, dominant, levels):
    """Disjoint clusters of near-duplicate 2-D boxes on a grid 100 px apart (boxes <= 40 px): the NMS of the union is the
    union of the per-cluster NMS.  Scores take `levels` values, so tie runs straddle multiples of the block size."""
    g = torch.Generator().manual_seed(seed)
    side = int(math.ceil(math.sqrt(n_clusters)))
    rows = []
    for c in range(n_clusters):
        cx, cy = 100.0 * (c % side), 100.0 * (c // side)
        xy = torch.tensor([cx, cy]) + torch.rand(per, 2, generator=g) * 6
        wh = torch.rand(1, 2, generator=g) * 20 + 15 + torch.rand(per, 2, generator=g) * 4
        cls = torch.randint(0, num_classes, (per, ), generator=g)
        if dominant:
            cls[torch.rand(per, generator=g) < dominant] = 0
        s = torch.floor(torch.rand(per, generator=g) * levels) / levels + 0.01
        rows.append((xy, wh, cls, s))
    return rows


@pytest.mark.parametrize("total,num_classes,dominant", [(5000, 1, None), (20000, 3, 0.9), (92000, 128, None),
                                                        (92000, 2, 0.95)])
def test_merge_large_disjoint_clusters_exact(total, num_classes, dominant):
    per = 23
    n_clusters = total // per
    rows = _cluster_boxes(7 + total + num_classes, n_clusters, per, num_classes, dominant, levels=12)
    A = 16
    cap = (n_clusters * per + A - 1) // A
    assert cap <= 5750
    buf = torch.zeros(A, cap, 24)
    counts = [0] * A
    flat = torch.zeros(n_clusters * per, 24)
    for c, (xy, wh, cls, s) in enumerate(rows):
        r = flat[c * per:(c + 1) * per]
        r[:, 0:2], r[:, 2:4], r[:, 4], r[:, 5] = xy, xy + wh, s, s
        r[:, 8], r[:, 12], r[:, 13], r[:, 14], r[:, 15:18] = 1.0, 320.0, 180.0, 10.0, 1.0
        r.view(torch.int32)[:, 6] = cls.to(torch.int32)
    flat.view(torch.int32)[:, 20] = torch.arange(flat.shape[0], dtype=torch.int32)  # Det::index: unique
    for a in range(A):
        part = flat[a * cap:(a + 1) * cap]
        buf[a, :part.shape[0]] = part
        counts[a] = part.shape[0]
    views = _identity_views(A)
    out, flags = run_merge(buf, counts, views, 0.5, 1, large=True)
    assert flags == 0
    # expectation: the one-CTA merge on each cluster (one view of `per` boxes), then the union in the merged order
    kept = []
    one_view = _identity_views(1)
    for c in range(n_clusters):
        r, f = run_merge(flat[c * per:(c + 1) * per].unsqueeze(0), [per], one_view, 0.5, 1, large=False)
        assert f == 0
        kept.append(r)
    ref = torch.cat(kept)
    idx = ref.view(torch.int32)[:, 20].long()
    order = sorted(range(ref.shape[0]), key=lambda i: (-float(ref[i, 5]), int(idx[i])))
    ref = ref[torch.tensor(order)]
    assert out.shape == ref.shape, (out.shape, ref.shape)
    o32, r32 = out.view(torch.int32).clone(), ref.view(torch.int32).clone()
    # `level` is the view index: the large call spreads the clusters over 16 views
    assert torch.equal(o32[:, 7].long(), o32[:, 20].long() // cap)
    o32[:, 7] = 0
    r32[:, 7] = 0
    assert torch.equal(o32, r32)
    assert ref.shape[0] < flat.shape[0]


def test_merge_large_scratch_garbage_and_determinism():
    seed, A, cap, counts, ncls, levels = 11, 16, 3000, [3000] * 15 + [1234], 4, 8
    buf = _view_dets(seed, A, cap, counts, ncls, levels, spread=3000.0)
    views = _identity_views(A, scales=[(1.0 + 0.01 * a, 1.0) for a in range(A)], flips=[a % 2 for a in range(A)])
    runs = [run_merge(buf, counts, views, 0.6, 1, large=True, poison=p) for p in (None, 0xFF, 0x00, None)]
    for out, flags in runs:
        assert flags == 0
        assert torch.equal(out.view(torch.int32), runs[0][0].view(torch.int32))
    s = runs[0][0][:, 5]
    assert runs[0][0].shape[0] > 1024 and torch.all(s[:-1] >= s[1:])


def test_merge_large_count_above_cap_flags():
    buf = _view_dets(12, 2, 64, [64, 64])
    out, flags = run_merge(buf, [64, 65], _identity_views(2), 0.5, 1, large=True)
    assert flags == 16 and out.shape[0] <= 128


# ------------------------------------------------------------------------------------------------ grouped BEV NMS
def run_large(buf, counts, Ks, poses, groups, num_groups, cap, thr, max_dets, pose_mode, with_global=True, poison=None,
              group_images=None):
    """run_kernel of test_group_bev_nms on dd3d_op_group_bev_nms_large."""
    _, L = _L()
    Bn = buf.shape[0]
    d_d, d_c = buf.cuda(), counts.cuda()
    d_K = Ks.reshape(Bn, Ks.shape[1], 9).contiguous().cuda()
    d_p = torch.tensor([list(q) + list(t) for q, t in poses], dtype=torch.float32).cuda() if poses is not None else None
    d_g = torch.tensor(groups, dtype=torch.int32).cuda()
    glob = torch.zeros(Bn, cap, 10, device="cuda") if with_global else None
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    if group_images is None:
        group_images = min(max(list(groups).count(g) for g in set(groups)), 16)
    nbytes = int(L.dd3d_op_group_bev_nms_large_scratch_bytes(Bn, cap, group_images))
    assert nbytes > 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    if poison is not None:
        scratch.fill_(poison)
    st = L.dd3d_op_group_bev_nms_large(_p(d_d), _p(d_c), _p(d_K), Ks.shape[1], _p(d_p), pose_mode, _p(d_g), num_groups,
                                       group_images, _p(glob), _p(scratch), _p(flags), Bn, cap, thr, max_dets, _stream())
    torch.cuda.synchronize()
    return st, d_d.cpu(), d_c.cpu(), glob.cpu() if glob is not None else None, int(flags.item())


def _same(a, b):
    st0, d0, c0, g0, f0 = a
    st1, d1, c1, g1, f1 = b
    assert st0 == st1 == 0 and f0 == f1
    assert torch.equal(c0, c1)
    for i, n in enumerate(c0.tolist()):
        assert torch.equal(d0[i, :n].view(torch.int32), d1[i, :n].view(torch.int32)), i
        if g0 is not None:
            assert torch.equal(g0[i, :n].view(torch.int32), g1[i, :n].view(torch.int32)), i


@pytest.mark.parametrize("name", sorted(GLOBAL_CASES))
@pytest.mark.parametrize("max_dets", [0, 10])
def test_group_large_equals_group_op_global(name, max_dets):
    seed, counts, groups, ng, cap, ncls, dom = GLOBAL_CASES[name]
    dets, Ks, poses = make_case(seed, counts, groups, num_classes=ncls, dominant=dom, num_views=3)
    buf, cnt_in, _ = pack(dets, Ks, cap)
    ref = run_kernel(buf, cnt_in, Ks, poses, groups, ng, cap, 0.3, max_dets, 0)
    out = run_large(buf, cnt_in, Ks, poses, groups, ng, cap, 0.3, max_dets, 0)
    _same(ref, out)


@pytest.mark.parametrize("thr", [0.3, 0.0])
def test_group_large_equals_group_op_camera(thr):
    counts = [1000, 731, 0, 1024]
    dets, Ks, _ = make_case(20, counts, [0, 1, 2, 3], num_classes=10, num_views=10, sort=True)
    buf, cnt_in, _ = pack(dets, Ks, 1024)
    ref = run_kernel(buf, cnt_in, Ks, None, [0, 1, 2, 3], 4, 1024, thr, 0, 1, with_global=False)
    out = run_large(buf, cnt_in, Ks, None, [0, 1, 2, 3], 4, 1024, thr, 0, 1, with_global=False)
    _same(ref, out)


def _bev_clusters(seed, n_clusters, per, num_classes, dominant, levels):
    """Camera-frame clusters of near-duplicate boxes on a 25 m grid (boxes <= 4 m, jitter 0.3 m): bounding circles far
    apart.  Scores take `levels` values: tie runs across multiples of the NMS block."""
    g = torch.Generator().manual_seed(seed)
    side = int(math.ceil(math.sqrt(n_clusters)))
    n = n_clusters * per
    c = torch.arange(n) // per
    base = torch.stack([25.0 * (c % side).float() - 12.5 * side, torch.zeros(n), 25.0 * (c // side).float() + 8.0], 1)
    t = base + torch.randn(n, 3, generator=g) * torch.tensor([0.3, 0.1, 0.3])
    q = torch.randn(n_clusters, 4, generator=g)
    q = (q / q.norm(dim=1, keepdim=True))[c] + torch.randn(n, 4, generator=g) * 0.02
    q = q / q.norm(dim=1, keepdim=True)
    size = (torch.rand(n_clusters, 3, generator=g) * 2 + 1)[c]
    cls = torch.randint(0, num_classes, (n, ), generator=g)
    if dominant:
        cls[torch.rand(n, generator=g) < dominant] = 0
    s = torch.floor(torch.rand(n, generator=g) * levels) / levels + 0.01
    return dict(quat=q, tvec=t, size=size, cls=cls, score3d=s, view=torch.zeros(n, dtype=torch.long))


@pytest.mark.parametrize("total,num_classes,dominant", [(5000, 1, None), (20000, 4, 0.9), (92000, 128, None),
                                                        (92000, 3, 0.95)])
def test_group_large_disjoint_clusters_exact(total, num_classes, dominant):
    per = 20
    n_clusters = total // per
    det = _bev_clusters(total + num_classes, n_clusters, per, num_classes, dominant, levels=10)
    K = torch.tensor([[700.0, 0.0, 320.0], [0.0, 690.0, 180.0], [0.0, 0.0, 1.0]])
    Ks = K.reshape(1, 1, 3, 3)
    n = n_clusters * per
    buf, cnt_in, _ = pack([det], Ks, n)
    out = run_large(buf, cnt_in, Ks, None, [0], 1, n, 0.3, 0, 1, with_global=False)
    assert out[0] == 0 and out[4] == 0
    # expectation: the grouped op with one cluster per image (group = image), survivors in slot order
    chunks = []
    for c0 in range(0, n_clusters, 256):
        m = min(256, n_clusters - c0)
        b = buf[0, c0 * per:(c0 + m) * per].reshape(m, per, 24).contiguous()
        st, d, c, _, f = run_kernel(b, torch.full((m, ), per, dtype=torch.int32), Ks.expand(m, 1, 3, 3), None,
                                    list(range(m)), m, per, 0.3, 0, 1, with_global=False)
        assert st == 0 and f == 0
        chunks += [d[i, :int(c[i])] for i in range(m)]
    ref = torch.cat(chunks)
    m = int(out[2][0])
    assert m == ref.shape[0] and m < n
    assert torch.equal(out[1][0, :m].view(torch.int32), ref.view(torch.int32))


def test_group_large_dense_cluster_vs_oracle():
    """One dense cluster: 3000 overlapping boxes of one class -- long greedy chains inside and across NMS blocks."""
    dets, Ks, _ = make_case(40, [3000], [0], num_classes=1, num_views=2, dup=0.6, sort=False)
    d = dets[0]
    d["tvec"] = d["tvec"] * torch.tensor([0.15, 1.0, 0.15]) + torch.tensor([0.0, 0.0, 6.0])
    buf, cnt_in, packed = pack(dets, Ks, 3000)
    st, out, cnt, _, flags = run_large(buf, cnt_in, Ks, None, [0], 1, 3000, 0.3, 0, 1, with_global=False)
    assert st == 0 and flags == 0
    keep = NT.bev_nms_camera(packed[0], 0.3)
    keep = keep.sort().values  # survivors keep their slot order
    m = int(cnt[0])
    assert m == keep.numel() and m < 3000 // 2
    assert torch.equal(out[0, :m, 5], packed[0]["score3d"][keep])
    assert torch.equal(out.view(torch.int32)[0, :m, 20].long(), keep)


def test_group_large_max_dets_across_groups_and_scratch():
    counts = [9000, 8000, 7000, 9500, 100, 0]
    groups = [0, 0, 0, 1, 1, 2]
    dets, Ks, poses = make_case(41, counts, groups, num_classes=5, num_views=4, dup=0.4)
    buf, cnt_in, _ = pack(dets, Ks, 9500)
    runs = [run_large(buf, cnt_in, Ks, poses, groups, 3, 9500, 0.3, 700, 0, poison=p) for p in (None, 0xFF, 0x00)]
    for r in runs:
        _same(runs[0], r)
    assert int(runs[0][2].sum()) == 700
    # the 700 best survivors of the call, each image's in slot order
    kept = torch.cat([runs[0][1][b, :int(runs[0][2][b]), 5] for b in range(len(counts))])
    assert kept.min() >= 0 and kept.numel() == 700


def test_group_large_capacity_flags():
    dets, Ks, poses = make_case(30, [20] * 17, [0] * 17, num_classes=3)
    buf, cnt_in, _ = pack(dets, Ks, 32)
    st, _, cnt, _, flags = run_large(buf, cnt_in, Ks, poses, [0] * 17, 1, 32, 0.3, 0, 0)
    assert st == 0 and flags == 32 and int(cnt[16]) == 0
    over = cnt_in[:2].clone()
    over[1] = 40
    st, _, cnt, _, flags = run_large(buf[:2], over, Ks[:2], poses[:2], [0, 0], 1, 32, 0.3, 0, 0)
    assert st == 0 and flags == 32


# ------------------------------------------------------------------------------------------------ wrappers
def _kitti_tta(mutate, monkeypatch=None, force_large=None):
    from dd3d_b200 import tta as tta_mod
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from oracle.gen_golden import tta_case
    cfg, x = tta_case()
    mutate(cfg)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    t = tta_mod.DD3DB200WithTTA(cfg, model)
    if force_large is not None:
        monkeypatch.setattr(t, "large_path", lambda: force_large)
    return t, x


def _instances_bytes(inst):
    return torch.cat([inst.pred_boxes.tensor, inst.scores_3d[:, None], inst.scores[:, None],
                      inst.pred_classes[:, None].float(), inst.pred_boxes3d.quat, inst.pred_boxes3d.depth.reshape(-1, 1)],
                     1).cpu()


def test_wrapper_large_path_equals_one_cta_path_on_the_fixture(monkeypatch):
    """The fixture config (6 views x POST_NMS_TOPK 100) fits the one-CTA ops; forced onto the large path it gives the same
    bits."""
    small, x = _kitti_tta(lambda cfg: None)
    assert not small.large_path()
    b = small([x])[0]["instances"]
    big, _ = _kitti_tta(lambda cfg: None, monkeypatch, force_large=True)
    a = big([x])[0]["instances"]
    assert small.overflow_flags() == 0 and big.overflow_flags() == 0 and len(a) > 100
    assert torch.equal(_instances_bytes(a), _instances_bytes(b))


def _golden_keys(box, cls):
    return [(int(c), ) + tuple(int(round(float(v) / 2.0)) for v in b) for b, c in zip(box, cls)]


@pytest.mark.parametrize("name", ["tta_large_nonms", "tta_large_nonms_bev", "tta_large_post200", "tta_large_16views"])
def test_wrapper_vs_emulating_oracle_and_reference_golden(name):
    """DD3DB200WithTTA on the large path against the bf16-emulating oracle and the reference's own DD3DWithTTA
    (tests/golden/<name>.npz): the tolerances of tests/test_tta.py, and the reference's output order -- descending
    scores_3d after the merged NMS / BEV NMS (merged_instances[keep]), view order without either."""
    import os
    import numpy as np
    from conftest import GOLDEN_DIR
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from dd3d_b200.tta import DD3DB200WithTTA
    from oracle import tta_large_oracle as TL
    from oracle.dd3d_oracle import DD3DOracle
    from util import quat_dist, rel_err
    cfg, x = TL.case(name)
    sd = make_state_dict(cfg)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    tta = DD3DB200WithTTA(cfg, model)
    assert tta.large_path()
    inst = tta([x])[0]["instances"]
    assert tta.overflow_flags() == 0
    g = np.load(os.path.join(GOLDEN_DIR, f"{name}.npz"))
    emu = TL.tta_forward(DD3DOracle(cfg, sd, emulate_bf16=True), x, cfg, nms_rotated=NT.nms_rotated)
    n, m, ng = len(inst), emu["score3d"].shape[0], g["scores_3d"].shape[0]
    assert abs(n - m) <= 0.1 * m and abs(n - ng) <= 0.15 * ng, (n, m, ng)
    s3 = inst.scores_3d.cpu()
    if name == "tta_large_nonms":
        assert n > 1024  # every candidate of every view
    else:
        assert torch.all(s3[:-1] >= s3[1:])  # the order of merged_instances[keep]
    ka, kb = _golden_keys(inst.pred_boxes.tensor.cpu(), inst.pred_classes.cpu()), _golden_keys(emu["box2d"], emu["cls"])
    # pairs on (class, box) keys that occur once on each side: without the 2-D NMS candidates of several levels share one
    from collections import Counter
    ca, cb = Counter(ka), Counter(kb)
    pos = {k: i for i, k in enumerate(kb) if cb[k] == 1}
    pairs = [(i, pos[k]) for i, k in enumerate(ka) if ca[k] == 1 and k in pos]
    assert len(pairs) >= (0.5 if name == "tta_large_nonms" else 0.7) * m
    ia, ib = (torch.tensor(p) for p in zip(*pairs))
    assert rel_err(inst.pred_boxes.tensor.cpu()[ia], emu["box2d"][ib], floor=16.0) < 0.1
    assert rel_err(s3[ia], emu["score3d"][ib], floor=0.05) < 0.2
    assert rel_err(inst.pred_boxes3d.depth.cpu()[ia].reshape(-1), emu["depth"][ib], floor=1.0) < 0.05
    assert quat_dist(inst.pred_boxes3d.quat.cpu()[ia], emu["quat"][ib]).median().item() < 0.05
    # the reference's own detections: the same (class, box) keys for most of them
    kg = set(_golden_keys(torch.as_tensor(g["boxes"]), torch.as_tensor(g["classes"])))
    assert sum(k in kg for k in ka) >= 0.7 * ng


def test_merge_sort_only_mode():
    """do_nms = 2: the concatenation sorted by scores_3d descending, ties in view order (stable argsort)."""
    buf = _view_dets(21, 6, 700, [700, 650, 0, 700, 3, 690], 5, levels=7)
    counts = [700, 650, 0, 700, 3, 690]
    views = _identity_views(6, flips=[a % 2 for a in range(6)])
    cat, f0 = run_merge(buf, counts, views, 0.5, 0, large=True)
    srt, f1 = run_merge(buf, counts, views, 0.5, 2, large=True)
    assert f0 == 0 and f1 == 0 and cat.shape[0] == sum(counts) > 1024
    order = torch.argsort(cat[:, 5], descending=True, stable=True)
    assert torch.equal(srt.view(torch.int32), cat[order].view(torch.int32))


def test_wrapper_raises_on_an_overflow_word():
    """A non-zero overflow word raises in the wrapper call itself: here the engine's own bit (more detections of a view
    than its output slots), folded into the call's word on the large path."""
    from oracle import tta_large_oracle as TL
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from dd3d_b200.tta import DD3DB200WithTTA
    cfg, x = TL.case("tta_large_post200")
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    tta = DD3DB200WithTTA(cfg, model)
    assert tta.large_path()
    model._release()
    model._desc.out_cap = 8  # far fewer slots than the views' detections
    with pytest.raises(RuntimeError, match="capacity exceeded"):
        tta([x])


def test_nuscenes_wrapper_bev_alone():
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import NuscenesDD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from dd3d_b200.tta import NuscenesDD3DB200WithTTA
    from oracle.gen_golden import NUSC_CASE, nusc_case_inputs
    cfg = get_cfg(NUSC_CASE[0], "nuscenes", meta_arch="NuscenesDD3D")
    cfg.DD3D.INFERENCE.DO_POSTPROCESS = False
    cfg.DD3D.INFERENCE.DO_NMS = False
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    cfg.TEST.AUG.MIN_SIZES = [96, 128]
    model = NuscenesDD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    t = NuscenesDD3DB200WithTTA(cfg, model)
    assert t.large_path()
    res = t(nusc_case_inputs())
    assert t.overflow_flags() == 0
    assert len(res) == 6 and sum(len(r["instances"]) for r in res) > 0
    assert all(r["instances"].has("pred_boxes3d_global") for r in res)
    for r in res:  # merged_instances[bev_nms keep], then the order-preserving sample aggregation: descending scores_3d
        s3 = r["instances"].scores_3d.cpu()
        assert torch.all(s3[:-1] >= s3[1:])


def test_shipped_config_makes_the_same_op_calls(monkeypatch):
    """The shipped configuration (one-CTA path): every library call of a TTA call is one the wrapper made before."""
    from dd3d_b200 import lib
    real = lib.load()
    calls = []

    class Rec:
        def __getattr__(self, name):
            fn = getattr(real, name)

            def wrapped(*a):
                calls.append(name)
                return fn(*a)
            return wrapped
    t, x = _kitti_tta(lambda cfg: None)
    assert not t.large_path()
    monkeypatch.setattr(lib, "load", lambda: Rec())
    t([x])
    ops = [c for c in calls if c.startswith("dd3d_op_")]
    assert ops == ["dd3d_op_tta_merged_cap", "dd3d_op_tta_merge_scratch_bytes", "dd3d_op_tta_merge"], ops
    assert not any(c.endswith("_large") for c in calls)
