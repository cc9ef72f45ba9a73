"""Grouped rotated BEV NMS (dd3d_op_group_bev_nms, csrc/bev_nms_group.cu): CPU pins of the test oracle's shortcuts, GPU
parity with the oracle on sets far beyond the one-CTA kernels' limits, capacity flags and determinism."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import nusc_tta_oracle as NT
from oracle import bev_nms_oracle as B
from util import quat_dist

CAM_TO_VEHICLE_WXYZ = (0.5, -0.5, 0.5, -0.5)  # CAMERA_TO_VEHICLE_ROTATION (bev_nms.py:27-32) as a quaternion


def _rig_pose(rs, group):
    """Camera (x right, y down, z forward) -> world of a nearly parallel rig: cameras of one group see overlapping boxes."""
    from dd3d_b200.structures import matrix_to_quaternion_wxyz
    yaw = math.radians(rs.uniform(-6, 6) + 40.0 * group)
    R = np.array([[math.sin(yaw), 0.0, math.cos(yaw)], [-math.cos(yaw), 0.0, math.sin(yaw)], [0.0, -1.0, 0.0]])
    t = [float(v) for v in rs.randn(3) * 0.5 + np.array([60.0 * group, -20.0 * group, 0.0])]
    return matrix_to_quaternion_wxyz(torch.tensor(R)), t


def make_case(seed, counts, groups, num_classes=10, dominant=None, num_views=1, dup=0.25, sort=False):
    """Seeded camera-frame detections per image: `counts[b]` boxes spread over a wide field, a fraction `dup` of them
    jittered copies of others (so suppression happens), per-view intrinsics, rig poses per group."""
    g = torch.Generator().manual_seed(seed)
    rs = np.random.RandomState(seed)
    Ks = torch.zeros(len(counts), num_views, 3, 3)
    dets, poses = [], []
    for b, n in enumerate(counts):
        for v in range(num_views):
            f = 700.0 + 40.0 * v
            Ks[b, v] = torch.tensor([[f, 0.0, 320.0 + 5 * v], [0.0, f * 0.98, 180.0 - 3 * v], [0.0, 0.0, 1.0]])
        q = torch.randn(n, 4, generator=g)
        q = q / q.norm(dim=1, keepdim=True)
        t = torch.randn(n, 3, generator=g) * torch.tensor([12.0, 0.5, 1.0])
        t[:, 2] = torch.rand(n, generator=g) * 45 + 4
        size = torch.rand(n, 3, generator=g) * 3 + 1
        m = int(n * dup)
        if m and n > m:
            src = torch.randint(0, n - m, (m, ), generator=g)
            t[n - m:] = t[src] + torch.randn(m, 3, generator=g) * 0.3
            q[n - m:] = q[src]
            size[n - m:] = size[src]
        cls = torch.randint(0, num_classes, (n, ), generator=g)
        if dominant is not None:
            cls[torch.rand(n, generator=g) < dominant] = 0
        if m and n > m:
            cls[n - m:] = cls[src]
        score = torch.rand(n, generator=g)
        view = torch.randint(0, num_views, (n, ), generator=g)
        if sort:
            o = torch.argsort(score, descending=True, stable=True)
            q, t, size, cls, score, view = q[o], t[o], size[o], cls[o], score[o], view[o]
        dets.append(dict(quat=q, tvec=t, size=size, cls=cls, score3d=score, view=view))
        poses.append(_rig_pose(rs, groups[b]))
    return dets, Ks, poses


def pack(dets, Ks, cap):
    """-> engine records [B][cap][24] (tvec through (proj_ctr, depth) and the detection's view K, level = view) and the
    oracle's dicts with the translation the kernel recomputes."""
    Bn = len(dets)
    buf = torch.zeros(Bn, cap, 24)
    counts = torch.zeros(Bn, dtype=torch.int32)
    packed = []
    inv = torch.linalg.inv(Ks.double()).float()
    for b, det in enumerate(dets):
        det = dict(det)
        n = det["quat"].shape[0]
        K, iK = Ks[b][det["view"]], inv[b][det["view"]]
        depth = det["tvec"][:, 2]
        uvw = torch.matmul(K, det["tvec"].unsqueeze(-1)).squeeze(-1)
        pc = uvw[:, :2] / uvw[:, 2:]
        det["tvec"] = torch.matmul(iK, torch.cat([pc, torch.ones(n, 1)], 1).unsqueeze(-1)).squeeze(-1) * depth[:, None]
        buf[b, :n, 5] = det["score3d"]
        buf[b, :n, 8:12] = det["quat"]
        buf[b, :n, 12:14] = pc
        buf[b, :n, 14] = depth
        buf[b, :n, 15:18] = det["size"]
        buf.view(torch.int32)[b, :n, 6] = det["cls"].to(torch.int32)
        buf.view(torch.int32)[b, :n, 7] = det["view"].to(torch.int32)
        buf.view(torch.int32)[b, :n, 20] = torch.arange(n, dtype=torch.int32)
        counts[b] = n
        packed.append(det)
    return buf, counts, packed


def run_kernel(buf, counts, Ks, poses, groups, num_groups, cap, thr, max_dets, pose_mode, with_global=True,
               poison=None, group_images=None):
    from dd3d_b200 import lib
    L = lib.load()
    Bn = buf.shape[0]
    d_d, d_c = buf.cuda(), counts.cuda()
    d_K = Ks.reshape(Bn, Ks.shape[1], 9).contiguous().cuda()
    d_p = torch.tensor([list(q) + list(t) for q, t in poses], dtype=torch.float32).cuda() if poses is not None else None
    d_g = torch.tensor(groups, dtype=torch.int32).cuda()
    glob = torch.zeros(Bn, cap, 10, device="cuda") if with_global else None
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    if group_images is None:  # the largest group of the call
        group_images = max(list(groups).count(g) for g in set(groups))
    group_images = min(group_images, 16)
    nbytes = int(L.dd3d_op_group_bev_nms_scratch_bytes(Bn, cap, group_images))
    assert nbytes > 0
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    if poison is not None:
        scratch.fill_(poison)
    st = L.dd3d_op_group_bev_nms(C.c_void_p(d_d.data_ptr()), C.c_void_p(d_c.data_ptr()), C.c_void_p(d_K.data_ptr()),
                                 Ks.shape[1], C.c_void_p(d_p.data_ptr()) if d_p is not None else None, pose_mode,
                                 C.c_void_p(d_g.data_ptr()), num_groups, group_images,
                                 C.c_void_p(glob.data_ptr()) if glob is not None else None,
                                 C.c_void_p(scratch.data_ptr()), C.c_void_p(flags.data_ptr()), Bn, cap, thr, max_dets,
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return st, d_d.cpu(), d_c.cpu(), glob.cpu() if glob is not None else None, int(flags.item())


def check_global(out, cnt, glob, ref, poses):
    total = 0
    for b, r in enumerate(ref):
        m = int(cnt[b])
        total += m
        assert m == r["score3d"].shape[0], (b, m, r["score3d"].shape[0])
        assert torch.equal(out[b, :m, 5], r["score3d"])  # same survivors in the same (original) order
        assert torch.equal(out.view(torch.int32)[b, :m, 20].long(), r["slot"])
        if m and glob is not None:
            q64, t64 = NT.to_global_f64(r["quat"], r["tvec"], *poses[b])
            assert quat_dist(glob[b, :m, 0:4].double(), q64).max().item() < 1e-5
            np.testing.assert_allclose(glob[b, :m, 4:7].double().numpy(), t64.numpy(), rtol=1e-5, atol=1e-4)
            np.testing.assert_allclose(glob[b, :m, 7:10].numpy(), r["size"].numpy(), rtol=0, atol=0)
    return total


def oracle_global(packed, groups, poses, thr, max_dets):
    dets = [dict(d, slot=torch.arange(d["quat"].shape[0])) for d in packed]
    return NT.sample_aggregate(dets, groups, poses, thr, max_dets)


GLOBAL_CASES = {
    # name: (seed, counts per image, groups, num_groups, cap, num_classes, dominant)
    "2x6x900": (10, [900 + 7 * i for i in range(12)], [0] * 6 + [1] * 6, 2, 1024, 10, None),
    "interleaved": (11, [850 - 11 * i for i in range(12)], [0, 0, 0, 1, 1, 1, 0, 0, 0, 1, 1, 1], 2, 1024, 10, None),
    "flood": (12, [300, 280, 310, 260, 290, 305], [0] * 6, 1, 512, 4, 0.9),
    "empty": (13, [0, 120, 0, 0, 0, 0, 90, 0, 200, 0, 0, 60], [0, 0, 1, 1, 2, 2, 0, 0, 3, 3, 0, 3], 5, 256, 5, None),
}



# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("seed,thr", [(0, 0.3), (1, 0.05), (2, 0.0)])
def test_shortcut_nms_equals_oracle(seed, thr):
    """The test oracle's circle shortcut changes nothing: same kept indices, same order as bev_nms_oracle.nms_rotated."""
    dets, _, poses = make_case(seed, [160, 140], [0, 0], num_classes=3)
    for d, (pq, pt) in zip(dets, poses):
        q, t = B.to_global(d["quat"], d["tvec"], pq, pt)
        rb = B.boxes3d_to_rotated_boxes(q, t, d["size"])
        assert torch.equal(NT.nms_rotated(rb, d["score3d"], d["cls"], thr), B.nms_rotated(rb, d["score3d"], d["cls"], thr))


def test_camera_rotated_boxes_equal_global_path_with_camera_pose():
    """bev_nms' default pose (CAMERA_TO_VEHICLE_ROTATION, no translation) == the global path through that pose."""
    dets, _, _ = make_case(3, [50], [0])
    d = dets[0]
    q, t = B.to_global(d["quat"], d["tvec"], CAM_TO_VEHICLE_WXYZ, (0.0, 0.0, 0.0))
    a = NT.camera_rotated_boxes(d["quat"], d["tvec"], d["size"])
    b = B.boxes3d_to_rotated_boxes(q, t, d["size"])
    np.testing.assert_allclose(a[:, :4].numpy(), b[:, :4].numpy(), rtol=1e-5, atol=1e-4)
    da = (a[:, 4] - b[:, 4] + 180.0) % 360.0 - 180.0
    assert da.abs().max().item() < 1e-3


@pytest.mark.parametrize("name,image,thr", [("2x6x900", 0, 0.3), ("flood", 0, 0.3), ("flood", 1, 0.0)])
def test_shortcut_nms_equals_oracle_on_kernel_cases(name, image, thr):
    """The same pin on whole images of the GPU cases below (900 boxes over 10 classes; a one-class flood)."""
    seed, counts, groups, ng, cap, ncls, dom = GLOBAL_CASES[name]
    dets, Ks, poses = make_case(seed, counts, groups, num_classes=ncls, dominant=dom, num_views=3)
    _, _, packed = pack(dets, Ks, cap)
    d, (pq, pt) = packed[image], poses[image]
    q, t = B.to_global(d["quat"], d["tvec"], pq, pt)
    rb = B.boxes3d_to_rotated_boxes(q, t, d["size"])
    keep = NT.nms_rotated(rb, d["score3d"], d["cls"], thr)
    assert torch.equal(keep, B.nms_rotated(rb, d["score3d"], d["cls"], thr))
    assert keep.numel() < d["score3d"].numel()


def test_fast_sample_aggregate_equals_oracle():
    import sys
    import os
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_nuscenes import aggregate_case
    for seed, max_dets in ((7, 1000), (8, 150)):
        dets, gids, poses = aggregate_case(seed)
        a = NT.sample_aggregate(dets, gids, poses, 0.3, max_dets)
        b = B.sample_aggregate(dets, gids, poses, 0.3, max_dets)
        for x, y in zip(a, b):
            assert torch.equal(x["score3d"], y["score3d"]) and torch.equal(x["tvec_global"], y["tvec_global"])


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name,max_dets", [("2x6x900", 0), ("2x6x900", 500), ("interleaved", 150), ("interleaved", 1),
                                           ("flood", 0), ("flood", 500), ("empty", 0), ("empty", 40)])
def test_group_bev_nms_global_vs_oracle(name, max_dets):
    seed, counts, groups, ng, cap, ncls, dom = GLOBAL_CASES[name]
    dets, Ks, poses = make_case(seed, counts, groups, num_classes=ncls, dominant=dom, num_views=3)
    buf, cnt_in, packed = pack(dets, Ks, cap)
    ref = oracle_global(packed, groups, poses, 0.3, max_dets)
    st, out, cnt, glob, flags = run_kernel(buf, cnt_in, Ks, poses, groups, ng, cap, 0.3, max_dets, 0)
    assert st == 0 and flags == 0
    total = check_global(out, cnt, glob, ref, poses)
    n_in = int(cnt_in.sum())
    assert total < n_in  # suppression happened
    if max_dets:
        assert total == max_dets  # every capped case has more survivors than max_dets: the cap binds across groups
    if name == "2x6x900":  # beyond both one-CTA kernels: > 256 per image, > 768 per group
        assert min(counts) > 256 and sum(counts[:6]) > 768
    if name == "flood":
        assert int((torch.cat([d["cls"] for d in dets]) == 0).sum()) >= 1500


@pytest.mark.gpu
def test_group_bev_nms_camera_mode_per_view_intrinsics():
    """Per-image bev_nms of merged TTA sets: group = image, camera-frame default pose, 10 views with their own K."""
    counts = [1000, 731, 0, 1024]
    dets, Ks, _ = make_case(20, counts, [0, 1, 2, 3], num_classes=10, num_views=10, sort=True)
    buf, cnt_in, packed = pack(dets, Ks, 1024)
    st, out, cnt, _, flags = run_kernel(buf, cnt_in, Ks, None, [0, 1, 2, 3], 4, 1024, 0.3, 0, 1, with_global=False)
    assert st == 0 and flags == 0
    for b, d in enumerate(packed):
        keep = NT.bev_nms_camera(d, 0.3)
        m = int(cnt[b])
        assert m == keep.numel(), (b, m, keep.numel())
        assert torch.equal(out[b, :m, 5], d["score3d"][keep])
        assert torch.equal(out.view(torch.int32)[b, :m, 7], d["view"][keep].to(torch.int32))
        if counts[b]:
            assert m < counts[b]


@pytest.mark.gpu
def test_group_bev_nms_capacity():
    from dd3d_b200 import lib
    L = lib.load()
    # 17 images in one group: flagged (bit 5 = 32), the call itself completes
    counts = [20] * 17
    dets, Ks, poses = make_case(30, counts, [0] * 17, num_classes=3)
    buf, cnt_in, _ = pack(dets, Ks, 32)
    st, _, cnt, _, flags = run_kernel(buf, cnt_in, Ks, poses, [0] * 17, 1, 32, 0.3, 0, 0)
    assert st == 0 and flags == 32
    assert int(cnt[16]) == 0 and int(cnt[:16].min()) > 0
    # 7 images in a group sized for 6
    st, _, cnt, _, flags = run_kernel(buf[:7], cnt_in[:7], Ks[:7], poses[:7], [0] * 7, 1, 32, 0.3, 0, 0, group_images=6)
    assert st == 0 and flags == 32 and int(cnt[6]) == 0
    # a count above cap: flagged instead of silently truncated
    over = cnt_in[:2].clone()
    over[1] = 40
    st, _, cnt, _, flags = run_kernel(buf[:2], over, Ks[:2], poses[:2], [0, 0], 1, 32, 0.3, 0, 0)
    assert st == 0 and flags == 32
    # arguments beyond the kernel's limits are refused on the host, before any launch
    assert L.dd3d_op_group_bev_nms_scratch_bytes(1, 2048, 1) < 0 and L.dd3d_op_group_bev_nms_scratch_bytes(257, 16, 1) < 0
    assert L.dd3d_op_group_bev_nms_scratch_bytes(4, 16, 17) < 0 and L.dd3d_op_group_bev_nms_scratch_bytes(4, 16, 0) < 0
    assert L.dd3d_op_group_bev_nms_scratch_bytes(12, 1024, 1) < L.dd3d_op_group_bev_nms_scratch_bytes(12, 1024, 6)
    dets, Ks, poses = make_case(31, [10, 10], [0, 0], num_classes=3)
    buf, cnt_in, _ = pack(dets, Ks, 2048)
    assert _refused(L, buf, cnt_in, Ks, poses, 2048) == -1


def _refused(L, buf, counts, Ks, poses, cap):
    d = buf.cuda()
    c = counts.cuda()
    k = Ks.reshape(buf.shape[0], -1).contiguous().cuda()
    p = torch.tensor([list(q) + list(t) for q, t in poses], dtype=torch.float32).cuda()
    g = torch.zeros(buf.shape[0], dtype=torch.int32, device="cuda")
    f = torch.zeros(1, dtype=torch.int32, device="cuda")
    s = torch.empty(256, dtype=torch.uint8, device="cuda")
    st = L.dd3d_op_group_bev_nms(C.c_void_p(d.data_ptr()), C.c_void_p(c.data_ptr()), C.c_void_p(k.data_ptr()), 1,
                                 C.c_void_p(p.data_ptr()), 0, C.c_void_p(g.data_ptr()), 1, 2, None, C.c_void_p(s.data_ptr()),
                                 C.c_void_p(f.data_ptr()), buf.shape[0], cap, 0.3, 0,
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert int(f.item()) == 0
    return st


@pytest.mark.gpu
def test_group_bev_nms_deterministic_and_scratch_independent():
    seed, counts, groups, ng, cap, ncls, dom = GLOBAL_CASES["2x6x900"]
    dets, Ks, poses = make_case(seed, counts, groups, num_classes=ncls, num_views=3)
    buf, cnt_in, _ = pack(dets, Ks, cap)
    runs = [run_kernel(buf, cnt_in, Ks, poses, groups, ng, cap, 0.3, 500, 0, poison=p) for p in (None, None, 0xFF, 0x00)]
    for st, out, cnt, glob, flags in runs:
        assert st == 0 and flags == 0
        assert torch.equal(out.view(torch.int32), runs[0][1].view(torch.int32))
        assert torch.equal(cnt, runs[0][2])
        assert torch.equal(glob.view(torch.int32), runs[0][3].view(torch.int32))
