"""GPU: the rotated BEV IoU (dd3d_op_rotated_iou, csrc/bev_geom.cuh) on the rectangle families of bev_geom_cases.py, and
the three BEV NMS kernels that threshold it (dd3d_op_bev_nms, dd3d_op_sample_aggregate, dd3d_op_group_bev_nms in camera
and global modes) on scenes of yaw-only boxes: rows of cars sharing edges, duplicates shifted along their heading on
either side of the threshold, the same object seen by two cameras of a sample or two TTA views, and tied scores_3d."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import bev_geom_cases as G
import nusc_tta_oracle as NT
from oracle import bev_nms_oracle as B
from test_group_bev_nms import _rig_pose, check_global, oracle_global, pack, run_kernel

BOUND = 1e-5
N = 1500


def _lib():
    from dd3d_b200 import lib
    return lib.load()


def gpu_iou(a, b):
    L = _lib()
    d_a, d_b = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    out = torch.full((a.shape[0], ), -1.0, device="cuda")
    st = L.dd3d_op_rotated_iou(C.c_void_p(d_a.data_ptr()), C.c_void_p(d_b.data_ptr()), a.shape[0],
                               C.c_void_p(out.data_ptr()), C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    return out.cpu().double().numpy()


# ------------------------------------------------------------------------------------------------ the IoU itself
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(G.FAMILIES))
def test_rotated_iou_family_vs_float64(name):
    a, b, _ = G.family(name, N, seed=1)
    ref = G.ref_clipper(a, b)
    ab, ba = gpu_iou(a, b), gpu_iou(b, a)
    err = np.abs(ab - ref)
    assert err.max() <= BOUND, (name, int((err > BOUND).sum()), float(err.max()), a[err.argmax()].tolist(),
                                b[err.argmax()].tolist(), float(ab[err.argmax()]), float(ref[err.argmax()]))
    assert ((ab >= 0) & (ab <= 1)).all() and ((ba >= 0) & (ba <= 1)).all()
    assert np.abs(ab - ba).max() <= BOUND
    if name == "identical":
        assert ab.min() >= 1 - BOUND


@pytest.mark.gpu
def test_rotated_iou_empty_call():
    L = _lib()
    assert L.dd3d_op_rotated_iou(None, None, 0, None, None) != 0  # null pointers are refused
    x = torch.zeros(5, device="cuda")
    assert L.dd3d_op_rotated_iou(C.c_void_p(x.data_ptr()), C.c_void_p(x.data_ptr()), 0, C.c_void_p(x.data_ptr()), None) == 0


# ------------------------------------------------------------------------------------------------ NMS scenes
def _rot_z(psi):
    c, s = math.cos(psi), math.sin(psi)
    return np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])


def _objects(rs, thr, origin, fwd, gaps):
    """Global yaw-only boxes (x, y, yaw, W, L, cls, score) in front of the rig; see the module docstring."""
    left = np.array([-fwd[1], fwd[0]])
    objs = []
    # rows of parked cars side by side (sharing long edges; 0.4 m apart with `gaps`), class 0; rows 16 m apart, so one
    # row never reaches another whatever its yaw
    for r in range(3):
        psi = rs.uniform(-math.pi, math.pi)
        W, Lh = rs.uniform(1.6, 2.2), rs.uniform(3.8, 5.2)
        step = W + (0.4 if gaps else 0.0)
        base = origin + fwd * (14.0 + 16.0 * r) + left * rs.uniform(-3, 3)
        n_w = np.array([-math.sin(psi), math.cos(psi)])
        for k in range(5):
            objs.append((base + (k - 2) * step * n_w, psi, W, Lh, 0, 0.2 + 0.5 * rs.rand()))
    # duplicates shifted along their heading: IoU (L - d) / (L + d) on both sides of the threshold, class 1; 22 m to the
    # side of the rows and 16 m from each other
    targets = [0.2, 0.0] if thr == 0.0 else [thr + 0.05, max(thr - 0.04, 0.01), thr + 0.2, 0.9]
    for j, iou in enumerate(targets):
        psi = rs.uniform(-math.pi, math.pi)
        W, Lh = rs.uniform(0.6, 2.5), rs.uniform(0.8, 6.0)
        d = Lh * (1 - iou) / (1 + iou) if iou > 0 else Lh + 0.5
        base = origin + fwd * (14.0 + 16.0 * j) + left * (22.0 + rs.uniform(-1, 1))
        h = np.array([math.cos(psi), math.sin(psi)])
        s = 0.3 + 0.6 * rs.rand()
        tie = j % 2 == 0  # tied scores_3d: the concatenation index decides which of the two survives
        objs.append((base, psi, W, Lh, 1, s))
        objs.append((base + d * h, psi, W, Lh, 1, s if tie else s - 0.05))
    return objs


def _record(obj, R_w, t_w, H=1.5):
    """A global box -> camera-frame quaternion / translation / size (W, L, H) through the camera pose."""
    from dd3d_b200.structures import matrix_to_quaternion_wxyz
    xy, psi, W, Lh, cls, score = obj
    R_c = R_w.T @ _rot_z(psi)
    t_c = R_w.T @ (np.array([xy[0], xy[1], 0.0]) - t_w)
    return torch.tensor(matrix_to_quaternion_wxyz(torch.tensor(R_c)), dtype=torch.float32), torch.tensor(t_c, dtype=torch.float32), \
        torch.tensor([W, Lh, H], dtype=torch.float32), cls, score


def make_scene(seed, thr, gaps=False, n_cams=3, num_views=1):
    """One sample group of `n_cams` overlapping cameras.  Camera 0 sees every object; camera 1 sees again the first box
    of every class-1 pair and two cars (cross-camera duplicates, one with a tied score); camera 2 sees the rest of the
    first row.  With num_views = 2 every detection of camera 0 is also reported under view 1 (a TTA duplicate)."""
    rs = np.random.RandomState(seed)
    poses = [_rig_pose(rs, 0) for _ in range(n_cams)]
    mats = []
    for q, t in poses:
        R = B.quaternion_to_matrix(torch.tensor(q, dtype=torch.float32)[None])[0].double().numpy()
        mats.append((R, np.array(t)))
    fwd = mats[0][0][:2, 2] / np.linalg.norm(mats[0][0][:2, 2])
    objs = _objects(rs, thr, mats[0][1][:2], fwd, gaps)
    pairs = [i for i, o in enumerate(objs) if o[4] == 1][::2]
    seen = [list(range(len(objs))), pairs + [0, 6], list(range(1, 5))]
    dets = []
    for cam in range(n_cams):
        rows = [(_record(objs[i], *mats[cam]), 0) for i in seen[cam]]
        if num_views == 2 and cam == 0:
            rows += [(r, 1) for r, _ in rows]
        q, t, sz, cl, sc = zip(*[r for r, _ in rows])
        score = torch.tensor(sc, dtype=torch.float32)
        if cam == 1:
            score[-1] = float(objs[6][5])  # tied with camera 0's copy of the same car
        d = dict(quat=torch.stack(q), tvec=torch.stack(t), size=torch.stack(sz), cls=torch.tensor(cl),
                 score3d=score, view=torch.tensor([v for _, v in rows]))
        o = torch.argsort(d["score3d"], descending=True, stable=True)  # the one-CTA kernel expects score order
        dets.append({k: v[o] for k, v in d.items()})
    Ks = torch.zeros(n_cams, num_views, 3, 3)
    for v in range(num_views):
        f = 1260.0 - 300.0 * v
        Ks[:, v] = torch.tensor([[f, 0.0, 800.0 - 160 * v], [0.0, f, 450.0 - 90 * v], [0.0, 0.0, 1.0]])
    buf, counts, packed = pack(dets, Ks, 64)
    assert all((d["tvec"][:, 2] > 1.0).all() for d in packed)
    return buf, counts, packed, Ks, poses


def _assert_clear_of_threshold(rects, cls, thr):
    """Every same-class pair: both float64 references agree and sit >= 1e-3 from thr (or are exactly 0 at thr 0)."""
    n = rects.shape[0]
    for i in range(n):
        for j in range(i + 1, n):
            if int(cls[i]) != int(cls[j]):
                continue
            a, b = rects[i].tolist(), rects[j].tolist()
            r1, r2 = B.rotated_iou(a, b), G.clipper_iou(a, b)
            if thr == 0.0 and r1 == 0.0 and r2 == 0.0:
                continue
            assert abs(r1 - r2) < 1e-4 and abs(r1 - thr) >= 1e-3, (i, j, r1, r2, thr)


def check_scene(packed, poses, thr):
    rects, cls = [], []
    for d, (pq, pt) in zip(packed, poses):
        q, t = B.to_global(d["quat"], d["tvec"], pq, pt)
        rects.append(B.boxes3d_to_rotated_boxes(q, t, d["size"]))
        cls.append(d["cls"])
        _assert_clear_of_threshold(NT.camera_rotated_boxes(d["quat"], d["tvec"], d["size"]), d["cls"], thr)
    _assert_clear_of_threshold(torch.cat(rects), torch.cat(cls), thr)


SCENES = [(0, 0.3, False), (1, 0.3, False), (2, 0.05, False), (3, 0.0, True), (4, 0.05, True)]


def test_scenes_are_clear_of_the_threshold():
    """CPU: the scene builder's guarantee (the GPU cases below compare keep sets exactly)."""
    for seed, thr, gaps in SCENES:
        _, _, packed, _, poses = make_scene(seed, thr, gaps)
        check_scene(packed, poses, thr)
        _, _, packed, _, _ = make_scene(seed, thr, gaps, num_views=2)
        for d in packed:
            _assert_clear_of_threshold(NT.camera_rotated_boxes(d["quat"], d["tvec"], d["size"]), d["cls"], thr)


def _slots(out, cnt, b):
    return out.view(torch.int32)[b, :int(cnt[b]), 20].long()


@pytest.mark.gpu
@pytest.mark.parametrize("seed,thr,gaps", SCENES)
@pytest.mark.parametrize("post", [0, 1])
def test_bev_nms_scene(seed, thr, gaps, post):
    L = _lib()
    buf, counts, packed, Ks, poses = make_scene(seed, thr, gaps)
    check_scene(packed, poses, thr)
    Bn, cap = buf.shape[0], buf.shape[1]
    # 2-D boxes inside the image, so the postprocess drops nothing and the survivors are the NMS keep set
    buf[:, :, 0:4] = torch.tensor([10.0, 20.0, 200.0, 220.0])
    sizes = torch.tensor([[900, 1600, 900, 1600]] * Bn, dtype=torch.int32)
    d_d, d_c = buf.cuda(), counts.cuda()
    d_K, d_p = Ks[:, 0].reshape(Bn, 9).contiguous().cuda(), torch.tensor([list(q) + list(t) for q, t in poses]).float().cuda()
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = L.dd3d_op_bev_nms(C.c_void_p(d_d.data_ptr()), C.c_void_p(d_c.data_ptr()), C.c_void_p(d_K.data_ptr()),
                           C.c_void_p(d_p.data_ptr()), C.c_void_p(sizes.cuda().data_ptr()), C.c_void_p(flags.data_ptr()),
                           Bn, cap, thr, post, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    assert int(flags.item()) == 0
    out, cnt = d_d.cpu(), d_c.cpu()
    for b, (d, (pq, pt)) in enumerate(zip(packed, poses)):
        keep = B.bev_nms_image(d, pq, pt, thr)
        assert torch.equal(_slots(out, cnt, b), keep), (b, _slots(out, cnt, b).tolist(), keep.tolist())
        cars = (d["cls"] == 0).sum()
        assert (d["cls"][keep] == 0).sum() == cars  # every car of every row survives


def _run_sample_aggregate(buf, counts, Ks, poses, thr, max_dets):
    L = _lib()
    Bn, cap = buf.shape[0], buf.shape[1]
    d_d, d_c = buf.cuda(), counts.cuda()
    d_K, d_p = Ks[:, 0].reshape(Bn, 9).contiguous().cuda(), torch.tensor([list(q) + list(t) for q, t in poses]).float().cuda()
    d_g = torch.zeros(Bn, dtype=torch.int32, device="cuda")
    glob = torch.zeros(Bn, cap, 10, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    scratch = torch.empty(int(L.dd3d_op_sample_aggregate_scratch_bytes(Bn, cap)), dtype=torch.uint8, device="cuda")
    st = L.dd3d_op_sample_aggregate(C.c_void_p(d_d.data_ptr()), C.c_void_p(d_c.data_ptr()), C.c_void_p(d_K.data_ptr()),
                                    C.c_void_p(d_p.data_ptr()), C.c_void_p(d_g.data_ptr()), 1, C.c_void_p(glob.data_ptr()),
                                    C.c_void_p(scratch.data_ptr()), C.c_void_p(flags.data_ptr()), Bn, cap, thr, max_dets,
                                    C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert st == 0
    torch.cuda.synchronize()
    assert int(flags.item()) == 0
    return d_d.cpu(), d_c.cpu(), glob.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("seed,thr,gaps", SCENES)
def test_sample_aggregate_and_group_global_scene(seed, thr, gaps):
    """The cameras of one sample: dd3d_op_sample_aggregate and dd3d_op_group_bev_nms (global mode) against the oracle
    and against each other, without a cap and with a max_dets that binds (across images, through tied scores)."""
    buf, counts, packed, Ks, poses = make_scene(seed, thr, gaps)
    check_scene(packed, poses, thr)
    groups = [0] * len(packed)
    free = oracle_global(packed, groups, poses, thr, 0)
    n_free = sum(int(r["slot"].numel()) for r in free)
    assert n_free < int(counts.sum())  # duplicates were suppressed
    for max_dets in (0, n_free - 3):
        ref = oracle_global(packed, groups, poses, thr, max_dets)
        out, cnt, glob = _run_sample_aggregate(buf, counts, Ks, poses, thr, max_dets)
        assert check_global(out, cnt, glob, ref, poses) == (max_dets or n_free)
        st, out2, cnt2, glob2, flags = run_kernel(buf, counts, Ks, poses, groups, 1, buf.shape[1], thr, max_dets, 0)
        assert st == 0 and flags == 0
        check_global(out2, cnt2, glob2, ref, poses)
        assert torch.equal(cnt, cnt2)
        for b in range(len(packed)):
            assert torch.equal(_slots(out, cnt, b), _slots(out2, cnt2, b))
        # every car survives when nothing caps the call: rows of side-by-side cars never suppress each other
        if not max_dets:
            cars = int((packed[0]["cls"] == 0).sum())  # camera 0 sees every car; the other cameras' copies go
            assert sum(int((r["cls"] == 0).sum()) for r in ref) == cars


@pytest.mark.gpu
@pytest.mark.parametrize("seed,thr,gaps", SCENES)
def test_group_camera_mode_tta_scene(seed, thr, gaps):
    """Merged TTA sets: every detection of camera 0 also under a second view with its own K, per-image camera-frame NMS."""
    buf, counts, packed, Ks, _ = make_scene(seed, thr, gaps, num_views=2)
    Bn = buf.shape[0]
    st, out, cnt, _, flags = run_kernel(buf, counts, Ks, None, list(range(Bn)), Bn, buf.shape[1], thr, 0, 1,
                                        with_global=False)
    assert st == 0 and flags == 0
    for b, d in enumerate(packed):
        keep = NT.bev_nms_camera(d, thr)
        assert torch.equal(_slots(out, cnt, b), torch.sort(keep).values), (b, _slots(out, cnt, b).tolist(), keep.tolist())
    assert int(cnt[0]) <= int(counts[0]) // 2  # each view-1 copy went
