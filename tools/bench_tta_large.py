"""Times the large-set TTA path (csrc/tta_large.cu) per image on KITTI-sized inputs (384x1272 mapped from 375x1242, 5 scales
x flip = 10 views), for V2-99 and DLA-34 with synthetic weights, in two configurations the one-CTA merge cannot hold:
  * no_nms_bev   DD3D.INFERENCE.DO_NMS False + DO_BEV_NMS True (per-view BEV NMS on every candidate, merged BEV NMS);
  * post_topk_200  FCOS2D.INFERENCE.POST_NMS_TOPK 200 (up to 2 000 merged detections).
Reports ms per image (CUDA events around whole wrapper calls), the merged-set size per image (after the merge) and the
output size, the device time of each operator of the merge / NMS steps (CUDA events around the C calls), and the card's
name and power limit read in the same run.  Synthetic weights give other candidate counts than a trained checkpoint:
read the times next to the counts (the synthetic weights give small merged sets).  `ops_92000_boxes`: the device time of
the two large-set operators alone on 92 000 synthetic boxes per image.  Prints one JSON line.  python tools/bench_tta_large.py [--images 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dd3d_b200 import lib as _lib  # noqa: E402
from dd3d_b200 import tta as tta_mod  # noqa: E402
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.meta_arch import DD3DB200  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict  # noqa: E402

TIMED = ("dd3d_op_tta_merge", "dd3d_op_tta_merge_large", "dd3d_op_bev_nms", "dd3d_op_bev_nms_large",
         "dd3d_op_group_bev_nms", "dd3d_op_group_bev_nms_large")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[0] if q.stdout else "")


class _Timer:
    """Proxy of the loaded library: CUDA events around every call of the operators in TIMED."""
    def __init__(self, real):
        self.real, self.events = real, []

    def __getattr__(self, name):
        fn = getattr(self.real, name)
        if name not in TIMED:
            return fn

        def timed(*a):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a)
            e1.record()
            self.events.append((name, e0, e1))
            return r
        return timed


def run(arch, mode, images):
    cfg = get_cfg(arch, "kitti_3d")
    cfg.DD3D.INFERENCE.DO_POSTPROCESS = False
    if mode == "no_nms_bev":
        cfg.DD3D.INFERENCE.DO_NMS = False
        cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    else:
        cfg.DD3D.FCOS2D.INFERENCE.POST_NMS_TOPK = 200
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    tta = tta_mod.DD3DB200WithTTA(cfg, model, world_size=8)  # TEST.IMS_PER_BATCH // 8 views per model call, as shipped
    assert tta.large_path()
    inputs = make_inputs(images + 1, 384, 1272, 721.5)
    pose = make_nusc_inputs(1, 8, 8, 100.0)[0]["pose"]
    for x in inputs:
        x["height"], x["width"] = 375, 1242
        x["pose"] = pose
    merged = []
    merge_image = tta._merge_image

    def counted_merge(x, out, n_out, *a, **k):
        r = merge_image(x, out, n_out, *a, **k)
        merged.append(n_out.clone())
        return r

    tta._merge_image = counted_merge
    real = _lib.load()
    timer = _Timer(real)
    _lib._lib = timer  # lib.load() returns the proxy
    try:
        tta([inputs[0]])  # warm-up: plans, resize tables, allocator
        torch.cuda.synchronize()
        timer.events.clear()
        merged.clear()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        n_out = 0
        for x in inputs[1:]:
            n_out += len(tta([x])[0]["instances"])
        e1.record()
        torch.cuda.synchronize()
    finally:
        _lib._lib = real
    op_ms = {}
    for name, a, b in timer.events:
        op_ms[name] = op_ms.get(name, 0.0) + a.elapsed_time(b) / images
    return {"ms_per_image": e0.elapsed_time(e1) / images,
            "merged_per_image": sum(int(m.sum()) for m in merged) / images,
            "out_per_image": n_out / images, "op_device_ms_per_image": op_ms, "overflow_flags": tta.overflow_flags()}


def large_ops(steps=5):
    """Device time of the two large-set operators on 92 000 synthetic boxes per image (16 views x 5 750): random boxes
    over a wide field, a third of them near-duplicates, 90 % in one class -- the worst case of the one-CTA-per-segment
    NMS (one segment holds most rows) -- plus the same with 128 classes."""
    import ctypes as C
    L = _lib.load()
    dev = "cuda"
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    res = {}
    for name, ncls, dom in (("one_class_90pct", 3, 0.9), ("classes_128", 128, None)):
        g = torch.Generator().manual_seed(5)
        A, cap = 16, 5750
        n = A * cap
        xy = torch.rand(n, 2, generator=g) * 4000
        m = n // 3
        xy[n - m:] = xy[:m] + torch.randn(m, 2, generator=g) * 2
        buf = torch.zeros(n, 24)
        buf[:, 0:2], buf[:, 2:4] = xy, xy + 30
        buf[:, 4] = buf[:, 5] = torch.rand(n, generator=g)
        buf[:, 8] = 1.0
        buf[:, 12], buf[:, 13] = xy[:, 0] * 0.1 + 100, 180.0
        buf[:, 14] = xy[:, 1] * 0.02 + 5
        buf[:, 15:18] = 1.5
        cls = torch.randint(0, ncls, (n, ), generator=g)
        if dom:
            cls[torch.rand(n, generator=g) < dom] = 0
        buf.view(torch.int32)[:, 6] = cls.to(torch.int32)
        buf.view(torch.int32)[:, 20] = torch.arange(n, dtype=torch.int32)
        d_in = buf.reshape(A, cap, 24).contiguous().to(dev)
        counts = torch.full((A, ), cap, dtype=torch.int32, device=dev)
        views = (_lib.TtaView * A)()
        for a in range(A):
            views[a].view_w, views[a].inv_sx[0], views[a].inv_sy[0], views[a].inv_sx[1], views[a].inv_sy[1] = \
                640.0, 1.0, 1.0, 1.0, 1.0
            for i, v in enumerate((700.0, 0.0, 320.0, 0.0, 690.0, 180.0, 0.0, 0.0, 1.0)):
                views[a].K_view[i] = views[a].K_orig[i] = v
        out = torch.empty(n, 24, device=dev)
        n_out = torch.zeros(2, dtype=torch.int32, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        ms_scr = torch.empty(int(L.dd3d_op_tta_merge_large_scratch_bytes(A, cap)), dtype=torch.uint8, device=dev)
        K = torch.tensor([700.0, 0.0, 320.0, 0.0, 690.0, 180.0, 0.0, 0.0, 1.0], device=dev).reshape(1, 1, 9)
        grp = torch.zeros(1, dtype=torch.int32, device=dev)
        gs_scr = torch.empty(int(L.dd3d_op_group_bev_nms_large_scratch_bytes(1, n, 1)), dtype=torch.uint8, device=dev)
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        times = {"merge_nms": 0.0, "group_bev_camera": 0.0}
        for it in range(steps + 1):
            e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            e[0].record()
            _lib.check(L.dd3d_op_tta_merge_large(p(d_in), p(counts), views, A, cap, 0.5, 1, p(ms_scr), p(out),
                                                 p(n_out), p(flags), stream))
            e[1].record()
            cat = d_in.reshape(1, n, 24).clone()
            cnt = torch.full((1, ), n, dtype=torch.int32, device=dev)
            e2 = torch.cuda.Event(enable_timing=True)
            e2.record()
            _lib.check(L.dd3d_op_group_bev_nms_large(p(cat), p(cnt), p(K), 1, None, 1, p(grp), 1, 1, None, p(gs_scr),
                                                     p(flags), 1, n, 0.3, 0, stream))
            e[2].record()
            torch.cuda.synchronize()
            if it:  # the first call configures the kernels
                times["merge_nms"] += e[0].elapsed_time(e[1]) / steps
                times["group_bev_camera"] += e2.elapsed_time(e[2]) / steps
        res[name] = dict(boxes=n, merge_survivors=int(n_out[0]), bev_survivors=int(cnt[0]),
                         device_ms=times, overflow_flags=int(flags.item()))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    line = {"metric": "tta_large_ms_per_image", "card": card(), "mapped_size": [384, 1272], "views": 10}
    for arch in ("v2_99", "dla34"):
        for mode in ("no_nms_bev", "post_topk_200"):
            line[f"{arch}_{mode}"] = run(arch, mode, args.images)
    line["ops_92000_boxes"] = large_ops()
    print(json.dumps(line))


if __name__ == "__main__":
    main()
