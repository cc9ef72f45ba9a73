"""Times the BEV NMS of DD3D.forward (DO_BEV_NMS) on the multi-CTA kernels and the DLA-34 KITTI forward with it.
Prints one JSON line.  python tools/bench_bev_nms.py [--steps 20]

  * bev_ms: device time (CUDA events) of one dd3d_op_bev_nms_large call at n = 1000 and 5750 boxes per image, B = 8 and
    32: seeded camera-frame boxes, 10 classes, scattered over 80 m x 80 m in front of the camera (some overlap, so the
    scan suppresses), in random order;
  * images_per_s: DLA-34 KITTI (384 x 1280, B = 8) end to end through DD3DB200.forward, default config next to
    DO_NMS False + DO_BEV_NMS (every candidate of an image enters the BEV NMS);
  * the card's name and power limit, read in the same run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dd3d_b200 import lib  # noqa: E402
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.meta_arch import DD3DB200  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402


def random_records(B, n, seed):
    """[B][n][24] engine records: boxes in front of a pinhole camera (tvec through proj_ctr and depth), K [B][9], poses."""
    g = torch.Generator().manual_seed(seed)
    K = torch.tensor([[721.5, 0.0, 640.0], [0.0, 721.5, 192.0], [0.0, 0.0, 1.0]])
    x = torch.rand(B, n, generator=g) * 80 - 40
    z = torch.rand(B, n, generator=g) * 80 + 5
    y = torch.rand(B, n, generator=g) * 2
    q = torch.randn(B, n, 4, generator=g)
    q[..., 1] = q[..., 3] = 0  # yaw about the camera's y axis
    q = q / q.norm(dim=-1, keepdim=True)
    buf = torch.zeros(B, n, 24)
    buf[..., 0:4] = torch.tensor([10.0, 20.0, 200.0, 220.0])
    buf[..., 5] = torch.rand(B, n, generator=g)
    buf[..., 8:12] = q
    buf[..., 12] = K[0, 0] * x / z + K[0, 2]
    buf[..., 13] = K[1, 1] * y / z + K[1, 2]
    buf[..., 14] = z
    buf[..., 15:18] = torch.rand(B, n, 3, generator=g) * 4 + 0.5
    buf.view(torch.int32)[..., 6] = torch.randint(0, 10, (B, n), generator=g, dtype=torch.int32)
    poses = torch.tensor([[1.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]]).repeat(B, 1)
    return buf, K.reshape(1, 9).repeat(B, 1), poses


def bev_ms(B, n, steps):
    L = lib.load()
    buf, K, poses = random_records(B, n, seed=B * 10000 + n)
    d_buf, d_K, d_p = buf.cuda(), K.cuda(), poses.cuda()
    d_sizes = torch.tensor([[384, 1280, 384, 1280]], dtype=torch.int32).repeat(B, 1).cuda()
    work = torch.empty_like(d_buf)
    counts = torch.full((B, ), n, dtype=torch.int32, device="cuda")
    cnt = torch.empty_like(counts)
    scratch = torch.empty(int(L.dd3d_op_bev_nms_large_scratch_bytes(B, n)), dtype=torch.uint8, device="cuda")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    ms = []
    for i in range(steps + 3):
        work.copy_(d_buf)  # the op works in place
        cnt.copy_(counts)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        lib.check(L.dd3d_op_bev_nms_large(C.c_void_p(work.data_ptr()), C.c_void_p(cnt.data_ptr()), C.c_void_p(d_K.data_ptr()),
                                          C.c_void_p(d_p.data_ptr()), C.c_void_p(d_sizes.data_ptr()),
                                          C.c_void_p(scratch.data_ptr()), C.c_void_p(flags.data_ptr()), B, n, 0.05, 1,
                                          C.c_void_p(stream)))
        e1.record()
        if i >= 3:
            ms.append((e0, e1))
    torch.cuda.synchronize()
    assert int(flags.item()) == 0
    t = sorted(a.elapsed_time(b) for a, b in ms)
    return dict(median=round(t[len(t) // 2], 4), min=round(t[0], 4), kept_per_image=round(float(cnt.float().mean()), 1))


def images_per_s(bev, steps, B=8):
    cfg = get_cfg("dla34", "kitti_3d")
    if bev:
        cfg.DD3D.INFERENCE.DO_NMS = False
        cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    inputs = make_inputs(B, 384, 1280, 721.5)
    for x in inputs:
        x["pose"] = ([1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 0.0])
    for _ in range(3):
        model(inputs)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        out = model(inputs)  # ends in the counts D2H: a device synchronise
    dt = time.perf_counter() - t0
    return dict(images_per_s=round(B * steps / dt, 1), detections_per_image=round(sum(len(o["instances"]) for o in out) / B, 1))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[0] if q.stdout else "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    line = {"card": card(), "bev_ms": {}}
    for B in (8, 32):
        for n in (1000, 5750):
            line["bev_ms"][f"B{B}_n{n}"] = bev_ms(B, n, args.steps)
    line["dla34_kitti_b8"] = {"default": images_per_s(False, args.steps), "no_nms_bev": images_per_s(True, args.steps)}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
