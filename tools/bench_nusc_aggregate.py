"""Times the NuscenesDD3D sample aggregation as the engine's last step (dd3d_set_sample_aggregate) on V2-99 NuscenesDD3D at
900x1600, 30 images (5 samples x 6 cameras) per call, synthetic weights:
  * default   the shipped config (POST_NMS_TOPK 100: the one-CTA path): ms per call of dd3d_forward with the step, against
              dd3d_forward without it followed by dd3d_op_sample_aggregate, two engines in the same process, alternating
              rounds (CUDA events around `--steps` calls after `--warmup`);
  * step      the device time of the aggregation step alone (its profile entry, median of `--reps` profiled forwards) and
              the boxes that enter it per sample, for the default config and the blocked path's configs: DO_NMS off,
              POST_NMS_TOPK 300 and 1000;
  * synthetic the blocked operator (dd3d_op_group_bev_nms_large, global mode, the kernels the step runs) on 34 500
              synthetic boxes per sample (30 images x 5 750 slots): 10 classes evenly, and 90 % of the boxes in one class.
Synthetic weights give other candidate counts than a trained checkpoint: read each time next to its box count.  The card's
name and power limit are read in the same run.  Prints one JSON line.
    python tools/bench_nusc_aggregate.py [--steps 20] [--warmup 5] [--rounds 2] [--reps 5]"""
import argparse
import ctypes as C
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dd3d_b200 import lib as _lib  # noqa: E402
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.meta_arch import NuscenesDD3DB200, group_indices  # noqa: E402
from dd3d_b200.synthetic import make_nusc_inputs, make_state_dict  # noqa: E402

SAMPLES, H, W, FOCAL = 5, 900, 1600, 1266.4
CONFIGS = {"default": {}, "no_nms": dict(DO_NMS=False), "post_300": dict(POST_NMS_TOPK=300),
           "post_1000": dict(POST_NMS_TOPK=1000)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[0] if q.stdout else "")


def make_cfg(over):
    cfg = get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D")
    for k, v in over.items():
        if k == "DO_NMS":
            cfg.DD3D.INFERENCE.DO_NMS = v
        else:
            setattr(cfg.DD3D.FCOS2D.INFERENCE, k, v)
    return cfg


class Route:
    """One engine on device-resident inputs: dd3d_forward with the step (step=True) or dd3d_forward followed by
    dd3d_op_sample_aggregate (step=False)."""
    def __init__(self, cfg, sd, inputs, step):
        L, dev = _lib.load(), torch.device("cuda")
        self.L, self.step = L, step
        m = NuscenesDD3DB200(cfg).to(dev)
        m.load_state_dict(sd)
        m.sample_aggregate_in_inference = step
        batch, K, sizes, shape, is_u8 = m._gather_inputs(inputs, dev)
        m._sync_options(True)
        m._plan(*shape)
        self.m, self.h, self.B, self.cap = m, m._handle, shape[0], m._desc.out_cap
        self.groups = group_indices([x["sample_token"] for x in inputs], 6)
        self.d_batch, self.d_K, self.d_sizes = batch.to(dev), K.to(dev), sizes.to(dev)
        self.dtype = _lib.IMG_U8 if is_u8 else _lib.IMG_F32
        self.out = torch.empty((self.B, self.cap, _lib.DET_WORDS), device=dev)
        self.counts = torch.zeros(self.B, dtype=torch.int32, device=dev)
        self.poses = m._gather_poses(inputs).to(dev)
        self.group = torch.tensor(self.groups, dtype=torch.int32, device=dev)
        self.glob = torch.zeros((self.B, self.cap, 10), device=dev)
        self.flags = torch.zeros(1, dtype=torch.int32, device=dev)
        self.scratch = torch.empty(int(L.dd3d_op_sample_aggregate_scratch_bytes(self.B, self.cap)) if not step else 1,
                                   dtype=torch.uint8, device=dev)
        if step:
            _lib.check(L.dd3d_set_poses(self.h, C.c_void_p(self.poses.data_ptr())), self.h)
            _lib.check(L.dd3d_set_groups(self.h, C.c_void_p(self.group.data_ptr()), max(self.groups) + 1), self.h)
            _lib.check(L.dd3d_set_global_out(self.h, C.c_void_p(self.glob.data_ptr())), self.h)

    def __call__(self):
        L, h, sp = self.L, self.h, C.c_void_p(torch.cuda.current_stream().cuda_stream)
        _lib.check(L.dd3d_forward(h, C.c_void_p(self.d_batch.data_ptr()), self.dtype, C.c_void_p(self.d_K.data_ptr()),
                                  C.c_void_p(self.d_sizes.data_ptr()), C.c_void_p(self.out.data_ptr()),
                                  C.c_void_p(self.counts.data_ptr()), sp), h)
        if not self.step:
            _lib.check(L.dd3d_op_sample_aggregate(
                C.c_void_p(self.out.data_ptr()), C.c_void_p(self.counts.data_ptr()), C.c_void_p(self.d_K.data_ptr()),
                C.c_void_p(self.poses.data_ptr()), C.c_void_p(self.group.data_ptr()), max(self.groups) + 1,
                C.c_void_p(self.glob.data_ptr()), C.c_void_p(self.scratch.data_ptr()), C.c_void_p(self.flags.data_ptr()),
                self.B, self.cap, float(self.m.bev_nms_iou_thresh), int(self.m.max_num_dets_per_sample or 0), sp), h)

    def time(self, steps, warmup):
        for _ in range(warmup):
            self()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            self()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def result(self):
        torch.cuda.synchronize()
        return self.out.cpu(), self.counts.cpu(), self.glob.cpu()


def compare_default(sd, inputs, args):
    cfg = make_cfg({})
    step, parent = Route(cfg, sd, inputs, True), Route(cfg, sd, inputs, False)
    rounds = []
    for _ in range(args.rounds):
        rounds.append(dict(step_ms=round(step.time(args.steps, args.warmup), 3),
                           parent_ms=round(parent.time(args.steps, args.warmup), 3)))
    (oa, ca, ga), (ob, cb, gb) = step.result(), parent.result()
    same = torch.equal(ca, cb) and all(
        torch.equal(oa[i, :n].view(torch.int32), ob[i, :n].view(torch.int32)) and
        torch.equal(ga[i, :n].view(torch.int32), gb[i, :n].view(torch.int32)) for i, n in enumerate(ca.tolist()))
    res = dict(rounds=rounds, bit_identical=bool(same), detections=int(ca.sum()),
               launches_step=_lib.load().dd3d_launches_per_forward(step.h),
               launches_parent=_lib.load().dd3d_launches_per_forward(parent.h) + 2,
               flags=int(step.m.overflow_flags()) | int(parent.flags.item()))
    del step, parent
    return res


def step_time(name, sd, inputs, args):
    cfg = make_cfg(CONFIGS[name])
    m = NuscenesDD3DB200(cfg).to("cuda")
    m.load_state_dict(sd)
    path = _lib.load().dd3d_sample_aggregate_path(m._desc)
    m.sample_aggregate_in_inference = False
    pre = m(inputs)
    groups = group_indices([x["sample_token"] for x in inputs], 6)
    per_sample = [0] * (max(groups) + 1)
    for g, o in zip(groups, pre):
        per_sample[g] += len(o["instances"])
    m.sample_aggregate_in_inference = True
    m(inputs)  # plan with the step
    ms = []
    m.set_profile(True)
    for _ in range(args.reps):
        out = m(inputs)
        ms.append(m.get_op_times()[-1][1])  # the last step of the forward: the aggregation (category "nms")
    m.set_profile(False)
    res = dict(path="one_cta" if path == _lib.AGG_PATH_ONE_CTA else "blocked", out_cap=int(m._desc.out_cap),
               boxes_per_sample=per_sample, survivors=sum(len(o["instances"]) for o in out),
               step_ms_median=round(statistics.median(ms), 3), step_ms=[round(v, 3) for v in ms],
               flags=int(m.overflow_flags()))
    m._release()
    return res


def synthetic_op(one_class_share, args):
    """dd3d_op_group_bev_nms_large in global mode on 30 images x 5 750 random boxes (5 groups of 6 images)."""
    L, dev = _lib.load(), torch.device("cuda")
    B, cap, ncls = 6 * SAMPLES, 5750, 10
    g = torch.Generator().manual_seed(11)
    d = torch.zeros(B, cap, _lib.DET_WORDS)
    di = d.view(torch.int32)
    yaw = torch.rand(B, cap, generator=g) * 6.2832
    d[..., 8], d[..., 10] = torch.cos(yaw / 2), torch.sin(yaw / 2)  # rotation about the camera's y axis
    d[..., 12] = torch.rand(B, cap, generator=g) * W
    d[..., 13] = 300 + torch.rand(B, cap, generator=g) * 300
    d[..., 14] = 5 + torch.rand(B, cap, generator=g) * 55
    d[..., 15], d[..., 16], d[..., 17] = 1.9, 4.6, 1.7
    d[..., 5] = torch.rand(B, cap, generator=g)
    cls = torch.randint(0, ncls, (B, cap), generator=g, dtype=torch.int32)
    cls[torch.rand(B, cap, generator=g) < one_class_share] = 0
    di[..., 6] = cls
    di[..., 20] = torch.arange(cap, dtype=torch.int32)
    K = torch.tensor([FOCAL, 0, W / 2, 0, FOCAL, H / 2, 0, 0, 1], dtype=torch.float32).repeat(B, 1)
    inputs = make_nusc_inputs(SAMPLES, 8, 8, FOCAL)
    poses = NuscenesDD3DB200._gather_poses(inputs).to(dev)
    group = torch.tensor([b // 6 for b in range(B)], dtype=torch.int32, device=dev)
    d_src, d_K = d.to(dev), K.to(dev)
    dets, counts = torch.empty_like(d_src), torch.empty(B, dtype=torch.int32, device=dev)
    glob = torch.empty((B, cap, 10), device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    scratch = torch.empty(int(L.dd3d_op_group_bev_nms_large_scratch_bytes(B, cap, 16)), dtype=torch.uint8, device=dev)
    sp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ms = []
    for r in range(args.reps + 1):
        dets.copy_(d_src)
        counts.fill_(cap)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _lib.check(L.dd3d_op_group_bev_nms_large(
            C.c_void_p(dets.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(d_K.data_ptr()), 1,
            C.c_void_p(poses.data_ptr()), _lib.POSE_GLOBAL, C.c_void_p(group.data_ptr()), SAMPLES, 16,
            C.c_void_p(glob.data_ptr()), C.c_void_p(scratch.data_ptr()), C.c_void_p(flags.data_ptr()), B, cap, 0.3, 500, sp))
        e1.record()
        torch.cuda.synchronize()
        if r:  # the first call loads the module
            ms.append(e0.elapsed_time(e1))
    return dict(boxes_per_sample=6 * cap, one_class_share=one_class_share, survivors=int(counts.sum()),
                ms_median=round(statistics.median(ms), 3), ms=[round(v, 3) for v in ms], flags=int(flags.item()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_nusc_aggregate.py measures on a CUDA device"
    sd = make_state_dict(make_cfg({}))
    inputs = make_nusc_inputs(SAMPLES, H, W, FOCAL, seed_base=1)
    for x in inputs:
        x["height"], x["width"] = H, W
    res = dict(card=card(), workload=f"v2_99 NuscenesDD3D bf16, {6 * SAMPLES} images ({SAMPLES} samples) {H}x{W}, "
                                     "synthetic weights")
    res["default"] = compare_default(sd, inputs, args)
    gc.collect()
    torch.cuda.empty_cache()
    res["step"] = {}
    for name in CONFIGS:
        res["step"][name] = step_time(name, sd, inputs, args)
        gc.collect()
        torch.cuda.empty_cache()
    res["synthetic_34500"] = [synthetic_op(0.0, args), synthetic_op(0.9, args)]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
