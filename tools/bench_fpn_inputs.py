"""Throughput of the default FPN inputs against another FE.FPN.IN_FEATURES list, with bench.py's method: seeded synthetic
weights and inputs, warm-up, CUDA events around `--steps` device forwards (dd3d_forward).  The configurations run in
alternation, `--rounds` times, so that drifting clocks hit all of them alike.  DLA-34 compares level3..5 with level2..5 and
DD3D.IN_FEATURES [p2..p6] (a stride-4 head level, which the default list does not have); V2-99 compares stage2..5 with
stage3..5 (no stride-4 FPN output, which also drops the p2 head).  A separate profiled forward gives the device time of every
op category, the launches, the op count and the workspace bytes.  Prints one JSON line per run and the card name / power
limit read in the same process.  V2-99 runs at bench.py's 32 x 900 x 1600 unless the plan does not fit in device memory; it
then halves the batch (the line says which batch ran).

    python tools/bench_fpn_inputs.py [--steps 20] [--warmup 5] [--rounds 2] [--archs dla34,v2_99]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (gpu_info only)

# the shapes of bench.py's two workloads
WORKLOADS = {"v2_99": (32, 900, 1600, "nuscenes"), "dla34": (8, 384, 1280, "kitti_3d")}
# arch -> the (FE.FPN.IN_FEATURES, DD3D.IN_FEATURES) run against the default (None, None)
OTHER = {"v2_99": (["stage3", "stage4", "stage5"], None),
         "dla34": (["level2", "level3", "level4", "level5"], ["p2", "p3", "p4", "p5", "p6"])}


def run(arch, lists, args, card):
    import torch
    from dd3d_b200 import lib
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_inputs, make_state_dict
    dev = torch.device("cuda", 0)
    B, H, W, dataset = WORKLOADS[arch]
    fpn_in, feats = lists
    cfg = get_cfg(arch, dataset, act_dtype=args.dtype, in_features=feats, fpn_in_features=fpn_in)
    model = DD3DB200(cfg).to(dev)
    model.load_state_dict(make_state_dict(cfg))
    L = lib.load()
    h = model._engine()
    free = torch.cuda.mem_get_info(dev)[0]
    while B > 1 and L.dd3d_workspace_bytes(h, B, H, W) > 0.8 * free:
        B //= 2
    inputs = make_inputs(B, H, W, 1266.4 if arch == "v2_99" else 721.5, seed_base=1)
    batch_t, K, sizes, shape, is_u8 = model._gather_inputs(inputs, dev)
    model._plan(*shape)
    d_batch, d_K, d_sizes = batch_t.to(dev), K.to(dev), sizes.to(dev)
    d_out = torch.empty((B, model._desc.out_cap, lib.DET_WORDS), dtype=torch.float32, device=dev)
    d_cnt = torch.empty((B, ), dtype=torch.int32, device=dev)
    sp = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    code = lib.IMG_U8 if is_u8 else lib.IMG_F32

    def step():
        lib.check(L.dd3d_forward(h, C.c_void_p(d_batch.data_ptr()), code, C.c_void_p(d_K.data_ptr()),
                                 C.c_void_p(d_sizes.data_ptr()), C.c_void_p(d_out.data_ptr()), C.c_void_p(d_cnt.data_ptr()),
                                 sp), h)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    model.set_profile(True)
    step()
    torch.cuda.synchronize()
    prof = model.get_profile()
    model.set_profile(False)
    line = {"arch": arch, "fpn_in_features": fpn_in or "default", "in_features": feats or "all", "batch": B, "shape": [H, W], "dtype": args.dtype,
            "images_per_s": B / (ms / 1e3), "ms_per_step": ms,
            "conv_ms": round(prof["conv_igemm"]["ms"] + prof["stem_conv"]["ms"], 3),
            "category_ms": {k: round(v["ms"], 3) for k, v in prof.items()},
            "launches": model.launches_per_forward(), "num_ops": L.dd3d_num_ops(h),
            "workspace_bytes": L.dd3d_workspace_bytes(h, B, H, W),
            "gpu": card["name"], "power_limit_w": card["power_limit_w"]}
    print(json.dumps(line), flush=True)
    model._release()
    del model
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--archs", default="dla34,v2_99")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_fpn_inputs: no CUDA device")
    card = bench.gpu_info(0)
    print(json.dumps({"gpu": card}), flush=True)
    for _ in range(args.rounds):
        for arch in args.archs.split(","):
            for lists in ((None, None), OTHER[arch]):
                run(arch, lists, args, card)


if __name__ == "__main__":
    main()
