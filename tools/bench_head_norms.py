"""Throughput of the FPN / FCOS head norms that DD3D.FCOS2D.NORM, DD3D.FCOS3D.NORM and FE.FPN.NORM select, with bench.py's
method: seeded synthetic weights and inputs, warm-up, CUDA events around `--steps` device forwards (dd3d_forward).  Heads:
"default" (per-level BN towers, BN FPN), "gn" (GroupNorm everywhere) and "none" (biased convs, no norm).  The layouts run
in alternation, `--rounds` times, so that drifting clocks hit all of them alike.  A separate profiled forward gives the time
of the elementwise category (GroupNorm statistics + apply, plus the DLA-34 top block's small relu) and its bytes, computed
from shapes.  Prints one JSON line per run and the card name / power limit read in the same process.

    python tools/bench_head_norms.py [--steps 20] [--warmup 5] [--rounds 2] [--archs v2_99,dla34] [--heads default,gn,none]
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
HEADS = {"default": {}, "gn": {"GN"}, "none": {""}}


def make_cfg(arch, heads, dtype):
    from dd3d_b200.config import get_cfg
    cfg = get_cfg(arch, WORKLOADS[arch][3], act_dtype=dtype)
    for norm in HEADS[heads]:
        cfg.DD3D.FCOS2D.NORM = cfg.DD3D.FCOS3D.NORM = cfg.FE.FPN.NORM = norm
    return cfg


def run(arch, heads, args, card):
    import torch
    from dd3d_b200 import lib
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_inputs, make_state_dict
    dev = torch.device("cuda", 0)
    B, H, W, _ = WORKLOADS[arch]
    cfg = make_cfg(arch, heads, args.dtype)
    model = DD3DB200(cfg).to(dev)
    model.load_state_dict(make_state_dict(cfg))
    inputs = make_inputs(B, H, W, 1266.4 if arch == "v2_99" else 721.5, seed_base=1)
    batch_t, K, sizes, shape, is_u8 = model._gather_inputs(inputs, dev)
    model._plan(*shape)
    h = model._handle
    L = lib.load()
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
    ew = prof["relu"]
    line = {"arch": arch, "heads": heads, "batch": B, "shape": [H, W], "dtype": args.dtype,
            "images_per_s": B / (ms / 1e3), "ms_per_step": ms,
            "gn_relu_ms": ew["ms"], "gn_relu_launches": ew["launches"], "gn_relu_gbytes": ew["bytes"] / 1e9,
            "gn_relu_gb_per_s": ew["bytes"] / (ew["ms"] * 1e6) if ew["ms"] > 0 else None,
            "conv_igemm_ms": prof["conv_igemm"]["ms"], "launches": model.launches_per_forward(),
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
    ap.add_argument("--archs", default="v2_99,dla34")
    ap.add_argument("--heads", default="default,gn,none")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_head_norms: no CUDA device")
    card = bench.gpu_info(0)
    print(json.dumps({"gpu": card}), flush=True)
    for _ in range(args.rounds):
        for arch in args.archs.split(","):
            for heads in args.heads.split(","):
                run(arch, heads, args, card)


if __name__ == "__main__":
    main()
