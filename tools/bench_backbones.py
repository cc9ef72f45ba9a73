"""Throughput of every VoVNetV2-eSE backbone FE.BACKBONE.NAME selects, with bench.py's method: seeded synthetic weights and
inputs, warm-up, CUDA events around `--steps` device forwards (dd3d_forward).  A separate profiled forward gives the summed
implicit-GEMM conv time and the depthwise conv time, with the depthwise bytes computed from shapes.  Prints one JSON line
per variant and the card name / power limit read in the same run.

    python tools/bench_backbones.py [--batch 32] [--height 900] [--width 1600] [--steps 20] [--warmup 5] [--archs a,b]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (gpu_info only)
from dd3d_b200.arch import VOVNET_SPECS  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--height", type=int, default=900)
    ap.add_argument("--width", type=int, default=1600)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--archs", default=",".join(VOVNET_SPECS))
    args = ap.parse_args()
    import torch
    from dd3d_b200 import lib
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_inputs, make_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("bench_backbones: no CUDA device")
    dev = torch.device("cuda", 0)
    card = bench.gpu_info(0)
    print(json.dumps({"gpu": card}), flush=True)
    B, H, W = args.batch, args.height, args.width
    inputs = make_inputs(B, H, W, 1266.4, seed_base=1)
    L = lib.load()
    for arch in args.archs.split(","):
        cfg = get_cfg(arch, "nuscenes", act_dtype=args.dtype)
        model = DD3DB200(cfg).to(dev)
        model.load_state_dict(make_state_dict(cfg))
        batch_t, K, sizes, shape, is_u8 = model._gather_inputs(inputs, dev)
        model._plan(*shape)
        h = model._handle
        cap = model._desc.out_cap
        d_batch, d_K, d_sizes = batch_t.to(dev), K.to(dev), sizes.to(dev)
        d_out = torch.empty((B, cap, lib.DET_WORDS), dtype=torch.float32, device=dev)
        d_cnt = torch.empty((B, ), dtype=torch.int32, device=dev)
        sp = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        code = lib.IMG_U8 if is_u8 else lib.IMG_F32

        def step():
            lib.check(L.dd3d_forward(h, C.c_void_p(d_batch.data_ptr()), code, C.c_void_p(d_K.data_ptr()),
                                     C.c_void_p(d_sizes.data_ptr()), C.c_void_p(d_out.data_ptr()),
                                     C.c_void_p(d_cnt.data_ptr()), sp), h)

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
        # profiled forward (separate from the timed window): per-op CUDA events
        model.set_profile(True)
        step()
        torch.cuda.synchronize()
        prof = model.get_profile()
        ops = model.get_op_times(with_op=True)
        model.set_profile(False)
        # the depthwise ops are the category-1 engine ops after stem_1 (engine op 0)
        dw_ms = sum(t for cat, t, _, op in ops if cat == "stem_conv" and op >= 1)
        dw_bytes = prof["stem_conv"]["bytes"] - _stem1_bytes(B, model)
        line = {"arch": arch, "name": VOVNET_SPECS[arch][0], "batch": B, "shape": [H, W], "dtype": args.dtype,
                "images_per_s": B / (ms / 1e3), "ms_per_step": ms,
                "conv_igemm_ms": prof["conv_igemm"]["ms"], "conv_igemm_tflops": prof["conv_igemm"]["flops"] / (prof["conv_igemm"]["ms"] * 1e9),
                "dw_ms": dw_ms if VOVNET_SPECS[arch][6] else 0.0,
                "dw_gbytes": dw_bytes / 1e9 if VOVNET_SPECS[arch][6] else 0.0,
                "dw_gb_per_s": (dw_bytes / (dw_ms * 1e6)) if VOVNET_SPECS[arch][6] and dw_ms > 0 else None,
                "launches": model.launches_per_forward(), "gpu": card["name"], "power_limit_w": card["power_limit_w"]}
        print(json.dumps(line), flush=True)
        model._release()
        del model
        torch.cuda.empty_cache()


def _stem1_bytes(B, model):
    """Bytes dd3d_get_profile books for VoVNet stem_1 (engine.cu Builder::stem): 8 B per input pixel, 2 B per output
    channel and pixel."""
    Hp, Wp = model._plan_key[1], model._plan_key[2]
    d = model.backbone.size_divisibility
    Hp, Wp = (Hp + d - 1) // d * d, (Wp + d - 1) // d * d
    return B * Hp * Wp * 8.0 + B * (Hp // 2) * (Wp // 2) * 64 * 2.0


if __name__ == "__main__":
    main()
