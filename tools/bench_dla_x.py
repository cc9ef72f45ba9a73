"""Throughput of the DLA-X networks FE.BACKBONE.NAME selects, with DLA-34 in the same run, at DLA-34's workload (KITTI,
8 x 384 x 1280), with bench.py's method: seeded synthetic weights and inputs, warm-up, CUDA events around `--steps` device
forwards (dd3d_forward).  A separate profiled forward gives the summed implicit-GEMM conv time and its useful TFLOP/s
(grouped convs book cout * cpg * 9 MACs per output pixel, not the issued block-diagonal ones), and the grouped-conv time with
its HBM bytes from shapes (16-bit input and output maps once).  Prints one JSON line per network and the card name / power
limit read in the same run.

    python tools/bench_dla_x.py [--batch 8] [--height 384] [--width 1280] [--steps 20] [--warmup 5] [--archs a,b]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (gpu_info only)
from dd3d_b200.arch import DLA_SPECS  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--height", type=int, default=384)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "fp16"])
    ap.add_argument("--archs", default=",".join(DLA_SPECS))
    args = ap.parse_args()
    import torch
    from dd3d_b200 import lib
    from dd3d_b200.config import get_cfg
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_inputs, make_state_dict

    if not torch.cuda.is_available():
        raise SystemExit("bench_dla_x: no CUDA device")
    dev = torch.device("cuda", 0)
    card = bench.gpu_info(0)
    print(json.dumps({"gpu": card}), flush=True)
    B, H, W = args.batch, args.height, args.width
    inputs = make_inputs(B, H, W, 721.5, seed_base=1)
    L = lib.load()
    for arch in args.archs.split(","):
        cfg = get_cfg(arch, "kitti_3d", act_dtype=args.dtype)
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
        conv_info = model.get_conv_info()
        by_op = {op: (t, fl) for _, t, fl, op in ops if op >= 0}
        g_ms = g_bytes = g_flops = 0.0
        per_cpg = {}
        for i, c in enumerate(conv_info):
            if c is None or not c["grouped"]:
                continue
            t, fl = by_op[i]
            o = model.get_tensor(f"op{i}")  # [B, Ho, Wo, C]
            nb = o.shape[0] * o.shape[1] * o.shape[2] * o.shape[3] * 2.0 * (1 + c["stride"] ** 2)  # input + output maps
            g_ms, g_bytes, g_flops = g_ms + t, g_bytes + nb, g_flops + fl
            cpg = c["cin"] // DLA_SPECS[arch][5]
            e = per_cpg.setdefault(cpg, [0.0, 0.0])
            e[0] += t
            e[1] += nb
        line = {"arch": arch, "name": DLA_SPECS[arch][0], "batch": B, "shape": [H, W], "dtype": args.dtype,
                "images_per_s": B / (ms / 1e3), "ms_per_step": ms,
                "conv_igemm_ms": prof["conv_igemm"]["ms"],
                "conv_igemm_tflops": prof["conv_igemm"]["flops"] / (prof["conv_igemm"]["ms"] * 1e9),
                "grouped_ms": g_ms, "grouped_gbytes": g_bytes / 1e9,
                "grouped_gb_per_s": g_bytes / (g_ms * 1e6) if g_ms > 0 else None,
                "grouped_tflops": g_flops / (g_ms * 1e9) if g_ms > 0 else None,
                "grouped_by_cpg": {str(k): {"ms": v[0], "gb_per_s": v[1] / (v[0] * 1e6) if v[0] > 0 else None}
                                   for k, v in sorted(per_cpg.items())},
                "launches": model.launches_per_forward(), "gpu": card["name"], "power_limit_w": card["power_limit_w"]}
        print(json.dumps(line), flush=True)
        model._release()
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
