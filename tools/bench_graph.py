"""Eager dd3d_forward against the captured forward (dd3d_graph_launch) on the same bound device buffers, synthetic weights:
  * dla34_b{1,2,8}   DLA-34 KITTI at 384x1280, B = 1, 2, 8;
  * v2_99_nusc6      V2-99 NuscenesDD3D, one sample of six 900x1600 cameras, DO_BEV_NMS and the sample aggregation.
Per configuration and path:
  * enqueue_us  host time of one call (perf_counter around `--burst` calls, no synchronisation; median over `--reps` bursts,
                each started on an idle device so the launch queue never blocks the host);
  * frame_ms    device time per frame (CUDA events around back-to-back frames for at least `--seconds` after warm-up);
the two paths alternate within `--rounds` rounds.  Also the kernel count of one forward, the graph's kernel nodes and
programmatic edges, and whether both paths return the same detections bit for bit.  The card's name, power limit and
max SM clock are read in the same run.  Prints one JSON line per configuration, then one with the card.
    python tools/bench_graph.py [--rounds 3] [--seconds 1] [--reps 50] [--burst 2] [--only dla34_b1,...]"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dd3d_b200 import lib as _lib  # noqa: E402
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.meta_arch import DD3DB200, NuscenesDD3DB200  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_nusc_inputs, make_state_dict  # noqa: E402


def _nusc_cfg():
    cfg = get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D")
    cfg.DD3D.INFERENCE.DO_BEV_NMS = True
    return cfg


# name -> (cfg factory, inputs factory)
CONFIGS = {
    "dla34_b1": (lambda: get_cfg("dla34", "kitti_3d"), lambda: make_inputs(1, 384, 1280, 721.5)),
    "dla34_b2": (lambda: get_cfg("dla34", "kitti_3d"), lambda: make_inputs(2, 384, 1280, 721.5)),
    "dla34_b8": (lambda: get_cfg("dla34", "kitti_3d"), lambda: make_inputs(8, 384, 1280, 721.5)),
    "v2_99_nusc6": (_nusc_cfg, lambda: make_nusc_inputs(1, 900, 1600, 1266.4)),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return dict(name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[0] if q.stdout else "")


class Paths:
    """One engine, its bound buffers, the eager call and the graph launch on them."""
    def __init__(self, name):
        make_cfg, make_case_inputs = CONFIGS[name]
        cfg = make_cfg()
        cls = NuscenesDD3DB200 if cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D" else DD3DB200
        m = cls(cfg).to("cuda")
        m.load_state_dict(make_state_dict(cfg))
        inputs = make_case_inputs()
        batch, K, sizes, _, is_u8 = m._gather_inputs(inputs, m.device)
        self.images, self.K, self.sizes = batch.cuda(), K.cuda(), sizes.cuda()
        poses = m._gather_poses(inputs).cuda() if "pose" in inputs[0] else None
        groups = getattr(m, "_groups", None)
        self.graph = m.capture_forward(self.images, self.K, self.sizes, poses=poses, groups=groups)
        self.m, self.h, self.L = m, m._handle, _lib.load()
        self.dtype = _lib.IMG_U8 if is_u8 else _lib.IMG_F32
        B, cap = self.images.shape[0], m._desc.out_cap
        self.out = torch.empty((B, cap, _lib.DET_WORDS), device="cuda")
        self.counts = torch.zeros(B, dtype=torch.int32, device="cuda")
        self.stream = torch.cuda.current_stream()
        self.sp = C.c_void_p(self.stream.cuda_stream)
        self.args = [C.c_void_p(t.data_ptr()) for t in (self.images, self.K, self.sizes, self.out, self.counts)]

    def eager(self):
        a = self.args
        st = self.L.dd3d_forward(self.h, a[0], self.dtype, a[1], a[2], a[3], a[4], self.sp)
        if st:
            _lib.check(st, self.h)

    def replay(self):
        st = self.L.dd3d_graph_launch(self.graph._graph, self.sp)
        if st:
            _lib.check(st, None)

    def results(self, fn):
        fn()
        torch.cuda.synchronize()
        B = self.out.shape[0]
        dets, counts, _ = self.graph.outputs() if fn == self.replay else (self.out, self.counts, None)
        c = counts[:B].cpu().clone()
        rows = [dets[b, :n].cpu().view(torch.int32).clone() for b, n in enumerate(c.tolist())]
        glob = self.graph.global_rows
        g = None if glob is None else [glob[b, :n].cpu().view(torch.int32).clone() for b, n in enumerate(c.tolist())]
        return c, rows, g


def enqueue_us(fn, reps, burst):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(burst):
            fn()
        ts.append((time.perf_counter() - t0) / burst * 1e6)
    torch.cuda.synchronize()
    return statistics.median(ts)


def frame_ms(fn, seconds, stream):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    n = max(10, int(seconds / max(time.perf_counter() - t0, 1e-6)) + 1)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(n):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / n, n


def run(name, args):
    p = Paths(name)
    for _ in range(args.warmup):
        p.eager()
        p.replay()
    ce, re_, ge = p.results(p.eager)
    cg, rg, gg = p.results(p.replay)
    same = torch.equal(ce, cg) and all(torch.equal(x, y) for x, y in zip(re_, rg)) and (
        ge is None or all(torch.equal(x, y) for x, y in zip(ge, gg)))
    rounds = []
    for _ in range(args.rounds):
        r = {}
        for path, fn in (("eager", p.eager), ("graph", p.replay)):
            r[f"{path}_enqueue_us"] = round(enqueue_us(fn, args.reps, args.burst), 2)
            ms, n = frame_ms(fn, args.seconds, p.stream)
            r[f"{path}_frame_ms"], r[f"{path}_frames"] = round(ms, 4), n
        rounds.append(r)
    med = {k: round(statistics.median(r[k] for r in rounds), 4) for k in rounds[0] if not k.endswith("_frames")}
    res = dict(config=name, B=int(p.images.shape[0]), H=int(p.images.shape[2]), W=int(p.images.shape[3]),
               launches_per_forward=int(p.m.launches_per_forward()), graph_kernel_nodes=int(p.graph.kernel_nodes),
               graph_programmatic_edges=int(p.graph.programmatic_edges), detections=int(ce.sum()),
               bit_identical=bool(same), median=med, rounds=rounds)
    p.graph.close()
    p.m._release()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--burst", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="", help="comma-separated subset of " + ",".join(CONFIGS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_graph: needs a CUDA device")
    names = [n for n in args.only.split(",") if n] or list(CONFIGS)
    for name in names:
        print(json.dumps(run(name, args)), flush=True)
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
