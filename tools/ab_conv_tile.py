"""A/B of a conv policy (dd3d_set_conv_policy) in one process: interleaved V2-99 forwards under two values of it, by default
the 256 x 128 pair tile off (policy "pair_tile" 0) against the default rule (-1); --policy stagger --old 0 times the
consumer-warpgroup skew off against its default.  Prints per conv launch (tagged by layer shape) the median device ms and
TFLOP/s of both, per-shape group totals, the step totals and their spread over the rounds.

    python tools/ab_conv_tile.py [--policy pair_tile] [--old 0] [--new -1] [--workload v2_99] [--batch 32] [--rounds 5]
                                 [--json out.json]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

import torch  # noqa: E402

from bench import WORKLOADS, gpu_info  # noqa: E402
from dd3d_b200 import lib  # noqa: E402
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.meta_arch import DD3DB200  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402


def tag(c):
    if c is None:
        return None
    kind = "halo" if c["halo"] else "3x3" if c["taps"] == 9 else "1x1"
    if c["stride"] == 2:
        kind += "/s2"
    return f"{kind} {c['cin']}->{c['cout_pad']}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="v2_99", choices=list(WORKLOADS))
    ap.add_argument("--batch", type=int, default=0, help="0: the workload's batch size")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    ap.add_argument("--policy", default="pair_tile", help="dd3d_set_conv_policy name")
    ap.add_argument("--old", type=int, default=0, help="policy value of the 'old' leg")
    ap.add_argument("--new", type=int, default=-1, help="policy value of the 'new' leg (-1: the default)")
    args = ap.parse_args()
    arch, ds, B, H, W, focal, _ = WORKLOADS[args.workload]
    B = args.batch or B
    cfg = get_cfg(arch, ds)
    sd = make_state_dict(cfg)
    inp = make_inputs(B, H, W, focal)
    L = lib.load()
    modes = {"old": args.old, "new": args.new}
    policy = args.policy.encode()
    models, info = {}, {}
    try:
        for name, mode in modes.items():  # the policy is read when the plan is made: one model (plan) per policy
            assert L.dd3d_set_conv_policy(policy, mode) == 0
            m = DD3DB200(cfg).to("cuda")
            m.load_state_dict(sd)
            for _ in range(3):
                m(inp)
            torch.cuda.synchronize()
            info[name] = m.get_conv_info()
            models[name] = m
    finally:
        L.dd3d_set_conv_policy(policy, -1)
    times = {n: [] for n in modes}
    steps = {n: [] for n in modes}
    walls = {n: [] for n in modes}
    flops = None
    for _ in range(args.rounds):
        for name, m in models.items():
            m.set_profile(True)
            m(inp)
            t = m.get_op_times(with_op=True)
            m.set_profile(False)
            times[name].append({op: ms for _, ms, _, op in t if op >= 0})
            steps[name].append(sum(ms for _, ms, _, _ in t))
            flops = {op: f for _, _, f, op in t if op >= 0}
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            m(inp)
            e1.record()
            torch.cuda.synchronize()
            walls[name].append(e0.elapsed_time(e1))
    med = {n: {op: statistics.median(r[op] for r in times[n]) for op in times[n][0]} for n in modes}
    rows, groups = [], {}
    for i, (c_old, c_new) in enumerate(zip(info["old"], info["new"])):
        if c_old is None:
            continue
        a, b, f = med["old"][i], med["new"][i], flops[i]
        k = tag(c_old)
        rows.append(dict(op=i, shape=k, pair=int(c_new["pair"]), old_ms=a, new_ms=b, gflop=f / 1e9))
        g = groups.setdefault((k, int(c_new["pair"])), [0, 0.0, 0.0, 0.0])
        g[0] += 1
        g[1] += a
        g[2] += b
        g[3] += f
    print(json.dumps(dict(gpu=gpu_info(0), workload=args.workload, batch=B, rounds=args.rounds, policy=args.policy,
                          old=args.old, new=args.new)))
    print(f"{'op':>4} {'shape':18} {'pair':>4} {'old ms':>8} {'new ms':>8} {'old TF/s':>8} {'new TF/s':>8} {'gain':>6}")
    for r in rows:
        tf = lambda ms: r["gflop"] / ms if ms > 0 else 0.0  # noqa: E731  GFLOP / ms = TFLOP/s
        print(f"{r['op']:4d} {r['shape']:18} {r['pair']:4d} {r['old_ms']:8.3f} {r['new_ms']:8.3f} {tf(r['old_ms']):8.1f} "
              f"{tf(r['new_ms']):8.1f} {100 * (1 - r['new_ms'] / r['old_ms']):5.1f}%")
    print("\nper shape (launches, old ms, new ms, old TF/s, new TF/s):")
    for (k, p), (n, a, b, f) in sorted(groups.items(), key=lambda kv: -kv[1][1]):
        print(f"  {k:18} pair={p} x{n:3d} {a:8.2f} {b:8.2f} {f / a / 1e9:7.1f} {f / b / 1e9:7.1f}")
    for n in modes:
        for what, s in (("sum of op times", steps[n]), ("forward incl. copies, unprofiled", walls[n])):
            print(f"{n:4}: {what}: median {statistics.median(s):.2f} ms, min {min(s):.2f}, max {max(s):.2f} "
                  f"over {len(s)} rounds")
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(dict(rows=rows, steps=steps, forwards=walls), fh)


if __name__ == "__main__":
    main()
