"""Dev tool: per-op device times of one forward (python tools/opprof.py v2_99 32)."""
import os, sys, torch
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from bench import WORKLOADS
from dd3d_b200.config import get_cfg
from dd3d_b200.meta_arch import DD3DB200
from dd3d_b200.synthetic import make_inputs, make_state_dict
wl = sys.argv[1]; B = int(sys.argv[2])
arch, ds, _, H, W, focal, _ = WORKLOADS[wl]
cfg = get_cfg(arch, ds)
m = DD3DB200(cfg).to("cuda"); m.load_state_dict(make_state_dict(cfg))
inp = make_inputs(B, H, W, focal)
for _ in range(3): m(inp)
m.set_profile(True)
acc = None
for _ in range(3):
    m(inp); t = m.get_op_times(with_op=True)
    acc = t if acc is None else [(a[0], a[1] + b[1], a[2], a[3]) for a, b in zip(acc, t)]
k = 0
for i, (c, ms, fl, _) in enumerate(acc):
    ms /= 3
    tf = fl / (ms * 1e-3) / 1e12 if ms > 0 and fl else 0
    if c == "conv_igemm":
        print(f"{i:4d} conv{k:4d} {ms:8.4f} ms {tf:8.1f} TF/s"); k += 1
    else:
        print(f"{i:4d} {c:9s} {ms:8.4f} ms")
