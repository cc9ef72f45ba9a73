"""Writes a JSON report (--out, default parity.json in the working directory): MEASURED end-to-end parity of the engine against the CPU oracle for every golden case
(small ragged cases + the BASELINE.json shapes) and both storage types.  GPU box only; the numbers the thresholds of
tests/test_parity_full_gpu.py / tests/test_e2e_gpu.py are derived from.

    python tools/parity_report.py [--cases dla34,v2_99,dla34_full,v2_99_full] [--dtypes bf16,fp16] [--out path]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, os.path.abspath(ROOT))
sys.path.insert(0, os.path.join(os.path.abspath(ROOT), "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="dla34,v2_99,dla34_full,v2_99_full")
    ap.add_argument("--dtypes", default="bf16,fp16")
    ap.add_argument("--out", default="parity.json")
    a = ap.parse_args()
    import torch
    from parity_lib import measure_case
    reports = []
    for case in a.cases.split(","):
        for dt in a.dtypes.split(","):
            t0 = time.time()
            rep = measure_case(case, dt)
            rep["seconds"] = round(time.time() - t0, 1)
            reports.append(rep)
            pn, po = rep["pre_nms"]["emu"], rep["post_nms"]["emu"]
            print(f"{case:11s} {dt}: maps worst rel-L2 {rep['maps']['emu']['worst_rel_l2']:.2e} (emu) "
                  f"{rep['maps'].get('fp32', {}).get('worst_rel_l2', float('nan')):.2e} (fp32) | hybrid sets "
                  f"{rep['hybrid']['candidate_sets_equal']} order {rep['hybrid']['kept_order_equal']} | pre-NMS match "
                  f"{pn['sets']['match_rate']:.4f} hard-miss {pn['sets']['missing_outside_margin']}+"
                  f"{pn['sets']['extra_outside_margin']} | post-NMS match emu {po['sets']['match_rate']:.3f} golden "
                  f"{rep['post_nms'].get('reference_golden', {}).get('sets', {}).get('match_rate', float('nan')):.3f} "
                  f"[{rep['seconds']} s]", flush=True)
    blob = dict(device=torch.cuda.get_device_name(0), torch=torch.__version__, reports=reports,
                note="errors: box / proj_ctr relative to the box size, score / score3d absolute, quat distance up to sign, "
                     "depth / size / tvec relative; emu = oracle emulating the engine's 16-bit storage (1 thread), fp32 = "
                     "pure fp32 oracle (= reference arithmetic), reference_golden = the reference's own forward run in the "
                     "build container (tests/golden)")
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(blob, f, indent=1)
    print("wrote", a.out)


if __name__ == "__main__":
    main()
