"""Times DD3DB200WithTTA (test-time augmentation fully on the device) on one synthetic nuScenes-sized image:
10 views (5 scales x flip) -> merged detections.  Prints one JSON line.  python tools/bench_tta.py [--arch v2_99]

--nusc: NuscenesDD3DB200WithTTA on --samples samples x 6 cameras (896x1593 mapped from 900x1600 originals, the shipped
TEST.AUG config): per-image merges, then the sample aggregation on the grouped BEV kernel; reports ms per sample, views/s,
merged detections per image, boxes entering the aggregation and the device time of the grouped BEV NMS (CUDA events)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from dd3d_b200.config import get_cfg  # noqa: E402
from dd3d_b200.meta_arch import DD3DB200  # noqa: E402
from dd3d_b200.synthetic import make_inputs, make_state_dict  # noqa: E402
from dd3d_b200.tta import DD3DB200WithTTA, NuscenesDD3DB200WithTTA  # noqa: E402


def bench_nusc(samples):
    from dd3d_b200.meta_arch import NuscenesDD3DB200
    from dd3d_b200.synthetic import make_nusc_inputs
    cfg = get_cfg("v2_99", "nuscenes", meta_arch="NuscenesDD3D")
    cfg.DD3D.INFERENCE.DO_POSTPROCESS = False
    model = NuscenesDD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    tta = NuscenesDD3DB200WithTTA(cfg, model, world_size=8)  # TEST.IMS_PER_BATCH // 8 views per model call, as shipped
    inputs = make_nusc_inputs(samples + 1, 896, 1593, 1266.4)
    for x in inputs:
        x["height"], x["width"] = 900, 1600
    stats = {"bev_ms": 0.0, "boxes_in": 0, "merged": 0}
    events = []
    group_bev = tta._group_bev_nms

    def timed_group_bev(out, counts, *a, **k):  # device time of every grouped BEV NMS call
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        if k.get("d_global") is not None:  # the sample aggregation: its input counts are the merged sets
            events.append(("in", counts[:out.shape[0]].clone()))
        e0.record()
        group_bev(out, counts, *a, **k)
        e1.record()
        events.append(("ev", e0, e1))

    tta._group_bev_nms = timed_group_bev
    tta(inputs[:6])  # warm-up: plans, resize tables, allocator
    torch.cuda.synchronize()
    events.clear()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n_out = 0
    for s in range(1, samples + 1):
        n_out += sum(len(o["instances"]) for o in tta(inputs[6 * s:6 * s + 6]))
    e1.record()
    torch.cuda.synchronize()
    for ev in events:
        if ev[0] == "ev":
            stats["bev_ms"] += ev[1].elapsed_time(ev[2])
        else:
            stats["boxes_in"] += int(ev[1].sum())
    ms = e0.elapsed_time(e1) / samples
    views = 6 * len(cfg.TEST.AUG.MIN_SIZES) * (2 if cfg.TEST.AUG.FLIP else 1)
    props = torch.cuda.get_device_properties(0)
    print(json.dumps({"metric": "nusc_tta_ms_per_sample", "value": ms, "views_per_sample": views,
                      "views_per_s": views / (ms * 1e-3), "device": props.name, "mapped_size": [896, 1593],
                      "min_sizes": list(cfg.TEST.AUG.MIN_SIZES), "views_per_model_call": tta.batch_size,
                      "merged_detections_per_image": stats["boxes_in"] / (6 * samples),
                      "aggregation_boxes_in_per_sample": stats["boxes_in"] / samples,
                      "detections_out_per_sample": n_out / samples,
                      "group_bev_nms_device_ms_per_sample": stats["bev_ms"] / samples,
                      "overflow_flags": tta.overflow_flags()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="v2_99", choices=["v2_99", "dla34"])
    ap.add_argument("--images", type=int, default=4)
    ap.add_argument("--nusc", action="store_true", help="NuscenesDD3D TTA with the sample aggregation")
    ap.add_argument("--samples", type=int, default=2)
    args = ap.parse_args()
    if args.nusc:
        return bench_nusc(args.samples)
    ds, H, W, focal = ("nuscenes", 896, 1593, 1266.4) if args.arch == "v2_99" else ("kitti_3d", 384, 1272, 721.5)
    cfg = get_cfg(args.arch, ds)
    cfg.DD3D.INFERENCE.DO_POSTPROCESS = False
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(make_state_dict(cfg))
    tta = DD3DB200WithTTA(cfg, model, world_size=8)  # TEST.IMS_PER_BATCH // 8 views per model call, as shipped
    inputs = make_inputs(args.images + 1, H, W, focal)
    for x in inputs:
        x["height"], x["width"] = (900, 1600) if args.arch == "v2_99" else (375, 1242)
    tta([inputs[0]])  # warm-up: plans, resize tables
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    n = 0
    for x in inputs[1:]:
        n += len(tta([x])[0]["instances"])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.images
    views = len(cfg.TEST.AUG.MIN_SIZES) * 2
    print(json.dumps({"metric": "tta_ms_per_image", "value": ms, "views_per_image": views,
                      "views_per_s": views / (ms * 1e-3), "arch": args.arch, "mapped_size": [H, W],
                      "min_sizes": list(cfg.TEST.AUG.MIN_SIZES), "views_per_model_call": tta.batch_size,
                      "merged_detections_per_image": n / args.images, "overflow_flags": tta.overflow_flags()}))


if __name__ == "__main__":
    main()
