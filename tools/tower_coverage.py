"""Share of the box3d (or box2d) tower the sparse tower computes (CPU, fp32 oracle):
python tools/tower_coverage.py [--images N] [--box2d].

For each image of the bench's V2-99 workload (900x1600, the same seeded images bench.py times) the seed pixels give, per tower
layer, the 16x8 conv tiles the engine's tower_tiles_kernel lists (csrc/tower_tiles.cu).  box3d tower: the seeds are the
oracle's pre-NMS candidates and layer i of `depth` runs on the tiles within Chebyshev distance depth - i of a seed.  box2d
tower (--box2d): the seeds are the pixels where some class passes PRE_NMS_THRESH alone (P) and layer i runs on the tiles
within depth - 1 - i, the predictor (list `depth`) on the tiles that hold a seed.  Prints the in-map pixels of the tower
layers' tiles per layer and their share of the dense depth x (head pixels).  tile_lists() is the rule
tests/test_tower_tiles.py checks against a brute-force receptive-field propagation."""
import argparse
import os
import sys

import numpy as np

TH, TW = 16, 8  # halo tile of the tower convs (conv_igemm.cuh kHaloTh x kHaloTw)


def tile_lists(cands, H, W, depth, th=TH, tw=TW, reach=None):
    """cands: (y, x) seed pixels of one level.  -> per list i < depth, the sorted row-major indices of the tiles within
    reach - i of a seed (reach: depth, or depth - 1 for the box2d tower and its predictor)."""
    reach = depth if reach is None else reach
    tiles_y, tiles_x = -(-H // th), -(-W // tw)
    ty, tx = np.arange(tiles_y), np.arange(tiles_x)
    y0, y1 = ty * th, np.minimum(ty * th + th, H) - 1
    x0, x1 = tx * tw, np.minimum(tx * tw + tw, W) - 1
    dist = np.full((tiles_y, tiles_x), 1 << 30, dtype=np.int64)
    for py, px in cands:
        dy = np.maximum(np.maximum(y0 - py, py - y1), 0)
        dx = np.maximum(np.maximum(x0 - px, px - x1), 0)
        dist = np.minimum(dist, np.maximum(dy[:, None], dx[None, :]))
    return [np.flatnonzero(dist.reshape(-1) <= reach - i) for i in range(depth)]


def class_pass_pixels(logits, C, thresh):
    """logits: [>= C, H, W] one level's cls map.  -> (y, x) of the pixels where some class has sigmoid(logit) > thresh
    (class_passes in csrc/detect.cuh)."""
    import torch
    ok = (torch.sigmoid(logits[:C].float()) > thresh).any(0).numpy()
    return np.argwhere(ok)


def tile_pixels(tiles, H, W, th=TH, tw=TW):
    tiles_x = -(-W // tw)
    ty, tx = tiles // tiles_x, tiles % tiles_x
    return int((np.minimum(th, H - ty * th) * np.minimum(tw, W - tx * tw)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--box2d", action="store_true", help="the box2d tower, seeded by the pixels that pass the threshold")
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    import torch
    from bench import WORKLOADS
    from dd3d_b200.config import get_cfg
    from dd3d_b200.synthetic import make_inputs, make_state_dict
    from oracle.dd3d_oracle import DD3DOracle

    arch, ds, B, H, W, focal, _ = WORKLOADS["v2_99"]
    cfg = get_cfg(arch, ds)
    depth = int(cfg.DD3D.FCOS2D.NUM_BOX_CONVS if args.box2d else cfg.DD3D.FCOS3D.NUM_CONVS)
    C, thresh = int(cfg.DD3D.NUM_CLASSES), float(cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH)
    oracle = DD3DOracle(cfg, make_state_dict(cfg), threads=args.threads or None)
    inputs = make_inputs(B, H, W, focal)
    shares = []
    for i in range(min(args.images, len(inputs))):
        with torch.no_grad():
            _, inter = oracle.forward(inputs[i:i + 1], return_intermediates=True)
        det = inter["pre_nms"][0]
        per_layer, dense, seeds = np.zeros(depth, dtype=np.int64), 0, 0
        for l, m in enumerate(inter["maps"]["logits"]):
            h, w = m.shape[-2:]
            dense += h * w
            if args.box2d:  # the box2d tower's lists + the predictor's, which is not counted
                yx = class_pass_pixels(m[0], C, thresh)
                lists = tile_lists(yx, h, w, depth + 1, reach=depth)[:depth]
            else:
                pix = det["pixel"][det["level"] == l].numpy()
                yx = np.stack([pix // w, pix % w], 1)
                lists = tile_lists(yx, h, w, depth)
            seeds += len(yx)
            per_layer += [tile_pixels(t, h, w) for t in lists]
        share = per_layer.sum() / (depth * dense)
        shares.append(share)
        print(f"image {i}: {seeds} {'pixels in P' if args.box2d else 'candidates'} ({len(det['pixel'])} candidates), "
              f"tile pixels per layer {' / '.join(map(str, per_layer))} of {dense}, share {100 * share:.1f} %", flush=True)
    print(f"mean share over {len(shares)} images: {100 * np.mean(shares):.1f} % (min {100 * min(shares):.1f}, "
          f"max {100 * max(shares):.1f})")


if __name__ == "__main__":
    main()
