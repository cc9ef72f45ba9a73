"""Share of the box3d (or box2d) tower the sparse tower computes (CPU, fp32 oracle):
python tools/tower_coverage.py [--images N] [--box2d] [--tile 16x8|8x8 ...].

For each image of the bench's V2-99 workload (900x1600, the same seeded images bench.py times) the seed pixels give, per tower
layer, the conv tiles (--tile, th x tw, default the engine's 8x8; repeat it to compare granularities on the same forwards)
that the engine's tower_tiles_kernel lists (csrc/tower_tiles.cu).  box3d tower: the seeds are the
oracle's pre-NMS candidates and layer i of `depth` runs on the tiles within Chebyshev distance depth - i of a seed.  box2d
tower (--box2d): the seeds are the pixels where some class passes PRE_NMS_THRESH alone (P) and layer i runs on the tiles
within depth - 1 - i, the predictor (list `depth`) on the tiles that hold a seed.  Prints the in-map pixels of the tower
layers' tiles per layer and their share of the dense depth x (head pixels).  tile_lists() is the rule
tests/test_tower_tiles.py checks against a brute-force receptive-field propagation."""
import argparse
import os
import sys

import numpy as np

TH, TW = 8, 8  # tile of the sparse tower convs (conv_igemm.cuh kListTile)
FAR = 1 << 30


def tile_dist(cands, H, W, th=TH, tw=TW):
    """cands: (y, x) seed pixels of one level.  -> [tiles_y][tiles_x] Chebyshev distance from the in-map part of each th x tw
    tile to the nearest seed (FAR: no seed)."""
    tiles_y, tiles_x = -(-H // th), -(-W // tw)
    ty, tx = np.arange(tiles_y), np.arange(tiles_x)
    y0, y1 = ty * th, np.minimum(ty * th + th, H) - 1
    x0, x1 = tx * tw, np.minimum(tx * tw + tw, W) - 1
    dist = np.full((tiles_y, tiles_x), FAR, dtype=np.int64)
    for py, px in cands:
        dy = np.maximum(np.maximum(y0 - py, py - y1), 0)
        dx = np.maximum(np.maximum(x0 - px, px - x1), 0)
        dist = np.minimum(dist, np.maximum(dy[:, None], dx[None, :]))
    return dist


def tile_lists(cands, H, W, depth, th=TH, tw=TW, reach=None):
    """cands: (y, x) seed pixels of one level.  -> per list i < depth, the sorted row-major indices of the tiles within
    reach - i of a seed (reach: depth, or depth - 1 for the box2d tower and its predictor)."""
    reach = depth if reach is None else reach
    dist = tile_dist(cands, H, W, th, tw)
    return [np.flatnonzero(dist.reshape(-1) <= reach - i) for i in range(depth)]


def predictor_tiles(cands, H, W):
    """The box2d predictor's list as tower_tiles_kernel derives it from the 8x8 distances: the sorted row-major indices of the
    16x8 tiles one of whose two 8x8 halves (tile rows 2 ty, 2 ty + 1) holds a seed."""
    d = tile_dist(cands, H, W, 8, 8)
    if d.shape[0] % 2:
        d = np.concatenate([d, np.full((1, d.shape[1]), FAR)])
    return np.flatnonzero(np.minimum(d[0::2], d[1::2]).reshape(-1) == 0)


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
    ap.add_argument("--tile", action="append", choices=["16x8", "8x8"],
                    help="tower tile th x tw (default 8x8); repeat to report several")
    args = ap.parse_args()
    tiles = [tuple(map(int, t.split("x"))) for t in (args.tile or ["8x8"])]
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
    shares = {t: [] for t in tiles}
    for i in range(min(args.images, len(inputs))):
        with torch.no_grad():
            _, inter = oracle.forward(inputs[i:i + 1], return_intermediates=True)
        det = inter["pre_nms"][0]
        per_layer, dense, seeds = {t: np.zeros(depth, dtype=np.int64) for t in tiles}, 0, 0
        for l, m in enumerate(inter["maps"]["logits"]):
            h, w = m.shape[-2:]
            dense += h * w
            if args.box2d:  # the box2d tower's lists; the predictor's (list `depth`) is not counted
                yx = class_pass_pixels(m[0], C, thresh)
            else:
                pix = det["pixel"][det["level"] == l].numpy()
                yx = np.stack([pix // w, pix % w], 1)
            seeds += len(yx)
            for th, tw in tiles:
                if args.box2d:
                    lists = tile_lists(yx, h, w, depth + 1, th, tw, reach=depth)[:depth]
                else:
                    lists = tile_lists(yx, h, w, depth, th, tw)
                per_layer[th, tw] += [tile_pixels(t, h, w, th, tw) for t in lists]
        what = "pixels in P" if args.box2d else "candidates"
        print(f"image {i}: {seeds} {what} ({len(det['pixel'])} candidates), dense {dense} pixels per layer", flush=True)
        for t in tiles:
            share = per_layer[t].sum() / (depth * dense)
            shares[t].append(share)
            print(f"  {t[0]}x{t[1]}: tile pixels per layer {' / '.join(map(str, per_layer[t]))}, per-layer share "
                  f"{' / '.join(f'{100 * v / dense:.1f}' for v in per_layer[t])} %, share {100 * share:.1f} %", flush=True)
    for t in tiles:
        s = shares[t]
        print(f"{t[0]}x{t[1]}: mean share over {len(s)} images: {100 * np.mean(s):.1f} % (min {100 * min(s):.1f}, "
              f"max {100 * max(s):.1f})")

if __name__ == "__main__":
    main()
