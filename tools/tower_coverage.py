"""Share of the box3d tower the sparse tower computes (CPU, fp32 oracle): python tools/tower_coverage.py [--images N].

For each image of the bench's V2-99 workload (900x1600, the same seeded images bench.py times) the oracle's pre-NMS candidates
give, per tower layer, the 16x8 conv tiles the engine's tower_tiles_kernel lists (csrc/tower_tiles.cu): layer i of `depth`
runs on the tiles within Chebyshev distance depth - i of a candidate.  Prints the in-map pixels of those tiles per layer and
their share of the dense depth x (head pixels).  tile_lists() is the rule tests/test_tower_tiles.py checks against a
brute-force receptive-field propagation."""
import argparse
import os
import sys

import numpy as np

TH, TW = 16, 8  # halo tile of the tower convs (conv_igemm.cuh kHaloTh x kHaloTw)


def tile_lists(cands, H, W, depth, th=TH, tw=TW):
    """cands: (y, x) pixels of one level's candidates.  -> per layer, the sorted row-major tile indices it computes."""
    tiles_y, tiles_x = -(-H // th), -(-W // tw)
    ty, tx = np.arange(tiles_y), np.arange(tiles_x)
    y0, y1 = ty * th, np.minimum(ty * th + th, H) - 1
    x0, x1 = tx * tw, np.minimum(tx * tw + tw, W) - 1
    dist = np.full((tiles_y, tiles_x), 1 << 30, dtype=np.int64)
    for py, px in cands:
        dy = np.maximum(np.maximum(y0 - py, py - y1), 0)
        dx = np.maximum(np.maximum(x0 - px, px - x1), 0)
        dist = np.minimum(dist, np.maximum(dy[:, None], dx[None, :]))
    return [np.flatnonzero(dist.reshape(-1) <= depth - i) for i in range(depth)]


def tile_pixels(tiles, H, W, th=TH, tw=TW):
    tiles_x = -(-W // tw)
    ty, tx = tiles // tiles_x, tiles % tiles_x
    return int((np.minimum(th, H - ty * th) * np.minimum(tw, W - tx * tw)).sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=32)
    ap.add_argument("--threads", type=int, default=0)
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
    import torch
    from bench import WORKLOADS
    from dd3d_b200.config import get_cfg
    from dd3d_b200.synthetic import make_inputs, make_state_dict
    from oracle.dd3d_oracle import DD3DOracle

    arch, ds, B, H, W, focal, _ = WORKLOADS["v2_99"]
    cfg = get_cfg(arch, ds)
    depth = int(cfg.DD3D.FCOS3D.NUM_CONVS)
    oracle = DD3DOracle(cfg, make_state_dict(cfg), threads=args.threads or None)
    inputs = make_inputs(B, H, W, focal)
    shares = []
    for i in range(min(args.images, len(inputs))):
        with torch.no_grad():
            _, inter = oracle.forward(inputs[i:i + 1], return_intermediates=True)
        det = inter["pre_nms"][0]
        per_layer, dense = np.zeros(depth, dtype=np.int64), 0
        for l, m in enumerate(inter["maps"]["logits"]):
            h, w = m.shape[-2:]
            dense += h * w
            pix = det["pixel"][det["level"] == l].numpy()
            lists = tile_lists(np.stack([pix // w, pix % w], 1), h, w, depth)
            per_layer += [tile_pixels(t, h, w) for t in lists]
        share = per_layer.sum() / (depth * dense)
        shares.append(share)
        print(f"image {i}: {len(det['pixel'])} candidates, tile pixels per layer {' / '.join(map(str, per_layer))} "
              f"of {dense}, share {100 * share:.1f} %", flush=True)
    print(f"mean share over {len(shares)} images: {100 * np.mean(shares):.1f} % (min {100 * min(shares):.1f}, "
          f"max {100 * max(shares):.1f})")


if __name__ == "__main__":
    main()
