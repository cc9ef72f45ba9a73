"""CPU oracle of NuscenesDD3DWithTTA (nuscenes_dd3d_tta.py) and of the BEV steps of test-time augmentation, built on the
pinned oracles (oracle/bev_nms_oracle.py, oracle/tta_oracle.py):
  * nms_rotated -- batched_nms_rotated with an exact shortcut: pairs whose bounding circles are apart are disjoint (IoU
    0) and skip the polygon clipper, so a few thousand boxes stay tractable; pinned equal to bev_nms_oracle.nms_rotated;
  * camera-frame bev_nms (bev_nms.py:51-133 with its default pose_cam_global = CAMERA_TO_VEHICLE_ROTATION);
  * sample_aggregate -- bev_nms_oracle.sample_aggregate on the shortcut NMS;
  * tta_forward / nusc_tta_forward -- the per-image TTA merge (+ BEV with DO_BEV_NMS) and the sample aggregation."""
import math

import numpy as np
import torch

from oracle import bev_nms_oracle as B
from oracle import tta_oracle as T
from oracle.dd3d_oracle import matrix_to_quaternion, pose_of, quaternion_to_matrix


def nms_rotated(boxes, scores, classes, thr):
    """Same contract and result as bev_nms_oracle.nms_rotated: kept indices in descending-score order."""
    n = int(scores.shape[0])
    order = torch.argsort(scores, descending=True, stable=True).numpy()
    rank = np.empty(n, dtype=np.int64)
    rank[order] = np.arange(n)
    bl = boxes.tolist()
    bx = np.asarray(bl, dtype=np.float64).reshape(n, 5)
    cls = np.asarray([int(c) for c in classes], dtype=np.int64)
    rad = 0.5 * np.hypot(bx[:, 2], bx[:, 3])
    removed = np.zeros(n, dtype=bool)
    keep = []
    for i in order.tolist():
        if removed[i]:
            continue
        keep.append(i)
        cand = ~removed & (cls == cls[i]) & (rank > rank[i])
        if thr >= 0:
            r = (rad + rad[i]) * 1.001 + 1e-4
            cand &= (bx[:, 0] - bx[i, 0]) ** 2 + (bx[:, 1] - bx[i, 1]) ** 2 <= r * r
        for j in np.nonzero(cand)[0].tolist():
            if B.rotated_iou(bl[i], bl[j]) > thr:
                removed[j] = True
    return torch.tensor(keep, dtype=torch.long)


def camera_rotated_boxes(quat, tvec, size):
    """boxes3d_to_rotated_boxes with pose_cam_global = CAMERA_TO_VEHICLE_ROTATION: camera-frame top surface, BEV (x, y) =
    (x_cam, -z_cam) (VEHICLE_TO_BEV_ROTATION @ CAMERA_TO_VEHICLE_ROTATION, first two rows)."""
    surf = B.corners3d(quat, tvec, size)[:, [0, 1, 5, 4], :]
    bev = torch.stack([surf[..., 0], -surf[..., 2]], -1)
    length = (bev[:, 0] - bev[:, 3]).norm(dim=1)
    width = (bev[:, 0] - bev[:, 1]).norm(dim=1)
    center = bev[:, [0, 2]].mean(dim=1)
    fwd = bev[:, 0] - bev[:, 3]
    angle = torch.atan2(fwd[:, 0], fwd[:, 1]) * (180.0 / math.pi)
    return torch.stack([center[:, 0], center[:, 1], width, length, angle], 1)


def bev_nms_camera(det, thr):
    """bev_nms(boxes3d, scores_3d, thr, class_idxs=pred_classes): kept indices in NMS output order (descending
    scores_3d), as merged_instances[keep] applies them."""
    if det["quat"].shape[0] == 0:
        return torch.zeros(0, dtype=torch.long)
    return nms_rotated(camera_rotated_boxes(det["quat"], det["tvec"], det["size"]), det["score3d"], det["cls"], thr)


def sample_aggregate(dets, group_ids, poses, thr, max_dets=None):
    """bev_nms_oracle.sample_aggregate with the shortcut NMS."""
    saved = B.nms_rotated
    B.nms_rotated = nms_rotated
    try:
        return B.sample_aggregate(dets, group_ids, poses, thr, max_dets)
    finally:
        B.nms_rotated = saved


def to_global_f64(quat, tvec, pose_quat, pose_tvec):
    """postprocessing.py:25-46 in float64 on the fp32 inputs (the pose rounded to fp32 as the kernels receive it): the
    yardstick for pred_boxes3d_global, free of the fp32 oracle's own rounding."""
    R_ws = quaternion_to_matrix(torch.tensor(pose_quat, dtype=torch.float32).double()[None])[0]
    R = torch.matmul(R_ws[None], quaternion_to_matrix(quat.double()))
    t = torch.matmul(tvec.double(), R_ws.T) + torch.tensor(pose_tvec, dtype=torch.float32).double()[None]
    return matrix_to_quaternion(R), t


def boxes3d_tvec(d):
    """Boxes3D.tvec (boxes3d.py:169-173): inv_K (proj_ctr, 1) * depth in fp32."""
    ph = torch.cat([d["proj_ctr"], torch.ones_like(d["proj_ctr"][:, :1])], 1).unsqueeze(-1)
    return torch.matmul(d["inv_K"], ph).squeeze(-1) * d["depth"].reshape(-1, 1)


def _with_nusc_fields(det, view, image_hw, orig_hw):
    out = T.invert_view(det, view, image_hw, orig_hw)
    for k in ("attr", "speed"):  # NuscenesDD3DWithTTA._get_augmented_instances carries them along
        if k in det:
            out[k] = det[k]
    return out


def tta_forward(oracle, x, cfg, bev_nms_thresh=None):
    """_inference_one_image of DD3DWithTTA / NuscenesDD3DWithTTA with a DD3DOracle as the model: the views in chunks of
    TEST.IMS_PER_BATCH (each view forward runs the per-image BEV NMS itself when the cfg has DO_BEV_NMS), the inverse
    transforms, one class-aware NMS on scores_3d and -- bev_nms_thresh -- the camera-frame bev_nms of the merged set."""
    aug = cfg.TEST.AUG
    image = x["image"]
    h, w = int(image.shape[1]), int(image.shape[2])
    orig = (int(x.get("height", h)), int(x.get("width", w)))
    views = T.make_views(image, orig, x["intrinsics"], aug.MIN_SIZES, aug.MAX_SIZE, aug.FLIP)
    outs = []
    bs = cfg.TEST.IMS_PER_BATCH
    for a0 in range(0, len(views), bs):
        chunk = [dict({k: x[k] for k in ("pose", "extrinsics") if k in x}, image=v["image"], intrinsics=v["intrinsics"])
                 for v in views[a0:a0 + bs]]
        outs.extend(oracle.forward(chunk, do_postprocess=False))
    inverted = []
    for a, (v, det) in enumerate(zip(views, outs)):
        v["index"] = a
        inverted.append(_with_nusc_fields(det, v, (h, w), orig))
    out = T.merge(inverted, cfg.DD3D.FCOS2D.INFERENCE.NMS_THRESH)
    out["tvec"] = boxes3d_tvec(out)
    if bev_nms_thresh is not None and out["score3d"].shape[0]:
        keep = bev_nms_camera(out, bev_nms_thresh)
        out = {k: v[keep] for k, v in out.items()}
    return out


def group_ids(inputs, num_images_per_sample):
    tokens = [x["sample_token"] for x in inputs]
    order = {t: i for i, t in enumerate(dict.fromkeys(tokens))}  # get_group_idxs, postprocessing.py:111-123
    if any(tokens.count(t) != num_images_per_sample for t in order):
        raise ValueError("Group sizes does not match with 'num_images_per_sample'.")
    return [order[t] for t in tokens]


def nusc_tta_forward(oracle, inputs, cfg, per_image=None):
    """NuscenesDD3DWithTTA.__call__: per-image TTA (per_image: precomputed merged sets), then nuscenes_sample_aggregate
    over the call with the global poses and MAX_NUM_DETS_PER_SAMPLE.  Returns per-image dicts with quat_global /
    tvec_global."""
    inf = cfg.DD3D.INFERENCE
    if per_image is None:
        per_image = [tta_forward(oracle, x, cfg, inf.BEV_NMS_IOU_THRESH if inf.DO_BEV_NMS else None) for x in inputs]
    gids = group_ids(inputs, cfg.DD3D.NUSC.INFERENCE.NUM_IMAGES_PER_SAMPLE)
    return sample_aggregate(per_image, gids, [pose_of({"pose": x["pose"]}) for x in inputs], inf.BEV_NMS_IOU_THRESH,
                            cfg.DD3D.NUSC.INFERENCE.MAX_NUM_DETS_PER_SAMPLE)
