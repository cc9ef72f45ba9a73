"""DD3DB200WithTTA -- mirror of the reference's test-time-augmentation wrapper (SURVEY.md 8f row 4).

``tridet.modeling.dd3d.test_time_augmentation.DD3DWithTTA`` (test_time_augmentation.py:89-239) takes one mapped dataset
dict per image, builds ``len(TEST.AUG.MIN_SIZES) * (2 if FLIP else 1)`` augmented views on the CPU (PIL resize + numpy
flip, ``DatasetMapperTTA`` :24-87), runs the model on them in chunks of ``TEST.IMS_PER_BATCH // world_size``, maps every
detection back with numpy loops (:190-239) and reduces with one NMS (:160-171).  Here the views are produced on the GPU by
the fused resize(+flip)+normalise kernel straight into the engine (``dd3d_forward_resized``), the detections never leave
the device until the end, and the inverse transforms + merged NMS are one kernel pair (``dd3d_op_tta_merge``).  The host
code below only restates the transform bookkeeping (shapes, fp32 factors, intrinsics) in the reference's order.
"""
import ctypes as C

import numpy as np
import torch
from torch import nn

from . import lib as _lib
from .meta_arch import DD3DB200, NuscenesDD3DB200, group_indices
from .structures import Boxes, Boxes3D, GenericBoxes3D, Instances


def build_views(image_hw, orig_hw, K_input, min_sizes, max_size, flip):
    """DatasetMapperTTA.__call__ (test_time_augmentation.py:50-87) + the inverse bookkeeping of
    _get_augmented_instances (:196-216) for one image.  Returns [(new_h, new_w, flip, lib.TtaView)]."""
    L = _lib.load()
    h, w = image_hw
    oh, ow = orig_hw
    K_input = np.asarray(K_input, dtype=np.float32).reshape(3, 3)
    pre = (oh, ow) != (h, w)  # pre_tfm = ResizeTransform(orig -> input) or NoOpTransform (:52-58)
    views = []
    nh_c, nw_c = C.c_int32(), C.c_int32()
    for min_size in min_sizes:
        _lib.check(L.dd3d_resize_shape(h, w, int(min_size), int(max_size), C.byref(nh_c), C.byref(nw_c)))
        nh, nw = nh_c.value, nw_c.value
        # apply_imresize_intrinsics (resize_transform.py:13-21)
        K_r = K_input * np.float32([nw / w, nh / h, 1]).reshape(3, 1)
        for f in ([0, 1] if flip else [0]):
            K_v = K_r.copy()
            if f:  # apply_hflip_intrinsics (flip_transform.py:8-10), width = width of the resized view
                K_v[0, 2] = nw - K_v[0, 2]
            # inv_tfm = (pre_tfm + tfms).inverse(): un-flip, un-resize, un-pre-resize (fvcore TransformList.inverse)
            K_o = K_v.copy()
            if f:
                K_o[0, 2] = nw - K_o[0, 2]
            K_o = K_o * np.float32([w / nw, h / nh, 1]).reshape(3, 1)
            if pre:
                K_o = K_o * np.float32([ow / w, oh / h, 1]).reshape(3, 1)
            v = _lib.TtaView()
            v.flip = f
            v.view_w = float(nw)
            # ResizeTransform.apply_coords of the inverses: coords * (new_w * 1.0 / w) with an fp32 coordinate array
            v.inv_sx[0], v.inv_sy[0] = np.float32(w * 1.0 / nw), np.float32(h * 1.0 / nh)
            v.inv_sx[1], v.inv_sy[1] = (np.float32(ow * 1.0 / w), np.float32(oh * 1.0 / h)) if pre else (1.0, 1.0)
            for i in range(9):
                v.K_view[i] = float(K_v.reshape(-1)[i])
                v.K_orig[i] = float(K_o.reshape(-1)[i])
            views.append((nh, nw, f, v))
    return views


class _DeviceTTA(nn.Module):
    """Shared device path of the TTA wrappers: per image, the augmented views through the engine in chunks, the optional
    per-view BEV NMS of the model's own forward, and the merge of the views into one device slot range."""
    def __init__(self, cfg, model, world_size):
        super().__init__()
        self.cfg = cfg
        self.model = model
        self.nms_thresh = cfg.DD3D.FCOS2D.INFERENCE.NMS_THRESH
        self.min_sizes = list(cfg.TEST.AUG.MIN_SIZES)
        self.max_size = cfg.TEST.AUG.MAX_SIZE
        self.flip = bool(cfg.TEST.AUG.FLIP)
        self.num_views = len(self.min_sizes) * (2 if self.flip else 1)
        self.batch_size = max(1, cfg.TEST.IMS_PER_BATCH // world_size)  # test_time_augmentation.py:116
        self.merged_bev_nms_in_inference = True  # test hook: False skips the BEV NMS of the merged sets (DO_BEV_NMS)

    def _do_bev_nms(self):
        """`not model.only_box2d and model.do_bev_nms` (core.py:137, nuscenes_dd3d_tta.py), read at call time like the
        reference.  The BEV kernels expect score-sorted sets: the engine's rule of DD3DB200._sync_options."""
        model = self.model
        bev = bool(model.do_bev_nms) and not model.only_box2d
        if bev and not model.do_nms:
            raise NotImplementedError("DO_BEV_NMS without DO_NMS: the BEV kernels expect the score-sorted output of the 2-D NMS")
        return bev

    def _merge_image(self, x, out, n_out, bev, stream):
        """Runs the views of one image and merges them into `out` [merged_cap][DET_WORDS] / `n_out` [1] (device, no sync).
        Returns (original (h, w), views)."""
        model, L = self.model, _lib.load()
        device = model.device
        image = torch.as_tensor(x["image"])
        if image.dtype != torch.uint8:
            raise ValueError("TTA resamples uint8 images (PIL path of ResizeTransform.apply_image)")
        h, w = int(image.shape[1]), int(image.shape[2])
        orig = (int(x.get("height", h)), int(x.get("width", w)))
        views = build_views((h, w), orig, x["intrinsics"], self.min_sizes, self.max_size, self.flip)
        A, cap = len(views), model._desc.out_cap
        hwc = image.to(device, non_blocking=True).permute(1, 2, 0).contiguous()
        dets = torch.empty((A, cap, _lib.DET_WORDS), dtype=torch.float32, device=device)
        counts = torch.empty((A, ), dtype=torch.int32, device=device)
        if bev:  # the model's own forward runs the per-image BEV NMS on every view (core.py:137-151, x["pose"])
            pose = model._gather_poses([x]).to(device, non_blocking=True)
        # chunks of `batch_size` views, each padded to the chunk's largest view like ImageList.from_tensors does for
        # one model(inputs) call (test_time_augmentation.py:118-133)
        for a0 in range(0, A, self.batch_size):
            chunk = views[a0:a0 + self.batch_size]
            B = len(chunk)
            model._plan(B, max(v[0] for v in chunk), max(v[1] for v in chunk))
            raw = hwc.unsqueeze(0).expand(B, h, w, 3).contiguous()
            raw_sizes = torch.tensor([[h, w]] * B, dtype=torch.int32)
            new_sizes = torch.tensor([[v[0], v[1]] for v in chunk], dtype=torch.int32)
            flips = torch.tensor([v[2] for v in chunk], dtype=torch.int32)
            K = torch.tensor([list(v[3].K_view) for v in chunk], dtype=torch.float32)
            sizes4 = torch.cat([new_sizes, new_sizes], 1).contiguous()
            _lib.check(L.dd3d_set_option(model._handle, b"do_postprocess", 0), model._handle)
            _lib.check(L.dd3d_set_option(model._handle, b"do_nms", int(model.do_nms)), model._handle)
            _lib.check(
                L.dd3d_forward_resized(model._handle, C.c_void_p(raw.data_ptr()), h, w, C.c_void_p(raw_sizes.data_ptr()),
                                       C.c_void_p(new_sizes.data_ptr()), C.c_void_p(flips.data_ptr()),
                                       C.c_void_p(K.data_ptr()), C.c_void_p(sizes4.data_ptr()),
                                       C.c_void_p(dets[a0].data_ptr()), C.c_void_p(counts[a0:].data_ptr()),
                                       C.c_void_p(stream)), model._handle)
            if self._engine_flags is not None:  # the engine's overflow word of this forward joins the call's word
                _lib.check(L.dd3d_copy_flags(model._handle, C.c_void_p(self._engine_flags.data_ptr()), C.c_void_p(stream)),
                           model._handle)
                self._flags |= self._engine_flags
            if bev:
                d_K, d_sizes = K.to(device, non_blocking=True), sizes4.to(device, non_blocking=True)
                d_pose = pose.expand(B, 7).contiguous()
                _lib.check(
                    L.dd3d_op_bev_nms(C.c_void_p(dets[a0].data_ptr()), C.c_void_p(counts[a0:].data_ptr()),
                                      C.c_void_p(d_K.data_ptr()), C.c_void_p(d_pose.data_ptr()),
                                      C.c_void_p(d_sizes.data_ptr()), C.c_void_p(self._flags.data_ptr()), B, cap,
                                      float(model.bev_nms_iou_thresh), 0, C.c_void_p(stream)), model._handle)
        scratch = torch.empty(int(L.dd3d_op_tta_merge_scratch_bytes(A, cap)), dtype=torch.uint8, device=device)
        varr = (_lib.TtaView * A)(*[v[3] for v in views])
        _lib.check(
            L.dd3d_op_tta_merge(C.c_void_p(dets.data_ptr()), C.c_void_p(counts.data_ptr()), varr, A, cap,
                                float(self.nms_thresh), int(model.do_nms), C.c_void_p(scratch.data_ptr()),
                                C.c_void_p(out.data_ptr()), C.c_void_p(n_out.data_ptr()),
                                C.c_void_p(self._flags.data_ptr()), C.c_void_p(stream)), model._handle)
        return orig, views

    def _group_bev_nms(self, out, counts, view_K, pose_mode, d_group, num_groups, group_images, d_poses=None,
                       d_global=None, max_dets=0, stream=None):
        """dd3d_op_group_bev_nms on out [B][merged_cap] / counts [B] (device, in place, no sync); groups of at most
        `group_images` images, which sizes the IoU bit matrix."""
        L = _lib.load()
        B, mcap = int(out.shape[0]), int(out.shape[1])
        scratch = torch.empty(int(_lib.check(L.dd3d_op_group_bev_nms_scratch_bytes(B, mcap, group_images))),
                              dtype=torch.uint8, device=out.device)
        _lib.check(
            L.dd3d_op_group_bev_nms(C.c_void_p(out.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(view_K.data_ptr()),
                                    int(view_K.shape[1]), C.c_void_p(d_poses.data_ptr()) if d_poses is not None else None,
                                    pose_mode, C.c_void_p(d_group.data_ptr()), num_groups, group_images,
                                    C.c_void_p(d_global.data_ptr()) if d_global is not None else None,
                                    C.c_void_p(scratch.data_ptr()), C.c_void_p(self._flags.data_ptr()), B, mcap,
                                    float(self.model.bev_nms_iou_thresh), int(max_dets), C.c_void_p(stream)))

    @staticmethod
    def _inv_K(views, device):
        # Boxes3D.from_vectors(vecs, orig_intrinsics): every detection keeps the inverse intrinsics recovered for its view
        return torch.stack([
            torch.linalg.inv(torch.tensor(list(v[3].K_orig), dtype=torch.float64).reshape(3, 3)).to(torch.float32)
            for v in views
        ]).to(device)

    @staticmethod
    def _view_K(views):
        return torch.tensor([list(v[3].K_orig) for v in views], dtype=torch.float32)


class DD3DB200WithTTA(_DeviceTTA):
    """Same constructor and call contract as DD3DWithTTA(cfg, model): ``__call__(batched_inputs)`` with mapped dataset
    dicts ("image" CHW uint8, "intrinsics", optional "height" / "width") -> ``[{"instances": Instances}]`` with
    pred_boxes, pred_boxes3d, pred_classes, scores, scores_3d on the original image, sorted by scores_3d.  With
    DD3D.INFERENCE.DO_BEV_NMS the views' forwards and the merged set go through the BEV NMS like the reference's
    (inputs then carry "pose" or "extrinsics").  The reference runs that branch only when each model call holds views
    of one scale (its per-view BEV step concatenates the call's Instances, and Instances.cat asserts one image size);
    here the per-view step is per image, so any TEST.IMS_PER_BATCH works and gives the per-view results the reference
    gives with one view per call."""
    def __init__(self, cfg, model, tta_mapper=None, world_size=1):
        assert isinstance(model, DD3DB200) and not isinstance(model, NuscenesDD3DB200), \
            "DD3DB200WithTTA only supports DD3DB200. Got a model of type {}".format(type(model))
        assert not model.postprocess_in_inference, \
            "To use test-time augmentation, `postprocess_in_inference` must be False."
        if tta_mapper is not None:
            raise NotImplementedError("custom tta_mapper: the views are generated on the device")
        super().__init__(cfg, model, world_size)
        self._engine_flags = None

    def __call__(self, batched_inputs):
        return [self._inference_one_image(x) for x in batched_inputs]

    @torch.no_grad()
    def _inference_one_image(self, x):
        model, L = self.model, _lib.load()
        device = model.device
        bev = self._do_bev_nms()
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            mcap = int(L.dd3d_op_tta_merged_cap(self.num_views, model._desc.out_cap))
            out = torch.empty((1, mcap, _lib.DET_WORDS), dtype=torch.float32, device=device)
            n_out = torch.zeros(1, dtype=torch.int32, device=device)
            self._flags = torch.zeros(1, dtype=torch.int32, device=device)
            orig, views = self._merge_image(x, out[0], n_out, bev, stream)
            if bev and self.merged_bev_nms_in_inference:  # bev_nms(merged_instances.pred_boxes3d, ...), camera frame
                view_K = self._view_K(views).unsqueeze(0).to(device, non_blocking=True)
                group = torch.zeros(1, dtype=torch.int32).to(device, non_blocking=True)
                self._group_bev_nms(out, n_out, view_K, _lib.POSE_CAMERA, group, 1, 1, stream=stream)
            n = int(n_out.item())  # the only synchronisation
        d, di = out[0, :n], out[0].view(torch.int32)[:n]
        inv_K = self._inv_K(views, device)
        inst = Instances(orig)
        inst.pred_boxes = Boxes(d[:, 0:4].clone())
        inst.pred_boxes3d = Boxes3D(d[:, 8:12].clone(), d[:, 12:14].clone(), d[:, 14:15].clone(), d[:, 15:18].clone(),
                                    inv_K[di[:, 7].to(torch.int64)])
        inst.pred_classes = di[:, 6].to(torch.int64)
        inst.scores = d[:, 4].clone()
        inst.scores_3d = d[:, 5].clone()
        return {"instances": inst}

    def overflow_flags(self):
        return self.model.overflow_flags() | int(self._flags.item())


class NuscenesDD3DB200WithTTA(_DeviceTTA):
    """Same constructor and call contract as NuscenesDD3DWithTTA(cfg, model) (nuscenes_dd3d_tta.py): per image the TTA
    merge of DD3DB200WithTTA (attributes and speeds carried along) and, with DO_BEV_NMS, the camera-frame BEV NMS of the
    merged set; then the sample aggregation over the whole call (get_group_idxs groups of NUM_IMAGES_PER_SAMPLE images,
    global poses, at most MAX_NUM_DETS_PER_SAMPLE survivors of the call).  Inputs carry "sample_token" and "pose".
    Outputs: pred_boxes, pred_boxes3d, pred_classes, scores, scores_3d, pred_attributes, pred_speeds,
    pred_boxes3d_global on the original image (model.sample_aggregate_in_inference = False, the model's test hook,
    returns the merged per-image sets before the aggregation, without pred_boxes3d_global).  All merged sets of the call live in one device buffer; the BEV steps run
    on the multi-CTA kernel (dd3d_op_group_bev_nms) and the call synchronises once."""
    MAX_IMAGES = 256  # images per call the grouped BEV kernel holds

    def __init__(self, cfg, model, tta_mapper=None, world_size=1):
        assert isinstance(model, NuscenesDD3DB200), \
            "NuscenesDD3DB200WithTTA only supports NuscenesDD3DB200. Got a model of type {}".format(type(model))
        assert not model.postprocess_in_inference, \
            "To use test-time augmentation, `postprocess_in_inference` must be False."
        if tta_mapper is not None:
            raise NotImplementedError("custom tta_mapper: the views are generated on the device")
        super().__init__(cfg, model, world_size)
        self._last_flags = 0

    @torch.no_grad()
    def __call__(self, batched_inputs):
        model, L = self.model, _lib.load()
        B = len(batched_inputs)
        groups = group_indices([x["sample_token"] for x in batched_inputs], model.num_images_per_sample)
        if B > self.MAX_IMAGES:
            raise ValueError(f"NuscenesDD3DB200WithTTA: at most {self.MAX_IMAGES} images per call, got {B}")
        poses = model._gather_poses([{"pose": x["pose"]} for x in batched_inputs])
        bev = self._do_bev_nms()
        device = model.device
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            mcap = int(L.dd3d_op_tta_merged_cap(self.num_views, model._desc.out_cap))
            out = torch.empty((B, mcap, _lib.DET_WORDS), dtype=torch.float32, device=device)
            counts = torch.zeros((B + 1, ), dtype=torch.int32, device=device)  # [B] counts + overflow word
            self._flags = torch.zeros(1, dtype=torch.int32, device=device)
            self._engine_flags = torch.zeros(1, dtype=torch.int32, device=device)
            origs, all_views = [], []
            for b, x in enumerate(batched_inputs):
                orig, views = self._merge_image(x, out[b], counts[b:b + 1], bev, stream)
                origs.append(orig)
                all_views.append(views)
            # nuscenes_sample_aggregate concatenates the Instances of the call: detectron2's Instances.cat asserts one
            # common image size
            assert len(set(origs)) == 1, "images of one call must share the original size"
            view_K = torch.stack([self._view_K(v) for v in all_views]).to(device, non_blocking=True)
            if bev and self.merged_bev_nms_in_inference:  # per image: group = image, camera-frame pose, no cap
                self._group_bev_nms(out, counts, view_K, _lib.POSE_CAMERA,
                                    torch.arange(B, dtype=torch.int32).to(device, non_blocking=True), B, 1, stream=stream)
            glob = None
            if model.sample_aggregate_in_inference:
                glob = torch.zeros((B, mcap, 10), dtype=torch.float32, device=device)
                self._group_bev_nms(out, counts, view_K, _lib.POSE_GLOBAL,
                                    torch.tensor(groups, dtype=torch.int32).to(device, non_blocking=True), max(groups) + 1,
                                    model.num_images_per_sample, d_poses=poses.to(device, non_blocking=True), d_global=glob,
                                    max_dets=int(model.max_num_dets_per_sample or 0), stream=stream)
            counts[B:] |= self._flags
            host = counts.cpu()  # the only synchronisation: B counts + the overflow word
        self._last_flags = int(host[-1])
        model._check_flags(self._last_flags)
        results = []
        ints = out.view(torch.int32)
        for b, n in enumerate(host[:-1].tolist()):
            d, di = out[b, :n], ints[b, :n]
            inv_K = self._inv_K(all_views[b], device)
            inst = Instances(origs[b])
            inst.pred_boxes = Boxes(d[:, 0:4].clone())
            inst.pred_boxes3d = Boxes3D(d[:, 8:12].clone(), d[:, 12:14].clone(), d[:, 14:15].clone(),
                                        d[:, 15:18].clone(), inv_K[di[:, 7].to(torch.int64)])
            inst.pred_classes = di[:, 6].to(torch.int64)
            inst.scores = d[:, 4].clone()
            inst.scores_3d = d[:, 5].clone()
            inst.pred_attributes = di[:, 21].to(torch.int64)
            inst.pred_speeds = d[:, 22].clone()
            if glob is not None:
                gb = glob[b, :n]
                inst.pred_boxes3d_global = GenericBoxes3D(gb[:, 0:4].clone(), gb[:, 4:7].clone(), gb[:, 7:10].clone())
            results.append({"instances": inst})
        return results

    def overflow_flags(self):
        """Overflow word of the last call (engine forwards, TTA merges, BEV steps); a non-zero word raised already."""
        return self._last_flags


# tridet/modeling/__init__.py TTA_MODELS, with the registered mirror names next to the reference's
TTA_MODELS = {
    "DD3D": DD3DB200WithTTA,
    "DD3DB200": DD3DB200WithTTA,
    "NuscenesDD3D": NuscenesDD3DB200WithTTA,
    "NuscenesDD3DB200": NuscenesDD3DB200WithTTA,
}


def build_tta_model(cfg, model):
    """build_tta_model (tridet/modeling/__init__.py): the TTA wrapper of cfg.MODEL.META_ARCHITECTURE around `model`,
    views split over the processes of the default process group like the reference's get_world_size()."""
    meta_arch = cfg.MODEL.META_ARCHITECTURE
    assert meta_arch in TTA_MODELS, f"Test-time augmentation model is not available: {meta_arch}"
    import torch.distributed as dist
    world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    return TTA_MODELS[meta_arch](cfg, model, world_size=world_size)
