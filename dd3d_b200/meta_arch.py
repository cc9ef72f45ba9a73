"""DD3DB200 -- drop-in mirror of the reference meta-architecture for inference.

Same constructor and call contract as ``tridet.modeling.dd3d.core.DD3D`` (core.py:18-164):
``DD3DB200(cfg)``, ``.to(device)``, ``load_state_dict(reference_state_dict)``,
``forward(batched_inputs: list[dict]) -> list[{"instances": Instances}]`` with the attributes callers toggle
(``postprocess_in_inference``, ``do_nms``, ``only_box2d``, ``num_classes``, ``device``,
``backbone.size_divisibility``).  All arithmetic runs in libdd3d_b200.so (hand-written sm_90a kernels for the H100) through the
C ABI in include/dd3d_b200.h; torch is used for device memory and streams only.  No CPU fallback exists.
"""
import ctypes as C
from types import SimpleNamespace

import torch
from torch import nn

from . import lib as _lib
from .arch import arch_of, check_fpn_channels, check_fpn_inputs, is_nuscenes_arch, param_specs, size_divisibility
from .structures import Boxes, Boxes3D, GenericBoxes3D, Instances

try:  # register next to the reference's DD3D when detectron2 is present (scripts/train.py:48 build_model)
    from detectron2.modeling.meta_arch.build import META_ARCH_REGISTRY  # type: ignore
except Exception:  # noqa: BLE001
    META_ARCH_REGISTRY = None


class DD3DB200(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        if is_nuscenes_arch(cfg) != isinstance(self, NuscenesDD3DB200):
            raise ValueError(f"MODEL.META_ARCHITECTURE = {cfg.MODEL.META_ARCHITECTURE} does not match {type(self).__name__}")
        self.arch = arch_of(cfg)  # raises KeyError for an unknown FE.BUILDER like the reference registry
        self.only_box2d = not cfg.MODEL.BOX3D_ON  # core.py:34-40
        self.num_classes = cfg.DD3D.NUM_CLASSES
        self.postprocess_in_inference = cfg.DD3D.INFERENCE.DO_POSTPROCESS
        self.do_nms = cfg.DD3D.INFERENCE.DO_NMS
        self.do_bev_nms = cfg.DD3D.INFERENCE.DO_BEV_NMS
        self.bev_nms_iou_thresh = cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH
        self.backbone = SimpleNamespace(size_divisibility=size_divisibility(cfg))
        self._specs = param_specs(cfg)  # the reference's own errors first (nn.GroupNorm's ValueError for GN widths)
        check_fpn_inputs(cfg)  # the top block's p5 lookup; FPN inputs of stride >= 4 and at most 5 head levels
        self._fpn_channels = check_fpn_channels(cfg)  # FE.FPN.OUT_CHANNELS: a multiple of 64 in [64, 512]
        if not 1 <= self.num_classes <= _lib.MAX_NUM_CLASSES:
            raise NotImplementedError(f"DD3D.NUM_CLASSES = {self.num_classes} is not supported: the engine builds 1 to "
                                      f"{_lib.MAX_NUM_CLASSES} classes")
        # above 16 classes the sizes travel through dd3d_set_canonical_sizes; missing rows raise IndexError here, where the
        # reference raises it at the first forward that predicts such a class (fcos3d.py:378)
        self._canon = None
        if cfg.MODEL.BOX3D_ON and self.num_classes > _lib.MAX_CLASSES:
            self._canon = _lib.canonical_sizes_from_cfg(cfg)
        self._state = None  # reference-keyed fp32 CPU tensors
        self._device = torch.device("cpu")
        self._desc = _lib.desc_from_cfg(cfg)
        self._layout = _lib.layout_from_cfg(cfg)
        self._fpn_inputs = _lib.fpn_inputs_from_cfg(cfg)  # FE.FPN.IN_FEATURES
        self._in_features = _lib.in_features_from_cfg(cfg)  # KeyError / NotImplementedError for lists the engine cannot run
        if cfg.DD3D.FCOS2D.USE_DEFORMABLE or (cfg.MODEL.BOX3D_ON and cfg.DD3D.FCOS3D.USE_DEFORMABLE):
            raise ValueError("Not supported yet.")  # fcos2d.py:51-52, fcos3d.py:77-78
        # param_specs raised the reference's errors for the FE.BACKBONE.NORM values it cannot build
        self._backbone_norm = _lib.BACKBONE_NORMS[cfg.FE.BACKBONE.NORM]
        self._handle = None
        self._plan_key = None
        self._host_bufs = None
        self._graph_synced = None  # attributes capture_forward last pushed to the engine
        self.training = False

    # ------------------------------------------------------------------ nn.Module surface the callers use
    @property
    def device(self):
        return self._device

    def to(self, device=None, *args, **kwargs):  # noqa: D401 - mirrors nn.Module.to for the device move
        if device is not None and not isinstance(device, torch.dtype):
            new = torch.device(device)
            if new.type == "cuda" and new.index is None:
                new = torch.device("cuda", torch.cuda.current_device())
            if new != self._device:
                self._release()  # the engine (weights, workspace, TMA descriptors) is bound to the device it was created on
            self._device = new
        return self

    def cuda(self, device=None):
        return self.to("cuda" if device is None else device)

    def train(self, mode=True):
        if mode:
            raise NotImplementedError("DD3DB200 is an inference engine; training uses the reference DD3D")
        return self

    def eval(self):
        return self

    def state_dict(self, *args, **kwargs):
        if self._state is None:
            return {k: torch.zeros(shape) for k, (shape, _) in self._specs.items()}
        return dict(self._state)

    def load_state_dict(self, state_dict, strict=True):
        """Accepts the reference DD3D state_dict (fvcore Checkpointer: ``{"model": state_dict}`` unwrapped)."""
        missing = [k for k in self._specs if k not in state_dict and not k.endswith("num_batches_tracked")]
        unexpected = [k for k in state_dict if k not in self._specs]
        if strict and (missing or unexpected):
            raise RuntimeError(f"Error(s) in loading state_dict for DD3DB200: missing {missing[:5]}, "
                               f"unexpected {unexpected[:5]}")
        for k, (shape, _) in self._specs.items():
            if k in state_dict and tuple(state_dict[k].shape) != tuple(shape):
                raise RuntimeError(f"size mismatch for {k}: {tuple(state_dict[k].shape)} vs {tuple(shape)}")
        self._state = {k: v.detach().to("cpu") for k, v in state_dict.items() if k in self._specs}
        self._release()
        return SimpleNamespace(missing_keys=missing, unexpected_keys=unexpected)

    # ------------------------------------------------------------------ engine lifetime
    def _release(self):
        if self._handle is not None:
            _lib.load().dd3d_destroy(self._handle)
        self._handle = None
        self._plan_key = None
        self._graph_synced = None

    def __del__(self):
        try:
            self._release()
        except Exception:  # noqa: BLE001
            pass

    def _engine_spec(self):
        """The config-to-ABI mapping: everything dd3d_create .. dd3d_finalize receive for this model, in call order
        (_engine makes the calls, save_model_file stores them)."""
        if self._state is None:
            raise RuntimeError("DD3DB200: load_state_dict() must be called before forward() or save_model_file()")
        # pixel mean/std travel in the state_dict like in the reference (core.py:54-55)
        for i in range(3):
            self._desc.pixel_mean[i] = float(self._state["pixel_mean"].reshape(-1)[i])
            self._desc.pixel_std[i] = float(self._state["pixel_std"].reshape(-1)[i])
        self._desc.do_nms = int(self.do_nms)

        def tensors():
            for name, t in self._state.items():
                if t.is_floating_point():
                    yield name, t.to(torch.float32).contiguous()

        return _lib.EngineSpec(self._desc, self._layout, self._backbone_norm, self._fpn_channels, self._fpn_inputs,
                               self._in_features, None if self._canon is None else (self.num_classes, self._canon), tensors)

    def _engine(self):
        if self._handle is not None:
            return self._handle
        if self._state is None:
            raise RuntimeError("DD3DB200: load_state_dict() must be called before forward()")
        if self._device.type != "cuda":
            raise RuntimeError("DD3DB200 runs on CUDA sm_90a (H100) only (model.to('cuda')); there is no CPU path")
        L = _lib.load()
        spec = self._engine_spec()
        handle = C.c_void_p()
        with torch.cuda.device(self._device):
            _lib.check(L.dd3d_create(C.byref(spec.desc), C.byref(handle)))
            _lib.check(L.dd3d_set_layout(handle, C.byref(spec.layout)), handle)
            _lib.check(L.dd3d_set_backbone_norm(handle, spec.backbone_norm), handle)
            _lib.check(L.dd3d_set_fpn_channels(handle, spec.fpn_channels), handle)
            if spec.fpn_inputs is not None:  # before dd3d_set_in_features, whose indices range over the FPN's outputs
                _lib.check(L.dd3d_set_fpn_inputs(handle, *spec.fpn_inputs), handle)
            if spec.in_features is not None:
                _lib.check(L.dd3d_set_in_features(handle, *spec.in_features), handle)
            if spec.canonical_sizes is not None:
                _lib.check(L.dd3d_set_canonical_sizes(handle, *spec.canonical_sizes), handle)
            for name, t in spec.tensors():
                shape = (C.c_int64 * max(t.dim(), 1))(*t.shape)
                _lib.check(L.dd3d_load_weight(handle, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()), handle)
            _lib.check(L.dd3d_finalize(handle), handle)
        self._handle = handle
        return handle

    def save_model_file(self, path):
        """Writes this model -- the engine's config values and the loaded state_dict's tensors -- to one self-contained
        file from which dd3d_create_from_file (include/dd3d_b200.h) builds the same engine in a C or C++ program, without
        Python, torch or the checkpoint.  Needs load_state_dict; no GPU.  The file holds do_nms as it is now and the
        output capacity the forward uses with it; postprocess_in_inference, do_bev_nms, the sample aggregation and the
        poses are run-time switches the caller sets per call, as on this model."""
        spec = self._engine_spec()
        desc = _lib.ModelDesc.from_buffer_copy(spec.desc)
        desc.out_cap = max(desc.out_cap, self._needed_out_cap())
        _lib.write_model_file(path, spec._replace(desc=desc))

    def _plan(self, B, Hs, Ws):
        key = (B, Hs, Ws)
        L = _lib.load()
        handle = self._engine()  # raises (no CPU path / weights not loaded) before any CUDA call
        # a switch that changes the op graph (do_bev_nms, or do_nms under it) makes the engine drop its plans
        if self._plan_key != key or L.dd3d_num_ops(handle) < 0:
            with torch.cuda.device(self._device):
                _lib.check(L.dd3d_plan(handle, B, Hs, Ws, None, 0), self._handle)
            self._plan_key = key
            self._host_bufs = None

    def _sync_options(self, postprocess_in_forward):
        """Pushes the attributes callers toggle at run time (postprocess_in_inference, do_nms, do_bev_nms:
        scripts/train.py:206-209, core.py:134-137) to the engine.  Without NMS (or without a post-NMS top-k) up to
        L * PRE_NMS_TOPK detections per image survive (L head levels): an engine planned with the small NMS-sized output buffer is rebuilt
        with the large one instead of silently truncating (the reference never truncates).  With do_bev_nms the engine
        runs the BEV NMS as its last op, then detector_postprocess (core.py:137-160)."""
        if self.do_bev_nms and self.only_box2d:
            self.do_bev_nms = False  # core.py:137: the BEV NMS needs the 3-D boxes
        need = self._needed_out_cap()
        if need > self._desc.out_cap:
            self._release()
            self._desc.out_cap = need
        L = _lib.load()
        h = self._engine()
        _lib.check(L.dd3d_set_option(h, b"do_postprocess", int(postprocess_in_forward)), h)
        _lib.check(L.dd3d_set_option(h, b"do_nms", int(self.do_nms)), h)
        _lib.check(L.dd3d_set_bev_nms(h, int(self.do_bev_nms), float(self.bev_nms_iou_thresh)), h)

    def _needed_out_cap(self):
        """Detection slots per image the forward needs at least under the current do_nms: every candidate without the NMS
        or its post-NMS top-k, else 0 (the desc's NMS-sized buffer)."""
        inf = self.cfg.DD3D.FCOS2D.INFERENCE
        return _lib.max_candidates(self.cfg) if (not self.do_nms or inf.POST_NMS_TOPK <= 0) else 0

    def _check_flags(self, flags):
        """Overflow word of the last forward (folded into the counts D2H): any set bit means the output differs from the
        reference's (which has no capacity limits) -- fail loudly instead of returning truncated detections."""
        self.last_overflow_flags = int(flags)
        if flags:
            names = {2: "more detections than out_cap slots", 4: "more than 256 boxes entered the BEV NMS of one image",
                     8: "sample aggregation capacity exceeded", 16: "more merged TTA detections than slots",
                     32: "grouped BEV NMS capacity exceeded", 64: "more than out_cap boxes entered the BEV NMS of one image"}
            raise RuntimeError("DD3DB200: detection capacity exceeded (" +
                               "; ".join(v for k, v in names.items() if flags & k) + f"; flags={int(flags)})")

    # ------------------------------------------------------------------ forward
    def _gather_inputs(self, batched_inputs, device):
        images = [x["image"] for x in batched_inputs]
        B = len(images)
        sizes_hw = [(int(im.shape[-2]), int(im.shape[-1])) for im in images]
        Hs, Ws = max(s[0] for s in sizes_hw), max(s[1] for s in sizes_hw)
        is_u8 = all(im.dtype == torch.uint8 for im in images)
        dtype = torch.uint8 if is_u8 else torch.float32
        if all(s == (Hs, Ws) for s in sizes_hw):
            batch = torch.stack([im.to(dtype) for im in images], 0)
        else:
            batch = torch.zeros((B, 3, Hs, Ws), dtype=dtype)
            for i, im in enumerate(images):
                batch[i, :, :im.shape[-2], :im.shape[-1]] = im.to(dtype)
        if "intrinsics" not in batched_inputs[0]:
            raise ValueError("DD3DB200 needs 'intrinsics' in every input (BOX3D_ON)")
        K = torch.stack([x["intrinsics"].to(torch.float32) for x in batched_inputs], 0)
        if torch.allclose(K[0].cpu(), torch.eye(3)):  # image_list.py:57-62
            raise ValueError("Intrinsics is Identity.")
        sizes = torch.empty((B, 4), dtype=torch.int32)
        for i, (x, (h, w)) in enumerate(zip(batched_inputs, sizes_hw)):
            if self.postprocess_in_inference:
                oh, ow = int(x.get("height", h)), int(x.get("width", w))
            else:
                oh, ow = h, w
            sizes[i] = torch.tensor([h, w, oh, ow], dtype=torch.int32)
        return batch, K.reshape(B, 9).contiguous(), sizes, (B, Hs, Ws), is_u8

    @staticmethod
    def _gather_poses(batched_inputs):
        """[B][7] sensor->global poses (w, x, y, z, tx, ty, tz) from input["pose"] / input["extrinsics"]
        (core.py:141-144): a tridet Pose (pyquaternion .quat.elements + .tvec), a (quat, tvec) pair, or a 4x4 matrix."""
        rows = []
        for x in batched_inputs:
            p = x["pose"] if "pose" in x else x["extrinsics"]
            if hasattr(p, "quat") and hasattr(p, "tvec"):
                q, t = [float(v) for v in p.quat.elements], [float(v) for v in p.tvec]
            elif isinstance(p, (tuple, list)) and len(p) == 2:
                q, t = [float(v) for v in p[0]], [float(v) for v in p[1]]
            else:
                m = torch.as_tensor(p, dtype=torch.float64)
                from .structures import matrix_to_quaternion_wxyz
                q, t = matrix_to_quaternion_wxyz(m[:3, :3]), [float(v) for v in m[:3, 3]]
            rows.append(q + t)
        return torch.tensor(rows, dtype=torch.float32)

    def _wrap(self, out, counts, K, sizes, device, global_boxes=None):
        """[B][cap][24] fp32 words + counts -> list[{"instances": Instances}] (fields: fcos2d.py:331-335, fcos3d.py:398;
        NuscenesDD3D adds pred_attributes / pred_speeds, nuscenes_dd3d.py:296-297, and pred_boxes3d_global,
        postprocessing.py:96-97)."""
        inv_K = torch.linalg.inv(K.reshape(-1, 3, 3).to(torch.float64)).to(torch.float32).to(device)
        results = []
        ints = out.view(torch.int32)
        for b, n in enumerate(counts.tolist()):
            d, di = out[b, :n], ints[b, :n]
            h, w, oh, ow = sizes[b].tolist()
            inst = Instances((oh, ow) if self.postprocess_in_inference else (h, w))
            inst.pred_boxes = Boxes(d[:, 0:4].clone())
            inst.scores = d[:, 4].clone()
            inst.pred_classes = di[:, 6].to(torch.int64)
            inst.locations = d[:, 18:20].clone()
            inst.fpn_levels = di[:, 7].to(torch.int64)
            if not self.only_box2d:  # core.py:117-125
                inst.pred_boxes3d = Boxes3D(d[:, 8:12].clone(), d[:, 12:14].clone(), d[:, 14:15].clone(),
                                            d[:, 15:18].clone(), inv_K[b][None].expand(n, 3, 3))
                inst.scores_3d = d[:, 5].clone()
            if self._desc.nuscenes_heads:
                inst.pred_attributes = di[:, 21].to(torch.int64)
                inst.pred_speeds = d[:, 22].clone()
            if global_boxes is not None:
                gb = global_boxes[b, :n]
                inst.pred_boxes3d_global = GenericBoxes3D(gb[:, 0:4].clone(), gb[:, 4:7].clone(), gb[:, 7:10].clone())
            results.append({"instances": inst})
        return results

    @torch.no_grad()
    def forward(self, batched_inputs):
        """Device path: inputs are moved to the GPU with torch, one small D2H (per-image counts) at the end."""
        return self._finish(self._forward_device(batched_inputs), batched_inputs)

    @torch.no_grad()
    def forward_raw(self, raw_inputs):
        """GPU input pipeline (SURVEY.md 8f row 3): takes what the dataset holds -- {"image_hwc": (H, W, 3) uint8 BGR
        array as cv2 reads it, "intrinsics": 3x3 of the original image, ...} -- and does the test-time work of
        DefaultDatasetMapper (dataset_mapper.py:100-153: ResizeShortestEdge to INPUT.RESIZE.MIN_SIZE_TEST with PIL-exact
        bilinear resampling, intrinsics rescale) on the device, fused with the model's normalisation.  Same outputs as
        ``forward([mapper(x) for x in raw_inputs])``; detections are mapped back to the original resolution."""
        return self._finish(self._forward_device_raw(raw_inputs), raw_inputs)

    def _finish(self, r, batched_inputs):
        host = r["counts"].cpu()  # the only sync: B counts + the overflow word
        self._check_flags(int(host[-1]))
        return self._wrap(r["out"], host[:-1], r["K"], r["sizes"], self._device)

    def _forward_device_raw(self, raw_inputs):
        device = self._device
        L = _lib.load()
        imgs = [torch.as_tensor(x["image_hwc"]) for x in raw_inputs]
        if not all(im.dtype == torch.uint8 and im.dim() == 3 and im.shape[2] == 3 for im in imgs):
            raise ValueError("forward_raw expects uint8 (H, W, 3) images")
        B = len(imgs)
        raw_h, raw_w = max(im.shape[0] for im in imgs), max(im.shape[1] for im in imgs)
        rs = self.cfg.INPUT.RESIZE
        min_size, max_size = (int(rs.MIN_SIZE_TEST), int(rs.MAX_SIZE_TEST)) if self.cfg.INPUT.AUG_ENABLED else (0, 0)
        raw_sizes = torch.tensor([[im.shape[0], im.shape[1]] for im in imgs], dtype=torch.int32)
        new_sizes = torch.zeros((B, 2), dtype=torch.int32)
        nh, nw = C.c_int32(), C.c_int32()
        for b in range(B):
            _lib.check(L.dd3d_resize_shape(int(raw_sizes[b, 0]), int(raw_sizes[b, 1]), min_size, max_size, C.byref(nh),
                                           C.byref(nw)))
            new_sizes[b, 0], new_sizes[b, 1] = nh.value, nw.value
        if all(tuple(im.shape) == (raw_h, raw_w, 3) for im in imgs):
            raw = torch.stack(imgs, 0)
        else:
            raw = torch.zeros((B, raw_h, raw_w, 3), dtype=torch.uint8)
            for b, im in enumerate(imgs):
                raw[b, :im.shape[0], :im.shape[1]] = im
        K0 = torch.stack([torch.as_tensor(x["intrinsics"], dtype=torch.float32) for x in raw_inputs], 0).reshape(B, 9).contiguous()
        if torch.allclose(K0[0].reshape(3, 3), torch.eye(3)):  # image_list.py:57-62
            raise ValueError("Intrinsics is Identity.")
        self._sync_options(self.postprocess_in_inference)
        self._plan(B, int(new_sizes[:, 0].max()), int(new_sizes[:, 1].max()))
        cap = self._desc.out_cap
        K = torch.empty((B, 9), dtype=torch.float32)
        with torch.cuda.device(device):
            d_poses = self._set_device_poses(raw_inputs)
            d_raw = raw.to(device, non_blocking=True)
            out = torch.empty((B, cap, _lib.DET_WORDS), dtype=torch.float32, device=device)
            counts = torch.zeros((B + 1, ), dtype=torch.int32, device=device)  # [B] counts + overflow word
            stream = torch.cuda.current_stream(device).cuda_stream
            _lib.check(
                L.dd3d_forward_raw(self._handle, C.c_void_p(d_raw.data_ptr()), raw_h, raw_w, C.c_void_p(raw_sizes.data_ptr()),
                                   C.c_void_p(K0.data_ptr()), min_size, max_size, C.c_void_p(out.data_ptr()),
                                   C.c_void_p(counts.data_ptr()), C.c_void_p(K.data_ptr()), None, C.c_void_p(stream)),
                self._handle)
            _lib.check(L.dd3d_copy_flags(self._handle, C.c_void_p(counts[B:].data_ptr()), C.c_void_p(stream)), self._handle)
            d_K = K.to(device, non_blocking=True)
        sizes = torch.cat([new_sizes, raw_sizes if self.postprocess_in_inference else new_sizes], 1)
        return dict(out=out, counts=counts, K=K, sizes=sizes, d_K=d_K, B=B, cap=cap, stream=stream, d_poses=d_poses)

    def _set_device_poses(self, batched_inputs):
        """With do_bev_nms: the [B][7] poses on the device, handed to the engine for the next forward (kept alive by the
        caller until that forward is enqueued)."""
        if not self.do_bev_nms:
            return None
        d_poses = self._gather_poses(batched_inputs).to(self._device, non_blocking=True)
        _lib.check(_lib.load().dd3d_set_poses(self._handle, C.c_void_p(d_poses.data_ptr())), self._handle)
        return d_poses

    def _set_host_poses(self, batched_inputs, slot):
        if self.do_bev_nms:
            poses = self._gather_poses(batched_inputs).contiguous()
            _lib.check(_lib.load().dd3d_set_host_poses(self._handle, int(slot), C.c_void_p(poses.data_ptr())), self._handle)

    def _forward_device(self, batched_inputs):
        device = self._device
        batch, K, sizes, shape, is_u8 = self._gather_inputs(batched_inputs, device)
        self._sync_options(self.postprocess_in_inference)
        self._plan(*shape)
        L = _lib.load()
        B = shape[0]
        cap = self._desc.out_cap
        with torch.cuda.device(device):
            d_batch = batch.to(device, non_blocking=True)
            d_K = K.to(device, non_blocking=True)
            d_sizes = sizes.to(device, non_blocking=True)
            d_poses = self._set_device_poses(batched_inputs)
            out = torch.empty((B, cap, _lib.DET_WORDS), dtype=torch.float32, device=device)
            counts = torch.zeros((B + 1, ), dtype=torch.int32, device=device)  # [B] counts + overflow word
            stream = torch.cuda.current_stream(device).cuda_stream
            _lib.check(
                L.dd3d_forward(self._handle, C.c_void_p(d_batch.data_ptr()), _lib.IMG_U8 if is_u8 else _lib.IMG_F32,
                               C.c_void_p(d_K.data_ptr()), C.c_void_p(d_sizes.data_ptr()), C.c_void_p(out.data_ptr()),
                               C.c_void_p(counts.data_ptr()), C.c_void_p(stream)), self._handle)
            _lib.check(L.dd3d_copy_flags(self._handle, C.c_void_p(counts[B:].data_ptr()), C.c_void_p(stream)), self._handle)
        return dict(out=out, counts=counts, K=K, sizes=sizes, d_K=d_K, B=B, cap=cap, stream=stream, d_poses=d_poses)

    def __call__(self, batched_inputs):
        return self.forward(batched_inputs)

    @torch.no_grad()
    def capture_forward(self, images_u8, intrinsics, sizes, poses=None, groups=None):
        """Records the forward on device buffers the caller keeps as a CUDA graph (dd3d_graph_create) and returns a
        CapturedForward: per frame, write the next images / intrinsics / sizes into the same tensors, then ``launch()``.
        images_u8: [B][3][Hs][Ws] uint8 (or float32); intrinsics: [B][3][3] or [B][9] float32; sizes: [B][4] int32 =
        (h, w, out_h, out_w) as dd3d_forward reads them.  With do_bev_nms (or the NuscenesDD3D sample aggregation) ``poses``
        is a [B][7] float32 device tensor and, for the aggregation, ``groups`` the group index of every image.  The
        attributes (postprocess_in_inference, do_nms, do_bev_nms) are taken as they are now; changing the engine's plan or
        options afterwards makes the graph stale (launch raises) -- forward() and the other paths push the options again,
        and with do_bev_nms or the aggregation so does every capture (it binds its poses)."""
        B = int(images_u8.shape[0]) if images_u8.dim() == 4 else -1
        tensors = dict(images=images_u8, intrinsics=intrinsics, sizes=sizes)
        shapes_ok = (B > 0 and images_u8.shape[1] == 3 and intrinsics.numel() == 9 * B and tuple(sizes.shape) == (B, 4)
                     and images_u8.dtype in (torch.uint8, torch.float32) and intrinsics.dtype == torch.float32
                     and sizes.dtype == torch.int32)
        if not shapes_ok:
            raise ValueError("capture_forward: images [B][3][H][W] uint8 / float32, intrinsics [B][9] float32 and sizes "
                             "[B][4] int32")
        for name, t in tensors.items():
            if t.device != self._device or not t.is_contiguous():
                raise ValueError(f"capture_forward: {name} must be a contiguous tensor on {self._device}")
        # every option call makes the engine's graphs stale: push the attributes only when they changed since the last
        # capture, so that several graphs of one shape can live side by side
        attrs = (self.postprocess_in_inference, self.do_nms, self.do_bev_nms, self.bev_nms_iou_thresh, self.only_box2d,
                 getattr(self, "sample_aggregate_in_inference", None))
        if self._handle is None or self._graph_synced != attrs:
            self._sync_options(self.postprocess_in_inference)
            self._graph_synced = attrs
        self._plan(B, int(images_u8.shape[2]), int(images_u8.shape[3]))
        L, h, cap = _lib.load(), self._handle, self._desc.out_cap
        with torch.cuda.device(self._device):
            keep = self._graph_bindings(B, poses, groups)
            out = torch.empty((B, cap, _lib.DET_WORDS), dtype=torch.float32, device=self._device)
            counts = torch.zeros((B + 1, ), dtype=torch.int32, device=self._device)  # [B] counts + overflow word
            stream = torch.cuda.current_stream(self._device).cuda_stream
            graph = C.c_void_p()
            status = L.dd3d_graph_create(h, C.c_void_p(images_u8.data_ptr()),
                                         _lib.IMG_U8 if images_u8.dtype == torch.uint8 else _lib.IMG_F32,
                                         C.c_void_p(intrinsics.data_ptr()), C.c_void_p(sizes.data_ptr()),
                                         C.c_void_p(out.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(stream),
                                         C.byref(graph))
            _lib.check(status, None)
        return CapturedForward(self, graph, out, counts, dict(tensors, **keep))

    def _graph_bindings(self, B, poses, groups):
        """The device buffers a captured forward reads besides its arguments, handed to the engine (dd3d_set_poses for the
        BEV NMS); returns them so that the graph keeps them alive."""
        return dict(poses=self._bind_poses(B, poses)) if self.do_bev_nms else {}

    def _bind_poses(self, B, poses):
        if poses is None or tuple(poses.shape) != (B, 7) or poses.dtype != torch.float32 or poses.device != self._device:
            raise ValueError(f"capture_forward needs poses: a [{B}][7] float32 tensor on {self._device}")
        poses = poses.contiguous()
        _lib.check(_lib.load().dd3d_set_poses(self._handle, C.c_void_p(poses.data_ptr())), self._handle)
        return poses

    @torch.no_grad()
    def forward_host(self, batched_inputs):
        """End-to-end path through HOST buffers: pinned staging -> dd3d_forward_host (H2D, kernels, D2H, sync)."""
        batch, K, sizes, shape, is_u8 = self._gather_inputs(batched_inputs, self._device)
        self._sync_options(self.postprocess_in_inference)
        self._plan(*shape)
        L = _lib.load()
        B = shape[0]
        cap = self._desc.out_cap
        hb = self._host_bufs
        if hb is None or hb["img"].shape != batch.shape or hb["img"].dtype != batch.dtype:
            hb = dict(img=torch.empty_like(batch).pin_memory(), K=torch.empty_like(K).pin_memory(),
                      sizes=torch.empty_like(sizes).pin_memory(),
                      out=torch.empty((B, cap, _lib.DET_WORDS), dtype=torch.float32).pin_memory(),
                      counts=torch.empty((B, ), dtype=torch.int32).pin_memory())
            self._host_bufs = hb
        hb["img"].copy_(batch)
        hb["K"].copy_(K)
        hb["sizes"].copy_(sizes)
        self._set_host_poses(batched_inputs, 0)
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _lib.check(
                L.dd3d_forward_host(self._handle, C.c_void_p(hb["img"].data_ptr()),
                                    _lib.IMG_U8 if is_u8 else _lib.IMG_F32, C.c_void_p(hb["K"].data_ptr()),
                                    C.c_void_p(hb["sizes"].data_ptr()), C.c_void_p(hb["out"].data_ptr()),
                                    C.c_void_p(hb["counts"].data_ptr()), C.c_void_p(stream)), self._handle)
        self._check_flags(self.overflow_flags())
        return self._wrap(hb["out"], hb["counts"], K, sizes, torch.device("cpu"), self._host_global_rows(0))

    @torch.no_grad()
    def submit_host(self, batched_inputs, slot=0):
        """Double-buffered host path (dd3d_submit_host): enqueues H2D -> kernels -> D2H for `slot` (0 / 1) and returns;
        ``wait_host(slot)`` returns the results.  Submitting the next batch to the other slot before waiting overlaps
        its H2D with the current batch's kernels.  All batches of a pipeline must share one plan shape."""
        batch, K, sizes, shape, is_u8 = self._gather_inputs(batched_inputs, self._device)
        self._sync_options(self.postprocess_in_inference)
        self._plan(*shape)
        L = _lib.load()
        B, cap = shape[0], self._desc.out_cap
        if not hasattr(self, "_slots"):
            self._slots = {}
        hb = self._slots.get(slot)
        if hb is None or hb["img"].shape != batch.shape or hb["img"].dtype != batch.dtype:
            hb = dict(img=torch.empty_like(batch).pin_memory(), K=torch.empty_like(K).pin_memory(),
                      sizes=torch.empty_like(sizes).pin_memory(),
                      out=torch.empty((B, cap, _lib.DET_WORDS), dtype=torch.float32).pin_memory(),
                      counts=torch.empty((B, ), dtype=torch.int32).pin_memory())
            self._slots[slot] = hb
        hb["img"].copy_(batch)
        hb["K"].copy_(K)
        hb["sizes"].copy_(sizes)
        hb["ctx"] = (K, sizes)
        self._set_host_poses(batched_inputs, slot)
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _lib.check(
                L.dd3d_submit_host(self._handle, int(slot), C.c_void_p(hb["img"].data_ptr()),
                                   _lib.IMG_U8 if is_u8 else _lib.IMG_F32, C.c_void_p(hb["K"].data_ptr()),
                                   C.c_void_p(hb["sizes"].data_ptr()), C.c_void_p(hb["out"].data_ptr()),
                                   C.c_void_p(hb["counts"].data_ptr()), C.c_void_p(stream)), self._handle)

    def wait_host(self, slot=0):
        hb = self._slots[slot]
        _lib.check(_lib.load().dd3d_wait_host(self._handle, int(slot)), self._handle)
        self._check_flags(self.overflow_flags())
        K, sizes = hb["ctx"]
        glob = self._host_global_rows(slot)
        return self._wrap(hb["out"].clone(), hb["counts"].clone(), K, sizes, torch.device("cpu"),
                          None if glob is None else glob.clone())

    def _host_global_rows(self, slot):
        """pred_boxes3d_global rows a host slot received (NuscenesDD3DB200 with the sample aggregation), else None."""
        return None

    # ------------------------------------------------------------------ introspection (stage-level parity tests)
    def get_tensor(self, name):
        """Device tensor of an engine-internal map after a forward: 'p0'..'p4', 'cls0'.., 'box0'.., 'b3d0'.., 'input'."""
        L = _lib.load()
        ptr = C.c_void_p()
        dims = (C.c_int32 * 6)()
        _lib.check(L.dd3d_get_tensor(self._handle, name.encode(), C.byref(ptr), C.byref(dims)), self._handle)
        B, H, W, Cc, pitch, eb = list(dims)
        # wrap device memory without copying through the CUDA array interface
        t = torch.as_tensor(_DevArray(ptr.value, (B, H, W, pitch), "<f4" if eb == 4 else "<i2"), device=self._device)
        if eb == 2:
            t = t.view(torch.float16 if self._desc.act_dtype == _lib.ACT_FP16 else torch.bfloat16)
        return t[..., :Cc]

    PROFILE_CATEGORIES = ("preprocess", "stem_conv", "conv_igemm", "maxpool", "ese", "relu", "decode", "nms")

    def set_engine_option(self, name, value):
        """dd3d_set_option pass-through for the switches that change the op graph or the workspace ("sparse_box3d",
        "workspace_reuse", "workspace_fill"): the next forward re-plans."""
        _lib.check(_lib.load().dd3d_set_option(self._engine(), name.encode(), int(value)), self._handle)
        self._plan_key = None
        self._graph_synced = None

    def set_profile(self, on):
        """Record CUDA events around every engine op of the following forwards (dd3d_get_profile)."""
        _lib.check(_lib.load().dd3d_set_option(self._engine(), b"profile", int(on)), self._handle)

    def get_profile(self):
        """{category: {ms, flops, bytes, launches}} of the last profiled forward."""
        ms, fl, by = (C.c_double * 8)(), (C.c_double * 8)(), (C.c_double * 8)()
        ln = (C.c_int32 * 8)()
        _lib.check(_lib.load().dd3d_get_profile(self._handle, ms, fl, by, ln), self._handle)
        return {n: dict(ms=ms[i], flops=fl[i], bytes=by[i], launches=ln[i]) for i, n in enumerate(self.PROFILE_CATEGORIES)}

    def get_op_times(self, max_ops=1024, with_op=False):
        """[(category, ms, algorithmic flops)] per step of the last profiled forward, in launch order.  with_op: each entry
        also carries the engine op the step ran (the index of get_conv_info), or -1 for the preprocess, tile-list, decode
        and NMS steps."""
        ms, cats, fl, ops = (C.c_float * max_ops)(), (C.c_int32 * max_ops)(), (C.c_double * max_ops)(), (C.c_int32 * max_ops)()
        n = _lib.check(_lib.load().dd3d_get_op_times(self._handle, ms, cats, fl, ops, max_ops), self._handle)
        return [(self.PROFILE_CATEGORIES[cats[i]], ms[i], fl[i]) + ((ops[i],) if with_op else ()) for i in range(n)]

    def get_conv_info(self, max_ops=1024):
        """Per engine op of the current plan, in launch order: None, or the conv's dict(taps, stride, cin, cout_pad, halo,
        pair, block_n, grouped) (dd3d_get_conv_info; grouped: the block-diagonal mode of a grouped 3x3)."""
        info = (C.c_int32 * (8 * max_ops))()
        n = _lib.check(_lib.load().dd3d_get_conv_info(self._handle, info, max_ops), self._handle)
        keys = ("taps", "stride", "cin", "cout_pad", "halo", "pair", "block_n")
        return [dict(zip(keys, info[8 * i + 1:8 * i + 8]), grouped=info[8 * i] == 2) if info[8 * i] else None
                for i in range(n)]

    def launches_per_forward(self):
        return _lib.load().dd3d_launches_per_forward(self._handle)

    def overflow_flags(self):
        flags = C.c_int32(0)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        _lib.check(_lib.load().dd3d_overflow_flags(self._handle, C.c_void_p(stream), C.byref(flags)), self._handle)
        return flags.value


def group_indices(sample_tokens, num_images_per_sample):
    """get_group_idxs (postprocessing.py:111-123): group index of every image, groups numbered in order of first
    appearance; every sample must have exactly `num_images_per_sample` images in the call."""
    order = {}
    for t in sample_tokens:
        order.setdefault(t, len(order))
    sizes = {t: 0 for t in order}
    for t in sample_tokens:
        sizes[t] += 1
    if not all(s == num_images_per_sample for s in sizes.values()):
        raise ValueError(f"Group sizes does not match with 'num_images_per_sample'. {sizes}")
    return [order[t] for t in sample_tokens]


class NuscenesDD3DB200(DD3DB200):
    """Mirror of ``tridet.modeling.dd3d.nuscenes_dd3d.NuscenesDD3D`` (nuscenes_dd3d.py:300-469) for inference: DD3D plus
    the attribute / speed predictors on the cls tower (fused into the cls predictor GEMM), ``pred_attributes`` /
    ``pred_speeds`` on every detection, and -- when ``postprocess_in_inference`` -- the cross-camera BEV NMS over the 6
    images of each nuScenes sample with at most MAX_NUM_DETS_PER_SAMPLE survivors (``pred_boxes3d_global`` added), run by
    the engine as the last step of every forward path (forward, forward_host, submit_host / wait_host, forward_raw).
    Inputs additionally carry "sample_token" and the global camera "pose"."""
    def __init__(self, cfg):
        super().__init__(cfg)
        self.num_images_per_sample = cfg.DD3D.NUSC.INFERENCE.NUM_IMAGES_PER_SAMPLE
        assert self.num_images_per_sample == 6  # nuscenes_dd3d.py:330
        assert cfg.DATALOADER.TEST.NUM_IMAGES_PER_GROUP == 6
        self.max_num_dets_per_sample = cfg.DD3D.NUSC.INFERENCE.MAX_NUM_DETS_PER_SAMPLE
        self.sample_aggregate_in_inference = True  # test hook: False returns the per-image detections before the aggregation
        self._groups = None  # group index of every image of the current call while the aggregation runs
        self._host_glob, self._host_glob_live = {}, {}  # per host slot: pinned global rows, filled by its last call

    def _aggregating(self, postprocess_in_forward=None):
        post = self.postprocess_in_inference if postprocess_in_forward is None else postprocess_in_forward
        return bool(post) and self.sample_aggregate_in_inference and not self.only_box2d

    def _check_groups(self, batched_inputs, out_sizes):
        """get_group_idxs (postprocessing.py:111-123) and the one common output size that detectron2's Instances.cat asserts
        when nuscenes_sample_aggregate concatenates the Instances of the call (postprocessing.py:95): host checks, raised
        before any device work.  Returns the group index of every image (None without the aggregation)."""
        if not self._aggregating():
            return None
        groups = group_indices([x["sample_token"] for x in batched_inputs], self.num_images_per_sample)
        assert len({tuple(int(v) for v in s) for s in out_sizes}) == 1, "images of one call must share the output size"
        return groups

    def _gather_inputs(self, batched_inputs, device):
        r = super()._gather_inputs(batched_inputs, device)
        self._groups = self._check_groups(batched_inputs, r[2][:, 2:].tolist())
        return r

    @torch.no_grad()
    def forward_raw(self, raw_inputs):
        # with postprocess_in_inference the output size of every image is its original (file) resolution
        self._groups = self._check_groups(raw_inputs, [tuple(x["image_hwc"].shape[:2]) for x in raw_inputs])
        return super().forward_raw(raw_inputs)

    def _sync_options(self, postprocess_in_forward):
        """The base switches, then the sample aggregation (nuscenes_dd3d.py:449-463) as the engine's last step whenever
        postprocess_in_inference is on; the engine drops its plans when the step turns on or off."""
        super()._sync_options(postprocess_in_forward)
        h = self._handle
        _lib.check(_lib.load().dd3d_set_sample_aggregate(h, int(self._aggregating(postprocess_in_forward)),
                                                         float(self.bev_nms_iou_thresh),
                                                         int(self.max_num_dets_per_sample or 0)), h)

    def _set_device_poses(self, batched_inputs):
        """With the sample aggregation: poses, group indices and the [B][cap][10] global-row buffer on the device, handed to
        the engine for the next forward.  Returns what must stay alive until that forward has run."""
        d_poses = super()._set_device_poses(batched_inputs)
        if self._groups is None:
            return SimpleNamespace(poses=d_poses, glob=None)
        L, h, device = _lib.load(), self._handle, self._device
        if d_poses is None:  # the BEV NMS did not hand them over already
            d_poses = self._gather_poses(batched_inputs).to(device, non_blocking=True)
            _lib.check(L.dd3d_set_poses(h, C.c_void_p(d_poses.data_ptr())), h)
        d_group = torch.tensor(self._groups, dtype=torch.int32).to(device, non_blocking=True)
        glob = torch.zeros((len(batched_inputs), self._desc.out_cap, _lib.GLOBAL_WORDS), dtype=torch.float32, device=device)
        _lib.check(L.dd3d_set_groups(h, C.c_void_p(d_group.data_ptr()), max(self._groups) + 1), h)
        _lib.check(L.dd3d_set_global_out(h, C.c_void_p(glob.data_ptr())), h)
        return SimpleNamespace(poses=d_poses, group=d_group, glob=glob)

    def _set_host_poses(self, batched_inputs, slot):
        """Host paths: poses and group indices copied by the engine, the slot's pinned global-row buffer registered."""
        self._host_glob_live[slot] = self._groups is not None
        if self._groups is None:
            return super()._set_host_poses(batched_inputs, slot)
        L, h = _lib.load(), self._handle
        poses = self._gather_poses(batched_inputs).contiguous()
        _lib.check(L.dd3d_set_host_poses(h, int(slot), C.c_void_p(poses.data_ptr())), h)
        groups = torch.tensor(self._groups, dtype=torch.int32)
        _lib.check(L.dd3d_set_host_groups(h, int(slot), C.c_void_p(groups.data_ptr()), max(self._groups) + 1), h)
        shape = (len(batched_inputs), self._desc.out_cap, _lib.GLOBAL_WORDS)
        glob = self._host_glob.get(slot)
        if glob is None or tuple(glob.shape) != shape:
            glob = torch.zeros(shape, dtype=torch.float32).pin_memory()
            self._host_glob[slot] = glob
        _lib.check(L.dd3d_set_host_global_out(h, int(slot), C.c_void_p(glob.data_ptr())), h)

    def _graph_bindings(self, B, poses, groups):
        """With the sample aggregation: the poses, the group indices and a [B][cap][10] global-row buffer
        (CapturedForward.global_rows) bound to the engine for the captured forward."""
        keep = super()._graph_bindings(B, poses, groups)
        if not self._aggregating():
            return keep
        if groups is None or len(groups) != B:
            raise ValueError(f"capture_forward with the sample aggregation needs the group index of each of the {B} images")
        L, h, device = _lib.load(), self._handle, self._device
        if "poses" not in keep:  # the BEV NMS did not bind them already
            keep["poses"] = self._bind_poses(B, poses)
        groups = [int(g) for g in groups]
        keep["group"] = torch.tensor(groups, dtype=torch.int32, device=device)
        keep["global_rows"] = torch.zeros((B, self._desc.out_cap, _lib.GLOBAL_WORDS), dtype=torch.float32, device=device)
        _lib.check(L.dd3d_set_groups(h, C.c_void_p(keep["group"].data_ptr()), max(groups) + 1), h)
        _lib.check(L.dd3d_set_global_out(h, C.c_void_p(keep["global_rows"].data_ptr())), h)
        return keep

    def _host_global_rows(self, slot):
        return self._host_glob.get(slot) if self._host_glob_live.get(slot) else None

    def _finish(self, r, batched_inputs):
        host = r["counts"].cpu()  # the only sync: B counts + the overflow word (bits 3 / 5: the aggregation's capacity)
        self._check_flags(int(host[-1]))
        return self._wrap(r["out"], host[:-1], r["K"], r["sizes"], self._device, r["d_poses"].glob)


class CapturedForward:
    """A forward recorded as a CUDA graph (DD3DB200.capture_forward): thin wrapper over dd3d_graph_launch /
    dd3d_graph_destroy.  ``launch(stream)`` replays it and copies the overflow word next to the counts; ``outputs()`` gives
    the live output tensors (dets [B][cap][24] fp32 words, counts [B] int32, flags [1] int32), valid once the launch's stream
    reaches them; ``global_rows`` is the [B][cap][10] pred_boxes3d_global buffer of the sample aggregation, or None."""
    def __init__(self, model, graph, out, counts, buffers):
        self._model, self._graph, self._out, self._counts, self._buffers = model, graph, out, counts, buffers
        self._handle = model._handle
        self.global_rows = buffers.get("global_rows")
        L = _lib.load()
        self.kernel_nodes = L.dd3d_graph_kernel_nodes(graph)
        self.programmatic_edges = L.dd3d_graph_programmatic_edges(graph)

    def launch(self, stream=None):
        if self._graph is None:
            raise RuntimeError("CapturedForward: launch after close()")
        L, device = _lib.load(), self._model.device
        if stream is None:
            stream = torch.cuda.current_stream(device)
        sp = C.c_void_p(stream.cuda_stream if isinstance(stream, torch.cuda.Stream) else stream)
        _lib.check(L.dd3d_graph_launch(self._graph, sp), None)
        B = self._out.shape[0]
        _lib.check(L.dd3d_copy_flags(self._handle, C.c_void_p(self._counts[B:].data_ptr()), sp), self._handle)

    def outputs(self):
        B = self._out.shape[0]
        return self._out, self._counts[:B], self._counts[B:]

    def close(self):
        if self._graph is not None:
            _lib.load().dd3d_graph_destroy(self._graph)
        self._graph = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class _DevArray:
    """Minimal __cuda_array_interface__ carrier so torch can alias engine-owned device memory."""
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}


if META_ARCH_REGISTRY is not None:  # pragma: no cover
    META_ARCH_REGISTRY.register(DD3DB200)
    META_ARCH_REGISTRY.register(NuscenesDD3DB200)
