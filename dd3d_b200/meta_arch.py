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
from .arch import arch_of, is_nuscenes_arch, param_specs, size_divisibility
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
        self._specs = param_specs(cfg)
        self._state = None  # reference-keyed fp32 CPU tensors
        self._device = torch.device("cpu")
        self._desc = _lib.desc_from_cfg(cfg)
        self._layout = _lib.layout_from_cfg(cfg)
        if cfg.DD3D.FCOS2D.USE_DEFORMABLE or (cfg.MODEL.BOX3D_ON and cfg.DD3D.FCOS3D.USE_DEFORMABLE):
            raise ValueError("Not supported yet.")  # fcos2d.py:51-52, fcos3d.py:77-78
        self._handle = None
        self._plan_key = None
        self._host_bufs = None
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

    def __del__(self):
        try:
            self._release()
        except Exception:  # noqa: BLE001
            pass

    def _engine(self):
        if self._handle is not None:
            return self._handle
        if self._state is None:
            raise RuntimeError("DD3DB200: load_state_dict() must be called before forward()")
        if self._device.type != "cuda":
            raise RuntimeError("DD3DB200 runs on CUDA sm_90a (H100) only (model.to('cuda')); there is no CPU path")
        L = _lib.load()
        # pixel mean/std travel in the state_dict like in the reference (core.py:54-55)
        for i in range(3):
            self._desc.pixel_mean[i] = float(self._state["pixel_mean"].reshape(-1)[i])
            self._desc.pixel_std[i] = float(self._state["pixel_std"].reshape(-1)[i])
        self._desc.do_nms = int(self.do_nms)
        handle = C.c_void_p()
        with torch.cuda.device(self._device):
            _lib.check(L.dd3d_create(C.byref(self._desc), C.byref(handle)))
            _lib.check(L.dd3d_set_layout(handle, C.byref(self._layout)), handle)
            for name, t in self._state.items():
                if not t.is_floating_point():
                    continue
                t = t.to(torch.float32).contiguous()
                shape = (C.c_int64 * max(t.dim(), 1))(*t.shape)
                _lib.check(L.dd3d_load_weight(handle, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()), handle)
            _lib.check(L.dd3d_finalize(handle), handle)
        self._handle = handle
        return handle

    def _plan(self, B, Hs, Ws):
        key = (B, Hs, Ws)
        if self._plan_key != key:
            L = _lib.load()
            handle = self._engine()  # raises (no CPU path / weights not loaded) before any CUDA call
            with torch.cuda.device(self._device):
                _lib.check(L.dd3d_plan(handle, B, Hs, Ws, None, 0), self._handle)
            self._plan_key = key
            self._host_bufs = None

    def _sync_options(self, postprocess_in_forward):
        """Pushes the attributes callers toggle at run time (postprocess_in_inference, do_nms: scripts/train.py:206-209,
        core.py:134) to the engine.  Without NMS (or without a post-NMS top-k) up to 5 * PRE_NMS_TOPK detections per image
        survive: an engine planned with the small NMS-sized output buffer is rebuilt with the large one instead of silently
        truncating (the reference never truncates)."""
        inf = self.cfg.DD3D.FCOS2D.INFERENCE
        if self.do_bev_nms and self.only_box2d:
            self.do_bev_nms = False  # core.py:137: the BEV NMS needs the 3-D boxes
        if self.do_bev_nms and not self.do_nms:
            raise NotImplementedError("DO_BEV_NMS without DO_NMS: the BEV kernel expects the score-sorted output of the 2-D NMS")
        need = 5 * inf.PRE_NMS_TOPK if (not self.do_nms or inf.POST_NMS_TOPK <= 0) else 0
        if need > self._desc.out_cap:
            self._release()
            self._desc.out_cap = need
        L = _lib.load()
        h = self._engine()
        _lib.check(L.dd3d_set_option(h, b"do_postprocess", int(postprocess_in_forward)), h)
        _lib.check(L.dd3d_set_option(h, b"do_nms", int(self.do_nms)), h)

    def _check_flags(self, flags):
        """Overflow word of the last forward (folded into the counts D2H): any set bit means the output differs from the
        reference's (which has no capacity limits) -- fail loudly instead of returning truncated detections."""
        self.last_overflow_flags = int(flags)
        if flags:
            names = {1: "more candidates tied at the k-th pre-NMS score than the boundary buffer holds",
                     2: "more detections than out_cap slots", 4: "more than 256 boxes entered the BEV NMS of one image",
                     8: "sample aggregation capacity exceeded", 16: "more merged TTA detections than slots",
                     32: "grouped BEV NMS capacity exceeded"}
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
        if self.do_bev_nms:
            raise NotImplementedError("forward_raw with DO_BEV_NMS: run the mapper-style forward()")
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
        return dict(out=out, counts=counts, K=K, sizes=sizes, d_K=d_K, B=B, cap=cap, stream=stream)

    def _forward_device(self, batched_inputs):
        device = self._device
        batch, K, sizes, shape, is_u8 = self._gather_inputs(batched_inputs, device)
        # with BEV NMS the rescale/clip happens after it (core.py:137-160): the BEV kernel applies it then
        self._sync_options(self.postprocess_in_inference and not self.do_bev_nms)
        self._plan(*shape)
        L = _lib.load()
        B = shape[0]
        cap = self._desc.out_cap
        with torch.cuda.device(device):
            d_batch = batch.to(device, non_blocking=True)
            d_K = K.to(device, non_blocking=True)
            d_sizes = sizes.to(device, non_blocking=True)
            out = torch.empty((B, cap, _lib.DET_WORDS), dtype=torch.float32, device=device)
            counts = torch.zeros((B + 1, ), dtype=torch.int32, device=device)  # [B] counts + overflow word
            stream = torch.cuda.current_stream(device).cuda_stream
            _lib.check(
                L.dd3d_forward(self._handle, C.c_void_p(d_batch.data_ptr()), _lib.IMG_U8 if is_u8 else _lib.IMG_F32,
                               C.c_void_p(d_K.data_ptr()), C.c_void_p(d_sizes.data_ptr()), C.c_void_p(out.data_ptr()),
                               C.c_void_p(counts.data_ptr()), C.c_void_p(stream)), self._handle)
            _lib.check(L.dd3d_copy_flags(self._handle, C.c_void_p(counts[B:].data_ptr()), C.c_void_p(stream)), self._handle)
            if self.do_bev_nms:
                d_poses = self._gather_poses(batched_inputs).to(device, non_blocking=True)
                self._bev_flags = torch.zeros(1, dtype=torch.int32, device=device)
                _lib.check(
                    L.dd3d_op_bev_nms(C.c_void_p(out.data_ptr()), C.c_void_p(counts.data_ptr()), C.c_void_p(d_K.data_ptr()),
                                      C.c_void_p(d_poses.data_ptr()), C.c_void_p(d_sizes.data_ptr()),
                                      C.c_void_p(self._bev_flags.data_ptr()), B, cap, float(self.bev_nms_iou_thresh),
                                      int(self.postprocess_in_inference), C.c_void_p(stream)), self._handle)
                counts[B:] |= self._bev_flags  # bit 2 rides in the same overflow word
        return dict(out=out, counts=counts, K=K, sizes=sizes, d_K=d_K, B=B, cap=cap, stream=stream)

    def __call__(self, batched_inputs):
        return self.forward(batched_inputs)

    @torch.no_grad()
    def forward_host(self, batched_inputs):
        """End-to-end path through HOST buffers: pinned staging -> dd3d_forward_host (H2D, kernels, D2H, sync)."""
        if self.do_bev_nms:  # the BEV NMS runs on the device buffers: device forward, then the results to the host
            return [{"instances": o["instances"].to("cpu")} for o in self.forward(batched_inputs)]
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
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream(self._device).cuda_stream
            _lib.check(
                L.dd3d_forward_host(self._handle, C.c_void_p(hb["img"].data_ptr()),
                                    _lib.IMG_U8 if is_u8 else _lib.IMG_F32, C.c_void_p(hb["K"].data_ptr()),
                                    C.c_void_p(hb["sizes"].data_ptr()), C.c_void_p(hb["out"].data_ptr()),
                                    C.c_void_p(hb["counts"].data_ptr()), C.c_void_p(stream)), self._handle)
        self._check_flags(self.overflow_flags())
        return self._wrap(hb["out"], hb["counts"], K, sizes, torch.device("cpu"))

    @torch.no_grad()
    def submit_host(self, batched_inputs, slot=0):
        """Double-buffered host path (dd3d_submit_host): enqueues H2D -> kernels -> D2H for `slot` (0 / 1) and returns;
        ``wait_host(slot)`` returns the results.  Submitting the next batch to the other slot before waiting overlaps
        its H2D with the current batch's kernels.  All batches of a pipeline must share one plan shape."""
        if self.do_bev_nms:
            raise NotImplementedError("submit_host with DO_BEV_NMS: use forward() / forward_host() (the BEV NMS kernel runs on "
                                      "the device buffers before the D2H)")
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
        return self._wrap(hb["out"].clone(), hb["counts"].clone(), K, sizes, torch.device("cpu"))

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
        """dd3d_set_option pass-through for the switches that change the op graph or the workspace ("dla_front",
        "workspace_reuse", "workspace_fill"): the next forward re-plans."""
        _lib.check(_lib.load().dd3d_set_option(self._engine(), name.encode(), int(value)), self._handle)
        self._plan_key = None

    def set_profile(self, on):
        """Record CUDA events around every engine op of the following forwards (dd3d_get_profile)."""
        _lib.check(_lib.load().dd3d_set_option(self._engine(), b"profile", int(on)), self._handle)

    def get_profile(self):
        """{category: {ms, flops, bytes, launches}} of the last profiled forward."""
        ms, fl, by = (C.c_double * 8)(), (C.c_double * 8)(), (C.c_double * 8)()
        ln = (C.c_int32 * 8)()
        _lib.check(_lib.load().dd3d_get_profile(self._handle, ms, fl, by, ln), self._handle)
        return {n: dict(ms=ms[i], flops=fl[i], bytes=by[i], launches=ln[i]) for i, n in enumerate(self.PROFILE_CATEGORIES)}

    def get_op_times(self, max_ops=1024):
        """[(category, ms, algorithmic flops)] per engine op of the last profiled forward, in launch order."""
        ms, cats, fl = (C.c_float * max_ops)(), (C.c_int32 * max_ops)(), (C.c_double * max_ops)()
        n = _lib.check(_lib.load().dd3d_get_op_times(self._handle, ms, cats, fl, max_ops), self._handle)
        return [(self.PROFILE_CATEGORIES[cats[i]], ms[i], fl[i]) for i in range(n)]

    def get_conv_info(self, max_ops=1024):
        """Per engine op of the current plan, in launch order: None, or the conv's dict(taps, stride, cin, cout_pad, halo,
        pair, block_n) (dd3d_get_conv_info)."""
        info = (C.c_int32 * (8 * max_ops))()
        n = _lib.check(_lib.load().dd3d_get_conv_info(self._handle, info, max_ops), self._handle)
        keys = ("taps", "stride", "cin", "cout_pad", "halo", "pair", "block_n")
        return [dict(zip(keys, info[8 * i + 1:8 * i + 8])) if info[8 * i] else None for i in range(n)]

    def launches_per_forward(self):
        return _lib.load().dd3d_launches_per_forward(self._handle)

    def overflow_flags(self):
        flags = C.c_int32(0)
        stream = torch.cuda.current_stream(self._device).cuda_stream
        _lib.check(_lib.load().dd3d_overflow_flags(self._handle, C.c_void_p(stream), C.byref(flags)), self._handle)
        f = flags.value
        if getattr(self, "_bev_flags", None) is not None:
            f |= int(self._bev_flags.item())
        return f


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
    images of each nuScenes sample with at most MAX_NUM_DETS_PER_SAMPLE survivors (``pred_boxes3d_global`` added).
    Inputs additionally carry "sample_token" and the global camera "pose"."""
    def __init__(self, cfg):
        super().__init__(cfg)
        self.num_images_per_sample = cfg.DD3D.NUSC.INFERENCE.NUM_IMAGES_PER_SAMPLE
        assert self.num_images_per_sample == 6  # nuscenes_dd3d.py:330
        assert cfg.DATALOADER.TEST.NUM_IMAGES_PER_GROUP == 6
        self.max_num_dets_per_sample = cfg.DD3D.NUSC.INFERENCE.MAX_NUM_DETS_PER_SAMPLE
        self.sample_aggregate_in_inference = True  # test hook: False returns the per-image detections before the aggregation

    def _finish(self, r, batched_inputs):
        glob = None
        if self.postprocess_in_inference and self.sample_aggregate_in_inference:
            L = _lib.load()
            device, B, cap = self._device, r["B"], r["cap"]
            groups = group_indices([x["sample_token"] for x in batched_inputs], self.num_images_per_sample)
            # nuscenes_sample_aggregate concatenates the Instances of the call (postprocessing.py:95); detectron2's
            # Instances.cat asserts one common (output) image size
            assert len({tuple(s[2:].tolist()) for s in r["sizes"]}) == 1, "images of one call must share the output size"
            with torch.cuda.device(device):
                d_poses = self._gather_poses([{"pose": x["pose"]} for x in batched_inputs]).to(device, non_blocking=True)
                d_group = torch.tensor(groups, dtype=torch.int32).to(device, non_blocking=True)
                glob = torch.zeros((B, cap, 10), dtype=torch.float32, device=device)
                scratch = torch.empty(int(L.dd3d_op_sample_aggregate_scratch_bytes(B, cap)), dtype=torch.uint8, device=device)
                self._agg_flags = torch.zeros(1, dtype=torch.int32, device=device)
                _lib.check(
                    L.dd3d_op_sample_aggregate(C.c_void_p(r["out"].data_ptr()), C.c_void_p(r["counts"].data_ptr()),
                                               C.c_void_p(r["d_K"].data_ptr()), C.c_void_p(d_poses.data_ptr()),
                                               C.c_void_p(d_group.data_ptr()), max(groups) + 1,
                                               C.c_void_p(glob.data_ptr()), C.c_void_p(scratch.data_ptr()),
                                               C.c_void_p(self._agg_flags.data_ptr()), B, cap,
                                               float(self.bev_nms_iou_thresh), int(self.max_num_dets_per_sample or 0),
                                               C.c_void_p(r["stream"])), self._handle)
            r["counts"][B:] |= self._agg_flags  # bit 3 rides in the same overflow word
        host = r["counts"].cpu()
        self._check_flags(int(host[-1]))
        return self._wrap(r["out"], host[:-1], r["K"], r["sizes"], self._device, glob)

    def forward_host(self, batched_inputs):
        """Host-buffer path: the sample aggregation needs the detections of all cameras on the device, so this is the
        device forward followed by the device->host copy of the results."""
        return [{"instances": o["instances"].to("cpu")} for o in self.forward(batched_inputs)]

    def overflow_flags(self):
        f = super().overflow_flags()
        if getattr(self, "_agg_flags", None) is not None:
            f |= int(self._agg_flags.item())
        return f


class _DevArray:
    """Minimal __cuda_array_interface__ carrier so torch can alias engine-owned device memory."""
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}


if META_ARCH_REGISTRY is not None:  # pragma: no cover
    META_ARCH_REGISTRY.register(DD3DB200)
    META_ARCH_REGISTRY.register(NuscenesDD3DB200)
