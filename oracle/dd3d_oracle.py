"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the DD3D inference hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this
module, and only as the checker / the CPU baseline.  The product path (dd3d_b200/) never imports it.

It is a plain-PyTorch (CPU, fp32) restatement of the reference's eval-mode ``DD3D.forward``
(/root/reference/tridet/modeling/dd3d/core.py:64-164) written functionally over the reference's
``state_dict`` key names.  Each function cites the reference file:line it follows.  Third-party arithmetic that
is NOT vendored under /root/reference (detectron2 FPN / FrozenBN / batched_nms / detector_postprocess,
pytorch3d quaternion conversions, torchvision nms) is restated from the published semantics listed in
SURVEY.md Appendix A.

Pinning: the reference ships no tests or golden vectors (SURVEY.md 4).  The oracle is pinned instead against
the reference's OWN modules executed in the build container under oracle/ref_standin.py
(tests/test_oracle_vs_reference.py, skipped where /root/reference is absent) and against the fixtures those
runs produced (tests/golden/*.npz, written by oracle/gen_golden.py).  The third-party pieces themselves remain
"parity unpinned" upstream (no pinned versions in the reference's Dockerfile) -- see DESIGN.md.

``emulate="bf16" | "fp16"`` (``emulate_bf16=True``) reproduces the CUDA engine's storage precision: conv weights
and every stored activation are rounded to that 16-bit type at the points where the engine stores it (after each conv
epilogue, after eSE scaling, after preprocessing); accumulation, BN affine, predictors' outputs, decode and NMS stay
fp32.  ``threads=1`` makes that emulation reproducible across processes (VERDICT r1 weak #4).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

EPS = 1e-7
BN_EPS = 1e-5


_EMU_DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16}


class DD3DOracle:
    def __init__(self, cfg, state_dict, emulate_bf16=False, emulate=None, threads=None):
        """emulate: None (pure fp32 = the reference), "bf16" or "fp16" (storage emulation of the engine's act_dtype;
        emulate_bf16=True is the older spelling of emulate="bf16").  threads: run forward() with this many intra-op
        threads (1 = accumulation order independent of the host's core count, so the storage emulation -- which amplifies
        1-ulp fp32 differences into 16-bit rounding flips -- reproduces bit for bit across processes and boxes)."""
        self.cfg = cfg
        self.sd = {k: v.detach().to(torch.float32).cpu() if v.is_floating_point() else v.detach().cpu()
                   for k, v in state_dict.items()}
        self.emu = emulate if emulate is not None else ("bf16" if emulate_bf16 else None)
        if self.emu is not None and self.emu not in _EMU_DTYPES:
            raise ValueError(f"emulate must be None, 'bf16' or 'fp16', got {self.emu!r}")
        self.threads = threads
        self.arch = "dla34" if cfg.FE.BUILDER == "build_fcos_dla_fpn_backbone_p67" else "v2_99"
        self.num_classes = cfg.DD3D.NUM_CLASSES
        if self.arch == "dla34":
            self.strides = [8, 16, 32, 64, 128]  # p3..p7 (dla.py:536-561)
            self.size_divisibility = 128  # FPN 32 * 4 (dla.py:559)
        else:
            self.strides = [4, 8, 16, 32, 64]  # p2..p6 (vovnet.py:428-454)
            self.size_divisibility = 64  # FPN 32 * 2 (vovnet.py:452)
        self.num_levels = 5
        self.nuscenes = cfg.MODEL.META_ARCHITECTURE == "NuscenesDD3D"  # nuscenes_dd3d.py:300-335

    # ------------------------------------------------------------------------------------------
    # primitives
    # ------------------------------------------------------------------------------------------
    def _q(self, x):
        return x.to(_EMU_DTYPES[self.emu]).to(torch.float32) if self.emu else x

    def _bn_affine(self, prefix):
        """FrozenBatchNorm2d / eval BatchNorm2d -> (scale, bias); detectron2 FrozenBatchNorm2d, eps=1e-5."""
        sd = self.sd
        scale = sd[prefix + ".weight"] * (sd[prefix + ".running_var"] + BN_EPS).rsqrt()
        bias = sd[prefix + ".bias"] - sd[prefix + ".running_mean"] * scale
        return scale, bias

    def conv(self, x, prefix, stride=1, relu=False, norm=None, residual=None, quant_out=True, wkey=None):
        """detectron2 ``Conv2d`` wrapper: conv -> norm -> (+residual) -> activation.
        `norm`: state_dict prefix of the BN to apply (default `<prefix>.norm` if present)."""
        sd = self.sd
        w = sd[(wkey or prefix) + ".weight"]
        k = w.shape[-1]
        if self.emu:
            w = self._q(w)
        y = F.conv2d(x, w, None, stride, (k - 1) // 2)
        cout = w.shape[0]
        scale = torch.ones(cout)
        bias = torch.zeros(cout)
        if (wkey or prefix) + ".bias" in sd:
            bias = sd[(wkey or prefix) + ".bias"].clone()
        nprefix = norm if norm is not None else prefix + ".norm"
        if nprefix + ".running_var" in sd:
            s, b = self._bn_affine(nprefix)
            bias = bias * s + b
            scale = s
        y = y * scale.view(1, -1, 1, 1) + bias.view(1, -1, 1, 1)
        if residual is not None:
            y = y + residual
        if relu:
            y = F.relu(y)
        return self._q(y) if quant_out else y

    # ------------------------------------------------------------------------------------------
    # preprocessing: core.py:61-72 + image_list.py:93-158
    # ------------------------------------------------------------------------------------------
    def preprocess(self, batched_inputs):
        mean = self.sd["pixel_mean"].view(3, 1, 1)
        std = self.sd["pixel_std"].view(3, 1, 1)
        images = [(x["image"].to(torch.float32) - mean) / std for x in batched_inputs]
        sizes = [(im.shape[-2], im.shape[-1]) for im in images]
        d = self.size_divisibility
        hmax = max(s[0] for s in sizes)
        wmax = max(s[1] for s in sizes)
        hp = (hmax + d - 1) // d * d
        wp = (wmax + d - 1) // d * d
        batch = torch.zeros(len(images), 3, hp, wp)  # pad value 0.0 AFTER normalisation
        for i, im in enumerate(images):
            batch[i, :, :im.shape[-2], :im.shape[-1]] = im
        intrinsics = torch.stack([x["intrinsics"].to(torch.float32) for x in batched_inputs], 0)
        if torch.allclose(intrinsics[0], torch.eye(3)):  # image_list.py:57-62
            raise ValueError("Intrinsics is Identity.")
        return self._q(batch), sizes, intrinsics

    # ------------------------------------------------------------------------------------------
    # DLA-34: dla.py:24-62 (BasicBlock), 146-167 (Root), 170-247 (Tree), 250-355 (DLA)
    # ------------------------------------------------------------------------------------------
    def _dla_block(self, x, p, stride, residual=None):
        if residual is None:
            residual = x
        out = self.conv(x, p + ".conv1", stride=stride, relu=True)
        out = self.conv(out, p + ".conv2", relu=True, residual=residual)
        return out

    def _dla_root(self, p, xs):
        # root_residual is False for DLA-34 (dla.py:359-361 passes no residual_root)
        return self.conv(torch.cat(xs, 1), p + ".conv", relu=True)

    def _dla_tree(self, x, p, levels, stride, level_root, in_ch, out_ch, children=None, residual=None):
        children = [] if children is None else children
        bottom = F.max_pool2d(x, stride, stride) if stride > 1 else x
        has_project = (in_ch != out_ch) and levels == 1
        residual = self.conv(bottom, p + ".project") if has_project else bottom
        if level_root:
            children.append(bottom)
        if levels == 1:
            x1 = self._dla_block(x, p + ".tree1", stride, residual)
            x2 = self._dla_block(x1, p + ".tree2", 1)
            return self._dla_root(p + ".root", [x2, x1] + children)
        x1 = self._dla_tree(x, p + ".tree1", levels - 1, stride, False, in_ch, out_ch)
        children.append(x1)
        return self._dla_tree(x1, p + ".tree2", levels - 1, 1, False, out_ch, out_ch, children=children)

    def dla34(self, x):
        p = "backbone.bottom_up"
        ch = [16, 32, 64, 128, 256, 512]
        levels = [1, 1, 1, 2, 2, 1]
        x = self.conv(x, p + ".base_layer", relu=True)
        x = self.conv(x, p + ".level0.0", relu=True)
        x = self.conv(x, p + ".level1.0", stride=2, relu=True)
        outs = {}
        x = self._dla_tree(x, p + ".level2", levels[2], 2, False, ch[1], ch[2])
        for lvl in (3, 4, 5):
            x = self._dla_tree(x, p + f".level{lvl}", levels[lvl], 2, True, ch[lvl - 1], ch[lvl])
            outs[f"level{lvl}"] = x
        return outs

    # ------------------------------------------------------------------------------------------
    # VoVNetV2-99-eSE: vovnet.py:79-87 (spec), 173-185 (eSE), 188-238 (OSA), 241-273 (stage), 276-367
    # ------------------------------------------------------------------------------------------
    def _vov_conv(self, x, p, name, stride=1):
        return self.conv(x, f"{p}.{name}/conv", stride=stride, relu=True, norm=f"{p}.{name}/norm")

    def _ese(self, x, p):
        sd = self.sd
        pooled = x.mean(dim=(2, 3), keepdim=True)
        y = F.conv2d(pooled, sd[p + ".fc.weight"], sd[p + ".fc.bias"])
        y = F.relu6(y + 3.0) / 6.0
        return x * y

    def _osa(self, x, p, name, identity):
        outs = [x]
        ident = x
        for i in range(5):
            x = self._vov_conv(x, f"{p}.layers.{i}", f"{name}_{i}")
            outs.append(x)
        xt = self._vov_conv(torch.cat(outs, 1), f"{p}.concat", f"{name}_concat")
        xt = self._ese(xt, p + ".ese")
        if identity:
            xt = xt + ident
        return self._q(xt)

    def v2_99(self, x):
        p = "backbone.bottom_up"
        x = self._vov_conv(x, p + ".stem", "stem_1", 2)
        x = self._vov_conv(x, p + ".stem", "stem_2", 1)
        x = self._vov_conv(x, p + ".stem", "stem_3", 2)
        outs = {}
        for si, nblocks in zip((2, 3, 4, 5), (1, 3, 9, 3)):
            if si != 2:
                x = F.max_pool2d(x, kernel_size=3, stride=2, ceil_mode=True)
            for b in range(nblocks):
                name = f"OSA{si}_{b + 1}"
                x = self._osa(x, f"{p}.stage{si}.{name}", name, identity=b > 0)
            outs[f"stage{si}"] = x
        return outs

    # ------------------------------------------------------------------------------------------
    # FPN: detectron2 FPN.forward (SURVEY Appendix A), LastLevelP6P7 / LastLevelP6 (vovnet.py:411-425)
    # ------------------------------------------------------------------------------------------
    def fpn(self, feats):
        p = "backbone"
        if self.arch == "dla34":
            names, stages = ["level3", "level4", "level5"], [3, 4, 5]
        else:
            names, stages = ["stage2", "stage3", "stage4", "stage5"], [2, 3, 4, 5]
        results = {}
        prev = None
        for name, st in zip(names[::-1], stages[::-1]):
            if prev is None:
                prev = self.conv(feats[name], f"{p}.fpn_lateral{st}")
            else:
                td = F.interpolate(prev, scale_factor=2.0, mode="nearest")
                prev = self.conv(feats[name], f"{p}.fpn_lateral{st}", residual=td)
            results[st] = self.conv(prev, f"{p}.fpn_output{st}")
        p6 = self.conv(results[5], f"{p}.top_block.p6", stride=2)
        outs = [results[s] for s in stages] + [p6]
        if self.arch == "dla34":
            outs.append(self.conv(self._q(F.relu(p6)), f"{p}.top_block.p7", stride=2))
        return outs

    # ------------------------------------------------------------------------------------------
    # heads: fcos2d.py:130-156, fcos3d.py:160-188 (ModuleListDial: level l uses norm l, normalization.py:30-40)
    # ------------------------------------------------------------------------------------------
    def _tower(self, x, p, lvl):
        for i in range(4):
            x = self.conv(x, f"{p}.{i}", relu=True, norm=f"{p}.{i}.norm.{lvl}")
        return x

    def heads(self, features):
        sd = self.sd
        f2, f3 = self.cfg.DD3D.FCOS2D, self.cfg.DD3D.FCOS3D
        box3d_on = bool(self.cfg.MODEL.BOX3D_ON)
        out = dict(logits=[], box2d_reg=[], centerness=[], quat=[], ctr=[], depth=[], size=[], conf=[])
        for l, f in enumerate(features):
            cls_t = self._tower(f, "fcos2d_head.cls_tower", l)
            box_t = self._tower(f, "fcos2d_head.box2d_tower", l)
            out["logits"].append(self.conv(cls_t, "fcos2d_head.cls_logits", quant_out=False))
            if self.nuscenes:  # nuscenes_dd3d.py:311-312,380-383: attribute logits / relu(speed) from the cls tower
                out.setdefault("attr", []).append(self.conv(cls_t, "attr_logits", quant_out=False))
                out.setdefault("speed", []).append(self.conv(cls_t, "speed", relu=True, quant_out=False))
            out["centerness"].append(self.conv(box_t, "fcos2d_head.centerness", quant_out=False))
            reg = self.conv(box_t, "fcos2d_head.box2d_reg", quant_out=False)
            if f2.USE_SCALE:  # fcos2d.py:145-152
                reg = reg * sd[f"fcos2d_head.scales_box2d_reg.{l}.scale"]
            out["box2d_reg"].append(F.relu(reg))
            if not box3d_on:  # core.py:34-40
                continue
            b3 = self._tower(f, "fcos3d_head.box3d_tower", l)
            i = l if f3.PER_LEVEL_PREDICTORS else 0  # fcos3d.py:166
            quat = self.conv(b3, f"fcos3d_head.box3d_quat.{i}", quant_out=False)
            ctr = self.conv(b3, f"fcos3d_head.box3d_ctr.{i}", quant_out=False)
            depth = self.conv(b3, f"fcos3d_head.box3d_depth.{i}", quant_out=False)
            size = self.conv(b3, f"fcos3d_head.box3d_size.{i}", quant_out=False)
            conf = self.conv(b3, f"fcos3d_head.box3d_conf.{i}", quant_out=False)
            if f3.USE_SCALE:  # fcos3d.py:175-180
                ctr = ctr * sd[f"fcos3d_head.scales_proj_ctr.{l}.scale"]
                size = size * sd[f"fcos3d_head.scales_size.{l}.scale"]
                conf = conf * sd[f"fcos3d_head.scales_conf.{l}.scale"]
                depth = depth * sd[f"fcos3d_head.scales_depth.{l}.scale"] + sd[f"fcos3d_head.offsets_depth.{l}.bias"]
            out["quat"].append(quat)
            out["ctr"].append(ctr)
            out["depth"].append(depth)
            out["size"].append(size)
            out["conf"].append(conf)
        return out

    # ------------------------------------------------------------------------------------------
    # decode: fcos2d.py:270-344, fcos3d.py:328-399 + 16-52, geometry.py:15-55,86-112, tensor2d.py:6-25
    # ------------------------------------------------------------------------------------------
    def locations(self, h, w, stride):
        ys, xs = torch.meshgrid(
            torch.arange(0, h * stride, stride, dtype=torch.float32),
            torch.arange(0, w * stride, stride, dtype=torch.float32), indexing="ij")
        loc = torch.stack((xs.reshape(-1), ys.reshape(-1)), 1)
        if self.cfg.DD3D.FEATURE_LOCATIONS_OFFSET == "half":
            loc = loc + stride // 2
        return loc

    def decode_level(self, maps, lvl, b, inv_K):
        """Candidates of image b at level lvl -> dict of per-candidate arrays (set semantics)."""
        cfg2 = self.cfg.DD3D.FCOS2D.INFERENCE
        C = self.num_classes
        logits = maps["logits"][lvl][b]
        h, w = logits.shape[-2:]
        scores = logits.permute(1, 2, 0).reshape(-1, C).sigmoid()
        ctrness = maps["centerness"][lvl][b].permute(1, 2, 0).reshape(-1).sigmoid()
        reg = maps["box2d_reg"][lvl][b].permute(1, 2, 0).reshape(-1, 4)
        if cfg2.THRESH_WITH_CTR:  # fcos2d.py:280-290: threshold the product, or the class score alone
            scores = scores * ctrness[:, None]
        mask = scores > cfg2.PRE_NMS_THRESH
        if not cfg2.THRESH_WITH_CTR:
            scores = scores * ctrness[:, None]
        cand = mask.nonzero(as_tuple=False)
        pix, cls = cand[:, 0], cand[:, 1]
        s = scores[mask]
        k = min(int(mask.sum()), cfg2.PRE_NMS_TOPK)
        if int(mask.sum()) > k:
            s, top = s.topk(k, sorted=False)
            pix, cls = pix[top], cls[top]
        loc = self.locations(h, w, self.strides[lvl])[pix]
        r = reg[pix]
        boxes = torch.stack([loc[:, 0] - r[:, 0], loc[:, 1] - r[:, 1], loc[:, 0] + r[:, 2], loc[:, 1] + r[:, 3]], 1)
        score2d = torch.sqrt(s)

        if not self.cfg.MODEL.BOX3D_ON:  # core.py:117-125: 2-D detector, the NMS is keyed on `scores`
            n = pix.shape[0]
            return dict(pixel=pix, cls=cls, level=torch.full_like(pix, lvl), box2d=boxes, score=score2d, score3d=score2d,
                        loc=loc, quat=torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1), proj_ctr=loc.clone(),
                        depth=torch.zeros(n), size=torch.zeros(n, 3), tvec=torch.zeros(n, 3))
        C3 = 1 if self.cfg.DD3D.FCOS3D.CLASS_AGNOSTIC_BOX3D else C  # fcos3d.py:333-352

        def gather(name, ncomp):
            m = maps[name][lvl][b].permute(1, 2, 0).reshape(-1, ncomp, C3)  # channel = comp*C3 + class
            return m[pix, :, cls if C3 > 1 else torch.zeros_like(cls)]

        quat = gather("quat", 4)
        ctr = gather("ctr", 2)
        depth = gather("depth", 1)[:, 0]
        size = gather("size", 3)
        conf = gather("conf", 1)[:, 0].sigmoid()
        canon = torch.tensor(self.cfg.DD3D.FCOS3D.CANONICAL_BOX3D_SIZES, dtype=torch.float32)[cls]
        box3d = predictions_to_boxes3d(quat, ctr, depth, size, loc, inv_K, canon, self.cfg.DD3D.FCOS3D)
        extra = {}
        if self.nuscenes:  # NuscenesInference, nuscenes_dd3d.py:268-298: argmax attribute, speed at the candidate pixel
            a = maps["attr"][lvl][b].permute(1, 2, 0).reshape(h * w, -1)[pix]
            extra["attr"] = a.argmax(dim=1) if a.shape[0] else torch.zeros(0, dtype=torch.long)
            extra["speed"] = maps["speed"][lvl][b].permute(1, 2, 0).reshape(-1)[pix]
        return dict(
            pixel=pix, cls=cls, level=torch.full_like(pix, lvl), box2d=boxes, score=score2d, score3d=score2d * conf,
            loc=loc, **box3d, **extra)

    # ------------------------------------------------------------------------------------------
    # NMS + top-k + postprocess: fcos2d.py:346-367, detectron2 batched_nms / detector_postprocess
    # ------------------------------------------------------------------------------------------
    def nms_topk_postprocess(self, det, image_size, out_size, do_postprocess=True):
        cfg2 = self.cfg.DD3D.FCOS2D.INFERENCE
        n = det["box2d"].shape[0]
        keep = torch.arange(n)
        if cfg2.NMS_THRESH > 0 and n > 0:
            keep = batched_nms_restated(det["box2d"], det["score3d"], det["cls"], cfg2.NMS_THRESH)
        det = {k: v[keep] for k, v in det.items()}
        n = det["box2d"].shape[0]
        if n > cfg2.POST_NMS_TOPK > 0:
            thr = torch.kthvalue(det["score"], n - cfg2.POST_NMS_TOPK + 1).values
            keep = torch.nonzero(det["score"] >= thr).squeeze(1)
            det = {k: v[keep] for k, v in det.items()}
        if do_postprocess:
            det = self.postprocess(det, image_size, out_size)
        return det

    @staticmethod
    def postprocess(det, image_size, out_size):
        """detectron2 detector_postprocess: scale to the output size, clip, drop empty boxes."""
        sx = out_size[1] / image_size[1]
        sy = out_size[0] / image_size[0]
        b = det["box2d"].clone()
        b[:, 0::2] *= sx
        b[:, 1::2] *= sy
        b[:, 0].clamp_(0, out_size[1])
        b[:, 2].clamp_(0, out_size[1])
        b[:, 1].clamp_(0, out_size[0])
        b[:, 3].clamp_(0, out_size[0])
        det = dict(det)
        det["box2d"] = b
        ne = ((b[:, 2] - b[:, 0]) > 0) & ((b[:, 3] - b[:, 1]) > 0)
        return {k: v[ne] for k, v in det.items()}

    # ------------------------------------------------------------------------------------------
    # whole forward
    # ------------------------------------------------------------------------------------------
    def backbone(self, batch):
        feats = self.dla34(batch) if self.arch == "dla34" else self.v2_99(batch)
        return self.fpn(feats)

    @torch.no_grad()
    def forward(self, batched_inputs, return_intermediates=False, do_postprocess=True):
        if self.threads is None:
            return self._forward(batched_inputs, return_intermediates, do_postprocess)
        prev = torch.get_num_threads()
        torch.set_num_threads(int(self.threads))
        try:
            return self._forward(batched_inputs, return_intermediates, do_postprocess)
        finally:
            torch.set_num_threads(prev)

    def _forward(self, batched_inputs, return_intermediates=False, do_postprocess=True):
        batch, sizes, K = self.preprocess(batched_inputs)
        feats = self.backbone(batch)
        maps = self.heads(feats)
        inv_K = torch.linalg.inv(K)
        results, pre_nms = [], []
        for b in range(batch.shape[0]):
            per_level = [self.decode_level(maps, l, b, inv_K[b]) for l in range(self.num_levels)]
            det = {k: torch.cat([d[k] for d in per_level], 0) for k in per_level[0]}
            pre_nms.append(det)
            out_size = (batched_inputs[b].get("height", sizes[b][0]), batched_inputs[b].get("width", sizes[b][1]))
            if self.cfg.DD3D.INFERENCE.DO_BEV_NMS:
                # core.py:134-160: 2-D NMS + top-k, then BEV NMS (per image = its own dummy group), then postprocess
                from oracle.bev_nms_oracle import bev_nms_image
                d = self.nms_topk_postprocess(dict(det), sizes[b], sizes[b], do_postprocess=False)
                pq, pt = pose_of(batched_inputs[b])
                keep = bev_nms_image(d, pq, pt, self.cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH)
                d = {k: v[keep] for k, v in d.items()}
                results.append(self.postprocess(d, sizes[b], out_size) if do_postprocess else d)
            else:
                results.append(self.nms_topk_postprocess(dict(det), sizes[b], out_size, do_postprocess))
        if self.nuscenes and do_postprocess:
            # nuscenes_dd3d.py:449-463: BEV NMS jointly over the cameras of each sample, <= MAX_NUM_DETS survivors
            from oracle.bev_nms_oracle import sample_aggregate
            tokens = [x["sample_token"] for x in batched_inputs]
            order = {t: i for i, t in enumerate(dict.fromkeys(tokens))}  # get_group_idxs, postprocessing.py:111-123
            nper = self.cfg.DD3D.NUSC.INFERENCE.NUM_IMAGES_PER_SAMPLE
            if any(tokens.count(t) != nper for t in order):
                raise ValueError("Group sizes does not match with 'num_images_per_sample'.")
            poses = [pose_of({"pose": x["pose"]}) for x in batched_inputs]
            results = sample_aggregate(results, [order[t] for t in tokens], poses,
                                       self.cfg.DD3D.INFERENCE.BEV_NMS_IOU_THRESH,
                                       self.cfg.DD3D.NUSC.INFERENCE.MAX_NUM_DETS_PER_SAMPLE)
        if return_intermediates:
            return results, dict(batch=batch, features=feats, maps=maps, pre_nms=pre_nms, inv_K=inv_K, sizes=sizes)
        return results


def pose_of(inp):
    """(quat wxyz, tvec) of input["pose"] / input["extrinsics"] (core.py:141-144): Pose-like object or a (quat, tvec) pair."""
    p = inp["pose"] if "pose" in inp else inp["extrinsics"]
    if hasattr(p, "quat"):
        return [float(v) for v in p.quat.elements], [float(v) for v in p.tvec]
    return [float(v) for v in p[0]], [float(v) for v in p[1]]


# ----------------------------------------------------------------------------------------------
# 3-D decode (free functions so kernel tests can call them directly)
# ----------------------------------------------------------------------------------------------
def quaternion_to_matrix(q):
    """pytorch3d.transforms.quaternion_to_matrix (real-first)."""
    r, i, j, k = q.unbind(-1)
    two_s = 2.0 / (q * q).sum(-1)
    o = torch.stack((1 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), 1 - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), 1 - two_s * (i * i + j * j)), -1)
    return o.reshape(q.shape[:-1] + (3, 3))


def matrix_to_quaternion(m):
    """pytorch3d >= 0.5 matrix_to_quaternion: best-conditioned candidate, no sign standardisation."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.reshape(-1, 9).unbind(-1)
    arg = torch.stack([1.0 + m00 + m11 + m22, 1.0 + m00 - m11 - m22, 1.0 - m00 + m11 - m22, 1.0 - m00 - m11 + m22], -1)
    q_abs = torch.where(arg > 0, torch.sqrt(arg.clamp(min=0)), torch.zeros_like(arg))
    cand = torch.stack([
        torch.stack([q_abs[:, 0]**2, m21 - m12, m02 - m20, m10 - m01], -1),
        torch.stack([m21 - m12, q_abs[:, 1]**2, m10 + m01, m02 + m20], -1),
        torch.stack([m02 - m20, m10 + m01, q_abs[:, 2]**2, m12 + m21], -1),
        torch.stack([m10 - m01, m20 + m02, m21 + m12, q_abs[:, 3]**2], -1),
    ], -2)
    cand = cand / (2.0 * q_abs[:, :, None].clamp(min=0.1))
    idx = q_abs.argmax(-1)
    return cand[torch.arange(cand.shape[0]), idx]


def unproject(points2d, inv_K):
    """geometry.py:86-112 with a single (3,3) inverse intrinsics."""
    ph = torch.cat([points2d, torch.ones(points2d.shape[0], 1)], 1)
    return ph @ inv_K.T


def allocentric_to_egocentric(quat, proj_ctr, inv_K):
    """geometry.py:15-55."""
    R_obj = quaternion_to_matrix(quat)
    ray = unproject(proj_ctr, inv_K)
    z = ray / ray.norm(dim=1, keepdim=True)
    y = torch.tensor([[0.0, 1.0, 0.0]]) - z[:, 1:2] * z
    y = y / y.norm(dim=1, keepdim=True)
    x = torch.cross(y, z, dim=1)
    R_l2g = torch.stack([x, y, z], -1)
    R = torch.bmm(R_l2g, R_obj)
    q = matrix_to_quaternion(R)
    n = q.norm(dim=1, keepdim=True)
    if q.shape[0] and not torch.allclose(n, torch.tensor(1.0), atol=1e-3):
        q = q / n.clamp(min=EPS)
    return q


def predictions_to_boxes3d(quat, ctr, depth, size, loc, inv_K, canon, cfg3d):
    """fcos3d.py:16-52 + Boxes3D.tvec (boxes3d.py:169-173)."""
    quat = quat / quat.norm(dim=1, keepdim=True).clamp(min=EPS)
    quat = quat / quat.norm(dim=1, keepdim=True)
    if cfg3d.SCALE_DEPTH_BY_FOCAL_LENGTHS:
        pixel_size = torch.sqrt(inv_K[0, 0]**2 + inv_K[1, 1]**2)
        depth = depth / (pixel_size * cfg3d.SCALE_DEPTH_BY_FOCAL_LENGTHS_FACTOR)
    if cfg3d.PREDICT_DISTANCE:
        depth = depth / unproject(loc, inv_K).norm(dim=1).clamp(min=EPS)
    depth = depth.clamp(cfg3d.MIN_DEPTH, cfg3d.MAX_DEPTH)
    proj_ctr = ctr + loc
    if cfg3d.PREDICT_ALLOCENTRIC_ROT:
        quat = allocentric_to_egocentric(quat, proj_ctr, inv_K)
    size = (size.tanh() + 1.0) * canon
    tvec = unproject(proj_ctr, inv_K) * depth[:, None]
    return dict(quat=quat, proj_ctr=proj_ctr, depth=depth, size=size, tvec=tvec)


def iou_matrix(b):
    area = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt = torch.max(b[:, None, :2], b[None, :, :2])
    rb = torch.min(b[:, None, 2:], b[None, :, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    return inter / (area[:, None] + area[None, :] - inter)


def batched_nms_restated(boxes, scores, idxs, thr):
    """detectron2 batched_nms -> torchvision batched_nms, per-class ("vanilla") form: greedy, sort by score
    descending (stable), suppress when IoU > thr (strict), only within the same class; returns kept indices in
    descending-score order.  Identical result set to the coordinate-offset form up to fp32 rounding of IoU."""
    n = boxes.shape[0]
    order = torch.argsort(scores, descending=True, stable=True)
    b = boxes[order]
    c = idxs[order]
    iou = iou_matrix(b)
    same = c[:, None] == c[None, :]
    sup = (iou > thr) & same
    removed = np.zeros(n, dtype=bool)
    sup_np = sup.numpy()
    keep = []
    for i in range(n):
        if removed[i]:
            continue
        keep.append(i)
        removed |= sup_np[i]
        removed[i] = True
    return order[torch.tensor(keep, dtype=torch.long)]
