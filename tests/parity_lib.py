"""Measured end-to-end parity of the CUDA engine against the CPU oracle (shared by tests/test_parity_full_gpu.py, which
asserts thresholds, and tools/parity_report.py, which writes the measured numbers as JSON).

For one seeded case (oracle/gen_golden.py: small ragged cases and the BASELINE.json shapes 1 x 384x1280 DLA-34 /
1 x 900x1600 V2-99) and one storage type (bf16 / fp16) it measures, all through the C ABI:

  maps      every FPN output and every head map: relative L2 / max-abs error vs the oracle emulating the same storage
            type (single thread -> reproducible) and vs the pure-fp32 oracle (= the reference, pinned in test_cpu_oracle).
  hybrid    the engine's decode + NMS kernels against the oracle's decode + NMS run on the ENGINE's own head maps:
            identical candidate sets per level, identical kept set and order, fields within 1e-4 -- at full size.  This is
            north_star's "decoded boxes / scores within 1e-3" for everything downstream of the conv stack.
  pre_nms   candidate-level comparison with the oracle's candidates (thousands of samples instead of <= 100 survivors):
            match rate by (level, pixel, class) and error statistics per field over the matched candidates, after
            SURVEY.md 8c-4's exclusion policy: a candidate whose score is within `delta` of the 0.05 threshold, or within
            `delta` of the level's k-th score when the top-k bites, may legitimately exist on one side only.
  post_nms  the same on the final detections (+ the reference's own golden vectors): match rate, field errors.
"""
import ctypes as C
import os

import numpy as np
import torch

from dd3d_b200 import lib
from util import det_key, match_by_key, quat_dist

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIELDS = ("box", "score", "score3d", "quat", "proj_ctr", "depth", "size", "tvec")


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def run_detect(desc, cls, box, b3d, K, sizes, level_hw, strides, topk):
    """dd3d_op_detect on device head maps (lists of 5 cuda tensors, engine layout); returns pre-NMS candidates and
    final detections on the host."""
    L = lib.load()
    B = K.shape[0]
    arr = lambda ts: (C.c_void_p * 5)(*[t.data_ptr() for t in ts])  # noqa: E731
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    scratch = torch.empty(L.dd3d_op_detect_scratch_bytes(B, topk), dtype=torch.uint8, device="cuda")
    pre = torch.zeros(B, 5 * topk, 24, dtype=torch.float32, device="cuda")
    pre_n = torch.zeros(B, 5, dtype=torch.int32, device="cuda")
    out = torch.zeros(B, desc.out_cap, 24, dtype=torch.float32, device="cuda")
    cnt = torch.zeros(B, dtype=torch.int32, device="cuda")
    hw = (C.c_int32 * 10)(*[v for q in level_hw for v in q])
    st = (C.c_int32 * 5)(*strides)
    Kd, sd = K.reshape(B, 9).contiguous().cuda(), sizes.cuda()
    r = L.dd3d_op_detect(C.byref(desc), B, hw, st, arr(cls), arr(box), arr(b3d), cls[0].shape[-1], b3d[0].shape[-1],
                         p(Kd), p(sd), p(scratch), p(pre), p(pre_n), p(out), p(cnt),
                         C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert r == 0
    torch.cuda.synchronize()
    return pre.cpu(), pre_n.cpu(), out.cpu(), cnt.cpu()


def oracle_maps(cls, box, b3d, Cn):
    """Engine-layout head maps [B,H,W,pitch] (host) -> the per-level NCHW tensors the oracle's decode_level consumes."""
    o = dict(logits=[], centerness=[], box2d_reg=[], quat=[], ctr=[], depth=[], size=[], conf=[])
    for c, bx, b3 in zip(cls, box, b3d):
        c, bx, b3 = c.permute(0, 3, 1, 2), bx.permute(0, 3, 1, 2), b3.permute(0, 3, 1, 2)
        o["logits"].append(c[:, :Cn])
        o["box2d_reg"].append(bx[:, 0:4])
        o["centerness"].append(bx[:, 4:5])
        o["quat"].append(b3[:, 0:4 * Cn])
        o["ctr"].append(b3[:, 4 * Cn:6 * Cn])
        o["depth"].append(b3[:, 6 * Cn:7 * Cn])
        o["size"].append(b3[:, 7 * Cn:10 * Cn])
        o["conf"].append(b3[:, 10 * Cn:11 * Cn])
    return o


def dets_from_words(w, K_inv):
    """[n][24] fp32 words of dd3d_det -> dict of fields (tvec rebuilt like Boxes3D.tvec, boxes3d.py:169-173)."""
    wi = w.view(torch.int32)
    pc, depth = w[:, 12:14], w[:, 14]
    ray = torch.cat([pc, torch.ones(pc.shape[0], 1)], 1) @ K_inv.T
    return dict(box=w[:, 0:4], score=w[:, 4], score3d=w[:, 5], cls=wi[:, 6].long(), level=wi[:, 7].long(),
                quat=w[:, 8:12], proj_ctr=pc, depth=depth, size=w[:, 15:18], loc=w[:, 18:20], index=wi[:, 20].long(),
                tvec=ray * depth[:, None])


def dets_from_oracle(d):
    return dict(box=d["box2d"], score=d["score"], score3d=d["score3d"], cls=d["cls"], level=d["level"], quat=d["quat"],
                proj_ctr=d["proj_ctr"], depth=d["depth"], size=d["size"], loc=d["loc"], tvec=d["tvec"])


def dets_from_instances(inst):
    b3 = inst.pred_boxes3d
    return dict(box=inst.pred_boxes.tensor.cpu(), score=inst.scores.cpu(), score3d=inst.scores_3d.cpu(),
                cls=inst.pred_classes.cpu(), level=inst.fpn_levels.cpu(), quat=b3.quat.cpu(), proj_ctr=b3.proj_ctr.cpu(),
                depth=b3.depth.cpu()[:, 0], size=b3.size.cpu(), loc=inst.locations.cpu(), tvec=b3.tvec.cpu())


def dets_from_golden(g, b):
    t = lambda k: torch.tensor(g[f"{k}{b}"])  # noqa: E731
    return dict(box=t("boxes"), score=t("scores"), score3d=t("scores_3d"), cls=t("classes"), level=t("levels"),
                quat=t("quat"), proj_ctr=t("proj_ctr"), depth=t("depth").reshape(-1), size=t("size"),
                loc=t("locations"), tvec=t("tvec"))


def keys_of(d):
    return [det_key(l, p, c) for l, p, c in zip(d["level"], d["loc"], d["cls"])]


def field_errors(a, b, ia, ib):
    """Per-field error vectors between matched detections a[ia] (engine) and b[ib] (reference).  box: |diff| / box size
    (pixels relative to max(w, h, 1)); score / score3d: absolute (they live in [0, 1]); quat: distance up to sign;
    proj_ctr: pixels relative to the box size; depth / size: relative; tvec: relative to |tvec|."""
    if len(ia) == 0:
        return {f: np.zeros(0) for f in FIELDS}
    rb = b["box"][ib].double()
    bs = torch.maximum(rb[:, 2] - rb[:, 0], rb[:, 3] - rb[:, 1]).clamp(min=1.0)
    e = {}
    e["box"] = ((a["box"][ia].double() - rb).abs().max(dim=1).values / bs).numpy()
    e["score"] = (a["score"][ia].double() - b["score"][ib].double()).abs().numpy()
    e["score3d"] = (a["score3d"][ia].double() - b["score3d"][ib].double()).abs().numpy()
    e["quat"] = quat_dist(a["quat"][ia].double(), b["quat"][ib].double()).numpy()
    e["proj_ctr"] = ((a["proj_ctr"][ia].double() - b["proj_ctr"][ib].double()).abs().max(dim=1).values / bs).numpy()
    e["depth"] = ((a["depth"][ia].double() - b["depth"][ib].double()).abs() / b["depth"][ib].double().abs()).numpy()
    e["size"] = ((a["size"][ia].double() - b["size"][ib].double()).abs() / b["size"][ib].double().abs()).max(dim=1).values.numpy()
    tn = b["tvec"][ib].double().norm(dim=1).clamp(min=1e-6)
    e["tvec"] = ((a["tvec"][ia].double() - b["tvec"][ib].double()).norm(dim=1) / tn).numpy()
    return e


def summarize(errs):
    out = {}
    for f, v in errs.items():
        out[f] = dict(median=float(np.median(v)), p99=float(np.percentile(v, 99)), max=float(v.max())) if len(v) else None
    return out


def compare_sets(a, b, margin_mask_a=None, margin_mask_b=None):
    """Match a (engine) against b (reference) by (level, location, class).  margin_mask_*: True where the entry sits inside
    an exclusion margin (SURVEY 8c-4): such entries do not count as misses."""
    ka, kb = keys_of(a), keys_of(b)
    ia, ib = match_by_key(ka, kb)
    na, nb = len(ka), len(kb)
    miss_b = np.setdiff1d(np.arange(nb), ib)  # reference entries the engine lacks
    miss_a = np.setdiff1d(np.arange(na), ia)  # engine entries the reference lacks
    if margin_mask_b is not None:
        hard_b = int((~margin_mask_b[miss_b]).sum())
    else:
        hard_b = len(miss_b)
    if margin_mask_a is not None:
        hard_a = int((~margin_mask_a[miss_a]).sum())
    else:
        hard_a = len(miss_a)
    return dict(n_engine=na, n_ref=nb, matched=len(ia), missing=len(miss_b), extra=len(miss_a),
                missing_outside_margin=hard_b, extra_outside_margin=hard_a,
                match_rate=len(ia) / max(nb, 1)), ia, ib


def margin_mask(d, level_counts, kth_scores, thresh, delta):
    """True where the candidate's raw score s = score^2 is within `delta` of the threshold, or -- on a level whose
    candidate count reached the top-k -- within `delta` of that level's smallest kept score."""
    s = d["score"].double()**2
    m = (s - thresh).abs() <= delta
    for l, (n_full, kth) in enumerate(zip(level_counts, kth_scores)):
        if n_full and kth is not None:
            m |= (d["level"] == l) & ((s - kth).abs() <= delta)
    return m.numpy()


def measure_case(name, dtype, emu_threads=1, want_fp32=True):
    """Runs the engine and the oracle(s) on one golden case; returns (report dict, raw pieces for assertions)."""
    from dd3d_b200.meta_arch import DD3DB200
    from dd3d_b200.synthetic import make_state_dict
    from oracle.dd3d_oracle import DD3DOracle  # checker only
    from oracle.gen_golden import case_cfg, case_inputs

    cfg = case_cfg(name, act_dtype=dtype)
    sd = make_state_dict(cfg)
    inputs = case_inputs(name)
    model = DD3DB200(cfg).to("cuda")
    model.load_state_dict(sd)
    # the box3d predictor evaluated only at the final 2-D candidates (csrc/b3d_sparse.cu; the engine's choice for large heads) ...
    model.set_engine_option("sparse_box3d", 1)
    out_sparse = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    sparse_dets = [dets_from_instances(o["instances"]) for o in out_sparse]
    # ... everything below (stage maps, operator-level decode + NMS on the engine's own maps) needs the dense 3-D maps
    model.set_engine_option("sparse_box3d", 0)
    out = model(inputs)
    torch.cuda.synchronize()
    assert model.overflow_flags() == 0
    Cn = cfg.DD3D.NUM_CLASSES
    B = len(inputs)
    rep = dict(case=name, dtype=dtype, images=B)
    # sparse vs dense predictor: same detections in the same order; the 3-D fields differ only by the fp32 summation order
    # of the two tensor paths (mma.sync vs wgmma) over K = 2304
    sv = dict(same_keys_and_order=True, n=0, max_err={f: 0.0 for f in FIELDS})
    for b in range(B):
        d_, s_ = dets_from_instances(out[b]["instances"]), sparse_dets[b]
        same = d_["box"].shape[0] == s_["box"].shape[0] and keys_of(d_) == keys_of(s_)
        sv["same_keys_and_order"] &= bool(same)
        if same and d_["box"].shape[0]:
            idx = np.arange(d_["box"].shape[0])
            e = field_errors(s_, d_, idx, idx)
            for f in FIELDS:
                sv["max_err"][f] = max(sv["max_err"][f], float(e[f].max()))
            sv["n"] += len(idx)
    rep["sparse_vs_dense_box3d"] = sv

    g_cls = [model.get_tensor(f"cls{l}") for l in range(5)]
    g_box = [model.get_tensor(f"box{l}") for l in range(5)]
    g_b3d = [model.get_tensor(f"b3d{l}") for l in range(5)]
    g_fpn = [model.get_tensor(f"p{l}").float().cpu().permute(0, 3, 1, 2) for l in range(5)]

    emu = DD3DOracle(cfg, sd, emulate=dtype, threads=emu_threads)
    ref_e, int_e = emu.forward(inputs, return_intermediates=True)
    refs = {"emu": (ref_e, int_e)}
    if want_fp32:
        refs["fp32"] = DD3DOracle(cfg, sd).forward(inputs, return_intermediates=True)

    # ---- maps
    x = model.get_tensor("input")[..., :3].float().cpu().permute(0, 3, 1, 2)
    rep["input_bit_exact"] = bool(torch.equal(x, int_e["batch"]))
    rep["maps"] = {}
    for tag, (_, inter) in refs.items():
        m = inter["maps"]
        rows = {}
        for l in range(5):
            cls = g_cls[l].cpu().permute(0, 3, 1, 2)[:, :Cn]
            box = g_box[l].cpu().permute(0, 3, 1, 2)
            b3d = g_b3d[l].cpu().permute(0, 3, 1, 2)[:, :11 * Cn]
            ref3d = torch.cat([m["quat"][l], m["ctr"][l], m["depth"][l], m["size"][l], m["conf"][l]], 1)
            rows[f"p{l}"] = rel_l2(g_fpn[l], inter["features"][l])
            rows[f"cls{l}"] = rel_l2(cls, m["logits"][l])
            rows[f"reg{l}"] = rel_l2(box[:, :4], m["box2d_reg"][l])
            rows[f"ctr{l}"] = rel_l2(box[:, 4:5], m["centerness"][l])
            rows[f"b3d{l}"] = rel_l2(b3d, ref3d)
            rows[f"cls{l}_maxabs"] = float((cls - m["logits"][l]).abs().max())
        rows["worst_rel_l2"] = max(v for k, v in rows.items() if not k.endswith("maxabs"))
        rep["maps"][tag] = rows

    # ---- hybrid: engine decode + NMS vs oracle decode + NMS on the ENGINE's head maps
    strides = emu.strides
    level_hw = [(int(t.shape[1]), int(t.shape[2])) for t in g_cls]
    topk = cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_TOPK
    thresh = cfg.DD3D.FCOS2D.INFERENCE.PRE_NMS_THRESH
    K = torch.stack([x_["intrinsics"].float() for x_ in inputs], 0)
    inv_K = torch.linalg.inv(K)
    sizes = torch.tensor([[x_["image"].shape[-2], x_["image"].shape[-1], int(x_.get("height", x_["image"].shape[-2])),
                           int(x_.get("width", x_["image"].shape[-1]))] for x_ in inputs], dtype=torch.int32)
    # get_tensor returns [..., :C] views of pitch-wide buffers: rebuild the pitch-wide contiguous maps for the operator
    def widen(t, pitch):
        w = torch.zeros(t.shape[:-1] + (pitch, ), dtype=t.dtype, device=t.device)
        w[..., :t.shape[-1]] = t
        return w
    cls_pitch = (Cn + 15) // 16 * 16
    b3d_pitch = (11 * Cn + 15) // 16 * 16
    d_cls = [widen(t, cls_pitch) for t in g_cls]
    d_box = [widen(t, 16) for t in g_box]
    d_b3d = [widen(t, b3d_pitch) for t in g_b3d]
    pre, pre_n, fin, cnt = run_detect(model._desc, d_cls, d_box, d_b3d, K, sizes, level_hw, strides, topk)
    omaps = oracle_maps([t.cpu() for t in d_cls], [t.cpu() for t in d_box], [t.cpu() for t in d_b3d], Cn)
    hyb = dict(candidate_sets_equal=True, kept_order_equal=True, max_err={f: 0.0 for f in FIELDS}, candidates=0, kept=0)
    eng_pre = []
    for b in range(B):
        per_level = [emu.decode_level(omaps, l, b, inv_K[b]) for l in range(5)]
        cand_b = []
        for l, d in enumerate(per_level):
            n = int(pre_n[b, l])
            got = dets_from_words(pre[b, l * topk:l * topk + n], inv_K[b])
            cand_b.append(got)
            idx_ref = (d["pixel"] * Cn + d["cls"])
            if n != d["box2d"].shape[0] or set(got["index"].tolist()) != set(idx_ref.tolist()):
                hyb["candidate_sets_equal"] = False
                continue
            if n == 0:
                continue
            o_ref, o_got = torch.argsort(idx_ref), torch.argsort(got["index"])
            e = field_errors(got, dets_from_oracle(d), o_got.numpy(), o_ref.numpy())
            for f in FIELDS:
                hyb["max_err"][f] = max(hyb["max_err"][f], float(e[f].max()))
            hyb["candidates"] += n
        eng_pre.append({k: torch.cat([c[k] for c in cand_b], 0) for k in cand_b[0]})
        det = {k: torch.cat([d[k] for d in per_level], 0) for k in per_level[0]}
        img, osz = (int(sizes[b, 0]), int(sizes[b, 1])), (int(sizes[b, 2]), int(sizes[b, 3]))
        ref = emu.nms_topk_postprocess(dict(det), img, osz)
        n = int(cnt[b])
        got = dets_from_words(fin[b, :n], inv_K[b])
        same = n == ref["box2d"].shape[0] and torch.equal(got["index"], ref["pixel"] * Cn + ref["cls"]) and \
            torch.equal(got["level"], ref["level"])
        hyb["kept_order_equal"] &= bool(same)
        hyb["kept"] += n
        # the engine's own forward must have produced exactly these detections
        inst = dets_from_instances(out[b]["instances"])
        hyb["forward_equals_operator"] = hyb.get("forward_equals_operator", True) and \
            bool(inst["box"].shape[0] == n and torch.equal(inst["box"], got["box"]) and torch.equal(inst["score3d"], got["score3d"]))
    rep["hybrid"] = hyb

    # ---- pre-NMS candidates and final detections vs the oracles (and the reference's golden vectors)
    delta = None
    rep["pre_nms"], rep["post_nms"] = {}, {}
    for tag, (ref, inter) in refs.items():
        # exclusion margin: the largest |score error| the measured map error can cause; taken from the matched candidates
        # themselves (99.9th percentile of |ds|), floored at SURVEY's 1e-4
        agg_cmp = dict(n_engine=0, n_ref=0, matched=0, missing=0, extra=0, missing_outside_margin=0, extra_outside_margin=0)
        errs = {f: [] for f in FIELDS}
        ds_all = []
        per_image = []
        for b in range(B):
            r = dets_from_oracle(inter["pre_nms"][b])
            e_ = eng_pre[b]
            _, ia, ib = compare_sets(e_, r)
            ds_all.append((e_["score"][ia].double()**2 - r["score"][ib].double()**2).abs().numpy())
            per_image.append((e_, r))
        ds = np.concatenate(ds_all) if ds_all else np.zeros(0)
        delta = max(1e-4, float(np.percentile(ds, 99.9)) if len(ds) else 1e-4)
        for b, (e_, r) in enumerate(per_image):
            def lvl_stats(d):
                counts, kth = [], []
                for l in range(5):
                    sel = d["level"] == l
                    n = int(sel.sum())
                    counts.append(n >= topk)
                    kth.append(float((d["score"][sel].double()**2).min()) if n >= topk else None)
                return counts, kth
            ce, ke = lvl_stats(e_)
            cr, kr = lvl_stats(r)
            cmp_, ia, ib = compare_sets(e_, r, margin_mask(e_, cr, kr, thresh, delta), margin_mask(r, ce, ke, thresh, delta))
            for k in agg_cmp:
                agg_cmp[k] += cmp_[k]
            fe = field_errors(e_, r, ia, ib)
            for f in FIELDS:
                errs[f].append(fe[f])
        agg_cmp["match_rate"] = agg_cmp["matched"] / max(agg_cmp["n_ref"], 1)
        agg_cmp["margin_delta_raw_score"] = delta
        rep["pre_nms"][tag] = dict(sets=agg_cmp, errors=summarize({f: np.concatenate(v) for f, v in errs.items()}))

        agg = dict(n_engine=0, n_ref=0, matched=0)
        errs = {f: [] for f in FIELDS}
        for b in range(B):
            e_ = dets_from_instances(out[b]["instances"])
            r = dets_from_oracle(ref[b])
            cmp_, ia, ib = compare_sets(e_, r)
            for k in agg:
                agg[k] += cmp_[k]
            fe = field_errors(e_, r, ia, ib)
            for f in FIELDS:
                errs[f].append(fe[f])
        agg["match_rate"] = agg["matched"] / max(agg["n_ref"], 1)
        rep["post_nms"][tag] = dict(sets=agg, errors=summarize({f: np.concatenate(v) for f, v in errs.items()}))

    gpath = os.path.join(GOLDEN_DIR, f"golden_{name}.npz")
    if os.path.exists(gpath):
        g = np.load(gpath)
        agg = dict(n_engine=0, n_ref=0, matched=0)
        errs = {f: [] for f in FIELDS}
        for b in range(B):
            e_ = dets_from_instances(out[b]["instances"])
            r = dets_from_golden(g, b)
            cmp_, ia, ib = compare_sets(e_, r)
            for k in agg:
                agg[k] += cmp_[k]
            fe = field_errors(e_, r, ia, ib)
            for f in FIELDS:
                errs[f].append(fe[f])
        agg["match_rate"] = agg["matched"] / max(agg["n_ref"], 1)
        rep["post_nms"]["reference_golden"] = dict(sets=agg, errors=summarize({f: np.concatenate(v) for f, v in errs.items()}))
    return rep
