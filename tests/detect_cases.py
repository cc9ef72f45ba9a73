"""Constructed head maps for the detection kernels (csrc/decode.cu: threshold + per-level top-k; csrc/nms.cu: class-aware
NMS + post-NMS top-k + rescale) and a host reference of the semantics they document.

The device computes sigmoid with expf, which is not correctly rounded, so the host cannot predict the bits of a score.  The
maps are built so that no ranking depends on those bits:
  * a class logit of +SAT gives a class score of exactly 1.0f, so the ranked score s is the centerness sigmoid alone;
    -SAT never passes; logit 0 gives exactly 0.5 (the at-threshold case);
  * distinct scores are hundreds of ulps apart and far from the threshold (`check_unambiguous`);
  * ties come only from identical inputs, which give bit-identical scores on the device;
  * the 3-D confidence logit is +SAT, so score_3d == score (= sqrt(s), correctly rounded on both sides).

Reference rules (`reference`):
  candidates   (pixel, class) with thresholded value > PRE_NMS_THRESH (s with THRESH_WITH_CTR, else the class score);
  top-k        per (image, level): order (s desc, index = pixel * C + class asc), keep the first PRE_NMS_TOPK;
  NMS          order (score_3d desc, level asc, index asc); greedy per class, suppress when the fp32 IoU
               inter / (a + b - inter) is > NMS_THRESH;
  post-NMS     keep survivors whose 2-D score is >= the POST_NMS_TOPK-th one (ties kept); scale, clip, drop empty boxes;
               the first out_cap are written, bit 1 of the flags when more survive.
`variant` switches one rule to a wrong one (the negative control of tests/test_detect_reference.py)."""
import numpy as np

SAT = 40.0
STRIDES_V2_99 = (4, 8, 16, 32, 64)
LEVELS_V2_99 = ((232, 400), (116, 200), (58, 100), (29, 50), (15, 25))  # 900x1600 padded to 928x1600
HIST_BINS, BOUNDARY_CAP = 2048, 4096
VARIANTS = ("thresh_ge", "index_desc", "boundary_trunc", "post_gt", "iou_ge")


def f32_bits(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


def bits_f32(k):
    return np.asarray(k, dtype=np.uint32).view(np.float32)


def logit(v):
    v = np.asarray(v, dtype=np.float64)
    return np.log(v / (1.0 - v)).astype(np.float32)


def sigmoid64(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, dtype=np.float64)))


def hist_params(thresh, with_ctr):
    """(thresh_bits, hist_shift) of decode_finalize_params."""
    t = np.float32(thresh if (thresh > 0 and with_ctr) else 0.0)
    tb = int(f32_bits(t))
    shift = 0
    while ((0x3F800000 - tb) >> shift) >= HIST_BINS:
        shift += 1
    return tb, shift


def bin_values(thresh, with_ctr, center, n, spacing_ulps):
    """n float scores `spacing_ulps` apart, all inside the histogram bin that holds `center`, >= 2000 ulps from its edges."""
    tb, shift = hist_params(thresh, with_ctr)
    k0 = ((int(f32_bits(np.float32(center))) - tb) >> shift) << shift
    span = (n - 1) * spacing_ulps
    assert span <= (1 << shift) - 4000, (n, spacing_ulps, shift)
    first = k0 + ((1 << shift) - span) // 2
    return bits_f32(np.arange(n, dtype=np.int64) * spacing_ulps + first + tb).astype(np.float64)


class Case:
    """Head maps of B images in the engine layout ([B][H*W][pitch] per level) plus the dd3d_model_desc fields the
    kernels read.  Every (pixel, class) starts at class logit -SAT (never a candidate)."""

    def __init__(self, C=10, level_hw=((64, 80), (32, 40), (16, 20), (8, 10), (4, 5)), strides=(8, 16, 32, 64, 128), B=1,
                 topk=1000, thresh=0.05, with_ctr=True, nms_thresh=0.75, post_topk=100, out_cap=128, class_agnostic=False):
        self.C, self.B, self.level_hw, self.strides = C, B, tuple(level_hw), tuple(strides)
        self.C3 = 1 if class_agnostic else C  # classes of the 3-D maps (CLASS_AGNOSTIC_BOX3D)
        self.topk, self.thresh, self.with_ctr = topk, thresh, with_ctr
        self.nms_thresh, self.post_topk, self.out_cap = nms_thresh, post_topk, out_cap
        self.cls_pitch = (C + 15) // 16 * 16
        self.b3d_pitch = (11 * self.C3 + 15) // 16 * 16
        self.cls, self.box, self.b3d = [], [], []
        for h, w in self.level_hw:
            cls = np.full((B, h * w, self.cls_pitch), -SAT, np.float32)
            box = np.zeros((B, h * w, 16), np.float32)
            box[..., 0:4] = 1.0  # 2x2-pixel boxes: disjoint unless a case says otherwise
            b3 = np.zeros((B, h * w, self.b3d_pitch), np.float32)
            C3 = self.C3
            b3[..., 0:C3] = 1.0               # quaternion w
            b3[..., 6 * C3:7 * C3] = 10.0     # depth
            b3[..., 10 * C3:11 * C3] = SAT    # 3-D confidence: score_3d == score
            self.cls.append(cls)
            self.box.append(box)
            self.b3d.append(b3)
        h0, w0 = self.level_hw[0]
        self.sizes = np.array([[h0 * self.strides[0], w0 * self.strides[0]] * 2] * B, np.int32)

    def put(self, b, l, pix, score, classes=(0,), cls_logit=SAT):
        """Pixels `pix` of (image b, level l) get centerness logit(score) (score in (0, 1), or a logit given as
        ('logit', x)) and class logit `cls_logit` at `classes`."""
        pix = np.atleast_1d(np.asarray(pix))
        x = np.asarray(score[1], np.float32) if isinstance(score, tuple) else logit(score)
        self.box[l][b, pix, 4] = x
        for c in classes:
            self.cls[l][b, pix, c] = cls_logit

    def level_scores(self, b, l):
        """(s, thresholded value) of every (pixel, class), [HW, C] float64."""
        cs = sigmoid64(self.cls[l][b, :, :self.C])
        s = cs * sigmoid64(self.box[l][b, :, 4])[:, None]
        return s, (s if self.with_ctr else cs)


def _topk_level(case, b, l, variant):
    s, t = case.level_scores(b, l)
    passing = (t >= case.thresh) if variant == "thresh_ge" else (t > case.thresh)
    pix, c = np.nonzero(passing)
    idx = pix * case.C + c
    sv = s[pix, c]
    if variant == "boundary_trunc":  # bin T capped at BOUNDARY_CAP entries taken in an arbitrary order
        tb, shift = hist_params(case.thresh, case.with_ctr)
        bins = np.minimum((f32_bits(sv.astype(np.float32)).astype(np.int64) - tb) >> shift, HIST_BINS - 1)
        if len(idx) > case.topk:
            hist = np.bincount(bins, minlength=HIST_BINS)
            above = np.cumsum(hist[::-1])[::-1]  # candidates in bins >= i
            T = int(np.nonzero(above >= case.topk)[0].max())
            inT = np.nonzero(bins == T)[0]
            if len(inT) > BOUNDARY_CAP:
                drop = np.random.default_rng(0).permutation(inT)[BOUNDARY_CAP:]
                keep = np.ones(len(idx), bool)
                keep[drop] = False
                idx, sv = idx[keep], sv[keep]
    order = np.lexsort((-idx if variant == "index_desc" else idx, -sv))[:case.topk]
    return idx[order], sv[order]


def reference(case, b, variant=None):
    """Per-level pre-NMS candidates (index arrays in rank order) and the final detections of image b:
    dict(pre=[idx per level], level, index, cls, box (scaled + clipped, fp32), score, n_written, flag_overflow)."""
    pre, lv, ix, sc = [], [], [], []
    for l in range(5):
        idx, sv = _topk_level(case, b, l, variant)
        pre.append(idx)
        lv.append(np.full(len(idx), l))
        ix.append(idx)
        sc.append(sv)
    level, index, s = np.concatenate(lv), np.concatenate(ix), np.concatenate(sc)
    cls = index % case.C
    boxes = np.zeros((len(index), 4), np.float32)
    for l in range(5):
        m = level == l
        pix = index[m] // case.C
        w, st = case.level_hw[l][1], case.strides[l]
        lx, ly = (pix % w * st).astype(np.float32), (pix // w * st).astype(np.float32)
        r = case.box[l][b, pix, 0:4]
        boxes[m] = np.stack([lx - r[:, 0], ly - r[:, 1], lx + r[:, 2], ly + r[:, 3]], 1)
    score = np.sqrt(s)  # score_3d == score (confidence 1.0)
    order = np.lexsort((index, level, -score))
    level, index, cls, boxes, score = level[order], index[order], cls[order], boxes[order], score[order]
    keep = _greedy_nms(boxes, cls, np.float32(case.nms_thresh), variant == "iou_ge")
    level, index, cls, boxes, score = level[keep], index[keep], cls[keep], boxes[keep], score[keep]
    if case.post_topk > 0 and len(score) > case.post_topk:
        kth = np.sort(score)[::-1][case.post_topk - 1]
        m = (score > kth) if variant == "post_gt" else (score >= kth)
        level, index, cls, boxes, score = level[m], index[m], cls[m], boxes[m], score[m]
    img_h, img_w, out_h, out_w = (int(v) for v in case.sizes[b])
    sx, sy = np.float32(out_w) / np.float32(img_w), np.float32(out_h) / np.float32(img_h)
    bx = boxes.copy()
    bx[:, 0::2] = np.minimum(np.maximum(bx[:, 0::2] * sx, np.float32(0)), np.float32(out_w))
    bx[:, 1::2] = np.minimum(np.maximum(bx[:, 1::2] * sy, np.float32(0)), np.float32(out_h))
    m = ((bx[:, 2] - bx[:, 0]) > 0) & ((bx[:, 3] - bx[:, 1]) > 0)
    level, index, cls, bx, score = level[m], index[m], cls[m], bx[m], score[m]
    n = min(len(index), case.out_cap)
    return dict(pre=pre, level=level[:n], index=index[:n], cls=cls[:n], box=bx[:n], score=score[:n], n_written=n,
                flag_overflow=len(index) > case.out_cap)


def iou_f32(a, b):
    """torchvision's IoU in fp32, one box a against boxes b [n, 4] (the operation order of iou_tv, csrc/nms.cu)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        area_a = (a[2] - a[0]) * (a[3] - a[1])
        area_b = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
        w = np.maximum(np.float32(0), np.minimum(a[2], b[:, 2]) - np.maximum(a[0], b[:, 0]))
        h = np.maximum(np.float32(0), np.minimum(a[3], b[:, 3]) - np.maximum(a[1], b[:, 1]))
        inter = w * h
        return inter / ((area_a + area_b) - inter)


def _greedy_nms(boxes, cls, thr, ge):
    n = len(boxes)
    removed = np.zeros(n, bool)
    for c in np.unique(cls):
        rows = np.nonzero(cls == c)[0]
        for k, i in enumerate(rows):
            if removed[i]:
                continue
            rest = rows[k + 1:]
            rest = rest[~removed[rest]]
            if len(rest):
                iou = iou_f32(boxes[i], boxes[rest])
                removed[rest[(iou >= thr) if ge else (iou > thr)]] = True
    return np.nonzero(~removed)[0]


def check_unambiguous(case, min_ulps=64):
    """The construction's promise: candidate scores are pairwise equal or >= min_ulps (fp32 ulps) apart, and
    thresholded values are equal to the threshold or >= min_ulps away from it -- so the device's score bits cannot
    change any ranking or threshold decision."""
    for b in range(case.B):
        vals = []
        for l in range(5):
            s, t = case.level_scores(b, l)
            near = np.abs(t - case.thresh) < min_ulps * np.spacing(np.float32(case.thresh))
            assert not (near & (t != case.thresh)).any(), (b, l, "value near the threshold")
            vals.append(s[t > case.thresh])
        v = np.unique(np.concatenate(vals))
        if len(v) > 1:
            gap = np.diff(v) / np.spacing(v[1:].astype(np.float32)).astype(np.float64)
            assert gap.min() >= min_ulps, (b, float(gap.min()))


# ------------------------------------------------------------------------------------------------ the constructed cases
def clustered(with_ctr, distinct, copies, topk=1000, extra=True, C=10):
    """`distinct` x `copies` scores inside ONE histogram bin at level 0 (> 4096 of them: more than the boundary buffer),
    plus, with `extra`, 310 candidates in higher bins and 300 in lower ones, and ties across classes of one pixel."""
    case = Case(C=C, level_hw=((80, 128), (40, 64), (20, 32), (10, 16), (5, 8)), topk=topk, with_ctr=with_ctr)
    vals = bin_values(case.thresh, with_ctr, 0.7, distinct, 300 if distinct > 1 else 1)
    scores = np.repeat(vals, copies)
    rng = np.random.default_rng(distinct * 7 + copies)
    pix = rng.permutation(80 * 128)
    n = len(scores)
    case.put(0, 0, pix[:n], scores[rng.permutation(n)] if distinct > 1 else scores)
    if extra:
        case.put(0, 0, pix[n:n + 310], np.linspace(0.9, 0.99, 310))  # 310: the k-th falls inside a group of copies
        case.put(0, 0, pix[n + 310:n + 610], np.linspace(0.2, 0.4, 300))
        case.put(0, 0, pix[n + 610:n + 620], vals[len(vals) // 2], classes=(1, 3, 4, 9))
    return case


def all_tied(with_ctr, topk=1000):
    """Every pixel of every level holds the same score for two classes: whole levels of identical scores."""
    case = Case(C=4, topk=topk, with_ctr=with_ctr)
    for l, (h, w) in enumerate(case.level_hw):
        case.put(0, l, np.arange(h * w), 0.6, classes=(0, 2))
    return case


def passing_count(n, topk):
    """Level 1 holds exactly n candidates with distinct scores (n = topk - 1, topk, topk + 1 or 0)."""
    case = Case(C=3, level_hw=((96, 128), (40, 50), (16, 20), (8, 10), (4, 5)), topk=topk)
    if n:
        case.put(0, 1, np.arange(n), np.linspace(0.95, 0.2, n), classes=(n % 3,))
    case.put(0, 0, [7, 9], 0.9, classes=(2,))
    return case


def at_threshold(with_ctr):
    """thresh = 0.5; a class logit 0 (class score exactly 0.5) or centerness logit 0 (s exactly 0.5) sits on it."""
    case = Case(C=4, thresh=0.5, with_ctr=with_ctr)
    case.put(0, 0, np.arange(0, 40), np.linspace(0.6, 0.9, 40))
    if with_ctr:
        case.put(0, 0, [50, 51], ("logit", 0.0), classes=(1, 2))           # s = 0.5: out
    else:
        case.put(0, 0, [50, 51], 0.9, classes=(1,), cls_logit=0.0)         # class score 0.5: out
        case.put(0, 0, [52], 0.9, classes=(3,))                             # class score 1, s = 0.9: in
    return case


def saturated(topk=64):
    """s = 1.0 exactly at several classes of several pixels (centerness logit +SAT): a tie broken by index."""
    case = Case(C=10, topk=topk)
    case.put(0, 0, np.arange(10, 40), ("logit", SAT), classes=(0, 3, 7, 9))
    case.put(0, 1, np.arange(0, 30), ("logit", SAT), classes=(2, 5))
    case.put(0, 0, np.arange(100, 300), np.linspace(0.3, 0.9, 200), classes=(1,))
    return case


def random_level(topk, seed, C=10):
    """Every level flooded with scores drawn from 37 values (ties across the k-th everywhere), each candidate pixel
    passing at a random subset of the classes."""
    case = Case(C=C, topk=topk)
    rng = np.random.default_rng(seed)
    vals = np.linspace(0.1, 0.95, 37)
    for l, (h, w) in enumerate(case.level_hw):
        pix = np.nonzero(rng.random(h * w) < 0.6)[0]
        case.put(0, l, pix, vals[rng.integers(0, len(vals), len(pix))], classes=())
        for c in range(C):
            case.cls[l][0, pix[rng.random(len(pix)) < 0.3], c] = SAT
    return case


def _set_box(case, l, pix, x1, y1, x2, y2):
    """Absolute box of level-l pixels `pix` of image 0 (through the regression channels)."""
    w, st = case.level_hw[l][1], case.strides[l]
    pix = np.atleast_1d(pix)
    lx, ly = (pix % w * st).astype(np.float32), (pix // w * st).astype(np.float32)
    case.box[l][0, pix, 0:4] = np.stack(np.broadcast_arrays(lx - x1, ly - y1, x2 - lx, y2 - ly), -1)


def iou_edges(nms_thresh):
    """One class of integer boxes at level 0, scores descending in this order:
      A [0, 16] x [0, 2] (area 32); B [0, 8] (IoU with A 0.5); C [0, 12] (0.75); D [0, 9] (0.5625); E [0, 13] (0.8125):
      at NMS_THRESH 0.5 B is kept (IoU exactly at the threshold) and C, D, E are suppressed; at 0.75 C is kept too;
      Z a zero-area box over G [100, 104] x [0, 2]: IoU 0, never suppresses;
      I an inverted box [204, 200] (area -8) over J [200, 204] (area 8): union 0, IoU 0 / 0 = NaN, never suppresses;
      K1, K2 two zero-area boxes at one point: NaN.  Empty boxes leave after the NMS (detector_postprocess)."""
    case = Case(C=2, level_hw=((8, 64), (4, 32), (2, 16), (1, 8), (1, 4)), nms_thresh=nms_thresh)
    rows = [(0, 0, 16, 2), (0, 0, 8, 2), (0, 0, 12, 2), (0, 0, 9, 2), (0, 0, 13, 2),
            (100, 0, 100, 0), (100, 0, 104, 2), (204, 0, 200, 2), (200, 0, 204, 2), (300, 0, 300, 0), (300, 0, 300, 0)]
    scores = (0.95, 0.93, 0.91, 0.89, 0.87, 0.99, 0.70, 0.97, 0.65, 0.96, 0.955)
    for p, (r, sc) in enumerate(zip(rows, scores)):
        _set_box(case, 0, p, *r)
        case.put(0, 0, [p], sc)
    return case


def class_sizes(sizes=(1, 63, 64, 65, 129)):
    """Class c holds sizes[c] boxes in a suppression chain, in score order: box i = [4i, 4i + 20] x [0, 8], so box i + 1
    overlaps it with IoU 0.67 (> 0.5) and box i + 2 with 0.43: greedy keeps every second box, across 64-box blocks --
    the segment and word edges of the multi-CTA NMS (nms_mask_kernel / nms_scan_kernel).  No post-NMS top-k."""
    case = Case(C=len(sizes), level_hw=((32, 160), (16, 80), (8, 40), (4, 20), (2, 10)), nms_thresh=0.5, post_topk=0,
                out_cap=256)
    for c, n in enumerate(sizes):
        pix = c * 4 * 160 + np.arange(n)  # level-0 pixel row 4c
        i = np.arange(n, dtype=np.float32)
        _set_box(case, 0, pix, 4 * i, 0, 4 * i + 20, 8)
        case.put(0, 0, pix, np.linspace(0.95, 0.3, n) if n > 1 else [0.8], classes=(c,))
    return case


def post_ties(n_tied):
    """90 candidates with distinct scores, then n_tied at one lower score (disjoint boxes): the 100th 2-D score is the
    tied one, so 90 + n_tied survive the post-NMS top-k; beyond out_cap (128) only the first 128 are written."""
    case = Case(C=3)
    case.put(0, 0, np.arange(90), np.linspace(0.9, 0.6, 90), classes=(0,))
    case.put(0, 1, np.arange(n_tied // 2), 0.4, classes=(1,))
    case.put(0, 2, np.arange(n_tied - n_tied // 2), 0.4, classes=(2,))
    return case


def level_ties():
    """The same ten scores at pixels 0-9 of every level, class 0: score_3d ties across levels.  Pixel 0 has the same
    box [-1, 1]^2 at every level, so the level-0 copy suppresses the others; the other pixels are apart and must come out
    in (score, level) order."""
    case = Case(C=2)
    for l in range(5):
        case.put(0, l, np.arange(10), np.linspace(0.9, 0.5, 10))
    return case


def big_batch(B=32):
    """B images at the V2-99 900x1600 level shapes, a different distribution per image: one-bin clusters beyond the
    boundary buffer, whole levels of one score, sparse random scores, nothing at all."""
    case = Case(C=10, level_hw=LEVELS_V2_99, strides=STRIDES_V2_99, B=B, class_agnostic=True)
    case.sizes[:] = (900, 1600, 900, 1600)
    for b in range(B):
        rng = np.random.default_rng(100 + b)
        kind = b % 4
        for l, (h, w) in enumerate(case.level_hw):
            if kind == 0 and l == 0:   # 60 values x 100 copies in one bin
                vals = np.repeat(bin_values(case.thresh, True, 0.55 + 0.01 * (b % 7), 60, 300), 100)
                pix = rng.permutation(h * w)[:len(vals)]
                case.put(b, l, pix, vals, classes=(b % 10,))
            elif kind == 1:            # every pixel of the level at one score, two classes
                case.put(b, l, np.arange(h * w), 0.3 + 0.1 * l, classes=(b % 10, (b + 3) % 10))
            elif kind == 2:            # sparse, 37 values
                pix = np.nonzero(rng.random(h * w) < 0.05)[0]
                case.put(b, l, pix, np.linspace(0.1, 0.95, 37)[rng.integers(0, 37, len(pix))], classes=(l, 5))
    return case
