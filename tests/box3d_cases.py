"""Constructed FCOS3D head maps for the 3-D box decode (decode_one, csrc/decode.cu) and a float64 reference of it.

Every test geometry sits on its own (image, level, pixel, class) of detect_cases.Case maps.  Its class and centerness
logits are +SAT, so its ranked score is exactly 1.0; every other (pixel, class) is -SAT.  Each level holds far fewer than
PRE_NMS_TOPK candidates, so every record is a candidate and is found by its `index` word.  All 11 * C3 3-D channels of
every pixel hold distinct values, the classes that are not candidates there included, and the padding of every map row is
NaN: a decode that reads a wrong column, or the padding, cannot give the right answer by accident.

Families (`fam` of a record), on B = 3 cameras (KITTI-like, nuScenes-like, and a synthetic K with fx != fy, skew and an
off-centre principal point):
  rotation   identity; yaw about the camera y axis at 0, +-45, +-90, +-180 degrees and +-1e-4 around each; yaw with pitch
             and roll up to +-30; random unit quaternions; near-ties of the four matrix_to_quaternion candidates; raw
             outputs scaled by 1e-8 .. 1e6; every one as q and -q; half of them projected at the principal point (where
             the local-to-global rotation is the identity);
  zero_quat  the exact-zero quaternion: NaN in `quat` (in the reference too), every other field finite and in bounds;
  ray        proj_ctr at the principal point, the image corners and edge midpoints, and up to one image size outside;
  extreme    rays 60 / 70 / 80 degrees off the optical axis;
  depth      (synthetic camera) depths that land on MIN_DEPTH / MAX_DEPTH, one float32 ulp inside and outside them, far
             beyond, zero and negative, through whatever focal / distance scaling the configuration applies;
  size       size logits 0, +-1, +-8, +-SAT, so that tanh + 1 is exactly 0 or 2 at +-SAT; canonical rows W != L != H.
The NuscenesDD3D attribute logits at the candidate pixels hold ties (torch.argmax takes the first maximum) and the speed
channel arbitrary values, -0.0 included.

box3d_ref64 restates predictions_to_boxes3d / allocentric_to_egocentric (fcos3d.py, geometry.py) and pytorch3d's quaternion
<-> matrix conversions in float64 on the same float32 inputs, with K inverted in float64.  `compare` holds a decode's
records (24-word Det rows) to it with the bounds below."""
import itertools

import numpy as np

import detect_cases as D

SAT = D.SAT
NC = 10
LEVEL_HW = ((19, 29), (10, 15), (5, 8), (3, 4), (2, 3))  # ragged: no level is a multiple of the next
STRIDES = (8, 16, 32, 64, 128)
MIN_DEPTH, MAX_DEPTH, DEPTH_FACTOR = np.float32(0.1), np.float32(80.0), np.float32(500.0)  # dd3d.yaml defaults
CAMERAS = (  # name, K, image width, height
    ("kitti", ((721.5377, 0.0, 609.5593), (0.0, 721.5377, 172.854), (0.0, 0.0, 1.0)), 1242, 375),
    ("nuscenes", ((1266.4172, 0.0, 816.267), (0.0, 1266.4172, 491.50708), (0.0, 0.0, 1.0)), 1600, 900),
    ("synthetic", ((903.25, 12.5, 270.75), (0.0, 655.5, 388.25), (0.0, 0.0, 1.0)), 800, 600),
)
K32 = np.array([np.array(k, np.float32).reshape(9) for _, k, _, _ in CAMERAS])
CANON = np.array([[0.6 + 0.13 * c, 1.9 + 0.41 * c, 1.2 + 0.07 * c] for c in range(NC)], np.float32)  # (W, L, H)
ATTR_PATTERNS = ((0.5, 0.5, 0.5), (1.25, 1.25, -2.0), (-2.0, 1.25, 1.25), (1.25, -2.0, 1.25), (-1.0, -1.0, 3.0),
                 (-0.0, 0.0, -1.0), (3.0, -1.0, 2.0))
SPEEDS = (0.0, -0.0, 7.25, -3.5, 1e-30, 123.456, -2.5e4)
FAMILIES = ("rotation", "zero_quat", "ray", "extreme", "depth", "size")

# Bounds against the float64 reference (tests/test_box3d_decode_gpu.py).  Bit-exact: box, proj_ctr, loc, score, cls,
# level, index, attr, speed, and depth where the reference clamps.
DEPTH_REL = 1e-6
SCORE3D_ULPS = 4
SIZE_REL_CANON = 2.0 ** -21
QUAT_NORM = 1e-6
QUAT_ROT = 4e-6
SIGN_MARGIN = 1e-3


def config(half=False, distance=False, allocentric=True, scale_depth=True, agnostic=False, nuscenes=False,
           box3d_on=True):
    return dict(half=half, distance=distance, allocentric=allocentric, scale_depth=scale_depth, agnostic=agnostic,
                nuscenes=nuscenes, box3d_on=box3d_on)


def _configs():
    out = {}
    names = ("half", "distance", "allocentric", "scale_depth")
    for bits in itertools.product((False, True), repeat=4):
        out["-".join(n for n, v in zip(names, bits) if v) or "egocentric"] = config(*bits)
    out["agnostic"] = config(agnostic=True)
    out["agnostic-half-distance"] = config(half=True, distance=True, agnostic=True)
    out["nuscenes"] = config(nuscenes=True)
    out["box3d_off"] = config(box3d_on=False)
    return out


CONFIGS = _configs()


# ------------------------------------------------------------------------------------------------ quaternions (float64)
def _axis_quat(axis, deg):
    """Rotation by `deg` about camera axis 0 (x), 1 (y) or 2 (z), real part first."""
    h = np.deg2rad(deg) / 2.0
    q = np.zeros(4)
    q[0], q[1 + axis] = np.cos(h), np.sin(h)
    return q


def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def quat_to_mat64(q):
    """[N, 4] (w, x, y, z), any norm -> [N, 3, 3] rotation matrices (the unit quaternion's), as pytorch3d's
    quaternion_to_matrix: entries scaled by 2 / |q|^2."""
    w, x, y, z = q.T
    s = 2.0 / (q * q).sum(1)
    return np.stack([1 - s * (y * y + z * z), s * (x * y - w * z), s * (x * z + w * y),
                     s * (x * y + w * z), 1 - s * (x * x + z * z), s * (y * z - w * x),
                     s * (x * z - w * y), s * (y * z + w * x), 1 - s * (x * x + y * y)], 1).reshape(-1, 3, 3)


def mat_to_quat64(R):
    """[N, 3, 3] -> ([N, 4], margin [N]) as pytorch3d's matrix_to_quaternion (>= 0.5): of the four candidates
    q_t = (column t of 4 q q^T) / (2 max(2|q_t|, 0.1)), with 2|q_t| = sqrt(1 +- m00 +- m11 +- m22) (0 where the argument
    is not positive), the one of the first largest |q_t|; no sign standardisation.  margin: the gap between the two
    largest 2|q_t| (the sign of the result flips between candidates whose components differ in sign)."""
    m = R.reshape(-1, 9)
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = m.T
    arg = np.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], 1)
    with np.errstate(invalid="ignore"):
        qa = np.where(arg > 0, np.sqrt(np.maximum(arg, 0)), 0.0)
    cols = np.stack([
        np.stack([qa[:, 0] ** 2, m21 - m12, m02 - m20, m10 - m01], 1),
        np.stack([m21 - m12, qa[:, 1] ** 2, m10 + m01, m02 + m20], 1),
        np.stack([m02 - m20, m10 + m01, qa[:, 2] ** 2, m12 + m21], 1),
        np.stack([m10 - m01, m20 + m02, m21 + m12, qa[:, 3] ** 2], 1)], 1)  # [N, candidate, component]
    best = np.argmax(qa, 1)  # first maximum
    n = np.arange(len(m))
    q = cols[n, best] / (2.0 * np.maximum(qa[n, best], 0.1))[:, None]
    top = np.sort(qa, 1)
    return q, top[:, 3] - top[:, 2]


# ------------------------------------------------------------------------------------------------ geometries
def _geometries(b, rng):
    """[(family, raw quaternion, proj_ctr target (u, v) or None, pre-clamp depth or None, size logits or None, conf logit
    or None)] of image b; None: drawn at random when the maps are filled."""
    _, _, W, H = CAMERAS[b]
    K = K32[b].astype(np.float64).reshape(3, 3)
    pp = (K[0, 2], K[1, 2])
    out = []
    qs = [np.array([1.0, 0, 0, 0])]
    for a in (0, 45, -45, 90, -90, 180, -180):
        for e in (0, 1e-4, -1e-4):
            qs.append(_axis_quat(1, a + e))
    for _ in range(10):
        qs.append(_qmul(_qmul(_axis_quat(1, rng.uniform(-180, 180)), _axis_quat(0, rng.uniform(-30, 30))),
                        _axis_quat(2, rng.uniform(-30, 30))))
    rand = [v / np.linalg.norm(v) for v in rng.standard_normal((10, 4))]
    qs += rand
    for base in ((1, 0, 1, 0), (1, 1, 0, 0), (1, 0, 0, 1), (0, 1, 1, 0), (0, 1, 0, 1), (0, 0, 1, 1), (1, 1, 1, 1)):
        for d in (0.0, 3e-7, -1e-4, 2e-3):
            v = np.array(base, np.float64)
            v[np.nonzero(v)[0][-1]] += d
            qs.append(v)
    for s in (1e-8, 1e-6, 1e-3, 1e3, 1e6):
        qs += [v * s for v in rand[:4]]
    for i, q in enumerate(qs):
        uv = pp if i % 2 == 0 else None
        out += [("rotation", q, uv, None, None, None), ("rotation", -q, uv, None, None, None)]
    out += [("zero_quat", np.zeros(4), uv, None, None, None) for uv in (pp, None)]

    pts = [pp, (0, 0), (W, 0), (0, H), (W, H), (W / 2, 0), (W / 2, H), (0, H / 2), (W, H / 2), (-W, -H), (2 * W, -H),
           (-W, 2 * H), (2 * W, 2 * H), (-W, pp[1]), (2 * W, pp[1]), (pp[0], -H), (pp[0], 2 * H)]
    for uv in pts:
        out += [("ray", rand[len(out) % 10], uv, None, None, None), ("ray", _axis_quat(1, 90), uv, None, None, None)]

    for alpha in (60, 70, 80):
        for phi in (0, 45, 90, 135, 180, 270):
            d = np.array([np.sin(np.deg2rad(alpha)) * np.cos(np.deg2rad(phi)),
                          np.sin(np.deg2rad(alpha)) * np.sin(np.deg2rad(phi)), np.cos(np.deg2rad(alpha))])
            p = K @ d
            out.append(("extreme", rand[(alpha + phi) % 10], (p[0] / p[2], p[1] / p[2]), None, None, None))

    if b == 2:  # the fx != fy camera
        lo, hi = MIN_DEPTH, MAX_DEPTH
        targets = [lo, hi, np.nextafter(lo, np.float32(0)), np.nextafter(lo, np.float32(1e9)),
                   np.nextafter(hi, np.float32(0)), np.nextafter(hi, np.float32(1e9)), lo * 0.5, lo * 1e-3, hi * 2,
                   hi * 1e4, 0.0, -3.0, 17.25]
        for t in targets:
            out += [("depth", rand[0], None, float(t), None, None), ("depth", rand[1], None, float(t), None, None)]

    L = (0.0, 1.0, -1.0, 8.0, -8.0, SAT, -SAT)
    for i in range(10):
        out.append(("size", rand[i], None, None, (L[i % 7], L[(i + 3) % 7], L[(i + 5) % 7]), None))
    return out


def _slots(rng):
    """(level, pixel) of one image: levels in turn, each level's last row and last column first."""
    order = []
    for h, w in LEVEL_HW:
        pix = rng.permutation(h * w)
        edge = (pix // w == h - 1) | (pix % w == w - 1)
        order.append(np.concatenate([pix[edge], pix[~edge]]))
    return [(l, int(o[k])) for k in range(max(map(len, order))) for l, o in enumerate(order) if k < len(o)]


def location(l, pix, half):
    """Feature location (x, y) of pixel `pix` at level l, float32 as the kernel computes it."""
    w, st = LEVEL_HW[l][1], STRIDES[l]
    lx, ly = np.float32(pix % w * st), np.float32(pix // w * st)
    if half:
        lx, ly = lx + np.float32(st // 2), ly + np.float32(st // 2)
    return lx, ly


def inv_K64(b):
    return np.linalg.inv(K32[b].astype(np.float64).reshape(3, 3))


def build(cfg, seed=0):
    """detect_cases.Case of the 3 cameras under configuration `cfg` (see CONFIGS) with the families above; attributes
    added: cfg, K [3, 9] float32, canon [NC, 3], rec: dict of record arrays b, l, pix, c, fam, sorted by (b, l, index)."""
    case = D.Case(C=NC, level_hw=LEVEL_HW, strides=STRIDES, B=len(CAMERAS), class_agnostic=cfg["agnostic"])
    case.cfg, case.K, case.canon = cfg, K32, CANON
    case.out_cap = 1024  # every 2-D score is 1.0: the post-NMS top-k keeps every NMS survivor, and all are written
    C3 = case.C3
    rng = np.random.default_rng(seed)
    B = case.B
    for l in range(5):
        n = case.cls[l].shape[1]
        case.cls[l][..., NC:] = np.nan                                    # row padding
        case.cls[l][..., NC:NC + 4] = rng.normal(0, 2, (B, n, 4))         # attribute logits, speed
        case.box[l][..., 0:4] = rng.uniform(0.25, 60.0, (B, n, 4))
        case.box[l][..., 4] = rng.normal(0, 1, (B, n))
        case.box[l][..., 5:] = np.nan
        case.b3d[l][...] = np.nan
        case.b3d[l][..., :11 * C3] = rng.normal(0, 3, (B, n, 11 * C3))
    rec = dict(b=[], l=[], pix=[], c=[], fam=[])
    k = 0
    for b in range(B):
        iK = inv_K64(b)
        _, _, W, H = CAMERAS[b]
        geoms = _geometries(b, rng)
        per_pixel = 1 if C3 == 1 else 3
        slots = _slots(rng)
        assert len(slots) * per_pixel >= len(geoms)
        for i, (fam, q, uv, depth, size, conf) in enumerate(geoms):
            l, pix = slots[i // per_pixel]
            j = i % per_pixel
            classes = (pix % NC, (pix + 5) % NC) if C3 == 1 else ((pix + 3 * j) % NC,)
            col = 0 if C3 == 1 else classes[0]
            lx, ly = location(l, pix, cfg["half"])
            if uv is None:
                uv = rng.uniform((0, 0), (W, H))
            if depth is None:
                depth = rng.uniform(2.0, 60.0)
            logit = depth
            if cfg["scale_depth"]:
                logit *= np.sqrt(iK[0, 0] ** 2 + iK[1, 1] ** 2) * np.float64(DEPTH_FACTOR)
            if cfg["distance"]:
                logit *= np.linalg.norm(iK @ np.array([lx, ly, 1.0]))
            size = rng.normal(0, 0.7, 3) if size is None else size
            conf = rng.uniform(-5, 5) if conf is None else conf
            vals = [*q, uv[0] - np.float64(lx), uv[1] - np.float64(ly), logit, *size, conf]
            for t, v in enumerate(vals):
                case.b3d[l][b, pix, t * C3 + col] = v
            case.box[l][b, pix, 4] = SAT
            case.cls[l][b, pix, NC:NC + 3] = ATTR_PATTERNS[k % len(ATTR_PATTERNS)]
            case.cls[l][b, pix, NC + 3] = SPEEDS[k % len(SPEEDS)]
            k += 1
            for c in classes:
                case.cls[l][b, pix, c] = SAT
                for key, v in zip(("b", "l", "pix", "c", "fam"), (b, l, pix, c, fam)):
                    rec[key].append(v)
    rec = {key: np.array(v) for key, v in rec.items()}
    rec["index"] = rec["pix"] * NC + rec["c"]
    order = np.lexsort((rec["index"], rec["l"], rec["b"]))
    case.rec = {key: v[order] for key, v in rec.items()}
    for b in range(B):
        for l in range(5):
            assert ((case.rec["b"] == b) & (case.rec["l"] == l)).sum() <= case.topk
    return case


# ------------------------------------------------------------------------------------------------ float64 reference
def box3d_ref64(case):
    """Float64 restatement of the decode of every record of `case`: dict(det [N, 24] float64 in the Det layout (integer
    words as values), depth_pre [N] (before the clamp), clamped [N] bool (the pre-clamp depth is beyond a bound by more
    than DEPTH_REL), margin [N] (mat_to_quat64's; inf where no matrix_to_quaternion runs), canon [N, 3], fam [N])."""
    cfg, r = case.cfg, case.rec
    N, C3 = len(r["b"]), case.C3
    col = np.zeros(N, int) if C3 == 1 else r["c"]
    g = np.array([case.b3d[l][b, p, np.arange(11) * C3 + c] for b, l, p, c in zip(r["b"], r["l"], r["pix"], col)],
                 np.float64).reshape(N, 11)
    reg = np.array([case.box[l][b, p, 0:4] for b, l, p in zip(r["b"], r["l"], r["pix"])], np.float64).reshape(N, 4)
    extra = np.array([case.cls[l][b, p, NC:NC + 4] for b, l, p in zip(r["b"], r["l"], r["pix"])]).reshape(N, 4)
    loc = np.array([location(l, p, cfg["half"]) for l, p in zip(r["l"], r["pix"])], np.float64).reshape(N, 2)
    iK = np.stack([inv_K64(b) for b in range(case.B)])[r["b"]]
    canon = case.canon[r["c"]].astype(np.float64)

    det = np.zeros((N, 24))
    det[:, 0:2] = loc - reg[:, 0:2]
    det[:, 2:4] = loc + reg[:, 2:4]
    det[:, 4] = 1.0  # sqrt(sigmoid(SAT) * sigmoid(SAT))
    det[:, 6], det[:, 7], det[:, 18:20], det[:, 20] = r["c"], r["l"], loc, r["index"]
    if cfg["nuscenes"]:
        det[:, 21] = np.argmax(extra[:, 0:3], 1)  # first maximum, like torch.argmax
        det[:, 22] = extra[:, 3]
    margin = np.full(N, np.inf)
    depth = np.zeros(N)
    if not cfg["box3d_on"]:  # core.py: 2-D detector, the 3-D fields are placeholders
        det[:, 5] = det[:, 4]
        det[:, 8] = 1.0
        det[:, 12:14] = loc
        return dict(det=det, depth_pre=depth, clamped=np.zeros(N, bool), margin=margin, canon=canon, fam=r["fam"])

    with np.errstate(invalid="ignore", divide="ignore"):
        q = g[:, 0:4] / np.maximum(np.linalg.norm(g[:, 0:4], axis=1), 1e-7)[:, None]
        q = q / np.linalg.norm(q, axis=1)[:, None]
        depth = g[:, 6].copy()
        if cfg["scale_depth"]:
            depth /= np.sqrt(iK[:, 0, 0] ** 2 + iK[:, 1, 1] ** 2) * np.float64(DEPTH_FACTOR)
        if cfg["distance"]:
            ray = np.einsum("nij,nj->ni", iK, np.concatenate([loc, np.ones((N, 1))], 1))
            depth /= np.maximum(np.linalg.norm(ray, axis=1), 1e-7)
        lo, hi = np.float64(MIN_DEPTH), np.float64(MAX_DEPTH)
        clamped = (depth < lo * (1 - DEPTH_REL)) | (depth > hi * (1 + DEPTH_REL))
        proj = g[:, 4:6] + loc
        if cfg["allocentric"]:
            ray = np.einsum("nij,nj->ni", iK, np.concatenate([proj, np.ones((N, 1))], 1))
            z = ray / np.linalg.norm(ray, axis=1)[:, None]
            y = np.array([0.0, 1.0, 0.0]) - z[:, 1:2] * z
            y /= np.linalg.norm(y, axis=1)[:, None]
            x = np.cross(y, z)
            R_l2g = np.stack([x, y, z], 2)  # columns x, y, z
            q, margin = mat_to_quat64(R_l2g @ quat_to_mat64(q))
            n = np.linalg.norm(q, axis=1)
            q = np.where((np.abs(n - 1) > 1e-3 + 1e-5)[:, None], q / np.maximum(n, 1e-7)[:, None], q)
    det[:, 5] = 1.0 / (1.0 + np.exp(-g[:, 10]))
    det[:, 8:12] = q
    det[:, 12:14] = proj
    det[:, 14] = np.clip(depth, lo, hi)
    det[:, 15:18] = (np.tanh(g[:, 7:10]) + 1.0) * canon
    return dict(det=det, depth_pre=depth, clamped=clamped, margin=margin, canon=canon, fam=r["fam"])


# ------------------------------------------------------------------------------------------------ bounds
EXACT_WORDS = dict(box=slice(0, 4), score=slice(4, 5), cls=slice(6, 7), level=slice(7, 8), proj_ctr=slice(12, 14),
                   loc=slice(18, 20), index=slice(20, 21), attr=slice(21, 22), speed=slice(22, 23))
INT_WORDS = (6, 7, 20, 21)
FIELDS = tuple(EXACT_WORDS) + ("depth", "score3d", "size", "quat_norm", "quat_rot", "quat_sign", "finite")


def _expected_words(ref):
    """Reference Det rows as the float32 / int32 words the kernel must write bit for bit, [N, 24] uint32."""
    det = ref["det"]
    w = det.astype(np.float32).view(np.uint32)
    for k in INT_WORDS:
        w[:, k] = det[:, k].astype(np.int32).view(np.uint32)
    return w


def compare(got, ref, box3d_on=True):
    """Holds `got` ([N, 24] float32 Det rows in the reference's record order) to the reference.  Returns
    (worst, fails): worst[(family, field)] = largest error (|delta| for bit-exact fields and depth at a clamp, relative for
    depth, ulps for score3d, |delta| / canon for size, |norm - 1|, rotation distance min(|q - r|, |q + r|) (about half the
    angle), 1 where q . r <= 0 away from a candidate tie), fails = [(family, field, records out of bound, worst)].  The `extreme` family's rotation
    distance is reported, not bounded; the `zero_quat` family's quaternion is NaN in the reference and is not compared."""
    got = np.ascontiguousarray(got, np.float32)
    gw, ew = got.view(np.uint32), _expected_words(ref)
    det = ref["det"]
    g64 = got.astype(np.float64)
    for k in INT_WORDS:
        g64[:, k] = gw[:, k].view(np.int32)
    err, bad = {}, {}
    with np.errstate(invalid="ignore", over="ignore"):
        for f, s in EXACT_WORDS.items():
            bad[f] = (gw[:, s] != ew[:, s]).any(1)
            err[f] = np.where(bad[f], np.nan_to_num(np.abs(g64[:, s] - det[:, s]).max(1), nan=np.inf), 0.0)
        d, dr = g64[:, 14], det[:, 14]
        if box3d_on:
            at = ref["clamped"]
            rel = np.abs(d - dr) / np.abs(dr)
            err["depth"] = np.where(at, np.abs(d - np.float32(dr)), rel)
            bad["depth"] = np.where(at, gw[:, 14] != ew[:, 14], ~(rel <= DEPTH_REL))
            ulp = np.spacing(det[:, 5].astype(np.float32)).astype(np.float64)
            err["score3d"] = np.abs(g64[:, 5] - det[:, 5]) / ulp
            bad["score3d"] = ~(err["score3d"] <= SCORE3D_ULPS)
            err["size"] = (np.abs(g64[:, 15:18] - det[:, 15:18]) / ref["canon"]).max(1)
            bad["size"] = ~(err["size"] <= SIZE_REL_CANON)
            q, r = g64[:, 8:12], det[:, 8:12]
            err["quat_norm"] = np.abs(np.linalg.norm(q, axis=1) - 1)
            err["quat_rot"] = np.minimum(np.linalg.norm(q - r, axis=1), np.linalg.norm(q + r, axis=1))
            pinned = ref["margin"] > SIGN_MARGIN
            err["quat_sign"] = np.where(pinned, ((q * r).sum(1) <= 0).astype(float), 0.0)
            nan_q = ref["fam"] == "zero_quat"
            extreme = ref["fam"] == "extreme"
            bad["quat_norm"] = ~nan_q & ~(err["quat_norm"] <= QUAT_NORM)
            bad["quat_rot"] = ~nan_q & ~extreme & ~(err["quat_rot"] <= QUAT_ROT)
            bad["quat_sign"] = ~nan_q & (err["quat_sign"] > 0)
            for f in ("quat_norm", "quat_rot", "quat_sign"):
                err[f] = np.where(nan_q, 0.0, err[f])
        else:  # 2-D detector: every placeholder is exact
            for f, s in (("depth", slice(14, 15)), ("score3d", slice(5, 6)), ("size", slice(15, 18)),
                         ("quat_norm", slice(8, 12))):
                bad[f] = (gw[:, s] != ew[:, s]).any(1)
                err[f] = bad[f].astype(float)
        other = np.ones(24, bool)
        other[8:12] = False
        other[23] = False
        nonfinite = ~np.isfinite(got[:, other]).all(1)
        if box3d_on:
            nonfinite |= (ref["fam"] != "zero_quat") & ~np.isfinite(got[:, 8:12]).all(1)
        err["finite"], bad["finite"] = nonfinite.astype(float), nonfinite
    worst, fails = {}, []
    fam = ref["fam"]
    for name in FAMILIES:
        m = fam == name
        if not m.any():
            continue
        for f in err:
            worst[(name, f)] = float(np.nan_to_num(err[f][m], nan=np.inf).max())
            nb = int(bad[f][m].sum())
            if nb:
                fails.append((name, f, nb, worst[(name, f)]))
    return worst, fails
