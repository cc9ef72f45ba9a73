"""CPU pins of the 3-D box decode bounds (tests/box3d_cases.py, tests/test_box3d_decode_gpu.py).

`decode32` restates decode_one (csrc/decode.cu) in float32 numpy, in its operation order (every operation rounded; the
device may contract some into FMAs).  It meets every bound of `box3d_cases.compare` on every family of every
configuration, so the bounds can be met in float32.  Each wrong variant of it breaks a bound on at least one named family,
so the families can tell it apart from the right decode.  box3d_ref64 itself agrees with the float32 oracle
(oracle/dd3d_oracle.py, pinned to the reference goldens)."""
import types

import numpy as np
import pytest
import torch

import box3d_cases as B3
from oracle import dd3d_oracle as O

f32 = np.float32
VARIANTS = {  # variant: (configuration, family, field) where it must break the bound
    "obj_l2g": ("allocentric-scale_depth", "ray", "quat_rot"),            # R_obj @ R_l2g
    "rows": ("allocentric-scale_depth", "ray", "quat_rot"),               # [x y z] as rows of R_l2g
    "last_max": ("nuscenes", "rotation", "attr"),                         # last maximum in both argmaxes
    "pixel_size_fx": ("allocentric-scale_depth", "depth", "depth"),       # pixel_size = sqrt(2) / fx
    "clamp_first": ("allocentric-scale_depth", "depth", "depth"),         # clamp, then the focal scaling
    "distance_at_proj": ("distance-allocentric", "rotation", "depth"),    # PREDICT_DISTANCE ray through proj_ctr
    "whl": ("allocentric-scale_depth", "size", "size"),                   # canonical (L, W, H) for (W, L, H)
    "agnostic_col_c": ("agnostic", "rotation", "quat_rot"),               # CLASS_AGNOSTIC_BOX3D reading column c
    "no_half": ("half-allocentric-scale_depth", "rotation", "loc"),       # FEATURE_LOCATIONS_OFFSET half dropped
}


def _gather(maps, pitch, rec, chans):
    """chans [N, k] channel offsets from each record's map row start, read from the flat [B][H*W][pitch] level arrays
    (an offset past the row reads the next pixel's row, as device memory would; past the last row, NaN)."""
    out = np.empty(chans.shape, f32)
    for l in range(5):
        m = rec["l"] == l
        hw = maps[l].shape[1]
        base = (rec["b"][m] * hw + rec["pix"][m]) * pitch
        flat = np.concatenate([maps[l].reshape(-1), np.full(2 * pitch, np.nan, f32)])
        out[m] = flat[base[:, None] + chans[m]]
    return out


def _sigmoid32(x):
    with np.errstate(over="ignore"):
        return f32(1) / (f32(1) + np.exp(-x))


def _matmul32(A, B):
    """[N, 3, 3] @ [N, 3, 3], each entry ((a0 b0 + a1 b1) + a2 b2) in float32."""
    return (A[:, :, 0, None] * B[:, None, 0, :] + A[:, :, 1, None] * B[:, None, 1, :]) + A[:, :, 2, None] * B[:, None, 2, :]


def _apply(M, u, v):
    """M @ (u, v, 1) for [N, 3, 3] float32 M."""
    return [(M[:, i, 0] * u + M[:, i, 1] * v) + M[:, i, 2] for i in range(3)]


def _norm4(q):
    return np.sqrt(((q[:, 0] * q[:, 0] + q[:, 1] * q[:, 1]) + q[:, 2] * q[:, 2]) + q[:, 3] * q[:, 3])


def _quat_to_mat32(q):
    r, i, j, k = q.T
    two_s = f32(2) / (((r * r + i * i) + j * j) + k * k)
    one = f32(1)
    return np.stack([one - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r),
                     two_s * (i * j + k * r), one - two_s * (i * i + k * k), two_s * (j * k - i * r),
                     two_s * (i * k - j * r), two_s * (j * k + i * r), one - two_s * (i * i + j * j)], 1).reshape(-1, 3, 3)


def _mat_to_quat32(R, last_max):
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = R.reshape(-1, 9).T
    one = f32(1)
    arg = np.stack([((one + m00) + m11) + m22, ((one + m00) - m11) - m22, ((one - m00) + m11) - m22,
                    ((one - m00) - m11) + m22], 1)
    qa = np.where(arg > 0, np.sqrt(np.maximum(arg, f32(0))), f32(0))
    best = 3 - np.argmax(qa[:, ::-1], 1) if last_max else np.argmax(qa, 1)
    sq = qa * qa
    cols = np.stack([np.stack([sq[:, 0], m21 - m12, m02 - m20, m10 - m01], 1),
                     np.stack([m21 - m12, sq[:, 1], m10 + m01, m02 + m20], 1),
                     np.stack([m02 - m20, m10 + m01, sq[:, 2], m12 + m21], 1),
                     np.stack([m10 - m01, m20 + m02, m21 + m12, sq[:, 3]], 1)], 1)
    n = np.arange(len(qa))
    return cols[n, best] / (f32(2) * np.maximum(qa[n, best], f32(0.1)))[:, None]


def decode32(case, variant=None):
    """decode_one of every record of `case` in float32 (record order of case.rec) -> [N, 24] float32 Det rows."""
    cfg, r = case.cfg, case.rec
    N, C3, C = len(r["b"]), case.C3, case.C
    half = cfg["half"] and variant != "no_half"
    loc = np.array([B3.location(l, p, half) for l, p in zip(r["l"], r["pix"])], f32).reshape(N, 2)
    lx, ly = loc[:, 0], loc[:, 1]
    det = np.zeros((N, 24), f32)
    di = det.view(np.int32)
    reg = _gather(case.box, 16, r, np.tile(np.arange(5), (N, 1)))
    det[:, 0], det[:, 1], det[:, 2], det[:, 3] = lx - reg[:, 0], ly - reg[:, 1], lx + reg[:, 2], ly + reg[:, 3]
    cls_logit = _gather(case.cls, case.cls_pitch, r, r["c"][:, None])[:, 0]
    score = np.sqrt(_sigmoid32(cls_logit) * _sigmoid32(reg[:, 4]))
    det[:, 4] = score
    di[:, 6], di[:, 7], di[:, 20] = r["c"], r["l"], r["index"]
    det[:, 18:20] = loc
    if cfg["nuscenes"]:
        a = _gather(case.cls, case.cls_pitch, r, np.tile(C + np.arange(4), (N, 1)))
        di[:, 21] = 2 - np.argmax(a[:, 2::-1], 1) if variant == "last_max" else np.argmax(a[:, 0:3], 1)
        det[:, 22] = a[:, 3]
    if not cfg["box3d_on"]:
        det[:, 5], det[:, 8], det[:, 12:14] = score, 1, loc
        return det
    col = r["c"] if (C3 > 1 or variant == "agnostic_col_c") else np.zeros(N, int)
    g = _gather(case.b3d, case.b3d_pitch, r, np.arange(11)[None, :] * C3 + col[:, None])
    det[:, 5] = score * _sigmoid32(g[:, 10])
    with np.errstate(invalid="ignore", divide="ignore"):
        q = g[:, 0:4]
        q = q / np.maximum(_norm4(q), f32(1e-7))[:, None]
        q = q / _norm4(q)[:, None]
        iK = np.stack([np.linalg.inv(case.K[b].astype(np.float64).reshape(3, 3)).astype(f32) for b in range(case.B)])
        iK = iK[r["b"]]
        depth = g[:, 6]
        lo, hi = B3.MIN_DEPTH, B3.MAX_DEPTH
        if variant == "clamp_first":
            depth = np.minimum(np.maximum(depth, lo), hi)
        if cfg["scale_depth"]:
            fy = iK[:, 0, 0] if variant == "pixel_size_fx" else iK[:, 1, 1]
            depth = depth / (np.sqrt(iK[:, 0, 0] * iK[:, 0, 0] + fy * fy) * B3.DEPTH_FACTOR)
        pcx, pcy = g[:, 4] + lx, g[:, 5] + ly
        if cfg["distance"]:
            ray = _apply(iK, pcx, pcy) if variant == "distance_at_proj" else _apply(iK, lx, ly)
            depth = depth / np.maximum(np.sqrt((ray[0] * ray[0] + ray[1] * ray[1]) + ray[2] * ray[2]), f32(1e-7))
        depth = np.minimum(np.maximum(depth, lo), hi)
        if cfg["allocentric"]:
            Ro = _quat_to_mat32(q)
            ray = _apply(iK, pcx, pcy)
            rn = np.sqrt((ray[0] * ray[0] + ray[1] * ray[1]) + ray[2] * ray[2])
            z = np.stack([ray[0] / rn, ray[1] / rn, ray[2] / rn], 1)
            y = np.stack([f32(0) - z[:, 1] * z[:, 0], f32(1) - z[:, 1] * z[:, 1], f32(0) - z[:, 1] * z[:, 2]], 1)
            y = y / np.sqrt((y[:, 0] * y[:, 0] + y[:, 1] * y[:, 1]) + y[:, 2] * y[:, 2])[:, None]
            x = np.stack([y[:, 1] * z[:, 2] - y[:, 2] * z[:, 1], y[:, 2] * z[:, 0] - y[:, 0] * z[:, 2],
                          y[:, 0] * z[:, 1] - y[:, 1] * z[:, 0]], 1)
            l2g = np.stack([x, y, z], 2)
            R = {"obj_l2g": lambda: _matmul32(Ro, l2g), "rows": lambda: _matmul32(l2g.transpose(0, 2, 1), Ro)}.get(
                variant, lambda: _matmul32(l2g, Ro))()
            q = _mat_to_quat32(R, variant == "last_max")
            qn = _norm4(q)
            fix = np.abs(qn - f32(1)) > f32(1e-3 + 1e-5)
            q = np.where(fix[:, None], q / np.maximum(qn, f32(1e-7))[:, None], q)
    det[:, 8:12] = q
    det[:, 12], det[:, 13] = pcx, pcy
    det[:, 14] = depth
    canon = case.canon[:, [1, 0, 2]] if variant == "whl" else case.canon
    det[:, 15:18] = (np.tanh(g[:, 7:10]) + f32(1)) * canon[r["c"]]
    return det


_cases = {}


def _case(name):
    if name not in _cases:
        case = B3.build(B3.CONFIGS[name])
        _cases[name] = (case, B3.box3d_ref64(case))
    return _cases[name]


@pytest.mark.parametrize("name", list(B3.CONFIGS))
def test_float32_restatement_meets_the_bounds(name):
    case, ref = _case(name)
    worst, fails = B3.compare(decode32(case), ref, case.cfg["box3d_on"])
    assert not fails, fails
    if case.cfg["box3d_on"]:
        print(name, {k: f"{v:.2e}" for k, v in worst.items() if k[1] in ("quat_rot", "depth", "size", "score3d")})


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_wrong_variant_breaks_a_named_family(variant):
    name, family, field = VARIANTS[variant]
    case, ref = _case(name)
    _, fails = B3.compare(decode32(case, variant), ref, case.cfg["box3d_on"])
    print(variant, "breaks", name, [f[:3] for f in fails])
    assert any(f[0] == family and f[1] == field for f in fails), (variant, fails)


def test_cases_are_built_as_documented():
    """Exactly the records are candidates, each at score 1.0; each level's last row and column hold one; every family is
    on every camera (depth on the synthetic one); the row padding is NaN; a record's 3-D column differs from the other
    class columns of its pixel; the depth family reaches both bounds."""
    for name in ("allocentric-scale_depth", "agnostic"):
        case, _ = _case(name)
        r = case.rec
        for l in range(5):
            for b in range(case.B):
                s, t = case.level_scores(b, l)
                m = (r["b"] == b) & (r["l"] == l)
                cand = np.nonzero(t > case.thresh)
                assert np.array_equal(np.sort(cand[0] * case.C + cand[1]), r["index"][m])
                assert (s[t > case.thresh] == 1.0).all()
                h, w = B3.LEVEL_HW[l]
                pix = r["pix"][m]
                assert ((pix // w) == h - 1).any() and ((pix % w) == w - 1).any(), (b, l)
        for fam in B3.FAMILIES:
            assert set(r["b"][r["fam"] == fam]) == ({2} if fam == "depth" else {0, 1, 2}), fam
        for l in range(5):
            assert np.isnan(case.b3d[l][..., 11 * case.C3:]).all() and np.isnan(case.cls[l][..., case.C + 4:]).all()
        if case.C3 > 1:  # a record's column differs from every other class column of its pixel
            for b, l, p, c in zip(r["b"], r["l"], r["pix"], r["c"]):
                cols = case.b3d[l][b, p, :11 * case.C3].reshape(11, case.C3)
                other = np.delete(cols, c, 1)
                cand = np.isin(np.delete(np.arange(case.C), c), r["c"][(r["b"] == b) & (r["l"] == l) & (r["pix"] == p)])
                assert (other[:, ~cand] != cols[:, c:c + 1]).all()  # non-candidate columns: every value
                assert (other[:, cand] != cols[:, c:c + 1]).any(0).all()  # candidate columns: some value
    for name, rtol in (("allocentric", 0), ("distance-allocentric-scale_depth", 1.2e-7)):  # exact / within an ulp
        case, ref = _case(name)
        d = ref["depth_pre"][ref["fam"] == "depth"]
        for bound in (B3.MIN_DEPTH, B3.MAX_DEPTH):
            assert (np.abs(d - bound) <= rtol * bound).sum() >= 2, (name, bound)
        assert ref["clamped"].sum() >= 10


def test_principal_point_rays_keep_the_rotation():
    """At the principal point the ray is the optical axis and R_l2g the identity: box3d_ref64's egocentric quaternion is
    the normalised raw output, up to sign and float64 rounding of the float32 proj_ctr; where the matrix_to_quaternion
    candidates are not near a tie the sign is the one making the largest component positive."""
    case, ref = _case("allocentric-scale_depth")
    r = case.rec
    K = case.K[r["b"]].astype(np.float64)
    m = (ref["fam"] == "rotation") & (np.abs(ref["det"][:, 12] - K[:, 2]) < 1e-3) & (np.abs(ref["det"][:, 13] - K[:, 5]) < 1e-3)
    assert m.sum() > 100
    raw = np.array([case.b3d[l][b, p, np.arange(4) * case.C3 + c] for b, l, p, c in
                    zip(r["b"][m], r["l"][m], r["pix"][m], r["c"][m])], np.float64)
    raw /= np.linalg.norm(raw, axis=1)[:, None]
    q = ref["det"][m, 8:12]
    assert np.minimum(np.abs(q - raw).max(1), np.abs(q + raw).max(1)).max() < 1e-5
    pinned = ref["margin"][m] > B3.SIGN_MARGIN
    big = np.argmax(np.abs(raw), 1)
    s = np.sign(raw[np.arange(len(raw)), big])
    assert np.abs(q[pinned] - (s[:, None] * raw)[pinned]).max() < 1e-5


@pytest.mark.parametrize("name", ["allocentric-scale_depth", "half-distance-allocentric-scale_depth", "distance",
                                  "agnostic-half-distance"])
def test_reference_agrees_with_the_float32_oracle(name):
    """box3d_ref64 against predictions_to_boxes3d of the float32 torch oracle (pinned to the reference goldens), image by
    image: quaternions within 1e-5 (same sign where the candidates are not near a tie), proj_ctr exactly, depth and size
    to float32 rounding.  The zero quaternion and the extreme rays are left out (NaN; float32 Gram-Schmidt error)."""
    case, ref = _case(name)
    cfg, r = case.cfg, case.rec
    cfg3d = types.SimpleNamespace(SCALE_DEPTH_BY_FOCAL_LENGTHS=cfg["scale_depth"], PREDICT_DISTANCE=cfg["distance"],
                                  PREDICT_ALLOCENTRIC_ROT=cfg["allocentric"],
                                  SCALE_DEPTH_BY_FOCAL_LENGTHS_FACTOR=float(B3.DEPTH_FACTOR),
                                  MIN_DEPTH=float(B3.MIN_DEPTH), MAX_DEPTH=float(B3.MAX_DEPTH))
    col = np.zeros(len(r["b"]), int) if case.C3 == 1 else r["c"]
    keep = ~np.isin(ref["fam"], ("zero_quat", "extreme"))
    for b in range(case.B):
        m = keep & (r["b"] == b)
        g = torch.tensor(np.array([case.b3d[l][b, p, np.arange(11) * case.C3 + c] for l, p, c in
                                   zip(r["l"][m], r["pix"][m], col[m])]))
        loc = torch.tensor(ref["det"][m, 18:20], dtype=torch.float32)
        iK = torch.linalg.inv(torch.tensor(case.K[b].reshape(3, 3)))
        o = O.predictions_to_boxes3d(g[:, 0:4], g[:, 4:6], g[:, 6], g[:, 7:10], loc, iK,
                                     torch.tensor(case.canon[r["c"][m]]), cfg3d)
        want = ref["det"][m]
        q, rq = o["quat"].double().numpy(), want[:, 8:12]
        assert np.minimum(np.abs(q - rq).max(1), np.abs(q + rq).max(1)).max() < 1e-5
        pinned = ref["margin"][m] > B3.SIGN_MARGIN
        assert np.abs(q - rq)[pinned].max() < 1e-5
        assert np.array_equal(o["proj_ctr"].numpy(), want[:, 12:14].astype(np.float32))
        np.testing.assert_allclose(o["depth"].double().numpy(), want[:, 14], rtol=2e-6)
        np.testing.assert_allclose(o["size"].double().numpy(), want[:, 15:18], rtol=0, atol=2e-6 * 5)
