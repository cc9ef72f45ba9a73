"""CPU pins of the rectangle families in bev_geom_cases.py: the two float64 references agree on every family and with the
families' closed forms, and a float32 restatement of detectron2's edge-intersection IoU -- parallel edges detected by an
absolute |det| <= 1e-14, the rule csrc/bev_geom.cuh followed before it clipped in the first box's frame -- breaks the
1e-5 bound the GPU tests hold the kernel to on the aligned and touching families (so those families can tell the two
apart)."""
import numpy as np
import pytest

import bev_geom_cases as G

N = 300
BOUND = 1e-5
f32 = np.float32


# ------------------------------------------------------------------------------------------------ float32 absolute-det rule
def _cross(a, b):
    return a[0] * b[1] - a[1] * b[0]


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1]


def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1])


def _vertices32(x, y, w, h, a):
    th = a * f32(0.01745329251994329577)
    c, s = np.cos(th) * f32(0.5), np.sin(th) * f32(0.5)
    p0 = (x + s * h + c * w, y + c * h - s * w)
    p1 = (x - s * h + c * w, y - c * h - s * w)
    return [p0, p1, (f32(2) * x - p0[0], f32(2) * y - p0[1]), (f32(2) * x - p1[0], f32(2) * y - p1[1])]


def absolute_det_iou32(b1, b2):
    """detectron2 single_box_iou_rotated in float32 without FMA contraction (every product rounded)."""
    b1, b2 = [f32(v) for v in b1], [f32(v) for v in b2]
    a1, a2 = b1[2] * b1[3], b2[2] * b2[3]
    if a1 < f32(1e-14) or a2 < f32(1e-14):
        return 0.0
    sx, sy = (b1[0] + b2[0]) * f32(0.5), (b1[1] + b2[1]) * f32(0.5)
    p1 = _vertices32(b1[0] - sx, b1[1] - sy, b1[2], b1[3], b1[4])
    p2 = _vertices32(b2[0] - sx, b2[1] - sy, b2[2], b2[3], b2[4])
    v1 = [_sub(p1[(i + 1) % 4], p1[i]) for i in range(4)]
    v2 = [_sub(p2[(i + 1) % 4], p2[i]) for i in range(4)]
    pts = []
    for i in range(4):
        for j in range(4):
            det = _cross(v2[j], v1[i])
            if abs(det) <= f32(1e-14):
                continue
            v12 = _sub(p2[j], p1[i])
            t1, t2 = _cross(v2[j], v12) / det, _cross(v1[i], v12) / det
            if 0 <= t1 <= 1 and 0 <= t2 <= 1:
                pts.append((p1[i][0] + v1[i][0] * t1, p1[i][1] + v1[i][1] * t1))
    for pa, pb, vb in ((p1, p2, v2), (p2, p1, v1)):
        AB, DA = vb[0], vb[3]
        for q in pa:
            AP = _sub(q, pb[0])
            if 0 <= _dot(AP, AB) <= _dot(AB, AB) and 0 <= -_dot(AP, DA) <= _dot(DA, DA):
                pts.append(q)
    if len(pts) <= 2:
        return 0.0
    # convex_hull_graham + polygon_area
    t = min(range(len(pts)), key=lambda k: (pts[k][1], pts[k][0]))
    q = [_sub(p, pts[t]) for p in pts]
    q[0], q[t] = q[t], q[0]
    dist = [_dot(v, v) for v in q]
    for i in range(2, len(q)):  # insertion sort by polar angle, as the device code
        qi, di, j = q[i], dist[i], i - 1
        while j >= 1:
            tmp = _cross(qi, q[j])
            if not ((di < dist[j]) if abs(tmp) < f32(1e-6) else (tmp > 0)):
                break
            q[j + 1], dist[j + 1] = q[j], dist[j]
            j -= 1
        q[j + 1], dist[j + 1] = qi, di
    k = 1
    while k < len(q) and dist[k] <= f32(1e-8):
        k += 1
    if k == len(q):
        return 0.0
    hull = [q[0], q[k]]
    for i in range(k + 1, len(q)):
        while len(hull) > 1 and _cross(_sub(q[i], hull[-2]), _sub(hull[-1], hull[-2])) >= 0:
            hull.pop()
        hull.append(q[i])
    if len(hull) <= 2:
        return 0.0
    inter = f32(0)
    for i in range(1, len(hull) - 1):
        inter += abs(_cross(_sub(hull[i], hull[0]), _sub(hull[i + 1], hull[0])))
    inter *= f32(0.5)
    return float(inter / (a1 + a2 - inter))


# ------------------------------------------------------------------------------------------------ tests
def _parallel(a, b):
    """Pairs whose angles differ by a multiple of 90 degrees (0 included): every edge of one is parallel to two of the
    other's."""
    d = np.abs(a[:, 4].astype(np.float64) - b[:, 4].astype(np.float64))
    return np.abs(d / 90.0 - np.round(d / 90.0)) < 1e-12


@pytest.mark.parametrize("name", list(G.FAMILIES))
def test_references_agree(name):
    """The oracle's detectron2 restatement and the independent clipper, both float64 on the same float32 rectangles,
    agree to 5e-6 wherever no two edges are exactly parallel.  With exactly parallel edges the oracle's restatement can
    misfire even in float64 (test_oracle_misfires_on_parallel_edges); the clipper matches the closed forms there, so the
    GPU bound is taken against the clipper."""
    a, b, exact = G.family(name, N)
    ref, clip = G.ref_iou(a, b), G.ref_clipper(a, b)
    off = np.abs(ref - clip) > 5e-6
    assert not (off & ~_parallel(a, b)).any(), (name, np.abs(ref - clip)[~_parallel(a, b)].max())
    assert np.abs(clip - G.ref_clipper(b, a)).max() <= 1e-9
    assert ((clip >= 0) & (clip <= 1 + 1e-12)).all()
    if exact is not None:
        # the closed form is of the float64 construction; float32 centres (<= 100 m) move it by ~1e-4 at most
        assert np.abs(clip - exact).max() <= 2e-4, name


def test_oracle_misfires_on_parallel_edges():
    """Why the clipper is the reference of the GPU bound: on exactly parallel edges (here a same-yaw shift at 180 degrees
    and one rectangle written at angle + 180) the oracle's skipped parallel intersections and its `<=` inside tests,
    on float64 rounding noise, drop vertices of the intersection."""
    shift = np.array([[-39.338764, 58.296268, 5.0787554, 2.558219, 180.0]], np.float32)
    moved = shift.copy()
    moved[0, 0] = -41.706585
    turned = np.array([[76.68627, -35.101944, 8.110873, 4.2402754, -89.999]], np.float32)
    turned_back = turned.copy()
    turned_back[0, 4] += np.float32(180.0)
    for a, b, exact in ((shift, moved, (5.0787554 - 2.367821) / (5.0787554 + 2.367821)), (turned, turned_back, 1.0)):
        assert abs(G.ref_clipper(a, b)[0] - exact) < 1e-5
        assert abs(G.ref_iou(a, b)[0] - exact) > 0.1


def test_issue_pair_shares_an_edge():
    a, b, _ = G.family("edge_sharing", 1)
    assert G.ref_iou(a, b)[0] < 1e-6 and G.ref_clipper(a, b)[0] < 1e-6


@pytest.mark.parametrize("name", ["shift_width", "shift_length", "special_angles", "thin_barriers"])
def test_absolute_det_rule_breaks_the_bound(name):
    """Negative control: the same families catch a float32 IoU that tests parallel edges with an absolute threshold."""
    a, b, _ = G.family(name, N)
    ref = G.ref_clipper(a, b)
    got = np.array([absolute_det_iou32(x, y) for x, y in zip(a, b)])
    assert np.abs(got - ref).max() > 1e-3, name
    assert (np.abs(got - ref) > BOUND).sum() >= 3, name
