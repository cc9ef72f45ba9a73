"""Rectangle-pair families for the rotated BEV IoU (csrc/bev_geom.cuh rotated_iou) and their float64 references.

Real detections are yaw-only boxes: duplicates share a yaw (flipped TTA views, overlapping nuScenes cameras) and parked
cars sit side by side, so BEV rectangles with parallel, collinear and touching edges are the common case, not an edge
case.  Each family returns float32 rectangles a, b of shape (n, 5) = (cx, cy, w, h, angle_deg) and, where one exists,
the closed-form IoU of the family (of the float64 construction, before the rectangles are rounded to float32).

Two float64 references of the same float32 rectangles, checked against each other on every family: the oracle's
restatement of detectron2's single_box_iou_rotated (oracle/bev_nms_oracle.py) and an independent Sutherland-Hodgman
polygon clipper."""
import math

import numpy as np

from oracle import bev_nms_oracle as B


# ------------------------------------------------------------------------------------------------ independent clipper
def rect_poly(box):
    return [(x, y) for x, y in B._vertices(tuple(float(v) for v in box))]


def clip_area(subject, clip):
    """Sutherland-Hodgman clipping of convex polygons (independent of the Graham-scan formulation of the oracle)."""
    def area2(p):
        return sum(p[i][0] * p[(i + 1) % len(p)][1] - p[(i + 1) % len(p)][0] * p[i][1] for i in range(len(p)))
    if area2(clip) < 0:
        clip = clip[::-1]
    out = subject
    for i in range(len(clip)):
        a, b = clip[i], clip[(i + 1) % len(clip)]
        inp, out = out, []
        if not inp:
            break

        def inside(p):
            return (b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0]) >= 0

        def inter(p, q):
            d1 = (b[0] - a[0]) * (p[1] - a[1]) - (b[1] - a[1]) * (p[0] - a[0])
            d2 = (b[0] - a[0]) * (q[1] - a[1]) - (b[1] - a[1]) * (q[0] - a[0])
            t = d1 / (d1 - d2)
            return (p[0] + t * (q[0] - p[0]), p[1] + t * (q[1] - p[1]))
        s = inp[-1]
        for e in inp:
            if inside(e):
                if not inside(s):
                    out.append(inter(s, e))
                out.append(e)
            elif inside(s):
                out.append(inter(s, e))
            s = e
    if len(out) < 3:
        return 0.0
    return abs(sum(out[i][0] * out[(i + 1) % len(out)][1] - out[(i + 1) % len(out)][0] * out[i][1]
                   for i in range(len(out)))) / 2.0


def clipper_iou(b1, b2):
    a1, a2 = float(b1[2]) * float(b1[3]), float(b2[2]) * float(b2[3])
    if a1 < 1e-14 or a2 < 1e-14:
        return 0.0
    # same centre shift as the oracle, so both see the rectangles at the same coordinate magnitude
    sx, sy = (float(b1[0]) + float(b2[0])) / 2.0, (float(b1[1]) + float(b2[1])) / 2.0
    c1 = (float(b1[0]) - sx, float(b1[1]) - sy) + tuple(float(v) for v in b1[2:])
    c2 = (float(b2[0]) - sx, float(b2[1]) - sy) + tuple(float(v) for v in b2[2:])
    inter = clip_area(rect_poly(c1), rect_poly(c2))
    return inter / (a1 + a2 - inter)


def ref_iou(a, b):
    """float64 IoU (the oracle's rotated_iou) of every float32 pair a[i], b[i]."""
    return np.array([B.rotated_iou(x, y) for x, y in zip(a, b)], dtype=np.float64)


def ref_clipper(a, b):
    return np.array([clipper_iou(x, y) for x, y in zip(a, b)], dtype=np.float64)


# ------------------------------------------------------------------------------------------------ families
def _axes(ang_deg):
    """Width axis u = (cos, -sin) and length axis v = (sin, cos) of a rectangle at angle_deg (detectron2's vertices)."""
    th = np.radians(ang_deg)
    return np.stack([np.cos(th), -np.sin(th)], -1), np.stack([np.sin(th), np.cos(th)], -1)


def _base(rs, n, side=(0.3, 12.0), extent=100.0, angles=None):
    ctr = rs.uniform(-extent, extent, (n, 2))
    w, h = rs.uniform(*side, n), rs.uniform(*side, n)
    ang = rs.uniform(-180.0, 180.0, n) if angles is None else angles
    return ctr, w, h, ang


def _pack(ctr, w, h, ang):
    return np.stack([ctr[:, 0], ctr[:, 1], w, h, ang], 1).astype(np.float32)


def _shifted(rs, n, fx, fy, side=(0.3, 12.0), extent=100.0, angles=None):
    """b = a moved by fx * w along its width axis and fy * h along its length axis, same size and yaw."""
    ctr, w, h, ang = _base(rs, n, side, extent, angles)
    u, v = _axes(ang)
    c2 = ctr + (fx * w)[:, None] * u + (fy * h)[:, None] * v
    ox, oy = np.clip(1.0 - np.abs(fx), 0, None), np.clip(1.0 - np.abs(fy), 0, None)
    inter = ox * oy
    return _pack(ctr, w, h, ang), _pack(c2, w, h, ang), inter / (2.0 - inter)


def fam_identical(rs, n):
    ctr, w, h, ang = _base(rs, n)
    a = _pack(ctr, w, h, ang)
    return a, a.copy(), np.ones(n)


def fam_shift_width(rs, n):
    return _shifted(rs, n, rs.uniform(0, 1.2, n), np.zeros(n))


def fam_shift_length(rs, n):
    return _shifted(rs, n, np.zeros(n), rs.uniform(0, 1.2, n))


def fam_shift_diagonal(rs, n):
    f = rs.uniform(0, 1.2, n)
    return _shifted(rs, n, f * rs.choice([-1, 1], n), f * rs.choice([-1, 1], n))


def fam_edge_sharing(rs, n):
    """Neighbours in a row: b is a moved by exactly one width or one length (the two share an edge)."""
    along_w = rs.rand(n) < 0.5
    sgn = rs.choice([-1.0, 1.0], n)
    a, b, exact = _shifted(rs, n, np.where(along_w, sgn, 0.0), np.where(along_w, 0.0, sgn))
    # the pair of adjacent cars whose float32 IoU came out as 1/3 under an absolute parallel-edge test
    a[0] = (-18.0995941, 25.1959438, 3.88634491, 0.601982296, 116.802948)
    b[0] = (-19.8520374, 21.7271385, 3.88634491, 0.601982296, 116.802948)
    return a, b, exact


def fam_corner_touching(rs, n):
    return _shifted(rs, n, rs.choice([-1.0, 1.0], n), rs.choice([-1.0, 1.0], n))


def fam_nested(rs, n):
    """b inside a, same yaw, anywhere inside (touching a's edges included): IoU = inner / outer."""
    ctr, w, h, ang = _base(rs, n, side=(1.0, 12.0))
    fw, fh = rs.uniform(0.05, 1.0, n), rs.uniform(0.05, 1.0, n)
    w2, h2 = w * fw, h * fh
    ox = rs.uniform(-1, 1, n) * (w - w2) / 2
    oy = rs.uniform(-1, 1, n) * (h - h2) / 2
    ox[: n // 4] = ((w - w2) / 2)[: n // 4]  # flush with an edge
    u, v = _axes(ang)
    c2 = ctr + ox[:, None] * u + oy[:, None] * v
    a, b = _pack(ctr, w, h, ang), _pack(c2, w2, h2, ang)
    swap = rs.rand(n) < 0.5  # either order
    a[swap], b[swap] = b[swap].copy(), a[swap].copy()
    return a, b, (w2 * h2) / (w * h)


def fam_perpendicular(rs, n):
    """Crosses: same centre, b turned by 90 degrees (its width along a's length)."""
    ctr, w, h, ang = _base(rs, n)
    w2, h2 = rs.uniform(0.3, 12.0, n), rs.uniform(0.3, 12.0, n)
    inter = np.minimum(w, h2) * np.minimum(h, w2)
    return _pack(ctr, w, h, ang), _pack(ctr, w2, h2, ang + rs.choice([-90.0, 90.0], n)), inter / (w * h + w2 * h2 - inter)


def fam_special_angles(rs, n):
    """Angles 0, +-90, +-180, 45 and k * 90 +- 1e-3 with same-yaw shifts, and one rectangle written at angle + 180 or
    with w, h swapped at angle + 90 (IoU 1)."""
    base = np.array([0.0, 90.0, -90.0, 180.0, -180.0, 45.0, -45.0, 135.0])
    near = np.array([k * 90.0 + d for k in range(-2, 3) for d in (-1e-3, 1e-3)])
    ang = rs.choice(np.concatenate([base, near]), n)
    m = n // 3
    a1, b1, e1 = _shifted(rs, m, rs.uniform(0, 1.2, m), rs.uniform(0, 1.2, m) * (rs.rand(m) < 0.5), angles=ang[:m])
    ctr, w, h, ang2 = _base(rs, n - m, angles=ang[m:])
    a2 = _pack(ctr, w, h, ang2)
    swap = rs.rand(n - m) < 0.5
    b2 = np.where(swap[:, None], _pack(ctr, h, w, ang2 + 90.0), _pack(ctr, w, h, ang2 + 180.0))
    return np.concatenate([a1, a2]), np.concatenate([b1, b2]), np.concatenate([e1, np.ones(n - m)])


def fam_thin_barriers(rs, n):
    """0.3 x 10 m barriers: same-yaw shifts along either axis and rows of them."""
    ctr, _, _, ang = _base(rs, n)
    w, h = np.full(n, 0.3), np.full(n, 10.0)
    fx = np.where(rs.rand(n) < 0.5, rs.uniform(0, 1.2, n), 0.0)
    fy = np.where(fx == 0, rs.uniform(0, 1.2, n), 0.0)
    fx[: n // 8] = 1.0  # a row of barriers side by side
    u, v = _axes(ang)
    c2 = ctr + (fx * w)[:, None] * u + (fy * h)[:, None] * v
    inter = np.clip(1 - fx, 0, None) * np.clip(1 - fy, 0, None)
    return _pack(ctr, w, h, ang), _pack(c2, w, h, ang), inter / (2 - inter)


def fam_cones(rs, n):
    f = rs.uniform(0, 1.2, n)
    return _shifted(rs, n, f * (rs.rand(n) < 0.5), f * (rs.rand(n) < 0.5), side=(0.2, 0.2))


def fam_far(rs, n):
    """Centres at +-2000 m (nuScenes global coordinates), same-yaw shifts and touching neighbours."""
    a, b, e = _shifted(rs, n, rs.uniform(-1.2, 1.2, n) * (rs.rand(n) < 0.7), rs.uniform(-1.2, 1.2, n) * (rs.rand(n) < 0.7))
    off = rs.choice([-2000.0, 2000.0], (n, 2)).astype(np.float32)
    a[:, :2] += off
    b[:, :2] += off
    return a, b, None  # rounding the centres at 2000 m moves the closed form by ~1e-4 m


def fam_degenerate(rs, n):
    """Zero and 1e-8 m sides against ordinary boxes and each other."""
    ctr, w, h, ang = _base(rs, n, extent=10.0)
    tiny = rs.choice([0.0, 1e-8], n)
    which = rs.rand(n) < 0.5
    w1, h1 = np.where(which, tiny, w), np.where(which, h, tiny)
    c2 = ctr + rs.uniform(-1, 1, (n, 2))
    w2, h2 = rs.uniform(0.3, 12.0, n), rs.uniform(0.3, 12.0, n)
    w2[: n // 4] = rs.choice([0.0, 1e-8], n // 4)
    a, b = _pack(ctr, w1, h1, ang), _pack(c2, w2, h2, rs.uniform(-180, 180, n))
    return a, b, None


def fam_tangent_circles(rs, n):
    """Bounding circles exactly tangent: centre distance = sum of the half diagonals (IoU 0)."""
    ctr, w, h, ang = _base(rs, n, extent=50.0)
    w2, h2 = rs.uniform(0.3, 12.0, n), rs.uniform(0.3, 12.0, n)
    ang2 = rs.uniform(-180, 180, n)
    r = 0.5 * np.hypot(w, h) + 0.5 * np.hypot(w2, h2)
    # half of the pairs point a corner of each box at the tangent point (the two rectangles touch there)
    corner = rs.rand(n) < 0.5
    phi = rs.uniform(0, 2 * np.pi, n)
    u, v = _axes(ang)
    dcorner = 0.5 * (w[:, None] * u + h[:, None] * v)
    phi = np.where(corner, np.arctan2(dcorner[:, 1], dcorner[:, 0]), phi)
    d = np.stack([np.cos(phi), np.sin(phi)], -1)
    c2 = ctr + r[:, None] * d
    ang2 = np.where(corner, _corner_angle(d, w2, h2), ang2)
    return _pack(ctr, w, h, ang), _pack(c2, w2, h2, ang2), np.zeros(n)


def _corner_angle(d, w, h):
    """Angle at which the corner centre + (w u + h v) / 2 lies along d, i.e. the corner - (w u + h v) / 2 faces -d."""
    # w u + h v = (w cos + h sin, -w sin + h cos) = R(-th) (w, h): its direction is atan2(h, w) - th
    return np.degrees(np.arctan2(h, w) - np.arctan2(d[:, 1], d[:, 0]))


def fam_random(rs, n):
    a = np.stack([rs.randn(n) * 2, rs.randn(n) * 2, rs.rand(n) * 4 + 0.5, rs.rand(n) * 4 + 0.5, rs.uniform(-180, 180, n)], 1)
    b = np.stack([rs.randn(n) * 2, rs.randn(n) * 2, rs.rand(n) * 4 + 0.5, rs.rand(n) * 4 + 0.5, rs.uniform(-180, 180, n)], 1)
    return a.astype(np.float32), b.astype(np.float32), None


FAMILIES = {
    "identical": fam_identical,
    "shift_width": fam_shift_width,
    "shift_length": fam_shift_length,
    "shift_diagonal": fam_shift_diagonal,
    "edge_sharing": fam_edge_sharing,
    "corner_touching": fam_corner_touching,
    "nested": fam_nested,
    "perpendicular": fam_perpendicular,
    "special_angles": fam_special_angles,
    "thin_barriers": fam_thin_barriers,
    "cones": fam_cones,
    "far": fam_far,
    "degenerate": fam_degenerate,
    "tangent_circles": fam_tangent_circles,
    "random": fam_random,
}


def family(name, n, seed=0):
    """-> (a, b, exact or None): n float32 pairs of the family, seeded by the family name and `seed`."""
    rs = np.random.RandomState((seed * 7919 + sum(map(ord, name)) * 104729) % (2 ** 31))
    return FAMILIES[name](rs, n)
