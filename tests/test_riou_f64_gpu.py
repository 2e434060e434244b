"""The three rotated-IoU kernels against float64 on degenerate geometry.

    riou_pairwise_kernel  (csrc/riou.cu, clamp_integral_area2)   rotated_iou_matrix, metrics.match_detections
    riou_paired_kernel    (csrc/riou.cu, clamp_integral_area)    skew_bbox_iou
    riou_grad_kernel      (csrc/riou_grad.cu)                    rotated_iou / riou_loss, value and gradient

Random boxes almost never put an edge exactly on another edge, a box exactly inside another, two boxes at exactly 0 or
pi/2 relative rotation, or a sliver at the culling slack.  Detection labels do all of that, so the pairs here are laid
out on purpose (seeded), each family in both role orders (a, b) and (b, a):

    F1 collinear   integer axis-aligned boxes sharing a full edge, part of an edge, a T-junction or a corner, equal-height
                   boxes on one centre line; then the same rotation (pi/4, +-pi/2, random) applied to both boxes, which
                   leaves the "shared" edges an fp32 rounding apart on either side
    F2 nested      b strictly inside a, inside and touching one or two edges, identical, identical but 1-4 ulps off
    F3 angles      relative rotations of exactly 0, +-pi/2, pi; w/h swapped at +pi/2 (the same box); theta outside
                   (-pi/2, pi/2]: +-pi, 3pi/2, 100pi; negative w or h
    F4 slivers     overlaps and gaps of 1e-7 .. 1e-1 of the box size, along an axis and along a diagonal, and a 45-degree
                   corner against an edge: both sides of the circle and separating-axis culls
    F5 scale       0.5-2 px boxes against 600 x 30 px boxes, aspect 1 and 50, zero-area boxes, NaN / +-inf anywhere
    F6 far         the F1 / F2 / F4 pairs moved to centres of 1e4 .. 1e5 px
    F7 generic     the near-overlap pairs of test_riou_loss_gpu.py, as a control

VALUE.  Every kernel's IoU (and GIoU for the two matrix / paired kernels) is compared with orc_skew_iou (float64 convex
clip of the fp32 inputs, oracle/rbox_oracle.c) under the project's IoU tolerance |got - want| <= 1e-4 |want| + 1e-6; a
touching or separated pair therefore has to come out <= 1e-6.

GRADIENT.  riou_grad_kernel's ga, gb (through rotated_iou(a, b).backward(w), weights positive, negative and zero) are
compared with one-sided differences of orc_skew_iou at steps h and 2h, evaluated on the pair moved by minus a's centre
(exact in float64; it keeps the far-from-origin differences free of canvas-scale cancellation).  With d+-(h) the forward /
backward differences:

  * a component is SMOOTH when |d+(h) - d-(h)| <= 2.5 max(|d+(2h) - d+(h)|, |d-(2h) - d-(h)|) + rounding, i.e. the two
    sides differ by no more than their own truncation error says (for a smooth function both sides are ~ h f''/2 away).
    There the kernel must match the Richardson central difference R = (4 D(h) - D(2h)) / 3 within
        bound + |D(h) - D(2h)| + |d+(h) - d-(h)| / 2 + rounding
    (the last two terms are the stencil's own spread: a kink inside the stencil that still passes the smoothness test
    moves R by no more than that);
  * otherwise the component sits on a KINK (the normal state of F1 / F2: a collinear edge, an identical box).  The kernel's
    value must lie in [min(d-, d+), max(d-, d+)] widened by bound + |d+(2h) - d+(h)| + |d-(2h) - d-(h)| + rounding.
    Every pair is checked; no kink is excused;
  * a pair with an invalid or zero-area box, or separated beyond twice the kernel's cull slack (8 u of the projections'
    scale), must give exactly zero.

The rounding term is 8 eps_f / h with eps_f = 2^-48 S (P_a + P_b) / U |w| (float64 clip of coordinates of size S,
perimeters P, union U).

The bound.  edge_terms(inner, outer) accumulates, per edge e of `inner`, the length L_e of the edge inside `outer`
(Liang-Barsky), its normal and its midpoint.  In fp32 the edge's start a = (ax, ay) and vector e = (ex, ey) in outer's
frame carry an absolute error

    eps_a <= C u S,   S = |rx| + |ry| + hw + hh + HW + HH,   u = 2^-24,

C = 16: sincosf is within 2 ulps, so the relative rotation (cd, sd) is within ~5u and moves the edge by 5u (hw + hh); the
frame offset (rx, ry) adds ~5u (|dx| + |dy|); the three-term sums and the edge vector 2 hw u add <= 4u S.  A crossing
t = (+-HW - a) / e therefore moves by

    dt <= C u S (1 + min(|t|, 2)) / |e|

which is large for near-parallel edges: that is the conditioning of the problem, not slack.  An axis-parallel edge
(e = 0) whose |a| is within C u S of HW may be wholly in or out.  Interval arithmetic over the crossings gives each edge's
[L_min, L_max] and dL_e = max deviation from the float64 L_e; then

    d(dI/dc)  <= sum dL_e + C u sum L_e                 (cx, cy; the rotation back to world adds < C u sum L_e)
    d(dI/dw)  <= 1/2 sum over the u = +-hw edges dL_e + C u sum L_e      (dI/dh likewise)
    d(dI/dth) <= S (sum dL_e + C u sum L_e)             (midpoint offsets |m - c| <= S)

and through k1 = w (U + I) / U^2, k2 = w I / U^2 (U = A_a + A_b - I), with dI_val the kernel's own error in the area I
(recovered exactly from the IoU it returns, the value having its own check):

    bound = |k1| d(dI) + |k1 dI| 2 dI_val / U + |w dA| dI_val (U + 2 I) / U^3 + C u (|k1 dI| + |k2 dA|)

(dA = h for the w component, w for h).  C was set from the derivation above, not from a run.  The worst ratio per kernel
and family is printed with -s.  On an H100 80GB HBM3 the worst gradient ratio is 0.60 (F6, a kink), the worst value
ratio 0.29 (paired IoU, thin boxes crossing; 0.27 for the pairwise kernel over all 7054^2 family pairs), and the file
runs in about 16 s.

Kernel faults these pairs cover: riou_grad_kernel gave small nonzero gradients for separated F4 / F6 pairs (the clamp
integral's rounding residue, through the union), and formed 0 * (edge terms) for dead pairs, NaN for a non-finite box;
the GIoU envelope lost 4e-4 at 1e5 px centres (test_values_vs_float64, F6).

A bound self-test puts six plausible bugs into stored outputs and requires each check to fail.  mAP matching
(ryolo_match_detections) is restated from the greedy loop of the reference's test.py over the kernel's own IoU matrix
and must agree bit for bit."""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

import helpers
from builders import overlapping_pairs

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 1e-6
U32 = 2.0 ** -24
C_BOUND = 16.0
ETA = 1e-5            # difference step, relative to the smallest box dimension of the pair
F32 = np.float32
PI = math.pi
REPORT = {}


def _report(kernel, family, ratio):
    key = (kernel, family)
    r = float(np.max(ratio)) if np.size(ratio) else 0.0
    REPORT[key] = max(REPORT.get(key, 0.0), r)


# ------------------------------------------------------------------------------------------------------------------
# families
# ------------------------------------------------------------------------------------------------------------------
def _rot_pair(a, b, phi):
    """rotate the pair rigidly by phi about a's centre (float64, then rounded to fp32 by the caller)"""
    a, b = a.astype(np.float64).copy(), b.astype(np.float64).copy()
    dx, dy = b[:, 0] - a[:, 0], b[:, 1] - a[:, 1]
    c, s = np.cos(phi), np.sin(phi)
    b[:, 0] = a[:, 0] + c * dx - s * dy
    b[:, 1] = a[:, 1] + s * dx + c * dy
    a[:, 4] += phi
    b[:, 4] += phi
    return a, b


def _in_frame(a, u, v):
    """world point of a's local (u, v) (float64)"""
    c, s = np.cos(a[:, 4]), np.sin(a[:, 4])
    return a[:, 0] + c * u - s * v, a[:, 1] + s * u + c * v


def _place(g, a, b, canvas=400.0):
    """move each pair to its own integer position on the canvas"""
    off = np.floor(g.uniform(50, canvas, (len(a), 2)))
    a, b = a.copy(), b.copy()
    a[:, :2] += off
    b[:, :2] += off
    return a, b


def fam_collinear(g):
    rows_a, rows_b = [], []
    for _ in range(24):
        wa, ha = 2 * g.integers(4, 40), 2 * g.integers(4, 20)
        wb, hb = 2 * g.integers(4, 40), 2 * g.integers(4, 20)
        a = [0.0, 0.0, wa, ha, 0.0]
        sx = (wa + wb) / 2
        cases = [
            [sx, 0.0, wb, ha, 0.0],                                 # full shared edge
            [sx, float(g.integers(-ha // 2, ha // 2)), wb, hb, 0.0],  # part of an edge
            [sx, (ha - hb) / 2, wb, hb, 0.0],                         # T-junction: corners of b on a's edge
            [sx, (ha + hb) / 2, wb, hb, 0.0],                         # corner only
            [float(g.integers(-wa // 2, wa // 2)), 0.0, wb, ha, 0.0],  # equal heights on one centre line, overlapping
            [float(g.integers(-wa // 2, wa // 2)), (ha + hb) / 2, wb, hb, 0.0],  # stacked: shared horizontal edge
            [float(g.integers(-wa // 2, wa // 2)), (ha - hb) / 2, wb, hb, 0.0],  # inside, flush with the top edge
        ]
        for bb in cases:
            rows_a.append(a)
            rows_b.append(bb)
    a, b = np.array(rows_a), np.array(rows_b)
    outs_a, outs_b = [a], [b]
    for phi in (PI / 4, PI / 2, -PI / 2, g.uniform(-PI, PI)):
        ra, rb = _rot_pair(a, b, phi)
        outs_a.append(ra)
        outs_b.append(rb)
    a, b = np.concatenate(outs_a), np.concatenate(outs_b)
    return _place(g, a, b)


def fam_nested(g):
    n = 48
    a = np.stack([np.zeros(n), np.zeros(n), g.uniform(20, 120, n), g.uniform(8, 40, n), g.uniform(-PI / 2, PI / 2, n)], 1)
    a[: n // 4, 4] = 0.0
    a[: n // 4, 2:4] = 2 * np.round(a[: n // 4, 2:4] / 2)
    rows_a, rows_b = [], []
    fr = g.uniform(0.2, 0.8, (n, 2))
    hw, hh = a[:, 2] / 2, a[:, 3] / 2
    bw, bh = a[:, 2] * fr[:, 0], a[:, 3] * fr[:, 1]
    # strictly inside, own rotation small enough to stay inside
    u = g.uniform(-0.5, 0.5, n) * (hw - bw / 2 - bh / 2).clip(0)
    v = g.uniform(-0.5, 0.5, n) * (hh - bh / 2 - bw / 2).clip(0)
    x, y = _in_frame(a, u, v)
    rows_a.append(a)
    rows_b.append(np.stack([x, y, bw * 0.5, bh * 0.5, a[:, 4] + g.uniform(-0.3, 0.3, n)], 1))
    # inside and touching one edge (u = hw - bw/2), two edges (a corner)
    x, y = _in_frame(a, hw - bw / 2, g.uniform(-0.3, 0.3, n) * (hh - bh / 2))
    rows_a.append(a)
    rows_b.append(np.stack([x, y, bw, bh, a[:, 4]], 1))
    x, y = _in_frame(a, -(hw - bw / 2), hh - bh / 2)
    rows_a.append(a)
    rows_b.append(np.stack([x, y, bw, bh, a[:, 4]], 1))
    # identical
    rows_a.append(a)
    rows_b.append(a.copy())
    a, b = np.concatenate(rows_a), np.concatenate(rows_b)
    a, b = _place(g, a, b)
    a32, b32 = a.astype(F32), b.astype(F32)
    # identical boxes 1..4 ulps apart in one parameter
    ident_a = a32[-n:]
    pa, pb = [], []
    for k in range(5):
        for steps in (1, 2, 4, -1, -3):
            bb = ident_a.copy()
            col = bb[:, k]
            for _ in range(abs(steps)):
                col = np.nextafter(col, F32(np.inf) if steps > 0 else F32(-np.inf))
            bb[:, k] = col
            pa.append(ident_a[:8])
            pb.append(bb[:8])
    return np.concatenate([a32] + pa), np.concatenate([b32] + pb)


def fam_angles(g):
    n = 24
    base = np.stack([np.zeros(n), np.zeros(n), g.uniform(20, 100, n), g.uniform(6, 30, n), np.zeros(n)], 1)
    off = np.stack([g.uniform(-0.4, 0.4, n) * base[:, 2], g.uniform(-0.4, 0.4, n) * base[:, 3]], 1)
    rows_a, rows_b = [], []
    hp = float(F32(PI / 2))
    for tb in (0.0, hp, -hp, float(F32(PI))):         # relative rotation exactly 0, +-pi/2, pi in fp32 (theta_a = 0)
        b = base.copy()
        b[:, :2] += off
        b[:, 4] = tb
        rows_a.append(base)
        rows_b.append(b)
    tha = g.uniform(-PI / 2, PI / 2, n)
    a = base.copy()
    a[:, 4] = tha
    b = a.copy()
    b[:, 2], b[:, 3] = a[:, 3], a[:, 2]                # w / h swapped at +pi/2: the same box
    b[:, 4] = (tha.astype(F32) + F32(PI / 2)).astype(np.float64)
    rows_a += [a, a]
    b2 = b.copy()
    b2[:, :2] += off * 0.5
    rows_b += [b, b2]
    for extra in (PI, -PI, 1.5 * PI, 100 * PI):        # theta outside (-pi/2, pi/2]
        b = a.copy()
        b[:, :2] += off * 0.3
        b[:, 4] = tha + extra
        rows_a.append(a)
        rows_b.append(b)
    a_neg = a.copy()
    a_neg[: n // 2, 2] *= -1                            # negative w
    a_neg[n // 2:, 3] *= -1                             # negative h
    b = a.copy()
    b[:, :2] += off * 0.5
    b[:, 4] += 0.2
    rows_a.append(a_neg)
    rows_b.append(b)
    b_neg = b.copy()
    b_neg[:, 2:4] *= -1
    rows_a.append(a)
    rows_b.append(b_neg)
    a, b = np.concatenate(rows_a), np.concatenate(rows_b)
    return _place(g, a, b)


def fam_slivers(g):
    rows_a, rows_b = [], []
    depths = [10.0 ** -k for k in range(7, 0, -1)]
    for d in depths:
        for sign in (1.0, -1.0):                      # overlap, gap
            n = 6
            a = np.stack([np.zeros(n), np.zeros(n), g.uniform(20, 80, n), g.uniform(8, 30, n),
                          g.uniform(-PI / 2, PI / 2, n)], 1)
            a[:2, 4] = 0.0
            b = a.copy()
            b[:, 2:4] *= g.uniform(0.6, 1.4, (n, 2))
            size = np.maximum(a[:, 2], a[:, 3])
            hwa, hha, hwb, hhb = a[:, 2] / 2, a[:, 3] / 2, b[:, 2] / 2, b[:, 3] / 2
            # along a's x axis
            x, y = _in_frame(a, hwa + hwb - sign * d * size, np.zeros(n))
            rows_a.append(a); rows_b.append(np.stack([x, y, b[:, 2], b[:, 3], a[:, 4]], 1))
            # along the diagonal: corners overlap by d in both axes
            x, y = _in_frame(a, hwa + hwb - sign * d * size, hha + hhb - sign * d * size)
            rows_a.append(a); rows_b.append(np.stack([x, y, b[:, 2], b[:, 3], a[:, 4]], 1))
            # b at 45 degrees, its corner against a's edge
            reach = (hwb + hhb) / math.sqrt(2.0)
            x, y = _in_frame(a, hwa + reach - sign * d * size, 0.3 * hha)
            rows_a.append(a); rows_b.append(np.stack([x, y, b[:, 2], b[:, 3], a[:, 4] + PI / 4], 1))
    a, b = np.concatenate(rows_a), np.concatenate(rows_b)
    return _place(g, a, b)


def fam_scale(g):
    rows_a, rows_b = [], []
    n = 40
    big = np.stack([np.zeros(n), np.zeros(n), np.full(n, 600.0), np.full(n, 30.0), g.uniform(-PI / 2, PI / 2, n)], 1)
    big[:8, 4] = 0.0
    sw = g.uniform(0.5, 2.0, (n, 2))
    u = g.uniform(-300, 300, n)
    v = g.uniform(-15, 15, n)
    v[::3] = 15.0 - sw[::3, 1] * g.uniform(-0.5, 0.5, len(v[::3]))    # across the long edge
    x, y = _in_frame(big, u, v)
    rows_a.append(big); rows_b.append(np.stack([x, y, sw[:, 0], sw[:, 1], g.uniform(-PI, PI, n)], 1))
    for aspect in (1.0, 50.0):
        m = 24
        area = g.uniform(200, 4000, m)
        w, h = np.sqrt(area * aspect), np.sqrt(area / aspect)
        a = np.stack([np.zeros(m), np.zeros(m), w, h, g.uniform(-PI / 2, PI / 2, m)], 1)
        b = a.copy()
        x, y = _in_frame(a, g.uniform(-0.5, 0.5, m) * w, g.uniform(-0.7, 0.7, m) * h)
        b[:, 0], b[:, 1] = x, y
        b[:, 4] += g.uniform(-0.05, 0.05, m)
        b[:, 2:4] *= g.uniform(0.8, 1.2, (m, 2))
        rows_a.append(a); rows_b.append(b)
    a, b = np.concatenate(rows_a), np.concatenate(rows_b)
    a, b = _place(g, a, b)
    # zero-area and non-finite boxes, against an overlapping valid box
    m = 8
    v = np.stack([np.full(m, 200.0), np.full(m, 200.0), np.full(m, 40.0), np.full(m, 20.0), g.uniform(-1, 1, m)], 1)
    bad_a, bad_b = [], []
    z = v.copy(); z[:3, 2] = 0.0; z[3:6, 3] = 0.0; z[6:, 2:4] = 0.0
    bad_a.append(v); bad_b.append(z)
    for k in range(5):
        for val in (np.nan, np.inf, -np.inf):
            bb = v[:1].copy()
            bb[0, 0] += 3.0
            bb[0, k] = val
            bad_a.append(v[:1]); bad_b.append(bb)
    ba, bb = np.concatenate(bad_a), np.concatenate(bad_b)
    return np.concatenate([a, ba]), np.concatenate([b, bb])


def fam_far(g, parts):
    a = np.concatenate([p[0] for p in parts]).astype(np.float64)
    b = np.concatenate([p[1] for p in parts]).astype(np.float64)
    off = np.floor(g.uniform(1e4, 1e5, (len(a), 2)))
    a[:, :2] += off
    b[:, :2] += off
    return a, b


def fam_generic():
    a, b = overlapping_pairs(160, 21)
    return a.numpy(), b.numpy()


@functools.lru_cache(maxsize=None)
def families():
    """name -> (a, b) fp32 [n, 5], each family in both role orders (built once; callers do not write into them)"""
    g = np.random.default_rng(2026)
    fams = {"F1 collinear": fam_collinear(g), "F2 nested": fam_nested(g), "F3 angles": fam_angles(g),
            "F4 slivers": fam_slivers(g), "F5 scale": fam_scale(g)}
    fams = {k: (np.asarray(a, F32), np.asarray(b, F32)) for k, (a, b) in fams.items()}
    fams["F6 far"] = tuple(np.asarray(x, F32) for x in fam_far(g, [fams["F1 collinear"], fams["F2 nested"],
                                                                    fams["F4 slivers"]]))
    fams["F7 generic"] = tuple(np.asarray(x, F32) for x in fam_generic())
    return {k: (np.concatenate([a, b]), np.concatenate([b, a])) for k, (a, b) in fams.items()}


# ------------------------------------------------------------------------------------------------------------------
# float64 oracle
# ------------------------------------------------------------------------------------------------------------------
_DBL5 = ctypes.c_double * 5


def _orc():
    return helpers.oracle().orc_skew_iou


def oracle_values(a, b, mode=0):
    f = _orc()
    out = np.empty(len(a))
    x, y = _DBL5(), _DBL5()
    for i in range(len(a)):
        x[:] = a[i].astype(np.float64).tolist()
        y[:] = b[i].astype(np.float64).tolist()
        out[i] = f(x, y, mode)
    return out


def value_ratio(got, want):
    return np.abs(got.astype(np.float64) - want) / (RTOL * np.abs(want) + ATOL)


# ------------------------------------------------------------------------------------------------------------------
# float64 restatement of edge_terms (csrc/riou_grad.cu) with the error analysis of the module docstring
# ------------------------------------------------------------------------------------------------------------------
def edge_geometry(inner, outer):
    """inner, outer float64 [N, 5].  Returns (dI [N, 5] world frame as the kernel orders it, ddI [N, 5] bound on the fp32
    error of dI, contrib [N, 4, 5] per-edge terms)."""
    cx, cy, th = inner[:, 0], inner[:, 1], inner[:, 4]
    w, h = np.abs(inner[:, 2]), np.abs(inner[:, 3])
    ocx, ocy, oth = outer[:, 0], outer[:, 1], outer[:, 4]
    W, H = np.abs(outer[:, 2]), np.abs(outer[:, 3])
    c, s, oc, os_ = np.cos(th), np.sin(th), np.cos(oth), np.sin(oth)
    dx, dy = cx - ocx, cy - ocy
    rx, ry = dx * oc + dy * os_, dy * oc - dx * os_
    cd, sd = oc * c + os_ * s, oc * s - os_ * c
    hw, hh, HW, HH = 0.5 * w, 0.5 * h, 0.5 * W, 0.5 * H
    ux, uy, vx, vy = cd, sd, -sd, cd
    S = np.abs(rx) + np.abs(ry) + hw + hh + HW + HH
    K = C_BOUND * U32 * S
    n = len(inner)
    contrib = np.zeros((n, 4, 5))
    dL_sum, L_sum, dL_w, dL_h = np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for e in range(4):
            if e == 0:
                ax, ay, ex, ey, nx, ny = rx - hw * ux - hh * vx, ry - hw * uy - hh * vy, 2 * hw * ux, 2 * hw * uy, -vx, -vy
            elif e == 1:
                ax, ay, ex, ey, nx, ny = rx + hw * ux - hh * vx, ry + hw * uy - hh * vy, 2 * hh * vx, 2 * hh * vy, ux, uy
            elif e == 2:
                ax, ay, ex, ey, nx, ny = rx + hw * ux + hh * vx, ry + hw * uy + hh * vy, -2 * hw * ux, -2 * hw * uy, vx, vy
            else:
                ax, ay, ex, ey, nx, ny = rx - hw * ux + hh * vx, ry - hw * uy + hh * vy, -2 * hh * vx, -2 * hh * vy, -ux, -uy
            elen = 2 * hh if e & 1 else 2 * hw
            t0, t1 = np.zeros(n), np.ones(n)
            t0lo, t0hi, t1lo, t1hi = np.zeros(n), np.zeros(n), np.ones(n), np.ones(n)
            for a_, e_, H_ in ((ax, ex, HW), (ay, ey, HH)):
                zero = e_ == 0
                ta, tb = (-H_ - a_) / e_, (H_ - a_) / e_
                lo, hi = np.minimum(ta, tb), np.maximum(ta, tb)
                dlo = K * (1 + np.minimum(np.abs(lo), 2)) / np.abs(e_)
                dhi = K * (1 + np.minimum(np.abs(hi), 2)) / np.abs(e_)
                lo_m, lo_p, hi_m, hi_p = lo - dlo, lo + dlo, hi - dhi, hi + dhi
                inside = np.abs(a_) <= H_
                sure = np.abs(np.abs(a_) - H_) > K
                zlo = np.where(inside, -np.inf, np.inf)
                zhi = np.where(inside, np.inf, -np.inf)
                lo = np.where(zero, zlo, lo)
                hi = np.where(zero, zhi, hi)
                lo_m = np.where(zero, np.where(sure, zlo, -np.inf), lo_m)
                lo_p = np.where(zero, np.where(sure, zlo, np.inf), lo_p)
                hi_m = np.where(zero, np.where(sure, zhi, -np.inf), hi_m)
                hi_p = np.where(zero, np.where(sure, zhi, np.inf), hi_p)
                t0, t1 = np.maximum(t0, lo), np.minimum(t1, hi)
                t0lo, t0hi = np.maximum(t0lo, lo_m), np.maximum(t0hi, lo_p)
                t1lo, t1hi = np.minimum(t1lo, hi_m), np.minimum(t1hi, hi_p)
            t0hi, t1lo = np.minimum(t0hi, 1.0), np.maximum(t1lo, 0.0)
            valid = t1 > t0
            L = np.where(valid, (t1 - t0) * elen, 0.0)
            Lmax = np.maximum(t1hi - t0lo, 0.0) * elen
            Lmin = np.maximum(t1lo - t0hi, 0.0) * elen
            dL = np.maximum(Lmax - L, L - Lmin)
            tm = 0.5 * (t0 + t1)
            mx, my = ax + tm * ex - rx, ay + tm * ey - ry
            gxl, gyl = L * nx, L * ny
            contrib[:, e, 0] = gxl * oc - gyl * os_
            contrib[:, e, 1] = gxl * os_ + gyl * oc
            contrib[:, e, 2 if e & 1 else 3] = 0.5 * L
            contrib[:, e, 4] = np.where(valid, L * (nx * (-my) + ny * mx), 0.0)
            dL_sum += dL
            L_sum += L
            if e & 1:
                dL_w += dL
            else:
                dL_h += dL
    dI = contrib.sum(1)
    r = C_BOUND * U32 * L_sum
    ddI = np.stack([dL_sum + r, dL_sum + r, 0.5 * dL_w + r, 0.5 * dL_h + r, S * (dL_sum + r)], 1)
    return dI, ddI, contrib


def grad_bound(inner, outer, iou_kernel, iou_ref, wt):
    """per-component bound on |kernel gradient - true gradient| for d IoU / d inner (module docstring)"""
    dI, ddI, _ = edge_geometry(inner, outer)
    Ai = np.abs(inner[:, 2] * inner[:, 3])
    Ao = np.abs(outer[:, 2] * outer[:, 3])
    tot = Ai + Ao
    I_ref = iou_ref * tot / (1 + iou_ref)
    I_k = iou_kernel.astype(np.float64) * tot / (1 + iou_kernel.astype(np.float64))
    dIv = np.abs(I_k - I_ref) + 4 * U32 * I_ref
    U = tot - I_ref
    k1 = wt * (U + I_ref) / U ** 2
    k2 = wt * I_ref / U ** 2
    dA = np.zeros_like(dI)
    dA[:, 2] = np.abs(inner[:, 3])
    dA[:, 3] = np.abs(inner[:, 2])
    aw = np.abs(wt)[:, None]
    b = (np.abs(k1)[:, None] * ddI + np.abs(k1 * 2 * dIv / U)[:, None] * np.abs(dI)
         + aw * dA * (dIv * (U + 2 * I_ref) / U ** 3)[:, None]
         + C_BOUND * U32 * (np.abs(k1)[:, None] * np.abs(dI) + np.abs(k2)[:, None] * dA))
    return b


# ------------------------------------------------------------------------------------------------------------------
# one-sided differences of the oracle
# ------------------------------------------------------------------------------------------------------------------
def oracle_differences(a, b, which, wt):
    """d IoU(a, b) / d(which box) by one-sided differences at steps h and 2h.  Returns dict of [N, 5] arrays."""
    f = _orc()
    n = len(a)
    A = a.astype(np.float64)
    B = b.astype(np.float64)
    out = {k: np.zeros((n, 5)) for k in ("dp1", "dm1", "dp2", "dm2", "D1", "D2", "rnd")}
    zero_all = np.ones(n, bool)
    x, y = _DBL5(), _DBL5()
    for i in range(n):
        pa, pb = A[i].copy(), B[i].copy()
        if not (np.isfinite(pa).all() and np.isfinite(pb).all() and pa[2] * pa[3] * pb[2] * pb[3] != 0):
            continue                                    # invalid or zero-area box: IoU 0 everywhere, exact zero checked
        ox, oy = pa[0], pa[1]
        pa[:2] -= (ox, oy)
        pb[:2] -= (ox, oy)
        dims = np.abs(np.array([pa[2], pa[3], pb[2], pb[3]]))
        s = dims.min()
        tgt = pa if which == "a" else pb
        other = pb if which == "a" else pa
        r_in = 0.5 * math.hypot(tgt[2], tgt[3])
        S = np.abs(pb[:2]).sum() + dims.sum()
        x[:] = pa.tolist()
        y[:] = pb.tolist()
        f0 = f(x, y, 0)
        area = dims[0] * dims[1] + dims[2] * dims[3]
        U = area - f0 * area / (1 + f0) if area > 0 else 1.0
        eps_f = 2.0 ** -48 * S * 2 * dims.sum() / max(U, 1e-300) * abs(wt[i])
        vals = np.zeros((5, 4))
        for k in range(5):
            h = ETA * s if k < 4 else ETA * s / r_in
            for j, st in enumerate((h, -h, 2 * h, -2 * h)):
                p = tgt.copy()
                p[k] += st
                if which == "a":
                    x[:] = p.tolist()
                    y[:] = other.tolist()
                else:
                    x[:] = other.tolist()
                    y[:] = p.tolist()
                vals[k, j] = f(x, y, 0)
            fp1, fm1, fp2, fm2 = vals[k]
            wi = wt[i]
            out["dp1"][i, k] = wi * (fp1 - f0) / h
            out["dm1"][i, k] = wi * (f0 - fm1) / h
            out["dp2"][i, k] = wi * (fp2 - f0) / (2 * h)
            out["dm2"][i, k] = wi * (f0 - fm2) / (2 * h)
            out["D1"][i, k] = wi * (fp1 - fm1) / (2 * h)
            out["D2"][i, k] = wi * (fp2 - fm2) / (4 * h)
            out["rnd"][i, k] = 8 * eps_f / h
        zero_all[i] = f0 == 0 and not vals.any()
    out["zero_all"] = zero_all
    return out


def grad_ratio(g, fd, bound):
    """g kernel gradient [N, 5]; returns (ratio [N, 5], smooth mask)"""
    dp1, dm1, dp2, dm2, D1, D2, rnd = (fd[k] for k in ("dp1", "dm1", "dp2", "dm2", "D1", "D2", "rnd"))
    spread = np.abs(dp1 - dm1)
    trunc = np.maximum(np.abs(dp2 - dp1), np.abs(dm2 - dm1))
    smooth = spread <= 2.5 * trunc + rnd
    R = (4 * D1 - D2) / 3
    tol_s = bound + np.abs(D1 - D2) + 0.5 * spread + rnd
    err_s = np.abs(g - R)
    lo, hi = np.minimum(dp1, dm1), np.maximum(dp1, dm1)
    tol_k = bound + np.abs(dp2 - dp1) + np.abs(dm2 - dm1) + rnd
    err_k = np.maximum(np.maximum(g - hi, lo - g), 0.0)
    err = np.where(smooth, err_s, err_k)
    tol = np.where(smooth, tol_s, tol_k)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / tol)
    return np.nan_to_num(ratio, nan=np.inf), smooth


# ------------------------------------------------------------------------------------------------------------------
# running the kernels
# ------------------------------------------------------------------------------------------------------------------
def _weights(n):
    w = np.array([1.0, -0.7, 0.0, 2.5, -1.9, 0.3], F32)
    return np.resize(w, n)


def _live(a, b):
    ok = np.isfinite(a).all(1) & np.isfinite(b).all(1)
    return ok & (a[:, 2] * a[:, 3] != 0) & (b[:, 2] * b[:, 3] != 0)


@pytest.fixture(scope="module")
def run():
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.iou import rotated_iou
    res = {}
    for name, (a, b) in families().items():
        ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        wt = _weights(len(a))
        r = dict(a=a, b=b, wt=wt.astype(np.float64))
        r["paired"] = pkg.skew_bbox_iou(ad, bd).cpu().numpy()
        r["paired_g"] = pkg.skew_bbox_iou(ad, bd, GIoU=True).cpu().numpy()
        ag, bg = ad.clone().requires_grad_(True), bd.clone().requires_grad_(True)
        iou = rotated_iou(ag, bg)
        (iou * torch.from_numpy(wt).cuda()).sum().backward()
        r["grad_val"] = iou.detach().cpu().numpy()
        r["ga"], r["gb"] = ag.grad.cpu().numpy(), bg.grad.cpu().numpy()
        # one side at a time: the same numbers
        for side in ("a", "b"):
            x = ad.clone().requires_grad_(side == "a")
            y = bd.clone().requires_grad_(side == "b")
            (rotated_iou(x, y) * torch.from_numpy(wt).cuda()).sum().backward()
            r["g%s_only" % side] = (x if side == "a" else y).grad.cpu().numpy()
            assert (y if side == "a" else x).grad is None
        r["want"] = oracle_values(a, b, 0)
        r["want_g"] = oracle_values(a, b, 1)
        res[name] = r
    return res


@pytest.fixture(scope="module")
def fd(run):
    out = {}
    for name, r in run.items():
        for which in ("a", "b"):
            out[name, which] = oracle_differences(r["a"], r["b"], which, r["wt"])
    return out


def separated(a, b):
    """float64 restatement of riou_grad.cu's `separated` with twice its slack: the pairs the kernel must cull whatever its
    own fp32 rounding (its gap and slack are both within 4 u of their scale)"""
    a, b = a.astype(np.float64), b.astype(np.float64)
    with np.errstate(invalid="ignore"):
        dx, dy = b[:, 0] - a[:, 0], b[:, 1] - a[:, 1]
        ca, sa, cb, sb = np.cos(a[:, 4]), np.sin(a[:, 4]), np.cos(b[:, 4]), np.sin(b[:, 4])
        C, S = np.abs(ca * cb + sa * sb), np.abs(ca * sb - sa * cb)
        ha, ka, hb, kb = (0.5 * np.abs(x) for x in (a[:, 2], a[:, 3], b[:, 2], b[:, 3]))
        slack = 8 * U32 * (np.abs(dx) + np.abs(dy) + ha + ka + hb + kb)
        gap = np.maximum.reduce([np.abs(dx * ca + dy * sa) - (ha + hb * C + kb * S),
                                 np.abs(dy * ca - dx * sa) - (ka + hb * S + kb * C),
                                 np.abs(dx * cb + dy * sb) - (hb + ha * C + ka * S),
                                 np.abs(dy * cb - dx * sb) - (kb + ha * S + ka * C)])
        return gap > 2 * slack


def _grad_checks(r, fdd, ga=None, gb=None):
    """ratio arrays for both sides plus the exact-zero violations.  Exact zeros are required where the kernel promises
    them: an invalid or zero-area box, or a pair separated beyond the kernel's cull slack.  A pair inside that slack whose
    oracle IoU is 0 on the whole stencil goes through the ordinary check (its references are 0; the bound covers what the
    clamp integral's rounding residue does through the union)."""
    a64, b64 = r["a"].astype(np.float64), r["b"].astype(np.float64)
    ga = r["ga"] if ga is None else ga
    gb = r["gb"] if gb is None else gb
    live = _live(r["a"], r["b"])
    sep = separated(r["a"], r["b"])
    ratios, zero_bad = [], 0
    for which, g, inner, outer in (("a", ga, a64, b64), ("b", gb, b64, a64)):
        f = fdd[which]
        dead = ~live | sep
        zero_bad += int(np.count_nonzero(g[dead] != 0) + np.count_nonzero(~np.isfinite(g)))
        rel = inner.copy()
        oth = outer.copy()
        with np.errstate(all="ignore"):
            rel[:, :2] -= a64[:, :2]
            oth[:, :2] -= a64[:, :2]
            bound = grad_bound(rel[live], oth[live], r["grad_val"][live], r["want"][live], r["wt"][live])
        ratio, smooth = grad_ratio(g[live].astype(np.float64), {k: v[live] for k, v in f.items() if k != "zero_all"},
                                   bound)
        ratio[sep[live]] = 0.0
        ratios.append(ratio)
    return ratios, zero_bad


# ------------------------------------------------------------------------------------------------------------------
# tests
# ------------------------------------------------------------------------------------------------------------------
def test_families_reach_the_degenerate_cases():
    fams = families()
    a, b = fams["F1 collinear"]
    want = oracle_values(a, b)
    assert (want == 0).sum() > 50 and (want > 0).sum() > 300          # touching and overlapping collinear pairs
    a, b = fams["F2 nested"]
    assert np.isclose(oracle_values(a, b), 1.0, atol=1e-6).sum() >= 96  # identical boxes, both orders
    a, b = fams["F5 scale"]
    assert (~np.isfinite(b)).any(1).sum() >= 15 and ((b[:, 2] * b[:, 3]) == 0).sum() >= 8


def test_values_vs_float64(run):
    worst = []
    for name, r in run.items():
        for kernel, got, want in (("paired iou", r["paired"], r["want"]), ("paired giou", r["paired_g"], r["want_g"]),
                                  ("grad value", r["grad_val"], r["want"])):
            ratio = value_ratio(got, want)
            _report(kernel, name, ratio)
            worst.append((float(ratio.max()), kernel, name, int(ratio.argmax())))
            assert np.isfinite(got).all()
    bad = [w for w in worst if not w[0] <= 1.0]
    assert not bad, bad


def _pairwise_check(a, b, mode, name, **kw):
    import rotate_yolov3_b200 as pkg
    got = pkg.rotated_iou_matrix(a, b, GIoU=bool(mode), **kw).cpu().numpy()
    an, bn = a.cpu().numpy()[:, :5], b.cpu().numpy()[:, :5]
    want = helpers.orc_skew_pairwise(an, bn, mode).astype(np.float64)
    ratio = value_ratio(got, want)
    _report("pairwise " + ("giou" if mode else "iou"), name, ratio)
    return ratio, got, want


@functools.lru_cache(maxsize=None)
def _all_pairs():
    fams = families()
    a = np.concatenate([v[0] for v in fams.values()])
    b = np.concatenate([v[1] for v in fams.values()])
    return a, b


def _circle_candidates(a, b, chunk=512):
    """(i, j) of every pair whose bounding circles come within 1e-3 of touching; all other pairs are disjoint"""
    ra = 0.5 * np.hypot(a[:, 2], a[:, 3]).astype(np.float64)
    rb = 0.5 * np.hypot(b[:, 2], b[:, 3]).astype(np.float64)
    ii, jj = [], []
    with np.errstate(invalid="ignore"):
        for i0 in range(0, len(a), chunk):
            sa = slice(i0, i0 + chunk)
            d2 = ((a[sa, None, :2].astype(np.float64) - b[None, :, :2]) ** 2).sum(-1)
            i, j = np.nonzero(d2 <= ((ra[sa, None] + rb[None, :]) * 1.001) ** 2)
            ii.append(i + i0)
            jj.append(j)
    return np.concatenate(ii), np.concatenate(jj)


def test_pairwise_all_families_matrix(run):
    """one matrix of every family box against every other: all 7054^2 pairs are checked.  The pairs within reach of each
    other's bounding circle (most of them accidental crossings of pairs placed near each other) go to the oracle; the rest
    are disjoint and must come out 0."""
    import rotate_yolov3_b200 as pkg
    a, b = _all_pairs()
    ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    ii, jj = _circle_candidates(a, b)
    assert len(ii) > 500000
    for mode in (0, 1):
        full = pkg.rotated_iou_matrix(ad, bd, GIoU=bool(mode)).cpu().numpy()
        want = helpers.orc_skew_paired(a[ii], b[jj], mode).astype(np.float64)
        ratio = value_ratio(full[ii, jj], want)
        full[ii, jj] = 0.0
        ratio_far = float(np.abs(full).max()) / ATOL
        _report("pairwise " + ("giou" if mode else "iou"), "all x all", np.array([ratio.max(), ratio_far]))
        k = int(np.argmax(ratio))
        assert ratio.max() <= 1.0, (mode, float(ratio.max()), int(ii[k]), int(jj[k]))
        assert ratio_far <= 1.0, (mode, ratio_far)


def test_thin_boxes_crossing_at_a_steep_angle():
    """A thin box (aspect ~50) crossed at a steep angle.  The clamp integral weights b's edges by ey in the frame box's
    normalised frame, and each breakpoint's rounding (~u in t) moves an edge's dY by ~u |ey|.  With the thin box's long
    side along x, |ey| reached ~50: the four named pairs are cross pairs of the all-families matrix, one of which missed the
    value contract on the device (1.02x, rcp.approx); a host restatement reaches 0.90 with IEEE reciprocals and 2.2 with
    reciprocals 1 ulp off.  canonical_frame (riou_area.cuh) turns the frame box so its long side runs along y; the host
    restatement then stays below 0.3 (0.6 with 1-ulp reciprocals) on all 7054^2 pairs.  All three kernels, both role
    orders, plus a seeded sweep of the same geometry."""
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.iou import rotated_iou
    fa, fb = _all_pairs()
    named = [(3610, 3630), (3614, 1792), (3627, 3630), (3725, 3720)]
    a = np.stack([fa[i] for i, _ in named])
    b = np.stack([fb[j] for _, j in named])
    assert (a[:, 2] / a[:, 3] > 35).all()
    g = np.random.default_rng(11)
    sweep_a, sweep_b = [], []
    for _ in range(256):
        L1, L2 = g.uniform(200, 500, 2)
        t1 = g.uniform(-PI, PI)
        t2 = t1 + g.choice([-1, 1]) * g.uniform(1.0, PI / 2)
        c = g.uniform(100, 500, 2)
        sweep_a.append([c[0], c[1], L1, L1 / g.uniform(40, 60), t1])
        off = g.uniform(-0.3, 0.3, 2) * [L1, L1 / 50]
        sweep_b.append([c[0] + off[0], c[1] + off[1], L2, L2 / g.uniform(40, 60), t2])
    a = np.concatenate([a, np.array(sweep_a, F32)])
    b = np.concatenate([b, np.array(sweep_b, F32)])
    a, b = np.concatenate([a, b]), np.concatenate([b, a])
    want = oracle_values(a, b)
    assert (want > 0).mean() > 0.9
    ad, bd = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    got = {"pairwise iou": np.diagonal(pkg.rotated_iou_matrix(ad, bd).cpu().numpy()),
           "paired iou": pkg.skew_bbox_iou(ad, bd).cpu().numpy(),
           "grad value": rotated_iou(ad, bd).detach().cpu().numpy()}
    for kernel, v in got.items():
        ratio = value_ratio(v, want)
        _report(kernel, "thin crossing", ratio)
        assert ratio.max() <= 1.0, (kernel, float(ratio.max()), int(ratio.argmax()))


def _full_tile():
    """32 rows x 128 columns that all overlap one another: degenerate shapes around one point"""
    g = np.random.default_rng(5)
    rows = []
    for i in range(32):
        th = [0.0, float(F32(PI / 2)), float(F32(PI)), g.uniform(-PI / 2, PI / 2)][i % 4]
        rows.append([300.0 + (i % 4), 300.0 + (i // 4) % 4, 2 * g.integers(20, 60), 2 * g.integers(10, 30), th])
    rows = np.array(rows, F32)
    cols = []
    for j in range(128):
        src = rows[j % 32].copy()
        kind = j // 32
        if kind == 0:
            cols.append(src)                                   # identical to a row
        elif kind == 1:
            src[0] += src[2] / 8
            cols.append(src)                                   # collinear: same centre line and height
        elif kind == 2:
            cols.append([src[0], src[1], src[3], src[2], src[4] + F32(PI / 2)])   # w/h swapped at +pi/2
        else:
            cols.append([300.0 + g.uniform(-3, 3), 300.0 + g.uniform(-3, 3), g.uniform(10, 50), g.uniform(10, 50),
                         g.uniform(-PI, PI)])
    return rows, np.array(cols, F32)


def test_pairwise_full_tile_all_pairs_survive():
    rows, cols = _full_tile()
    for mode in (0, 1):
        ratio, got, want = _pairwise_check(torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda(), mode, "full tile")
        assert (want > 1e-3).all() and (got > 0).all()           # all 4096 pairs reach the integral: 16 A2 rounds
        assert ratio.max() <= 1.0, ratio.max()


@pytest.mark.parametrize("n", [1, 31, 33])
@pytest.mark.parametrize("m", [1, 127, 129, 256])
def test_pairwise_shapes(n, m):
    """scalar write-back (m = 1, 127, 129) and the __stcs vector write-back (m = 256), partial row tiles"""
    a, b = _all_pairs()
    g = np.random.default_rng(n * 1000 + m)
    keep = np.isfinite(a).all(1) & np.isfinite(b).all(1)
    idx = g.permutation(np.flatnonzero(keep))
    ai, bi = idx[:n], idx[:m]                           # the first min(n, m) rows and columns are family pairs
    for mode in (0, 1):
        ratio, _, want = _pairwise_check(torch.from_numpy(a[ai]).cuda(), torch.from_numpy(b[bi]).cuda(), mode,
                                         "shapes")
        assert ratio.max() <= 1.0, (mode, ratio.max())


def test_pairwise_strided_rows():
    a, b = _all_pairs()
    n, m = 200, 300
    bufa = torch.randn(n, 11).cuda()
    bufa[:, 2:7] = torch.from_numpy(a[:n]).cuda()
    bufb = torch.randn(2 * m, 7).cuda()
    bufb[::2, :5] = torch.from_numpy(b[:m]).cuda()
    av, bv = bufa[:, 2:9], bufb[::2]                   # [N, 7] row views with strides 11 and 14
    assert av.stride(0) == 11 and bv.stride(0) == 14
    for mode in (0, 1):
        ratio, got, _ = _pairwise_check(av, bv, mode, "strided")
        assert ratio.max() <= 1.0
        import rotate_yolov3_b200 as pkg
        dense = pkg.rotated_iou_matrix(av[:, :5].contiguous(), bv[:, :5].contiguous(), GIoU=bool(mode)).cpu().numpy()
        assert np.array_equal(got, dense)


def test_gradient_vs_float64_differences(run, fd):
    worst = {}
    bad = []
    zeros_bad = 0
    n_kink = n_smooth = 0
    for name, r in run.items():
        ratios, zb = _grad_checks(r, {"a": fd[name, "a"], "b": fd[name, "b"]})
        zeros_bad += zb
        for which, ratio in zip("ab", ratios):
            _report("grad d/d" + which, name, ratio)
            worst[name, which] = float(ratio.max()) if ratio.size else 0.0
            if not worst[name, which] <= 1.0:
                i, k = np.unravel_index(np.argmax(ratio), ratio.shape)
                bad.append((name, which, worst[name, which], int(i), int(k)))
        assert np.array_equal(r["ga"], r["ga_only"]) and np.array_equal(r["gb"], r["gb_only"])
    for name in run:
        for which in "ab":
            f = fd[name, which]
            sm = np.abs(f["dp1"] - f["dm1"]) <= 2.5 * np.maximum(np.abs(f["dp2"] - f["dp1"]),
                                                                  np.abs(f["dm2"] - f["dm1"])) + f["rnd"]
            n_kink += int((~sm).sum())
            n_smooth += int(sm.sum())
    print("\nriou gradient: %d smooth components, %d on kinks" % (n_smooth, n_kink))
    assert zeros_bad == 0
    assert not bad, bad
    assert n_kink > 500                                     # the families do sit on kinks


def test_gradient_zero_and_finite_on_dead_pairs(run):
    r = run["F5 scale"]
    dead = ~_live(r["a"], r["b"])
    assert dead.sum() >= 23
    for g in (r["ga"], r["gb"]):
        assert np.isfinite(g).all()
        assert (g[dead] == 0).all(), g[dead]
    assert (r["grad_val"][dead] == 0).all()
    n_sep = 0
    for name in ("F4 slivers", "F6 far"):                 # gaps of 1e-6 .. 1e-1 of the box size
        r = run[name]
        sep = separated(r["a"], r["b"])
        n_sep += int(sep.sum())
        assert (r["ga"][sep] == 0).all() and (r["gb"][sep] == 0).all() and (r["grad_val"][sep] == 0).all()
    assert n_sep >= 500


def test_bound_self_test(run, fd):
    """plausible bugs put into stored outputs: each check must fail"""
    import rotate_yolov3_b200 as pkg
    name = "F7 generic"
    r = run[name]
    fdd = {"a": fd[name, "a"], "b": fd[name, "b"]}

    def worst(**kw):
        ratios, zb = _grad_checks(r, fdd, **kw)
        return max(float(x.max()) for x in ratios), zb

    base, zb = worst()
    assert base <= 1.0 and zb == 0
    a64, b64 = r["a"].astype(np.float64), r["b"].astype(np.float64)
    rel_a, rel_b = a64.copy(), b64.copy()
    rel_b[:, :2] -= a64[:, :2]
    rel_a[:, :2] = 0.0
    # 1. one edge's term dropped from ga (a pair with weight 1 and a partly clipped edge)
    _, _, contrib = edge_geometry(rel_a, rel_b)
    iou = r["want"]
    tot = np.abs(a64[:, 2] * a64[:, 3]) + np.abs(b64[:, 2] * b64[:, 3])
    I = iou * tot / (1 + iou)
    U = tot - I
    k1 = r["wt"] * (U + I) / U ** 2
    found = 0
    for i in np.flatnonzero((r["wt"] != 0) & (iou > 0.05))[:40]:
        e = int(np.argmax(np.abs(contrib[i, :, 4])))
        ga = r["ga"].copy()
        ga[i] -= (k1[i] * contrib[i, e] * np.array([1, 1, np.sign(r["a"][i, 2]), np.sign(r["a"][i, 3]), 1])).astype(F32)
        found += worst(ga=ga)[0] > 1.0
    assert found >= 35, found
    # 2. theta components scaled by 1 + 1e-3
    ga = r["ga"].copy()
    ga[:, 4] *= F32(1.001)
    assert worst(ga=ga)[0] > 1.0
    # 3. ga and gb swapped
    assert worst(ga=r["gb"], gb=r["ga"])[0] > 1.0
    # 4. sign(w) ignored (F3 holds negative widths and heights)
    r3 = run["F3 angles"]
    neg = r3["a"][:, 2] < 0
    assert neg.sum() >= 12
    ga = r3["ga"].copy()
    ga[neg, 2] *= -1
    ratios, _ = _grad_checks(r3, {"a": fd["F3 angles", "a"], "b": fd["F3 angles", "b"]}, ga=ga)
    assert ratios[0].max() > 1.0
    # 5. one overlapping pair culled to 0 in a pairwise tile
    rows, cols = _full_tile()
    got = pkg.rotated_iou_matrix(torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda()).cpu().numpy()
    want = helpers.orc_skew_pairwise(rows, cols, 0).astype(np.float64)
    assert value_ratio(got, want).max() <= 1.0
    got[17, 77] = 0.0
    assert value_ratio(got, want).max() > 1.0
    # 6. the paired kernel's value replaced by its fp32 intersection over a's area
    p = r["paired"]
    aa = np.abs(r["a"][:, 2] * r["a"][:, 3])
    inter = (p * (aa + np.abs(r["b"][:, 2] * r["b"][:, 3])) / (1 + p)).astype(F32)
    assert value_ratio(inter / aa, r["want"]).max() > 1.0


def test_zz_report(run, fd):
    """prints the worst ratio per kernel and family (run with -s); runs after the checks that fill the table"""
    print("\nworst ratio (<= 1 passes)")
    for (kernel, family), v in sorted(REPORT.items()):
        print("  %-14s %-14s %.3g" % (kernel, family, v))
    assert all(v <= 1.0 for v in REPORT.values())


# ------------------------------------------------------------------------------------------------------------------
# mAP matching
# ------------------------------------------------------------------------------------------------------------------
def _greedy(iou, pcls, tcls, thr):
    """test.py:134-151 over a given IoU matrix: class-restricted first argmax, each target claimed once, stop once every
    target is claimed"""
    correct, detected, stopped = [0] * len(pcls), [], False
    for i in range(len(pcls)):
        if len(detected) == len(tcls):
            stopped = True
            break
        if float(pcls[i]) not in set(tcls.tolist()):
            continue
        m = np.flatnonzero(tcls == pcls[i])
        row = iou[i, m]
        bi = int(np.argmax(row))
        if row[bi] > thr and int(m[bi]) not in detected:
            correct[i] = 1
            detected.append(int(m[bi]))
    return correct, stopped       # stopped: the early break fired with predictions left


@pytest.mark.parametrize("t", [1, 31, 32, 33, 100, 257])
def test_match_detections_restates_greedy_loop(t):
    import rotate_yolov3_b200 as pkg
    from rotate_yolov3_b200.metrics import match_detections
    g = np.random.default_rng(t)
    tb = helpers.gen_boxes(t, 300 + t, 300.0).numpy()
    tcls = g.integers(0, 3, t).astype(F32)
    if t > 1:                                           # duplicate targets: ties within a lane's stride and across lanes
        nd = max(1, t // 4)
        src = g.integers(0, t, nd)
        dst = (src + g.choice([1, 32, 33, 64], nd)) % t
        tb[dst] = tb[src]
        tcls[dst] = tcls[src]
    p = 3 * t + 7
    pick = g.integers(0, t, p)
    pb = tb[pick] + g.normal(0, 1, (p, 5)).astype(F32) * np.array([2, 2, 2, 2, 0.02], F32)
    pb[: t // 3 + 1] = tb[pick[: t // 3 + 1]]           # exact copies: IoU 1 ties with duplicates
    pb[-(p // 5):] = helpers.gen_boxes(p // 5, 7 + t, 300.0).numpy()
    pcls = np.where(g.random(p) < 0.8, tcls[pick], g.integers(0, 5, p)).astype(F32)   # classes 3, 4 have no targets
    conf = np.sort(g.random(p).astype(F32))[::-1]
    pred = np.concatenate([pb, conf[:, None], np.ones((p, 1), F32), pcls[:, None]], 1).astype(F32)
    pd = torch.from_numpy(pred).cuda()
    iou = pkg.rotated_iou_matrix(pd[:, :5].contiguous(), torch.from_numpy(tb).cuda()).cpu().numpy()
    present = np.unique(iou[(iou > 0.05) & (iou < 0.99)])
    thresholds = [0.5, float(present[len(present) // 2]) if len(present) else 0.3, 0.0]
    for thr in thresholds:
        want, _ = _greedy(iou, pcls, tcls, F32(thr))
        got = match_detections(pd, torch.from_numpy(tb).cuda(), torch.from_numpy(tcls).cuda(), iou_thres=thr)
        assert got == want, (t, thr)
    # the early stop: distinct targets, each matched by an exact copy in order, then predictions that would still match
    tu = helpers.gen_boxes(t, 900 + t, 300.0 * max(1, t) ** 0.5).numpy()
    tu_cls = g.integers(0, 3, t).astype(F32)
    order = np.concatenate([np.arange(t), g.integers(0, t, 5)])
    pred2 = np.concatenate([tu[order], np.ones((len(order), 2), F32), tu_cls[order, None]], 1).astype(F32)
    iou2 = pkg.rotated_iou_matrix(torch.from_numpy(pred2[:, :5]).cuda(), torch.from_numpy(tu).cuda()).cpu().numpy()
    want, stopped = _greedy(iou2, pred2[:, 7], tu_cls, F32(0.5))
    assert stopped and sum(want) == t
    got = match_detections(torch.from_numpy(pred2).cuda(), torch.from_numpy(tu).cuda(), torch.from_numpy(tu_cls).cuda(),
                           iou_thres=0.5)
    assert got == want
    # P = 0, T = 0
    assert match_detections(pd[:0], torch.from_numpy(tb).cuda(), torch.from_numpy(tcls).cuda()) == []
    assert match_detections(pd, torch.zeros((0, 5)).cuda(), torch.zeros(0).cuda()) == [0] * p


# ------------------------------------------------------------------------------------------------------------------
# wide rows through backward, and the out= contract of rotated_iou_matrix
# ------------------------------------------------------------------------------------------------------------------
def test_riou_loss_backpropagates_through_wide_and_strided_rows():
    from rotate_yolov3_b200.iou import riou_loss, rotated_iou
    a, b = overlapping_pairs(64, 31)
    a7 = torch.cat([a, torch.randn(64, 2)], 1).cuda()
    b7 = torch.cat([b, torch.randn(64, 2)], 1).cuda()
    w = torch.linspace(-1, 1, 64).cuda()
    a5, b5 = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    (rotated_iou(a5, b5) * w).sum().backward()
    pa, pb = a7.clone().requires_grad_(True), b7.clone().requires_grad_(True)
    (rotated_iou(pa, pb) * w).sum().backward()
    assert pa.grad.shape == (64, 7) and pb.grad.shape == (64, 7)
    assert torch.equal(pa.grad[:, :5], a5.grad) and torch.equal(pb.grad[:, :5], b5.grad)
    assert not pa.grad[:, 5:].any() and not pb.grad[:, 5:].any()
    # riou_loss on [N, 7] rows, float64 rows, and non-contiguous views (column slice, transposed storage)
    pd = a7.double().requires_grad_(True)
    riou_loss(pd, b7.double()).backward()
    assert pd.grad.dtype == torch.float64 and pd.grad.shape == (64, 7) and not pd.grad[:, 5:].any()
    buf = torch.randn(64, 9).cuda()
    buf[:, 1:6] = a.cuda()
    leaf = buf.clone().requires_grad_(True)
    tr = b7.t().contiguous().requires_grad_(True)          # [7, N]; tr.t() is a non-contiguous [N, 7]
    loss = riou_loss(leaf[:, 1:8], tr.t(), reduction="sum")
    loss.backward()
    ref_a, ref_b = a.cuda().requires_grad_(True), b.cuda().requires_grad_(True)
    riou_loss(ref_a, ref_b, reduction="sum").backward()
    assert torch.equal(leaf.grad[:, 1:6], ref_a.grad) and not leaf.grad[:, 0].any() and not leaf.grad[:, 6:].any()
    assert torch.equal(tr.grad.t()[:, :5], ref_b.grad) and not tr.grad[5:].any()


def test_rotated_iou_matrix_rejects_a_bad_out():
    import rotate_yolov3_b200 as pkg
    a, b = helpers.gen_boxes(20, 1, 100.0).cuda(), helpers.gen_boxes(12, 2, 100.0).cuda()
    want = pkg.rotated_iou_matrix(a, b)
    out = torch.empty(20, 12).cuda()
    assert pkg.rotated_iou_matrix(a, b, out=out) is out and torch.equal(out, want)
    # every bad buffer below is at least as large as [N, M] fp32, so even an unchecked write would stay in bounds
    for bad in (torch.zeros(20, 12, dtype=torch.float64).cuda(),      # float64
                torch.zeros(12, 20).cuda().t(),                        # transposed view
                torch.zeros(20, 15).cuda()[:, :12],                    # column slice of a wider buffer
                torch.zeros(21, 12).cuda()):                           # [N + 1, M]
        keep = bad.clone()
        with pytest.raises(ValueError):
            pkg.rotated_iou_matrix(a, b, out=bad)
        assert torch.equal(bad, keep)
