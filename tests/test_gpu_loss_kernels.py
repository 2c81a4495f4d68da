"""Kernel-level tests of the MMPI loss path (csrc/loss.cu: di_match_cost_f32, di_hungarian_f32, di_heuristic_assign_f32,
di_loss_targets_f32, di_gaussian_heatmap_f32, di_mmpi_losses_f32) against references written from each operation's
definition, at the inputs where this code branches: coincident and touching box edges, tied assignment costs, map
borders, saturated logits and clamps.  The C entry points are called directly; every output goes into a SENT-filled
canvas (accumulators into a zeroed one with SENT pads), and every word outside the output must keep its bits.
U = 2^-24 is the fp32 unit roundoff.

Rotated IoU.  The float64 reference is not the kernel's algorithm (Sutherland-Hodgman clipping of one rectangle by the
other, which oracle/loss.py also uses) but a line integral: the area of A n B is the sum of x dy along the pieces of
A's edges inside B and of B's edges inside A, each edge clipped Cyrus-Beck style.  A piece lying on the other box's
edge line counts once, from A, when the two edges run the same way, and not at all when they run opposite ways (boxes
touching along an edge).  The reference is itself checked against closed forms (axis-aligned dyadic boxes, concentric
boxes of one yaw) and against oracle.loss.rotated_intersection_area on random boxes.  Kernel bar: the kernel rounds A's
corners relative to B's centre (centre difference 1 U, cosf / sinf 2 ulp, two products and two adds: <= 8 U S, with
S = |centre distance| + R_A + R_B and R the half diagonals); a corner or clipped point moved by e changes the area by at
most e times the intersection's perimeter (<= 4 S), and the shoelace sum of <= 8 cross products of coordinates <= S
rounds by <= 32 U S^2: 64 U S^2 on the area.  IoU = o3 / union moves by at most 2 oh darea / union, and its own fp32
steps by 8 U: bar = 128 U S^2 oh / union + 8 U.  Identical boxes must give 1 within that bar.

Matching cost.  FocalLossCost takes p = sigmoid(x) in fp32, as the reference's tensors do: the reference restates that
rounding (p = fp32(sigmoid64(x))) and then follows the definition in float64.  The kernel's p = 1 / (1 + expf(-x)) is
within 4 U p of it, and equal where p rounds to exactly 1 (x >= 30 here).  One exception: at x = -100, expf(100)
overflows and the kernel's p is 0 where the reference's is a denormal near 3.6e-44; both give log(p + eps) = log(eps)
and (1 - p)^gamma = 1, and the p^gamma of the other term changes by less than 1e-80, far inside the bar.  The cost bar
is the change of the cost over p +- 4 U p, plus 8 U of each log / pow term; the BEV L1 cost has two divisions per
coordinate (4 U of each quotient), the 3-D L1 cost one fp32 sum of nb terms (nb U); the total adds 2 U of each part
and iou_w times the IoU bar.

Hungarian assignment.  scipy.optimize.linear_sum_assignment is the reference's own solver, so it is the reference here,
ties included: on costs of small integers, constant and duplicated rows, at G <, ==, > P and past the 32-lane loops, the
kernel's gt_inds must equal scipy's, its float64 total must equal scipy's exactly, and max_overlaps must be the bits of
the matched pairs' IoUs.  Padded cost and IoU columns (j >= n_gt) hold NaN.

Heuristic assignment.  Centres on an integer grid make every squared distance an exact fp32 integer, so the kernel's
sqrtf and the reference's fp32 sqrt round the same value, and ties and the `<= dist_thre` test are exact.  The reference
is a plain restatement of hungarian_assigner.py:60-91 (first minimum, earlier box wins a tie, claims nearer than the
10000 an unclaimed prediction starts with).  Overlaps: the IoU bar above.

Targets.  Labels, label weights, bbox weights, clamped IoUs, num_pos and pos_cnt are exact.  Encoded boxes are within
2 ulp of float64 (a subtraction and a division; logf 1 ulp, sinf / cosf 2 ulp).  iou_sum is accumulated with float
atomics in no fixed order, so it is not bit-reproducible: bar (n - 1) U sum|ov|.

Heat map.  The radius is oracle.loss.gaussian_radius on the fp32 width and length, as the reference computes it; the
window is oracle.loss.draw_heatmap_gaussian with Python's slicing (negative stops included), the values float64
gaussian_2d rounded to fp32.  The map must be equal bit for bit.

Losses.  Each output is held to its float64 sum: clip_sigmoid's clamp [1e-4, 1 - 1e-4] and the sigmoid focal loss's
max(., FLT_MIN) are restated on the fp32 p; each term gets 16 U of its magnitude plus its change when the sigmoid,
before the clamp, moves by +- 4 U of itself (the fp32 1 - p is ill conditioned just inside the clamp, where this
dominates; a p the clamp pins, such as every logit of +-30 or +-100, is exact), the box L1 terms 16 U; the per-block
double sums add nothing that matters.  Every bar must stay below 1e-5 of its output, so that a dropped or repeated
element of a grid-stride loop shows.  Two calls on the same inputs must give the same bits.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from kernel_check import SENT, _capi, same_bits

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
FLT_MIN = float(np.finfo(np.float32).tiny)
SENT64 = (SENT << 32) | SENT
PC = (-54.0, -54.0, -5.0, 54.0, 54.0, 3.0)


def dev():
    return torch.device('cuda:0')


def _p(t):
    from deepinteraction_b200 import ops
    return ops._ptr(t)


def _f(vals):
    return (ctypes.c_float * len(vals))(*[float(v) for v in vals])


def f32(x):
    return np.float64(np.float32(x))


class Canvas:
    """n words of `dtype` at offset `pad` of a buffer whose other words hold SENT (SENT64 for int64); `fill` sets the
    words of the view (zeros for the accumulators the entry points add into)."""

    def __init__(self, n, dtype=torch.float32, fill=None, pad=16):
        self.n, self.pad, self.dtype = n, pad, dtype
        wide = dtype in (torch.int64, torch.float64)
        self.buf = torch.full((n + 2 * pad,), SENT64 if wide else SENT, dtype=torch.int64 if wide else torch.int32,
                              device=dev()).view(dtype)
        self.view = self.buf[pad:pad + n]
        if fill is not None:
            self.view.fill_(fill)

    def intact(self):
        b = self.buf.view(torch.int64 if self.dtype in (torch.int64, torch.float64) else torch.int32)
        s = SENT64 if b.dtype == torch.int64 else SENT
        return bool((b[:self.pad] == s).all()) and bool((b[self.pad + self.n:] == s).all())


# ---------------------------------------------------------------------------------------------------------------------
# float64 references: rotated intersection by a line integral, 3-D IoU
# ---------------------------------------------------------------------------------------------------------------------
def corners64(b):
    """[N, 5] (x, y, dx, dy, yaw) -> [N, 4, 2] corners, counter-clockwise; x' = x cos + y sin, y' = -x sin + y cos."""
    x, y, dx, dy, r = (b[:, k] for k in range(5))
    c, s = np.cos(r), np.sin(r)
    out = np.empty((b.shape[0], 4, 2))
    for k, (sx, sy) in enumerate(((-1, -1), (1, -1), (1, 1), (-1, 1))):
        lx, ly = sx * dx / 2, sy * dy / 2
        out[:, k, 0] = lx * c + ly * s + x
        out[:, k, 1] = -lx * s + ly * c + y
    return out


def _edge_integral(P, Q, own):
    """sum over the edges of P of the integral of x dy along the part of the edge inside the convex CCW polygon Q
    (Cyrus-Beck).  A part on an edge line of Q is kept only when `own` and the two edges run the same way."""
    p0 = P
    d = np.roll(P, -1, axis=1) - P                                          # [N, 4, 2]
    n = P.shape[0]
    tmin, tmax = np.zeros((n, 4)), np.ones((n, 4))
    keep = np.ones((n, 4), bool)
    for f in range(4):
        q0 = Q[:, f][:, None]
        e = (Q[:, (f + 1) % 4] - Q[:, f])[:, None]                           # [N, 1, 2]
        num = e[..., 0] * (p0[..., 1] - q0[..., 1]) - e[..., 1] * (p0[..., 0] - q0[..., 0])
        den = e[..., 0] * d[..., 1] - e[..., 1] * d[..., 0]
        par = den == 0
        same = (e[..., 0] * d[..., 0] + e[..., 1] * d[..., 1]) > 0
        keep &= ~(par & (num < 0))
        keep &= ~(par & (num == 0) & ~(same & own))
        t = np.where(par, 0.0, -num / np.where(par, 1.0, den))
        tmin = np.where(~par & (den > 0), np.maximum(tmin, t), tmin)
        tmax = np.where(~par & (den < 0), np.minimum(tmax, t), tmax)
    keep &= tmin < tmax
    a, b = p0 + tmin[..., None] * d, p0 + tmax[..., None] * d
    return np.where(keep, 0.5 * (a[..., 0] + b[..., 0]) * (b[..., 1] - a[..., 1]), 0.0).sum(1)


def bev_area64(a5, b5):
    """Intersection area of rectangles a5[i] and b5[i] ([N, 5] float64), in b's own frame: b's edges are then exact, and
    an edge of a of the same yaw is exactly parallel to them."""
    a5, b5 = np.array(a5, np.float64), np.array(b5, np.float64)
    c, s = np.cos(b5[:, 4]), np.sin(b5[:, 4])
    dx, dy = a5[:, 0] - b5[:, 0], a5[:, 1] - b5[:, 1]
    a5 = np.c_[c * dx - s * dy, s * dx + c * dy, a5[:, 2:4], a5[:, 4] - b5[:, 4]]
    b5 = np.c_[np.zeros((len(b5), 2)), b5[:, 2:4], np.zeros(len(b5))]
    A, B = corners64(a5), corners64(b5)
    area = _edge_integral(A, B, True) + _edge_integral(B, A, False)
    return np.where((a5[:, 2] * a5[:, 3] == 0) | (b5[:, 2] * b5[:, 3] == 0), 0.0, area)    # a flat box has no area


def iou3d64(p, g):
    """3-D IoU of the pairs p[i], g[i] ([N, >= 7], x, y, z_bottom, dx, dy, dz, yaw) -> (iou, bar)."""
    p, g = np.asarray(p, np.float64), np.asarray(g, np.float64)
    oh = np.maximum(np.minimum(p[:, 2] + p[:, 5], g[:, 2] + g[:, 5]) - np.maximum(p[:, 2], g[:, 2]), 0.0)
    area = bev_area64(p[:, [0, 1, 3, 4, 6]], g[:, [0, 1, 3, 4, 6]])
    o3 = area * oh
    union = np.maximum(p[:, 3] * p[:, 4] * p[:, 5] + g[:, 3] * g[:, 4] * g[:, 5] - o3, f32(1e-8))
    S = np.hypot(p[:, 0] - g[:, 0], p[:, 1] - g[:, 1]) + 0.5 * (np.hypot(p[:, 3], p[:, 4]) + np.hypot(g[:, 3], g[:, 4]))
    return o3 / union, 128 * U * S * S * oh / union + 8 * U


def test_line_integral_reference_matches_closed_forms_and_oracle():
    """The IoU reference against exact areas (axis-aligned dyadic boxes, concentric boxes of one yaw) and against the
    oracle's clipping on random boxes, which also pins the yaw convention."""
    import oracle.loss as ol
    rng = np.random.default_rng(5)
    # axis-aligned, dyadic: the exact overlap is the product of the interval overlaps (the clip parameters t round)
    a = np.c_[rng.integers(-16, 16, (200, 2)) / 8, rng.integers(1, 24, (200, 2)) / 4, np.zeros(200)]
    b = np.c_[rng.integers(-16, 16, (200, 2)) / 8, rng.integers(1, 24, (200, 2)) / 4, np.zeros(200)]
    ov = lambda c0, w0, c1, w1: np.maximum(np.minimum(c0 + w0 / 2, c1 + w1 / 2) - np.maximum(c0 - w0 / 2, c1 - w1 / 2), 0)
    want = ov(a[:, 0], a[:, 2], b[:, 0], b[:, 2]) * ov(a[:, 1], a[:, 3], b[:, 1], b[:, 3])
    assert np.abs(bev_area64(a, b) - want).max() < 1e-13
    # concentric boxes of one yaw (nested, crossed, equal): min(dx) * min(dy)
    yaw = rng.uniform(-4, 4, 100)
    a = np.c_[rng.uniform(-50, 50, (100, 2)), rng.integers(1, 9, (100, 2)) / 2, yaw]
    b = np.c_[a[:, :2], rng.integers(1, 9, (100, 2)) / 2, yaw]
    want = np.minimum(a[:, 2], b[:, 2]) * np.minimum(a[:, 3], b[:, 3])
    assert np.abs(bev_area64(a, b) - want).max() < 1e-12 * 64
    # random boxes: the oracle's Sutherland-Hodgman clipping
    a = np.c_[rng.uniform(-3, 3, (300, 2)), rng.uniform(0.5, 5, (300, 2)), rng.uniform(-4, 4, 300)]
    b = np.c_[rng.uniform(-3, 3, (300, 2)), rng.uniform(0.5, 5, (300, 2)), rng.uniform(-4, 4, 300)]
    got = bev_area64(a, b)
    want = np.array([ol.rotated_intersection_area(a[i:i + 1], b[i:i + 1])[0, 0] for i in range(300)])
    assert np.abs(got - want).max() < 1e-12 and (got > 0.5).sum() > 50


# ---------------------------------------------------------------------------------------------------------------------
# 1. rotated 3-D IoU and matching costs (di_match_cost_f32)
# ---------------------------------------------------------------------------------------------------------------------
def box(x, y, dx, dy, yaw, z=-1.0, dz=1.5, v=(0.5, -0.25)):
    return [x, y, z, dx, dy, dz, yaw, v[0], v[1]]


def iou_pairs():
    """(pred, gt, exact IoU or None) -- the edge cases of the rotated intersection."""
    pi = math.pi
    cases = []
    for k, yaw in enumerate((0.0, pi / 2, -pi / 2, pi, -pi, 0.3, -2.9, 1e-7, 2.0 * pi, 1.1)):
        x, y = (54.0, -54.0) if k % 2 else (-53.75, 37.5 + k)
        cases.append((box(x, y, 4.0, 1.75, yaw), box(x, y, 4.0, 1.75, yaw), 1.0))            # identical
        cases.append((box(x, y, 4.5, 2.0, yaw + pi), box(x, y, 4.5, 2.0, yaw), 1.0))        # yaw + pi
        cases.append((box(x, y, 2.0, 4.5, yaw + pi / 2), box(x, y, 4.5, 2.0, yaw), 1.0))    # swapped, + pi / 2
    # concentric, nested with shared edges (same dx, or same dy), yaw 0 and odd
    for yaw in (0.0, 0.7, -pi / 2):
        cases.append((box(10.0, 5.0, 4.0, 2.0, yaw), box(10.0, 5.0, 4.0, 1.0, yaw), 0.5))
        cases.append((box(-7.0, 3.0, 2.0, 3.0, yaw), box(-7.0, 3.0, 1.0, 3.0, yaw), 0.5))
        cases.append((box(1.0, 1.0, 2.0, 2.0, yaw), box(1.0, 1.0, 4.0, 1.0, yaw), 1.0 / 3.0))
    # touching along an edge, at a corner, and one box shifted half its length along the shared edge line
    cases.append((box(0.0, 0.0, 2.0, 2.0, 0.0), box(2.0, 0.0, 2.0, 2.0, 0.0), 0.0))
    cases.append((box(0.0, 0.0, 2.0, 2.0, 0.0), box(2.0, 2.0, 2.0, 2.0, 0.0), 0.0))
    cases.append((box(0.0, 0.0, 2.0, 2.0, 0.0), box(2.0, 1.0, 2.0, 2.0, 0.0), 0.0))
    cases.append((box(0.0, 0.0, 2.0, 2.0, 0.0), box(1.0, 1.0, 2.0, 2.0, 0.0), 1.0 / 7.0))
    cases.append((box(5.0, 5.0, 3.0, 1.0, 0.9), box(5.0 + 2.0 * math.sin(0.9), 5.0 + 2.0 * math.cos(0.9), 3.0, 3.0, 0.9), None))
    # corners pointing at each other along the diagonal, centres t (R_A + R_B) apart: the circumscribed circles (the
    # kernel's rejection test) just apart, just overlapping, corners overlapping by 0.15 x 0.075 m, by half the boxes
    for t in (1.0 + 1e-6, 1.0 - 1e-6, 0.95, 0.5):
        d = t * (math.hypot(2.0, 1.0) + math.hypot(4.0, 2.0)) / (2.0 * math.sqrt(5.0))
        cases.append((box(0.0, 0.0, 2.0, 1.0, 0.0), box(2.0 * d, d, 4.0, 2.0, 0.0), None))
    # height: touching in z, overlapping in z
    cases.append((box(3.0, 3.0, 2.0, 2.0, 0.2, z=0.0, dz=1.0), box(3.0, 3.0, 2.0, 2.0, 0.2, z=1.0, dz=1.0), 0.0))
    cases.append((box(3.0, 3.0, 2.0, 2.0, 0.2, z=0.0, dz=1.0), box(3.0, 3.0, 2.0, 2.0, 0.2, z=0.5, dz=1.0), 1.0 / 3.0))
    # zero-volume boxes: the union's 1e-8 clamp
    cases.append((box(1.0, 1.0, 0.0, 2.0, 0.0), box(1.0, 1.0, 0.0, 2.0, 0.0), 0.0))
    cases.append((box(1.0, 1.0, 2.0, 2.0, 0.0, dz=0.0), box(1.0, 1.0, 2.0, 2.0, 0.0, dz=0.0), 0.0))
    # thin boxes, aspect ratio 100: crossed, parallel and offset, identical at odd yaws
    cases.append((box(-20.0, 8.0, 10.0, 0.1, 0.4), box(-20.0, 8.0, 10.0, 0.1, 0.4 + pi / 2), None))
    cases.append((box(-20.0, 8.0, 10.0, 0.1, 0.4), box(-20.0 + 0.05 * math.sin(0.4), 8.0 + 0.05 * math.cos(0.4), 10.0, 0.1, 0.4), None))
    cases.append((box(33.3, -41.7, 10.0, 0.1, 2.2), box(33.3, -41.7, 10.0, 0.1, 2.2), 1.0))
    cases.append((box(33.3, -41.7, 0.1, 10.0, -0.8), box(33.3, -41.7, 10.0, 0.1, -0.8 + pi / 2), 1.0))
    return cases


LOGITS = (0.0, -0.0, 5.0, -5.0, 30.0, -30.0, 100.0, -100.0)


def cost_ref(pred, score, gt, lab, cp):
    """float64 cost of every (pred, gt) pair: FocalLossCost on fp32 sigmoid, BEV / 3-D L1, IoU3DCost -> (cost, bar)."""
    cls_w, alpha, gamma, eps, reg_w, kind, iou_w = cp[:7]
    x0, y0, xr, yr = cp[7:]
    x = score.astype(np.float64)[lab].T                                      # [P, G] logit of each gt's class
    p = f32(1.0 / (1.0 + np.exp(-x)))
    dp = np.where(p < 1.0, 4 * U * p, 0.0)

    def cls(p):
        neg = -np.log(1 - p + f32(eps)) * (1 - alpha) * p ** gamma
        pos = -np.log(p + f32(eps)) * alpha * (1 - p) ** gamma
        return (pos - neg) * cls_w, (np.abs(pos) + np.abs(neg)) * abs(cls_w)
    c_cls, mag = cls(p)
    cb = np.maximum(np.abs(cls(np.minimum(p + dp, 1.0))[0] - c_cls), np.abs(cls(np.maximum(p - dp, 0.0))[0] - c_cls)) + 8 * U * mag
    P, G = pred.astype(np.float64), gt.astype(np.float64)
    if kind == 0:
        qx, qy = (P[:, 0] - x0) / xr, (P[:, 1] - y0) / yr
        gx, gy = (G[:, 0] - x0) / xr, (G[:, 1] - y0) / yr
        c_reg = np.abs(qx[:, None] - gx) + np.abs(qy[:, None] - gy)
        rb = 4 * U * (np.abs(qx[:, None]) + np.abs(gx) + np.abs(qy[:, None]) + np.abs(gy))
    else:
        c_reg = np.abs(P[:, None, :] - G[None]).sum(-1)
        rb = P.shape[1] * U * (np.abs(P[:, None, :]) + np.abs(G[None])).sum(-1)
    c_reg, rb = c_reg * reg_w, rb * reg_w
    ii = np.repeat(np.arange(P.shape[0]), G.shape[0])
    jj = np.tile(np.arange(G.shape[0]), P.shape[0])
    u, ub = (t.reshape(P.shape[0], G.shape[0]) for t in iou3d64(P[ii], G[jj]))
    cost = c_cls + c_reg - u * iou_w
    bar = cb + rb + ub * iou_w + 2 * U * (np.abs(c_cls) + np.abs(c_reg) + np.abs(u * iou_w))
    return cost, bar, u, ub


@pytest.mark.parametrize('nb,kind', [(9, 0), (9, 1), (7, 0), (7, 1)])
def test_match_cost_edges(nb, kind):
    """Every (pred, gt) pair of two samples: the IoU edge cases on the diagonal, random boxes around them; logits at
    +-0, +-5, +-30, +-100; LP = 150 (two 128-blocks, the second partial); the second sample has n_gt < Gmax with
    NaN-filled ground-truth rows, which must never be read (their cost and IoU words keep SENT)."""
    rng = np.random.default_rng(17 + nb + kind)
    pairs = iou_pairs()
    K, LP, B = 10, 150, 2
    n_pairs = len(pairs)
    Gmax = n_pairs
    n_gt = [n_pairs, 23]
    preds = np.zeros((B, LP, 9), np.float32)
    gts = np.full((B, Gmax, 9), np.nan, np.float32)
    for b in range(B):
        preds[b] = np.c_[rng.uniform(-40, 40, (LP, 2)), rng.uniform(-2, 0, LP), rng.uniform(0.5, 5, (LP, 3)),
                         rng.uniform(-3.2, 3.2, LP), rng.normal(size=(LP, 2))]
        order = rng.permutation(n_pairs) if b else np.arange(n_pairs)
        for j in range(n_gt[b]):
            pr, g, _ = pairs[order[j]]
            preds[b, 7 + j], gts[b, j] = pr, g
        # a few predictions right on top of a ground-truth box, so the sums mix non-zero IoUs
        preds[b, 120:130] = gts[b, :10] + rng.normal(size=(10, 9)).astype(np.float32) * 0.2
        preds[b, 120:130, 3:6] = np.abs(preds[b, 120:130, 3:6]) + 0.5
    labels = np.zeros((B, Gmax), np.int32)
    for b in range(B):
        labels[b, :n_gt[b]] = rng.integers(0, K, n_gt[b])
    score = rng.choice(LOGITS, (B, K, LP)).astype(np.float32)
    score[:, :, ::3] = rng.normal(size=(B, K, (LP + 2) // 3)) * 2
    cp = (2.0, 0.25, 2.0, 1e-12, 0.25, kind, 0.25, PC[0], PC[1], PC[3] - PC[0], PC[4] - PC[1])
    pd = torch.from_numpy(preds[:, :, :nb].copy()).to(dev())
    gd = torch.from_numpy(gts[:, :, :nb].copy()).to(dev())
    sd, ld, nd = torch.from_numpy(score).to(dev()), torch.from_numpy(labels).to(dev()), torch.tensor(n_gt, dtype=torch.int32, device=dev())
    cost, iou = Canvas(B * LP * Gmax), Canvas(B * LP * Gmax)
    _capi('di_match_cost_f32', _p(pd), nb, _p(sd), K, _p(gd), _p(ld), _p(nd), B, LP, Gmax, _f(cp), _p(cost.view), _p(iou.view))
    assert cost.intact() and iou.intact()
    cg, ig = cost.view.view(B, LP, Gmax).cpu(), iou.view.view(B, LP, Gmax).cpu()
    for b in range(B):
        G = n_gt[b]
        pad_c, pad_i = cg[b, :, G:].view(torch.int32), ig[b, :, G:].view(torch.int32)
        assert bool((pad_c == SENT).all()) and bool((pad_i == SENT).all())
        want, bar, u, ub = cost_ref(preds[b, :, :nb], score[b], gts[b, :G, :nb], labels[b, :G], cp)
        gi, gc = ig[b, :, :G].double().numpy(), cg[b, :, :G].double().numpy()
        assert np.isfinite(gi).all() and np.isfinite(gc).all()
        bad = np.argwhere(np.abs(gi - u) > ub)
        assert bad.size == 0, [(i, j, gi[i, j], u[i, j], ub[i, j]) for i, j in bad[:8]]
        bad = np.argwhere(np.abs(gc - want) > bar)
        assert bad.size == 0, [(i, j, gc[i, j], want[i, j], bar[i, j]) for i, j in bad[:8]]
        print(f'sample {b}: IoU worst |err| / bar {float((np.abs(gi - u) / ub).max()):.3f}, '
              f'cost worst |err| / bar {float((np.abs(gc - want) / bar).max()):.3f}')
        if b == 0:                 # the case pairs: exact values, where a closed form gives one
            for j, (_, _, ex) in enumerate(pairs):
                if ex is not None:
                    assert abs(gi[7 + j, j] - ex) <= ub[7 + j, j], (j, gi[7 + j, j], ex)
    assert (ig[0, 7:7 + n_pairs, :n_pairs].diagonal() > 0.99).sum() >= 32


def test_iou_yaw_convention_matches_oracle():
    """One generic, asymmetric configuration against oracle.loss.BboxOverlaps3D: a mirrored yaw would change every value."""
    import oracle.loss as ol
    p = torch.tensor([box(0.3, 0.2, 4.0, 1.5, 0.6), box(-0.4, 0.5, 3.0, 1.0, -1.2), box(0.0, -0.6, 5.0, 2.0, 2.5)])
    g = torch.tensor([box(0.0, 0.0, 4.2, 1.8, 0.35), box(0.5, -0.2, 2.5, 2.5, -0.9)])
    want = ol.BboxOverlaps3D()(p.double(), g.double())
    mirror = ol.BboxOverlaps3D()(p.double() * torch.tensor([1.0] * 6 + [-1.0, 1.0, 1.0], dtype=torch.float64), g.double())
    assert float((want - mirror).abs().min()) > 0.005
    B, LP, G, K = 1, 3, 2, 2
    cost, iou = Canvas(LP * G), Canvas(LP * G)
    pd, gd = p[None].contiguous().to(dev()), g[None].contiguous().to(dev())
    sd = torch.zeros(B, K, LP, device=dev())
    ld, nd = torch.zeros(B, G, dtype=torch.int32, device=dev()), torch.tensor([G], dtype=torch.int32, device=dev())
    _capi('di_match_cost_f32', _p(pd), 9, _p(sd), K, _p(gd), _p(ld), _p(nd), B, LP, G,
          _f((1, 0.25, 2, 1e-12, 1, 0, 1) + (PC[0], PC[1], 108.0, 108.0)), _p(cost.view), _p(iou.view))
    got = iou.view.view(LP, G).double().cpu()
    assert float((got - want).abs().max()) < 2e-6 and float(want.min()) > 0.05


# ---------------------------------------------------------------------------------------------------------------------
# 2. Hungarian assignment (di_hungarian_f32)
# ---------------------------------------------------------------------------------------------------------------------
def _cost_matrix(kind, P, G, rng):
    if kind == 'int3':
        return rng.integers(0, 4, (P, G)).astype(np.float32)
    if kind == 'int1':
        return rng.integers(0, 2, (P, G)).astype(np.float32)
    if kind == 'const':
        return np.full((P, G), -1.5, np.float32)
    if kind == 'dup':              # a few distinct proposals and boxes, repeated
        base = rng.integers(-3, 4, (max(1, P // 6), max(1, G // 4))).astype(np.float32)
        return base[rng.integers(0, base.shape[0], P)][:, rng.integers(0, base.shape[1], G)]
    raise ValueError(kind)


def run_hungarian(costs, ious, n_gt, L, P):
    """costs / ious [B, L*P, Gmax] (NaN beyond n_gt) -> gt_inds [B, L*P], max_overlaps [B, L*P] (checked canvases)."""
    B, LP, Gmax = costs.shape
    cd, idv = torch.from_numpy(costs).to(dev()), torch.from_numpy(ious).to(dev())
    nd = torch.tensor(n_gt, dtype=torch.int32, device=dev())
    gi, mo = Canvas(B * LP, torch.int64), Canvas(B * LP)
    _capi('di_hungarian_f32', _p(cd), _p(idv), _p(nd), B, L, P, Gmax, _p(gi.view), _p(mo.view))
    assert gi.intact() and mo.intact()
    return gi.view.view(B, LP).cpu().numpy(), mo.view.view(B, LP).cpu()


HUNGARIAN_CASES = [
    ('int3', 20, (7, 20, 33)),
    ('int1', 40, (40, 0, 1, 39, 41)),
    ('int3', 70, (33, 70, 100, 64)),
    ('const', 35, (35, 12, 50, 1)),
    ('dup', 48, (20, 48, 60, 5)),
    ('int1', 7, (3, 7, 12)),
]


@pytest.mark.parametrize('kind,P,Gs', HUNGARIAN_CASES)
def test_hungarian_ties_match_scipy(kind, P, Gs):
    """Tied costs (small integers, constants, duplicated proposals and boxes) at G <, ==, > P, one and no box, sizes past
    the 32-lane loops, 3 layers: the assignment is scipy's, with scipy's total, and max_overlaps the matched IoUs' bits."""
    from scipy.optimize import linear_sum_assignment
    rng = np.random.default_rng(P * 31 + len(Gs))
    L, B = 3, len(Gs)
    Gmax = max(Gs) + 3
    costs = np.full((B, L * P, Gmax), np.nan, np.float32)
    ious = np.full((B, L * P, Gmax), np.nan, np.float32)
    for b, G in enumerate(Gs):
        for l in range(L):
            costs[b, l * P:(l + 1) * P, :G] = _cost_matrix(kind, P, G, rng)
            ious[b, l * P:(l + 1) * P, :G] = rng.random((P, G), np.float32)
    gi, mo = run_hungarian(costs, ious, list(Gs), L, P)
    for b, G in enumerate(Gs):
        for l in range(L):
            sl = slice(l * P, (l + 1) * P)
            c, got = costs[b, sl, :G].astype(np.float64), gi[b, sl]
            want = np.zeros(P, np.int64)
            if G:
                r, cc = linear_sum_assignment(c)
                want[r] = cc + 1
            rows = np.nonzero(got)[0]
            cols = got[rows] - 1
            assert len(rows) == min(P, G) and len(set(cols.tolist())) == len(cols) and (cols < G).all(), (b, l)
            tot = lambda m: c[np.nonzero(m)[0], m[np.nonzero(m)[0]] - 1].sum()
            assert tot(got) == tot(want), (b, l, tot(got), tot(want))
            assert np.array_equal(got, want), (b, l, np.nonzero(got != want)[0][:8])
            wov = torch.zeros(P)
            wov[torch.from_numpy(rows)] = torch.from_numpy(ious[b, sl][rows, cols])
            assert same_bits(mo[b, sl], wov)


def test_hungarian_large_problem():
    """P = 1000 proposals, 400 boxes of integer costs (shared memory 1000 x 48 bytes): scipy's assignment."""
    from scipy.optimize import linear_sum_assignment
    rng = np.random.default_rng(3)
    P, G = 1000, 400
    costs = rng.integers(0, 8, (1, P, G)).astype(np.float32)
    ious = rng.random((1, P, G), np.float32)
    gi, mo = run_hungarian(costs, ious, [G], 1, P)
    r, c = linear_sum_assignment(costs[0].astype(np.float64))
    want = np.zeros(P, np.int64)
    want[r] = c + 1
    assert np.array_equal(gi[0], want)
    assert same_bits(mo[0][torch.from_numpy(r)], torch.from_numpy(ious[0, r, c]))


# ---------------------------------------------------------------------------------------------------------------------
# 3. heuristic assignment (di_heuristic_assign_f32)
# ---------------------------------------------------------------------------------------------------------------------
def heuristic_ref(pred, gt, gl, ql, thre):
    """hungarian_assigner.py:60-91 in fp32 numpy (exact here: integer squared distances)."""
    d2 = ((pred[None, :, :2] - gt[:, None, :2]) ** 2).sum(-1).astype(np.float32)
    dist = np.sqrt(d2).astype(np.float32)
    if ql is not None:
        dist = (dist + (ql[None] != gl[:, None]).astype(np.float32) * np.float32(thre)).astype(np.float32)
    nearest = dist.argmin(1)
    P = pred.shape[0]
    inds, vals, labels = np.zeros(P, np.int64), np.full(P, 10000, np.float32), np.full(P, -1.0, np.float32)
    for g in range(gt.shape[0]):
        p = nearest[g]
        if dist[g, p] <= np.float32(thre) and dist[g, p] < vals[p]:
            vals[p], inds[p], labels[p] = dist[g, p], g + 1, gl[g]
    return inds, labels


@pytest.mark.parametrize('case', ['wrap', 'wrap_labels', 'ties', 'ties_labels', 'far'])
def test_heuristic_assign_edges(case):
    """P, G > 256 (both block loops wrap); tied nearest distances (first minimum); a distance exactly dist_thre; two boxes
    at one distance from one prediction (the earlier wins); the class penalty with and without query_labels; and a
    dist_thre above 10000, where the reference's initial 10000 decides."""
    rng = np.random.default_rng(len(case))
    if case.startswith('wrap'):
        P, G, thre = 300, 270, 5.0
        pred = np.c_[rng.integers(-60, 61, (P, 2)), rng.uniform(-2, 0, P), rng.uniform(1, 4, (P, 3)), rng.uniform(-3, 3, P)]
        gt = np.c_[rng.integers(-60, 61, (G, 2)), rng.uniform(-2, 0, G), rng.uniform(1, 4, (G, 3)), rng.uniform(-3, 3, G)]
        gt[:60, :2] = pred[rng.integers(0, P, 60), :2] + rng.choice([0, 3, 4, -3], (60, 2))
    elif case.startswith('ties'):
        # box 0 at the origin: proposals 1 and 2 both at distance 5; box 1 at (6, 8): proposal 1 at distance 5 too;
        # box 2 at (20, 0): proposal 3 at exactly dist_thre = 5; box 3 at (40, 0): proposal 4 at 5, of another class
        P, G, thre = 6, 4, 5.0
        xy = np.array([[50, 50], [3, 4], [-4, 3], [25, 0], [40, 5], [-50, -50]], np.float64)
        pred = np.c_[xy, np.full(P, -1.0), np.full((P, 3), 2.0), np.zeros(P)]
        gt = np.c_[np.array([[0, 0], [6, 8], [20, 0], [40, 0]], np.float64), np.full(G, -1.0), np.full((G, 3), 2.0), np.zeros(G)]
    else:
        # box 0's nearest proposal (3) lies 13 * 1024 > 10000 away, within dist_thre: the reference leaves it unclaimed
        P, G, thre = 5, 3, 20000.0
        pred = np.c_[np.array([[0, 0], [14, 0], [-9, 0], [0, 12], [1, 1]], np.float64) * 1024, np.full(P, -1.0),
                     np.full((P, 3), 2.0), np.zeros(P)]
        gt = np.c_[np.array([[0, 25], [-9, 1], [14, 2]], np.float64) * 1024, np.full(G, -1.0), np.full((G, 3), 2.0), np.zeros(G)]
    pred, gt = np.c_[pred, np.zeros((P, 2))].astype(np.float32), np.c_[gt, np.zeros((G, 2))].astype(np.float32)
    gl = rng.integers(0, 4, G).astype(np.int32)
    ql = rng.integers(0, 4, P).astype(np.int32) if case == 'wrap_labels' else None
    if case.startswith('ties'):
        gl = np.array([0, 0, 1, 2], np.int32)
        ql = np.array([0, 0, 0, 1, 1, 0], np.int32) if case == 'ties_labels' else None
    inds, labels = heuristic_ref(pred, gt, gl, ql, thre)
    assert (inds > 0).sum() >= 2
    pd, gd, gld = (torch.from_numpy(t).to(dev()) for t in (pred, gt, gl))
    qd = torch.from_numpy(ql).to(dev()) if ql is not None else None
    work = Canvas(2 * G, torch.int32)
    gi, ov, lab = Canvas(P, torch.int64), Canvas(P), Canvas(P)
    _capi('di_heuristic_assign_f32', _p(pd), 9, P, _p(gd), _p(gld), G, _p(qd), float(thre), _p(gi.view), _p(ov.view),
          _p(lab.view), _p(work.view))
    assert gi.intact() and ov.intact() and lab.intact() and work.intact()
    got = gi.view.cpu().numpy()
    assert np.array_equal(got, inds), np.nonzero(got != inds)[0][:8]
    assert np.array_equal(lab.view.cpu().numpy(), labels)
    hit = np.nonzero(inds)[0]
    want, bar = np.zeros(P), np.zeros(P)
    if hit.size:
        want[hit], bar[hit] = iou3d64(gt[inds[hit] - 1], pred[hit])
    o = ov.view.double().cpu().numpy()
    assert (np.abs(o - want) <= bar).all() and (o[inds == 0] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# 4. targets (di_loss_targets_f32)
# ---------------------------------------------------------------------------------------------------------------------
def ulp32(x):
    return np.spacing(np.abs(x).astype(np.float32)).astype(np.float64)


@pytest.mark.parametrize('mode,code,pos_weight,L,npos', [
    (0, 10, 0.0, 1, 'some'), (1, 10, -1.0, 6, 'some'), (2, 8, 2.5, 3, 'some'), (1, 8, 1.0, 4, 'some'),
    (2, 10, 0.0, 6, 'none'), (0, 8, 3.0, 2, 'all')])
def test_loss_targets(mode, code, pos_weight, L, npos):
    """Mask modes 0 (a mask is passed and must be ignored), 1 (even layers use mask l / 2) and 2; code 8 and 10;
    pos_weight <= 0 and > 0 (truncated to an integer weight); no positives, all positives; max_overlaps outside [0, 1];
    padded ground-truth rows NaN."""
    rng = np.random.default_rng(L * 7 + code + mode)
    B, P, K = 2, 37, 10
    nb = 9 if code == 10 else int(rng.choice([7, 9]))
    Gmax, n_gt = 12, [9, 4]
    gt = np.full((B, Gmax, nb), np.nan, np.float32)
    gl = np.full((B, Gmax), -7, np.int32)
    for b in range(B):
        n = n_gt[b]
        gt[b, :n] = np.c_[rng.uniform(-54, 54, (n, 2)), rng.uniform(-3, 1, n), rng.uniform(0.2, 12, (n, 3)),
                          rng.uniform(-3.5, 3.5, n), rng.normal(size=(n, 2))][:, :nb]
        gl[b, :n] = rng.integers(0, K, n)
    gt[0, 0, 6] = 0.0
    gi = np.zeros((B, L * P), np.int64)
    if npos != 'none':
        for b in range(B):
            gi[b] = rng.integers(1, n_gt[b] + 1, L * P) * (rng.random(L * P) < (1.0 if npos == 'all' else 0.3))
    mo = rng.uniform(-0.5, 1.5, (B, L * P)).astype(np.float32)
    mo[:, :4] = [-1e-30, 0.0, 1.0, 1.0 + 2 ** -23]
    n_masks = {0: 1, 1: (L + 1) // 2, 2: L}[mode]
    mask = (rng.random((n_masks, B, P)) < 0.7).astype(np.uint8)
    coder4 = (8 * 0.075, 8 * 0.075, PC[0], PC[1])
    gid, mod, gtd, gld, maskd = (torch.from_numpy(np.ascontiguousarray(a)).to(dev()) for a in (gi, mo, gt, gl, mask))
    n = B * L * P
    labels, label_w = Canvas(n, torch.int64), Canvas(n, torch.int64)
    bt, bw, ious = Canvas(n * code), Canvas(n * code), Canvas(n)
    num_pos, iou_sum, pos_cnt = Canvas(L, fill=0.0), Canvas(B, fill=0.0), Canvas(B, torch.int32, fill=0)
    _capi('di_loss_targets_f32', _p(gid), _p(mod), _p(gtd), _p(gld), Gmax, _p(maskd), mode, B, L, P, nb, code, K,
          float(pos_weight), _f(coder4), _p(labels.view), _p(label_w.view), _p(bt.view), _p(bw.view), _p(ious.view),
          _p(num_pos.view), _p(iou_sum.view), _p(pos_cnt.view))
    for c in (labels, label_w, bt, bw, ious, num_pos, iou_sum, pos_cnt):
        assert c.intact()
    # reference
    mk = np.ones((B, L, P))
    for l in range(L):
        if mode == 1 and l % 2 == 0:
            mk[:, l] = mask[l // 2]
        elif mode == 2:
            mk[:, l] = mask[l]
    mk = mk.reshape(B, L * P)
    pos = gi > 0
    g = np.zeros((B, L * P, nb))
    lab_w = np.where(pos, gl[np.arange(B)[:, None], np.maximum(gi - 1, 0)], K)
    for b in range(B):
        g[b][pos[b]] = gt[b, gi[b][pos[b]] - 1]
    pw = 1.0 if pos_weight <= 0 else pos_weight
    want_lw = np.where(pos, np.trunc(np.float32(pw) * mk), mk).astype(np.int64)
    enc = np.stack([(g[..., 0] - f32(coder4[2])) / f32(coder4[0]), (g[..., 1] - f32(coder4[3])) / f32(coder4[1]),
                    g[..., 2] + 0.5 * g[..., 5], np.log(np.where(pos, g[..., 3], 1)), np.log(np.where(pos, g[..., 4], 1)),
                    np.log(np.where(pos, g[..., 5], 1)), np.sin(g[..., 6]), np.cos(g[..., 6])]
                   + ([g[..., 7], g[..., 8]] if code == 10 else []), -1)
    enc = np.where(pos[..., None], enc, 0.0)
    assert np.array_equal(labels.view.cpu().numpy().reshape(B, L * P), lab_w)
    assert np.array_equal(label_w.view.cpu().numpy().reshape(B, L * P), want_lw)
    assert same_bits(bw.view.cpu().view(B, L * P, code), torch.from_numpy(np.repeat((mk * pos)[..., None], code, -1)).float())
    got = bt.view.cpu().double().numpy().reshape(B, L * P, code)
    assert (np.abs(got - enc) <= 2 * ulp32(enc)).all(), np.argwhere(np.abs(got - enc) > 2 * ulp32(enc))[:8]
    assert same_bits(ious.view.cpu().view(B, L * P) + 0.0, torch.from_numpy(np.clip(mo, 0, 1)) + 0.0)
    want_np = (mk * pos).reshape(B, L, P).sum((0, 2))
    assert np.array_equal(num_pos.view.cpu().double().numpy(), want_np)
    assert np.array_equal(pos_cnt.view.cpu().numpy(), pos.sum(1))
    ov = np.where(pos, np.clip(mo, 0, 1), 0.0)
    s = iou_sum.view.cpu().double().numpy()
    assert (np.abs(s - ov.sum(1)) <= (pos.sum(1) + 1) * U * ov.sum(1)).all()


# ---------------------------------------------------------------------------------------------------------------------
# 5. gaussian heat-map targets (di_gaussian_heatmap_f32)
# ---------------------------------------------------------------------------------------------------------------------
VX, VY, OSF, X0, Y0 = 0.075, 0.1, 8, -54.0, -40.0
HX, HY = 56, 40                             # map X, Y (non-square; cells 0.6 m x 0.8 m)


def heat_ref(gt, gl, n_gt, K, min_radius, overlap):
    """deepinteraction_decoder.py:443-476 with oracle.loss.gaussian_radius / draw_heatmap_gaussian, fp32 tensors."""
    import oracle.loss as ol
    B = gt.shape[0]
    heat = torch.zeros(B, K, HY, HX)
    vox, rng = torch.tensor([VX, VY]), torch.tensor([X0, Y0])
    for b in range(B):
        g = torch.from_numpy(gt[b])
        for i in range(n_gt[b]):
            width, length = g[i][3] / vox[0] / OSF, g[i][4] / vox[1] / OSF
            if width > 0 and length > 0:
                radius = max(min_radius, int(ol.gaussian_radius((length, width), min_overlap=overlap)))
                cx, cy = (g[i][0] - rng[0]) / vox[0] / OSF, (g[i][1] - rng[1]) / vox[1] / OSF
                ci = torch.tensor([cx, cy], dtype=torch.float32).to(torch.int32)
                ol.draw_heatmap_gaussian(heat[b, int(gl[b, i])], ci, radius)
    return heat


def _at(cx, cy, w, l, yaw=0.0):
    """A box whose centre lies at map coordinates (cx, cy) and whose footprint is w x l cells."""
    return [X0 + cx * VX * OSF, Y0 + cy * VY * OSF, -1.0, w * VX * OSF, l * VY * OSF, 1.5, yaw, 0.0, 0.0]


def heat_boxes(radius_of):
    """(box, class) cases; radius_of(w, l) is the reference radius of a w x l cell footprint."""
    c = []
    for k, cx in ((2, 10.5), (3, 30.5), (4, 45.5)):   # footprints whose radius lands just below / just above 2, 3, 4
        ws = np.arange(3.0, 14.0, 0.01)
        r = np.array([radius_of(w, 0.8 * w) for w in ws])
        below, above = ws[(r > k - 0.01) & (r < k - 0.001)][0], ws[(r > k + 0.001) & (r < k + 0.01)][0]
        c += [(_at(cx, 20.5, below, 0.8 * below), 0), (_at(cx, 28.5, above, 0.8 * above), 0)]
    for cx in (0.5, HX - 0.5, 0.0, HX - 1e-3):     # on the borders
        c += [(_at(cx, 15.5, 6, 5), 1)]
    for cy in (0.25, HY - 0.5):
        c += [(_at(25.5, cy, 6, 5), 1)]
    for cx in (-0.7, -1.3, -2.5, -4.5, -9.5, -40.0, HX + 0.5, HX + 2.5, HX + 4.5, HX + 30.0):   # outside, x
        c += [(_at(cx, 8.5, 8, 7), 2)]
    for cy in (-0.7, -1.3, -3.5, -12.5, HY + 1.5, HY + 3.5, HY + 12.0):                       # outside, y
        c += [(_at(40.5, cy, 8, 7), 2)]
    c += [(_at(-3.5, -2.5, 9, 9), 0), (_at(HX + 2.5, HY + 1.5, 9, 9), 0)]                       # outside, corners
    c += [(_at(20.5, 30.5, 9, 9), 1), (_at(22.5, 31.5, 7, 9), 1), (_at(21.5, 30.5, 5, 4), 1)]  # same class, overlapping
    c += [(_at(20.5, 30.5, 6, 6), 2), (_at(45.5, 33.5, 0.3, 0.2), 2), (_at(47.5, 33.5, 0.01, 3), 0)]  # min_radius binds
    c += [(_at(5.5, 5.5, 0.0, 4), 0), (_at(6.5, 6.5, 4, -1), 1), (_at(7.5, 7.5, -2, -2), 2)]    # skipped
    return c


@pytest.mark.parametrize('min_radius', [2, 0])
def test_gaussian_heatmap_edges(min_radius):
    import oracle.loss as ol
    K, overlap = 3, 0.1

    def radius_of(w, l):
        return float(ol.gaussian_radius((torch.tensor(l, dtype=torch.float64), torch.tensor(w, dtype=torch.float64)), overlap))
    cases = heat_boxes(radius_of)
    B, n = 2, len(cases)
    Gmax = n + 3
    gt = np.zeros((B, Gmax, 9), np.float32)
    gl = np.zeros((B, Gmax), np.int32)
    n_gt = [n, n - 9]
    for b in range(B):
        order = np.arange(n) if b == 0 else np.random.default_rng(1).permutation(n)
        for j in range(Gmax):
            bx, k = cases[order[j]] if j < n_gt[b] else (_at(28.5, 20.5, 12, 12), 0)   # padding: a valid box, never drawn
            gt[b, j], gl[b, j] = bx, k
    want = heat_ref(gt, gl, n_gt, K, min_radius, overlap)
    heat = Canvas(B * K * HY * HX, fill=0.0)
    gd, gld = torch.from_numpy(gt).to(dev()), torch.from_numpy(gl).to(dev())
    nd = torch.tensor(n_gt, dtype=torch.int32, device=dev())
    _capi('di_gaussian_heatmap_f32', _p(gd), 9, _p(gld), _p(nd), B, Gmax, K, HY, HX,
          _f([VX, VY, X0, Y0, OSF, min_radius, overlap]), _p(heat.view))
    assert heat.intact()
    got = heat.view.view(B, K, HY, HX).cpu()
    assert same_bits(got, want), float((got - want).abs().max())
    assert int((want == 1).sum()) >= 20 and float(want[0, :, :, 0].max()) > 0 and float(want[0, :, 0, :].max()) > 0


# ---------------------------------------------------------------------------------------------------------------------
# 6. losses (di_mmpi_losses_f32)
# ---------------------------------------------------------------------------------------------------------------------
def _sig32(x):
    return f32(1.0 / (1.0 + np.exp(-x.astype(np.float64))))


def _with_bar(f, s, ds, lo=0.0, hi=1.0):
    """(f(p), |change of f over clip(s +- ds)| + 16 U |f(p)|) with p = clip(s, lo, hi): s is the sigmoid before the
    clamp, so a p that the clamp pins is not charged for the sigmoid's rounding."""
    v = f(np.clip(s, lo, hi))
    d = np.maximum(np.abs(f(np.clip(s + ds, lo, hi)) - v), np.abs(f(np.clip(s - ds, lo, hi)) - v))
    return v, d + 16 * U * np.abs(v)


def losses_ref(d, B, K, L, P, code, cw, gamma, alpha, ga, gg, w3):
    lo, hi = f32(1e-4), f32(np.float32(1) - np.float32(1e-4))
    x, t = d['logit'].astype(np.float64), d['target'].astype(np.float64)
    s = _sig32(d['logit'])
    posw, negw = (t == 1.0).astype(np.float64), (1 - t) ** gg
    fh = lambda p: -np.log(p + 1e-12) * (1 - p) ** ga * posw - np.log(1 - p + 1e-12) * p ** ga * negw
    th, bh = _with_bar(fh, s, 4 * U * s, lo, hi)
    cnt = max(posw.sum(), 1.0)
    out, bar = [th.sum() / cnt * w3[0]], [bh.sum() / cnt * w3[0]]
    LP = L * P
    for l in range(L):
        sl = slice(l * P, (l + 1) * P)
        s = d['score'][:, :, sl]                                              # [B, K, P]
        p = _sig32(s)
        lab, w = d['labels'][:, sl], d['label_w'][:, sl].astype(np.float64)
        one = (lab[:, None, :] == np.arange(K)[None, :, None])
        fc = lambda p: np.where(one, -alpha * (1 - p) ** gamma * np.log(np.maximum(p, FLT_MIN)),
                                -(1 - alpha) * p ** gamma * np.log(np.maximum(1 - p, FLT_MIN))) * w[:, None, :]
        tc, bc = _with_bar(fc, p, np.where(p < 1.0, 4 * U * p, 0.0))
        pr = np.concatenate([d['center'], d['height'], d['dim'], d['rot']] + ([d['vel']] if code == 10 else []), 1)[:, :, sl]
        tb = np.abs(pr.astype(np.float64) - d['bbox_t'][:, sl].transpose(0, 2, 1)) * d['bbox_w'][:, sl].transpose(0, 2, 1) \
            * np.array(cw[:code], np.float32).astype(np.float64)[None, :, None]
        af = max(float(d['num_pos'][l]), 1.0)
        out += [tc.sum() / af * w3[1], tb.sum() / af * w3[2]]
        bar += [bc.sum() / af * w3[1], 16 * U * tb.sum() / af * w3[2]]
    m = (d['iou_sum'].astype(np.float64) / np.maximum(d['pos_cnt'], 1)).mean()
    out, bar = np.array(out + [m]), np.array(bar + [4 * U * m])
    return out, bar + 2 * U * np.abs(out)


LOSS_CASES = [  # n_heat, B, K, L, P, code
    (100, 1, 3, 1, 50, 10),
    (70001, 2, 10, 3, 40, 8),
    (2 * 3 * 180 * 180, 2, 3, 1, 9000, 10),
]


@pytest.mark.parametrize('n_heat,B,K,L,P,code', LOSS_CASES)
def test_mmpi_losses(n_heat, B, K, L, P, code):
    """n_heat below 256, not a multiple of 256 x 256 and above the grid stride; B P above 64 x 256 rows; logits +-100
    and +-30 (the FLT_MIN and 1e-4 clamps); targets exactly 1, 0 and between; label weights 0, 1, 2; background label K;
    code 8 with vel = NULL; a layer with num_pos = 0; and the same bits from a second call."""
    rng = np.random.default_rng(n_heat)
    LP = L * P
    sat = lambda shape: np.where(rng.random(shape) < 0.3, rng.choice(LOGITS, shape), rng.normal(size=shape) * 2).astype(np.float32)
    tgt = rng.random(n_heat).astype(np.float32)
    r = rng.random(n_heat)
    tgt[r < 0.3], tgt[(r >= 0.3) & (r < 0.35)] = 0.0, 1.0
    d = dict(logit=sat(n_heat), target=tgt, score=sat((B, K, LP)), center=rng.normal(size=(B, 2, LP)) * 50,
             height=rng.normal(size=(B, 1, LP)), dim=rng.normal(size=(B, 3, LP)), rot=rng.normal(size=(B, 2, LP)),
             vel=rng.normal(size=(B, 2, LP)), labels=rng.integers(0, K + 1, (B, LP)), label_w=rng.integers(0, 3, (B, LP)),
             bbox_t=rng.normal(size=(B, LP, code)) * 20, bbox_w=(rng.random((B, LP, code)) < 0.6) * rng.choice([1.0, 0.5], (B, LP, code)),
             num_pos=rng.integers(0, 30, L), iou_sum=rng.random(B) * 5, pos_cnt=rng.integers(0, 9, B))
    d['logit'][:8], d['target'][:8] = [100, -100, 30, -30, 100, -100, 0, 0], [1, 1, 1, 1, 0, 0, 1, 0]
    d['num_pos'][0] = 0
    d = {k: np.ascontiguousarray(v, dtype=np.int64 if k in ('labels', 'label_w') else np.int32 if k == 'pos_cnt'
                                 else np.float32) for k, v in d.items()}
    cw = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.2, 0.2][:code] + [0.0] * (10 - code)
    gamma, alpha, ga, gg, w3 = 2.0, 0.25, 2.0, 4.0, (1.0, 1.0, 0.25)
    want, bar = losses_ref(d, B, K, L, P, code, cw, gamma, alpha, ga, gg, w3)
    t = {k: torch.from_numpy(v).to(dev()) for k, v in d.items()}
    vel = t['vel'] if code == 10 else None
    outs = []
    for _ in range(2):
        work, out = Canvas(2 * 256 + L * 2 * 64, torch.float64), Canvas(2 + 2 * L)
        _capi('di_mmpi_losses_f32', _p(t['logit']), _p(t['target']), n_heat, _p(t['score']), _p(t['center']), _p(t['height']),
              _p(t['dim']), _p(t['rot']), _p(vel), _p(t['labels']), _p(t['label_w']), _p(t['bbox_t']), _p(t['bbox_w']),
              _p(t['num_pos']), _p(t['iou_sum']), _p(t['pos_cnt']), B, K, L, P, code, _f(cw), _f([gamma, alpha]), _f([ga, gg]),
              _f(w3), _p(work.view), _p(out.view))
        assert work.intact() and out.intact()
        outs.append(out.view.cpu())
    assert same_bits(outs[0], outs[1])
    got = outs[0].double().numpy()
    print('|err| / bar per output', np.round(np.abs(got - want) / bar, 3))
    assert (np.abs(got - want) <= bar).all(), list(zip(got, want, bar))
    assert (bar <= 1e-5 * np.abs(want)).all(), list(zip(want, bar))
