"""Kernel-level tests of the MMPI decoder's proposal, RoI and box kernels (csrc/decoder.cu) against references written
from each operation's definition in float64: heat-map NMS, top-k, query init, the prediction finish of both decoders, RoI
generation (image and BEV mode), RoIAlignV2, DynamicConv, the box coder and circle NMS.  The oracle's code is used
where it is a plain statement of the operation (oracle.geometry.roi_align / lidar_box_corners, the oracle's
TransFusionBBoxCoder and circle_nms), evaluated in float64.

Inputs.  The geometry is dyadic: power-of-two camera scales, camera rows of small dyadic numbers, centres and heights on
a 1/8 grid, RoI extents of 7 * 2^-j on a 1/4 grid, NMS centres on a 1/8 grid.  The fp32 kernels and the float64
references then compute the same on-image tests, sampling positions, range tests and squared distances exactly, and
make the same discrete decisions, also for the cases placed exactly on a boundary (a centre on the image edge, a
RoIAlign sample at -1 or at H, an NMS pair at the threshold distance).  Where a test needs scores whose fp32 rounding
decides a tie (heat-map NMS, top-k), the reference is applied to the kernel's own fp32 scores, and those scores are
checked separately against float64.

Exact outputs.  win, onbits, RoI map indices, labels, keep masks, top-k indices and NMS survivors must be equal.  query
init and the prediction finish only move or add data: they are held to bit equality against torch evaluating the same
fp32 adds.

Float outputs.  row_err (kernel_check.py) takes, per output row, max|got - want| over the magnitude of the terms
summed into that row.  The kernels use fp32 FFMA and fp32 expf / atan2f / cosf / sinf / logf (a few ulp each); their
rows carry a few units of 2^-24 times a sqrt of the term count (at most 128 terms here): about 1e-6 of the row scale.
TOL = 1e-5 leaves a 10x margin.  For DynamicConv the scale of a LayerNorm output is the scale of its input divided by
the row's standard deviation (times |gamma|, plus |beta|): an absolute error d of the input becomes d / std after the
normalisation, so rows with a large mean and a small spread are judged by what fp32 can deliver for them.
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from kernel_check import _capi, row_err, same_bits

pytestmark = pytest.mark.gpu

TOL = 1e-5
F32_EPS = float(np.float32(1e-5))       # the clamp of the projected depth, as the kernel's fp32 constant


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _p(t):
    return _ops()._ptr(t)


def _mask32(m):
    """A 32-bit class mask as the C int the ABI takes."""
    return m - (1 << 32) if m >= 1 << 31 else m


def _rejects(name, *args):
    with pytest.raises(RuntimeError):
        _capi(name, *args)


# ---------------------------------------------------------------------------------------------------------------------
# 1. heat-map fusion + NMS
# ---------------------------------------------------------------------------------------------------------------------
def _nms_ref(hc, ks, no_nms):
    """Max-pool NMS of deepinteraction_decoder.py:230-239 on scores hc [B,K,H,W]: a score survives iff it equals the
    maximum of its ks x ks window; the border ring of width ks // 2 has local max 0 (drops every positive score); the
    classes in no_nms keep every score."""
    B, K, H, W = hc.shape
    r = ks // 2
    lm = torch.zeros_like(hc)
    if H > 2 * r and W > 2 * r:
        lm[:, :, r:H - r, r:W - r] = F.max_pool2d(hc, ks, 1, 0)
    for c in range(K):
        if (no_nms >> c) & 1:
            lm[:, c] = hc[:, c]
    return torch.where(hc == lm, hc, torch.zeros(()))


NMS_CASES = [  # B, K, H, W, ld, ks, no_nms
    (2, 10, 180, 180, 10, 3, (1 << 8) | (1 << 9)),       # base decoder
    (2, 10, 36, 44, 12, 3, (1 << 8) | (1 << 9)),         # small scene, padded logit rows
    (2, 10, 36, 44, 12, 5, (1 << 8) | (1 << 9)),
    (1, 32, 9, 13, 40, 3, 1 | (1 << 31)),                # K = 32: the whole no_nms mask, ld > K
    (1, 4, 5, 5, 4, 5, 0),                               # map as large as the window: one pixel inside the ring
    (1, 3, 3, 4, 5, 5, 1 << 1),                          # map smaller than the window
    (2, 2, 1, 1, 2, 3, 0),
]


@pytest.mark.parametrize('case', NMS_CASES, ids=lambda c: 'B%dK%d_%dx%d_ld%d_ks%d' % c[:6])
def test_heatmap_nms_matches_definition(case):
    ops = _ops()
    B, K, H, W, ld, ks, no_nms = case
    g = torch.Generator().manual_seed(H * W + ks)
    # logits on a 1/4 grid: equal (a, b) pairs make plateaus of equal scores; painted 2x2 plateaus above every other
    # score must survive whole
    a = torch.randint(-8, 9, (B, H, W, ld), generator=g).float() / 4
    b = torch.randint(-8, 9, (B, H, W, ld), generator=g).float() / 4
    for y0, x0 in ((H // 2, W // 3), (H // 3, (2 * W) // 3)):
        a[:, y0:y0 + 2, x0:x0 + 2, :] = 3.0
        b[:, y0:y0 + 2, x0:x0 + 2, :] = 2.5
    ad, bd = a.to(dev()), b.to(dev())
    hc, _ = ops.heatmap_nms(ad, bd, K, ks, _mask32((1 << K) - 1))      # every class without NMS: the raw scores
    hc = hc.cpu().view(B, K, H, W)
    want64 = ((a.double().sigmoid() + b.double().sigmoid()) / 2)[..., :K].permute(0, 3, 1, 2)
    assert float((hc.double() - want64).abs().max()) < 2 ** -22
    out, dense = ops.heatmap_nms(ad, bd, K, ks, _mask32(no_nms))
    assert torch.equal(dense.cpu(), b[..., :K].permute(0, 3, 1, 2))
    assert same_bits(out.cpu().view(B, K, H, W), _nms_ref(hc, ks, no_nms))
    if H * W * K >= 50:
        top = ops.topk(out.view(B, -1), 50).cpu().long()
        assert torch.equal(top, _topk_ref(out.cpu().view(B, -1), 50))


# ---------------------------------------------------------------------------------------------------------------------
# 2. top-k
# ---------------------------------------------------------------------------------------------------------------------
def _topk_ref(s, k):
    """Indices of the k largest scores, descending, ties by ascending index."""
    return torch.from_numpy(np.argsort(-s.double().numpy(), axis=-1, kind='stable')[:, :k].copy())


def _topk_scores(name, g):
    if name == 'base_heat':                      # 2 x 10 x 180 x 180 heat map: mostly zeros, values on a coarse grid
        s = torch.randint(1, 200, (2, 324000), generator=g).float() / 256
        return s * (torch.rand(2, 324000, generator=g) < 0.1), 200
    if name == 'ties_5000':                      # 300 ties at 0.5 cut at 198, two larger values, zeros
        s = torch.zeros(1, 5000)
        s[0, torch.randperm(5000, generator=g)[:300]] = 0.5
        s[0, 7], s[0, 4000] = 0.9, 0.7
        return s, 200
    if name == 'k_eq_n':
        return torch.rand(3, 64, generator=g) * 1e-6, 64
    if name == 'zeros_2048':                     # 2048 ties at the cut, k = 1024
        return torch.zeros(2, 2048), 1024
    if name == 'zeros_65537':                    # two levels, every slice all ties, short last slice
        return torch.zeros(1, 65537), 1024
    if name == 'few_positive_65537':             # fewer than k positive scores: the rest are zeros in index order
        s = torch.zeros(2, 65537)
        s[:, torch.randperm(65537, generator=g)[:100]] = torch.rand(100, generator=g) + 0.5
        return s, 1024
    if name.startswith('ties_over_1024'):        # 1100 ties at the cut below 500 larger values
        n = int(name.split('_')[-1])
        s = torch.full((1, n), 0.25)
        perm = torch.randperm(n, generator=g)
        s[0, perm[:500]] = 0.75
        s[0, perm[500:1600]] = 0.5
        return s, 1024
    if name == 'random_100000':
        return torch.rand(2, 100000, generator=g), 1024
    raise KeyError(name)


TOPK_CASES = ['base_heat', 'ties_5000', 'k_eq_n', 'zeros_2048', 'zeros_65537', 'few_positive_65537',
              'ties_over_1024_30000', 'ties_over_1024_70000', 'random_100000']


@pytest.mark.parametrize('name', TOPK_CASES)
def test_topk_matches_stable_argsort(name):
    ops = _ops()
    g = torch.Generator().manual_seed(len(name))
    s, k = _topk_scores(name, g)
    B, n = s.shape
    want = _topk_ref(s, k)
    sd = s.to(dev())
    got = ops.topk(sd, k).cpu().long()                 # two levels (64 slices) from n = 65536
    assert torch.equal(got, want), (got != want).nonzero()[:5].tolist()
    # the entry point with other slice counts, the single-level path and slices shorter than k included
    for slices in (0, 2, 7, 64):
        if slices * k > (1 << 20):
            continue
        idx = torch.empty(B, k, dtype=torch.int32, device=dev())
        work = torch.empty(max(1, B * slices * k * 2), device=dev())
        _capi('di_topk_f32', _p(sd), _p(idx), B, n, k, _p(work) if slices else None, slices)
        assert torch.equal(idx.cpu().long(), want), slices


def test_topk_few_positive_with_short_slices():
    """Slices shorter than k pad their candidates with index -1; no pad may be returned while real indices remain."""
    g = torch.Generator().manual_seed(11)
    s = torch.zeros(2, 1500)
    s[:, torch.randperm(1500, generator=g)[:40]] = 0.5
    want = _topk_ref(s, 1024)
    idx = torch.empty(2, 1024, dtype=torch.int32, device=dev())
    work = torch.empty(2 * 2 * 1024 * 2, device=dev())
    _capi('di_topk_f32', _p(s.to(dev())), _p(idx), 2, 1500, 1024, _p(work), 2)
    assert torch.equal(idx.cpu().long(), want)


# ---------------------------------------------------------------------------------------------------------------------
# 3. query init and the prediction finish (data movement: bit equality)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('shape', [(2, 200, 180, 180, 128, 10), (1, 7, 3, 1, 300, 32), (3, 5, 4, 6, 4, 2)],
                         ids=lambda s: 'B%dP%d_%dx%d_C%dK%d' % s)
def test_query_init_bit_exact(shape):
    ops = _ops()
    B, P, H, W, C, K = shape
    HW = H * W
    g = torch.Generator().manual_seed(P * C)
    feat, heat = torch.randn(B, HW, C, generator=g), torch.rand(B, K, HW, generator=g)
    wce_t, bce = torch.randn(K, C, generator=g), torch.randn(C, generator=g)
    top = torch.randint(0, K * HW, (B, P), generator=g)
    edges = torch.tensor([0, HW - 1, HW % (K * HW), K * HW - 1, (K - 1) * HW])      # first / last class and pixel
    top[:, :min(P, 5)] = edges[:min(P, 5)]
    top = top.int()
    qfeat, qpos, labels, qscore = ops.query_init(feat.to(dev()), top.to(dev()), heat.to(dev()), wce_t.to(dev()),
                                                 bce.to(dev()), W)
    t = top.long()
    cls, pix = t // HW, t % HW
    bi = torch.arange(B)[:, None]
    want = (feat[bi, pix] + wce_t[cls]) + bce                                # [B, P, C], fp32 adds in kernel order
    assert same_bits(qfeat, want.reshape(B * P, C))
    assert same_bits(qpos, torch.stack([(pix % W).float() + 0.5, (pix // W).float() + 0.5], -1).reshape(B * P, 2))
    assert torch.equal(labels.cpu(), cls.int())
    assert same_bits(qscore, heat[bi[:, None], torch.arange(K)[None, :, None], pix[:, None, :]])


@pytest.mark.parametrize('M,NP', [(400, 20), (1, 10), (129, 2)])
def test_pred_finish_bit_exact(M, NP):
    ops = _ops()
    g = torch.Generator().manual_seed(M)
    pred, qpos, first = (torch.randn(M, n, generator=g) for n in (NP, 2, NP))
    win = torch.randint(-1, 6, (M,), generator=g).int()
    win[0] = -1
    for with_first in (False, True):
        p, q = pred.to(dev()), qpos.to(dev())
        ops.pred_finish(p, q, first.to(dev()) if with_first else None, win.to(dev()) if with_first else None)
        want = pred.clone()
        want[:, :2] = pred[:, :2] + qpos
        if with_first:
            want[win < 0] = first[win < 0]
        assert same_bits(p, want) and same_bits(q, want[:, :2].contiguous()), with_first


@pytest.mark.parametrize('M,NP', [(400, 20), (1, 10), (129, 2)])
def test_pred_finish_pp_bit_exact(M, NP):
    ops = _ops()
    g = torch.Generator().manual_seed(M + 1)
    pred, qpos, look, first = (torch.randn(M, n, generator=g) for n in (NP, 2, 2, NP))
    win = torch.randint(-1, 6, (M,), generator=g).int()
    keep0 = torch.randint(0, 2, (M,), generator=g).int()
    for first_layer, with_win in ((1, True), (0, True), (0, False)):
        p, q, lk, kp = pred.to(dev()), qpos.to(dev()), look.to(dev()), keep0.to(dev())
        ops.pred_finish_pp(p, q, lk, first.to(dev()), win.to(dev()) if with_win else None, kp, first_layer)
        keep = torch.ones(M, dtype=torch.int32) if first_layer else keep0.clone()
        if with_win:
            keep = keep & (win >= 0).int()
        want = pred.clone()
        want[:, :2] = pred[:, :2] + look
        want[keep == 0] = first[keep == 0]
        tag = (first_layer, with_win)
        assert torch.equal(kp.cpu(), keep), tag
        assert same_bits(lk, pred[:, :2] + qpos), tag
        assert same_bits(p, want) and same_bits(q, want[:, :2].contiguous()), tag


# ---------------------------------------------------------------------------------------------------------------------
# 4. RoI generation (image mode 0, BEV mode 1)
# ---------------------------------------------------------------------------------------------------------------------
# params10: box centre (sx, sy, ox, oy) differs from the centre path (csx, cox, used for x AND y, as the reference does)
PRM = dict(sx=0.5, sy=0.25, ox=-32.0, oy=-16.0, csx=0.5, cox=-32.0, h_pad=64.0, w_pad=128.0, bev_scale=0.5, bev_off=-32.0)
P10 = [PRM[k] for k in ('sx', 'sy', 'ox', 'oy', 'csx', 'cox', 'h_pad', 'w_pad', 'bev_scale', 'bev_off')]


def _cameras(B, V):
    """[B, V, 3, 4] lidar -> image rows: views look along +x, +y, -x, -y (views 4..7 again, other focal length and
    principal point), depth = the lidar coordinate along the view axis, so every centre's depth is a grid value."""
    Ms = []
    for v in range(V):
        f, cu, cv = (32.0, 64.0, 32.0) if v < 4 else (16.0, 48.0, 40.0)
        ax, sg = [(0, 1.0), (1, 1.0), (0, -1.0), (1, -1.0)][v % 4]
        lat = 1 - ax
        M = torch.zeros(3, 4)
        M[2, ax] = sg                                            # depth
        M[0, ax], M[0, lat] = cu * sg, -f * sg if ax == 0 else f * sg
        M[1, ax], M[1, 2] = cv * sg, -f
        Ms.append(M)
    return torch.stack(Ms)[None].expand(B, V, 3, 4).contiguous()


def _rois_pred(B, P, g, NP=10, lone_view=False):
    """pred rows [B*P, NP]: centre cells on a 1/4 grid (lidar |x|, |y| in [8, 28], so no box corner comes near depth 0),
    heights on a 1/8 grid, log-dims in [-1, 0.5], rotation (sin, cos) pairs incl. (0, 1) and (0, 0).  The last sample's
    first rows put centres exactly on the image edges of view 0 (depth 8) and 1/8 inside them.  With lone_view, sample 0
    has one single query at x < 0 (views 2 and 6 see one query each and must be skipped)."""
    pred = torch.zeros(B * P, NP)
    side = torch.where(torch.rand(B * P, 2, generator=g) < 0.5, -1.0, 1.0)
    xy = side * (8 + torch.randint(0, 161, (B * P, 2), generator=g).float() / 8)
    z = torch.randint(-16, 17, (B * P,), generator=g).float() / 8
    if lone_view:
        xy[:P, 0] = xy[:P, 0].abs()
        xy[0] = torch.tensor([-16.0, 1.0])
        z[0] = 0.0
    # view 0 at depth 8: u = 64 - 4 y (0 at y = 16, 128 at y = -16), w = 32 - 4 z (0 at z = 8, 64 at z = -8)
    edge = [(16.0, 0.0), (15.875, 0.0), (-16.0, 0.0), (-15.875, 0.0), (0.0, 8.0), (0.0, 7.875), (0.0, -8.0), (0.0, -7.875)]
    for i, (y, zz) in enumerate(edge[:P - 1]):              # sample 0 (no crop, no flip), after its first row
        xy[1 + i] = torch.tensor([8.0, y])
        z[1 + i] = zz
    pred[:, 0] = (xy[:, 0] - PRM['cox']) / PRM['csx']
    pred[:, 1] = (xy[:, 1] - PRM['cox']) / PRM['csx']
    pred[:, 2] = z
    pred[:, 3:6] = torch.rand(B * P, 3, generator=g) * 1.5 - 1.0
    rot = torch.randn(B * P, 2, generator=g)
    rot[::5] = torch.tensor([0.0, 1.0])
    rot[1::7] = 0.0
    pred[:, 6:8] = rot
    pred[:, 8:] = torch.randn(B * P, NP - 8, generator=g)
    return pred


def _project(M, pts, ax):
    """pts [N, 3] float64 -> image (u, w) of the 3x4 rows M, depth clamped to the kernel's 1e-5, crop and flip of ax."""
    p = torch.cat([pts, torch.ones(len(pts), 1, dtype=pts.dtype)], 1) @ M.double().t()
    c = p[:, 2].clamp(min=F32_EPS)
    u, w = p[:, 0] / c - float(ax[0]), p[:, 1] / c - float(ax[1])
    if float(ax[2]) != 0:
        u = float(ax[3]) - u
    return u, w


def _boxes64(pred, dim_scale=1.0):
    from oracle.geometry import lidar_box_corners
    p = pred.double()
    dims = p[:, 3:6].exp() * dim_scale
    box = torch.stack([p[:, 0] * PRM['sx'] + PRM['ox'], p[:, 1] * PRM['sy'] + PRM['oy'],
                       p[:, 2] - p[:, 5].exp() * 0.5, dims[:, 0], dims[:, 1], dims[:, 2],
                       torch.atan2(p[:, 6], p[:, 7])], 1)
    return lidar_box_corners(box)                               # [N, 8, 3]; BEV mode (dims doubled) reads x, y only


def _rois_ref(pred, proj, aux, B, P, V):
    """decoder_utils.py:660-741: per view, the box centre (test_cfg scale / offset for x and y, raw height) is on the
    image iff 0 < u < w_pad and 0 < w < h_pad; a view with at most one query on it is skipped; a query takes the last
    view it is on; its RoI is the bounding rectangle of the 8 projected corners in that view."""
    corners = _boxes64(pred)
    p = pred.double()
    ctr = torch.stack([p[:, 0] * PRM['csx'] + PRM['cox'], p[:, 1] * PRM['csx'] + PRM['cox'], p[:, 2]], 1)
    win = torch.full((B * P,), -1, dtype=torch.int32)
    bits = torch.zeros(B * P, dtype=torch.int32)
    rois = torch.zeros(B * P, 5, dtype=torch.float64)
    rois[:, 0] = -1
    for b in range(B):
        sl = slice(b * P, (b + 1) * P)
        for v in range(V):
            u, w = _project(proj[b, v], ctr[sl], aux[b])
            on = (u > 0) & (u < PRM['w_pad']) & (w > 0) & (w < PRM['h_pad'])
            if int(on.sum()) <= 1:
                continue
            cu, cw = _project(proj[b, v], corners[sl].reshape(-1, 3), aux[b])
            cu, cw = cu.view(P, 8), cw.view(P, 8)
            rect = torch.stack([cu.min(1).values, cw.min(1).values, cu.max(1).values, cw.max(1).values], 1)
            idx = on.nonzero().squeeze(1) + b * P
            win[idx], bits[idx] = v, bits[idx] | (1 << v)
            rois[idx, 0] = b * V + v
            rois[idx, 1:] = rect[on]
    return rois, win, bits


RCNN_CASES = [(2, 200, 6), (1, 1, 6), (2, 33, 8), (1, 1024, 8), (2, 8, 2)]


@pytest.mark.parametrize('BPV', RCNN_CASES, ids=lambda c: 'B%dP%dV%d' % c)
def test_rcnn_rois_image_mode_matches_definition(BPV):
    ops = _ops()
    B, P, V = BPV
    g = torch.Generator().manual_seed(P * V)
    pred = _rois_pred(B, P, g, lone_view=P > 8)
    proj = _cameras(B, V)
    aux = torch.tensor([[0.0, 0.0, 0.0, 0.0], [8.0, 4.0, 1.0, 136.0]])[torch.arange(B) % 2]   # crop x/y, flip, orig_w
    rois, win, onbits = ops.rcnn_rois(pred.to(dev()), B, P, V, 0, P10, proj.to(dev()), aux.contiguous().to(dev()))
    want, wwin, wbits = _rois_ref(pred, proj, aux, B, P, V)
    assert torch.equal(win.cpu(), wwin)
    assert torch.equal(onbits.cpu(), wbits)
    assert torch.equal(rois.cpu()[:, 0], want[:, 0].float())
    assert bool((rois.cpu()[wwin < 0, 1:] == 0).all())
    assert row_err(rois[:, 1:], want[:, 1:], want[:, 1:].abs()) < TOL
    if P > 8:
        assert int(wwin[0]) == -1 and int(wbits[0]) == 0, 'the one query of views 2 and 6 must be skipped'
        assert bool((wwin >= 0).any())


@pytest.mark.parametrize('BPV', [(2, 200, 6), (1, 1, 1), (1, 1024, 8)], ids=lambda c: 'B%dP%dV%d' % c)
def test_rcnn_rois_bev_mode_matches_definition(BPV):
    ops = _ops()
    B, P, V = BPV
    pred = _rois_pred(B, P, torch.Generator().manual_seed(P + 3))
    rois, win, onbits = ops.rcnn_rois(pred.to(dev()), B, P, V, 1, P10)
    c = (_boxes64(pred, 2.0)[..., :2] - PRM['bev_off']) / PRM['bev_scale']          # doubled dims, x and y by index 0
    want = torch.stack([c[..., 0].min(1).values, c[..., 1].min(1).values, c[..., 0].max(1).values,
                        c[..., 1].max(1).values], 1)
    assert torch.equal(win.cpu(), torch.zeros(B * P, dtype=torch.int32))
    assert torch.equal(onbits.cpu(), torch.ones(B * P, dtype=torch.int32))
    assert torch.equal(rois.cpu()[:, 0], torch.arange(B).repeat_interleave(P).float())
    assert row_err(rois[:, 1:], want, want.abs()) < TOL


# ---------------------------------------------------------------------------------------------------------------------
# 5. RoIAlignV2
# ---------------------------------------------------------------------------------------------------------------------
def _axis_spans(n):
    """(lo, hi) of RoI extents in map pixels (x * scale - 0.5) along an axis of n pixels: zero-width RoIs whose samples
    sit exactly at -1, in [-1, 0), at 0, n - 1, n - 0.5, n and beyond; inverted RoIs; widths 7 * 2^-j."""
    return [(-1.0, -1.0), (-1.5, -1.5), (-0.75, -0.75), (0.0, 0.0), (n - 1.0, n - 1.0), (n - 0.5, n - 0.5),
            (float(n), float(n)), (n + 0.25, n + 0.25), (5.0, 1.5), (0.5, 4.0), (-3.5, 3.5), (n - 7.0, n + 7.0),
            (-1.0, 13.0), (0.25, 28.25)]


def _edge_rois(n_maps, H, W, scale):
    """[R, 5] RoIs (map index, x0, y0, x1, y1) in input coordinates: every y span with every x span on every map."""
    ys, xs = _axis_spans(H), _axis_spans(W)
    r = []
    for m in range(n_maps):
        for y0, y1 in ys:
            for x0, x1 in xs:
                r.append([m, (x0 + 0.5) / scale, (y0 + 0.5) / scale, (x1 + 0.5) / scale, (y1 + 0.5) / scale])
    return torch.tensor(r, dtype=torch.float32)


def _roi_align_ref(maps_nchw, rois, scale):
    """[R, 49, C] float64: oracle.geometry.roi_align, and the same of |maps| (the summed |terms| of every output), 16
    RoIs per call (the oracle holds C x 196 samples per RoI in float64); rows with map index -1 are zero."""
    from oracle.geometry import roi_align
    C = maps_nchw.shape[1]
    out = torch.zeros(rois.shape[0], 49, 2 * C, dtype=torch.float64)
    for m in range(maps_nchw.shape[0]):
        sel = (rois[:, 0] == m).nonzero().squeeze(1)
        fm = torch.cat([maps_nchw[m], maps_nchw[m].abs()]).double()
        for part in sel.split(16):
            out[part] = roi_align(fm, rois[part, 1:].double(), 7, scale, 2).flatten(2).transpose(1, 2)
    return out[..., :C], out[..., C:]


ROI_CASES = [  # n_maps, H, W, C, scale
    (12, 112, 200, 128, 0.25),            # base image maps (B = 2 x 6 views)
    (2, 180, 180, 128, 1.0),              # base BEV map
    (2, 9, 13, 4, 1.0), (2, 9, 13, 132, 0.25), (2, 9, 13, 256, 1.0), (2, 9, 13, 260, 0.5), (2, 9, 13, 384, 1.0),
    (2, 9, 13, 512, 0.25), (1, 5, 1, 64, 1.0), (1, 1, 6, 128, 1.0),
]


@pytest.mark.parametrize('case', ROI_CASES, ids=lambda c: 'n%d_%dx%d_C%d_s%g' % c)
def test_roi_align_matches_oracle(case):
    ops = _ops()
    n_maps, H, W, C, scale = case
    g = torch.Generator().manual_seed(H * C + W)
    maps = torch.randn(n_maps, C, H, W, generator=g)
    rois = _edge_rois(1, H, W, scale)
    rnd = torch.cat([torch.randint(0, n_maps, (64, 1), generator=g).float(),
                     (torch.randint(-8, 4 * max(H, W) + 8, (64, 2), generator=g).float() / 4 + 0.5) / scale], 1)
    ext = torch.randint(0, 6, (64, 2), generator=g).float()
    rnd = torch.cat([rnd, rnd[:, 1:3] + 7 * 2.0 ** (ext - 2) / scale], 1)             # widths 7 * 2^-j
    dead = torch.tensor([[-1.0, 0.0, 0.0, 10.0, 10.0]])
    rois = torch.cat([rois, rnd, dead])
    got = ops.roi_align(maps.permute(0, 2, 3, 1).contiguous().to(dev()), rois.to(dev()), scale)
    want, mag = _roi_align_ref(maps, rois, scale)
    assert row_err(got, want, mag) < TOL
    assert bool((got[-1] == 0).all())
    # NaN corners: every sample of the RoI is NaN and skipped -> an exactly zero row
    nan = float('nan')
    bad = torch.tensor([[0, nan, 1.0, 8.0, 8.0], [0, 1.0, nan, 8.0, 8.0], [0, 1.0, 1.0, nan, 8.0], [0, 1.0, 1.0, 8.0, nan]])
    assert bool((ops.roi_align(maps.permute(0, 2, 3, 1).contiguous().to(dev()), bad.to(dev()), scale) == 0).all())


def test_roi_align_old_rois_match_oracle():
    """Six RoIs of the small scene's image maps (3 x 128 x 28 x 50, scale 1/4), including one with map index -1."""
    ops = _ops()
    g = torch.Generator().manual_seed(5)
    maps = torch.randn(3, 128, 28, 50, generator=g)
    rois = torch.tensor([[0, 8.0, 12.0, 70.0, 49.0], [1, -30.0, -10.0, 20.0, 30.0], [2, 150.0, 60.0, 230.0, 140.0],
                         [1, 40.0, 40.0, 40.0, 40.0], [-1, 0.0, 0.0, 10.0, 10.0], [0, 190.0, 100.0, 260.0, 150.0]])
    got = ops.roi_align(maps.permute(0, 2, 3, 1).contiguous().to(dev()), rois.to(dev()), 0.25)
    assert row_err(got, *_roi_align_ref(maps, rois, 0.25)) < TOL
    assert float(got[4].abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------------------------------
# 6. DynamicConv
# ---------------------------------------------------------------------------------------------------------------------
def _ln_relu_ref(x, terms, g, b, eps):
    """relu(LayerNorm(x) g + b) in float64 and the error scale of its outputs: the row's largest summed |term| over
    sqrt(var + eps), times |g|, plus |b|."""
    mu = x.mean(-1, keepdim=True)
    sd = ((x - mu).pow(2).mean(-1, keepdim=True) + eps).sqrt()
    y = F.relu((x - mu) / sd * g + b)
    return y, terms.amax(-1, keepdim=True) / sd * g.abs() + b.abs()


def _dynconv_ref(roi, params, g1, b1, g2, b2, eps=1e-5):
    n = roi.shape[0]
    F0, P1, P2 = roi.double(), params[:, :16384].double().view(n, 128, 128), params[:, 16384:].double().view(n, 128, 128)
    y1, s1 = _ln_relu_ref(F0 @ P1, F0.abs() @ P1.abs(), g1.double(), b1.double(), eps)
    y2, s2 = _ln_relu_ref(y1 @ P2, (y1.abs() + s1) @ P2.abs(), g2.double(), b2.double(), eps)
    return y2.flatten(1), s2.flatten(1)


@pytest.mark.parametrize('n', [1, 37, 400, 2000])
def test_dynconv_matches_float64(n):
    ops = _ops()
    d = dev()
    g = torch.Generator().manual_seed(n)
    gd = torch.Generator(device=d).manual_seed(n)
    if n == 37:                                   # the oracle module's parameter generator and norms
        import oracle.mmpi as om
        torch.manual_seed(6)
        m = om.DynamicConv().eval()
        with torch.no_grad():
            params = m.dynamic_layer(torch.randn(1, n, 128, generator=g))[0].contiguous().to(d)
        norms = [t.detach().clone() for t in (m.norm1.weight, m.norm1.bias, m.norm2.weight, m.norm2.bias)]
    else:
        params = torch.randn(n, 2 * 128 * 128, generator=gd, device=d) / 11
        norms = [torch.rand(128, generator=g) + 0.5, torch.randn(128, generator=g) * 0.5,
                 torch.rand(128, generator=g) + 0.5, torch.randn(128, generator=g) * 0.5]
    roi = torch.randn(n, 49, 128, generator=gd, device=d)
    roi[0, :7] = 0.0                              # zero-variance rows of the first LayerNorm
    if n > 1:
        roi[1] = 64.0 + torch.randn(49, 128, generator=gd, device=d) * 0.5   # large mean, small spread
        params[1, :16384] = 1.0 / 16 + params[1, :16384] / 8
        roi[n - 1] = 0.0                                                     # a whole query of zero rows
    got = ops.dynconv(roi, params, *(t.to(d) for t in norms))
    # every query is independent: up to 400 are checked, always the first two and the last
    rows = torch.arange(n) if n <= 400 else torch.cat([torch.tensor([0, 1, n - 1]), torch.randperm(n - 3, generator=g)[:397] + 2])
    want, scale = _dynconv_ref(roi[rows.to(d)].cpu(), params[rows.to(d)].cpu(), *norms)
    got = got[rows.to(d)]
    assert row_err(got, want, scale, width=128) < TOL


# ---------------------------------------------------------------------------------------------------------------------
# 7. box coder
# ---------------------------------------------------------------------------------------------------------------------
CODER = dict(sx=0.5, sy=0.25, ox=-32.0, oy=-16.0)
RANGE = [-20.0, -10.0, -3.0, 20.0, 10.0, 3.0]


def _coder64(code_size=10):
    from oracle.mmpi import TransFusionBBoxCoder
    return TransFusionBBoxCoder([CODER['ox'], CODER['oy']], 1, [CODER['sx'], CODER['sy']], RANGE, 0.25, code_size)


def _coder_inputs(B, K, P, g):
    """[B, k, P] heads: heat on a 1/8 grid (arg-max ties), centres / heights on a 1/8 grid; the first rows of every
    sample sit exactly on each face of the post-centre range and 1/8 outside it (dims 0 -> dz = 1 exactly)."""
    heat = torch.randint(-16, 17, (B, K, P), generator=g).float() / 8
    center = torch.randint(-400, 401, (B, 2, P), generator=g).float() / 8
    height = torch.randint(-40, 41, (B, 1, P), generator=g).float() / 8
    dim = torch.randn(B, 3, P, generator=g) * 0.3
    rot = torch.randn(B, 2, P, generator=g)
    rot[..., ::4] = 0.0                                                     # atan2(0, 0)
    vel = torch.randn(B, 2, P, generator=g)
    cx = lambda x: (x - CODER['ox']) / CODER['sx']
    cy = lambda y: (y - CODER['oy']) / CODER['sy']
    faces = [(cx(-20), cy(0), 0.5), (cx(20), cy(0), 0.5), (cx(0), cy(-10), 0.5), (cx(0), cy(10), 0.5),
             (cx(0), cy(0), -2.5), (cx(0), cy(0), 3.5), (cx(-20.125), cy(0), 0.5), (cx(20.125), cy(0), 0.5),
             (cx(0), cy(-10.125), 0.5), (cx(0), cy(10.125), 0.5), (cx(0), cy(0), -2.625), (cx(0), cy(0), 3.625)]
    for i, (x, y, h) in enumerate(faces[:P]):
        center[:, 0, i], center[:, 1, i], height[:, 0, i], dim[:, :, i] = x, y, h, 0.0
        heat[:, :, i] = 0.0
        heat[:, i % K, i] = 0.375 if i % 2 else 0.25                        # score exactly at / above the threshold
    return heat, rot, dim, center, height, vel


@pytest.mark.parametrize('BKP', [(2, 10, 200), (1, 10, 1), (1, 3, 37)], ids=lambda c: 'B%dK%dP%d' % c)
@pytest.mark.parametrize('variant', ['plain', 'vel_range_thr', 'qscore'])
def test_bbox_decode_matches_coder(BKP, variant):
    ops = _ops()
    B, K, P = BKP
    g = torch.Generator().manual_seed(P * K)
    heat, rot, dim, center, height, vel = _coder_inputs(B, K, P, g)
    use_vel = variant != 'plain'
    rng, thr = (RANGE, 0.25) if variant == 'vel_range_thr' else (None, None)
    qs = ql = None
    s64 = heat.double()
    if variant == 'qscore':
        qs = torch.rand(B, K, P, generator=g)
        ql = torch.randint(0, K, (B, P), generator=g)
        qs[:, :, 0] = 0.0                                                   # every product 0: class 0
        s64 = s64.sigmoid() * qs.double() * F.one_hot(ql, K).permute(0, 2, 1).double()
    dv = lambda t: None if t is None else t.to(dev())
    boxes, scores, labels, keep = ops.bbox_decode(*(dv(t) for t in (heat, rot, dim, center, height)),
                                                  dv(vel) if use_vel else None, *CODER.values(), post_range=rng,
                                                  score_thr=thr, qscore=dv(qs), qlabel=dv(ql))
    want_lab = torch.from_numpy(np.argmax(s64.numpy(), axis=1))              # first maximum
    want_sc = s64.max(1).values
    want_box = _coder64().decode_boxes(rot.double(), dim.double(), center.double(), height.double(),
                                       vel.double() if use_vel else None)
    assert torch.equal(labels.cpu().long(), want_lab)
    if variant == 'qscore':
        assert row_err(scores[..., None], want_sc[..., None], want_sc[..., None]) < TOL
    else:
        assert torch.equal(scores.cpu(), heat.max(1).values)
    assert row_err(boxes, want_box, want_box.abs()) < TOL
    want_keep = torch.ones(B, P, dtype=torch.bool)
    if rng is not None:
        r = torch.tensor(rng, dtype=torch.float64)
        want_keep = (want_box[..., :3] >= r[:3]).all(-1) & (want_box[..., :3] <= r[3:]).all(-1) & (want_sc > thr)
        if P >= 12:
            assert want_keep[:, 1:6:2].all() and not want_keep[:, 6:12].any() and not want_keep[:, 0:6:2].any()
    assert torch.equal(keep.cpu(), want_keep)


@pytest.mark.parametrize('code', [8, 10])
def test_bbox_encode_matches_coder(code):
    ops = _ops()
    g = torch.Generator().manual_seed(code)
    heat, rot, dim, center, height, vel = _coder_inputs(1, 10, 300, g)
    boxes = _coder64().decode_boxes(rot.double(), dim.double(), center.double(), height.double(), vel.double())[0]
    boxes = boxes.float() if code == 10 else boxes[:, :7].float()
    got = ops.bbox_encode(boxes.to(dev()), code, *CODER.values())
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        want = _coder64(code).encode(boxes.double())
    finally:
        torch.set_default_dtype(prev)
    assert row_err(got, want, want.abs()) < TOL


# ---------------------------------------------------------------------------------------------------------------------
# 8. circle NMS
# ---------------------------------------------------------------------------------------------------------------------
def _nms_want(boxes, scores, labels, keep, class_mask, thresh, post_max):
    from oracle.mmpi import circle_nms
    out = keep.clone()
    for b in range(boxes.shape[0]):
        cand = (keep[b] & ((torch.tensor(class_mask) >> labels[b].long()) & 1).bool()).nonzero().squeeze(1)
        dets = torch.cat([boxes[b, cand, :2], scores[b, cand, None]], 1).double().numpy()
        kept = set(cand[circle_nms(dets, float(np.float32(thresh)), post_max)].tolist()) if len(cand) else set()
        for i in cand.tolist():
            out[b, i] = i in kept
    return out


@pytest.mark.parametrize('P', [200, 1024, 7])
@pytest.mark.parametrize('task', [(1 << 8, 0.25, 83), (1 << 9, 0.175, 83), (0x3ff, 0.25, 5), (0x3ff, 1.0, 1000)],
                         ids=['cls8', 'cls9_r0.175', 'all_post5', 'all_r1'])
def test_circle_nms_matches_oracle(P, task):
    ops = _ops()
    class_mask, thresh, post_max = task
    g = torch.Generator().manual_seed(P + post_max)
    B = 2
    # centres on a 1/8 grid inside a few 2 x 2 m clusters: many pairs at squared distance exactly 1/4 and 1
    ctr = torch.randint(0, 4, (B, P, 2), generator=g).float() * 8
    boxes = torch.randn(B, P, 9, generator=g)
    boxes[..., :2] = ctr + torch.randint(0, 17, (B, P, 2), generator=g).float() / 8
    scores = torch.randint(1, 5, (B, P), generator=g).float() / 4              # 4 levels: many ties
    labels = torch.randint(0, 10, (B, P), generator=g).int()
    labels[:, :P // 2] = 8 + (torch.arange(P // 2) % 2).int()
    keep = torch.rand(B, P, generator=g) < 0.85
    got = ops.circle_nms(boxes.to(dev()), scores.to(dev()), labels.to(dev()), keep.to(dev()), class_mask, thresh, post_max)
    want = _nms_want(boxes, scores, labels, keep, class_mask, thresh, post_max)
    assert torch.equal(got.cpu(), want)
    assert P < 50 or bool((want != keep).any())


# ---------------------------------------------------------------------------------------------------------------------
# 9. documented limits: rejected before any launch
# ---------------------------------------------------------------------------------------------------------------------
def test_documented_limits_are_rejected():
    d = dev()
    buf = torch.zeros(1 << 16, device=d)
    ibuf = torch.zeros(1 << 14, dtype=torch.int32, device=d)
    prm = (ctypes.c_float * 10)(*P10)
    # rcnn_rois: P <= 1024, V <= 8
    _rejects('di_rcnn_rois_f32', _p(buf), 10, _p(buf), _p(buf), _p(buf), _p(ibuf), _p(ibuf), 1, 1025, 6, 0, prm)
    _rejects('di_rcnn_rois_f32', _p(buf), 10, _p(buf), _p(buf), _p(buf), _p(ibuf), _p(ibuf), 1, 8, 9, 0, prm)
    # roi_align: C % 4 == 0, C <= 512
    for C in (6, 130, 516):
        _rejects('di_roi_align_f32', _p(buf), _p(buf), _p(buf), 1, 2, 2, C, 1.0)
    # dynconv: 16-byte aligned roi and params
    mis = ctypes.c_void_p(buf.data_ptr() + 4)
    for roi, par in ((mis, _p(buf)), (_p(buf), mis)):
        _rejects('di_dynconv_f32', roi, par, _p(buf), _p(buf), _p(buf), _p(buf), _p(buf), 1, 1e-5)
    # circle NMS: P <= 1024
    _rejects('di_circle_nms_f32', _p(buf), 9, _p(buf), _p(ibuf), _p(ibuf), 1, 1025, 0x3ff, 0.25, 83)
    # top-k: k <= 1024, k <= n
    _rejects('di_topk_f32', _p(buf), _p(ibuf), 1, 4096, 1025, None, 0)
    _rejects('di_topk_f32', _p(buf), _p(ibuf), 1, 100, 101, None, 0)
