"""Backward of the base decoder's ImageRCNNBlock (backward.image_rcnn_backward, backward.ImageRCNNFunction) and the
view-group mask of the small-attention gradient (di_mha_small_bwd_f32 with onbits / win) against float64 autograd.

The block's self-attention runs within view groups: query i with win[i] = w >= 0 attends over the keys j of its sample
with bit w of onbits[j]; a query with win < 0 outputs the constant 0.  The kernel is compared with dense attention under
that explicit mask, per row of dq / dk / dv at max(1e-5, 5x the error fp32 autograd makes).  The whole block is compared
with autograd through oracle.mmpi.ImageRCNNBlock._tail run per (sample, live view) group, as the reference runs it, at
max(1e-4, 5x the fp32 error) like the PointRCNNBlock test.  The index-valued decisions (win, onbits, the RoI rectangles)
are the product's own (di_rcnn_rois_f32, pinned by test_rcnn_rois_image_mode_matches_definition), so the oracle is driven
with them rather than re-deriving them from projected floats.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import record_calls, same_bits

pytestmark = pytest.mark.gpu

TOL = 1e-4
C, H = 128, 8


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


def _row_err(got, want):
    """max over rows of max|got - want| / max|want| on that row; a row whose reference is all zero must be exactly zero."""
    g, w = got.double().cpu().reshape(got.shape[0], -1), want.double().cpu().reshape(want.shape[0], -1)
    den = w.abs().amax(1)
    err = (g - w).abs().amax(1)
    return float(torch.where(den > 0, err / den.clamp_min(1e-300), err * 1e30).max())


# ---------------------------------------------------------------------------------------------------------------------
# 1. the masked small-attention gradient
# ---------------------------------------------------------------------------------------------------------------------
def _groups(raw, V):
    """Per-query raw view bits of one sample -> (onbits, win) as di_rcnn_rois_f32 derives them: a view is live when more
    than one query is on it, onbits keeps the live bits, win is the last live view (-1 if none)."""
    cnt = [sum((r >> v) & 1 for r in raw) for v in range(V)]
    live = sum(1 << v for v in range(V) if cnt[v] > 1)
    onbits = [r & live for r in raw]
    win = [max([v for v in range(V) if (o >> v) & 1], default=-1) for o in onbits]
    return onbits, win


def _mask_draw(B, P, V, g):
    """(onbits, win) int32 [B*P] with, in every sample: a view with exactly one query (view V-1: not live, so it is in no
    group), queries with win = -1, a query on two views (with V >= 3 both live; with 2 views the second is the lone
    view V-1), with V >= 3 a live group in which no query wins (every query on view 0 is also on view 1, which comes
    later), and a key seen only by a group in which no query wins (bit V-1; the key's own win is -1).  P = 2 is the one
    hand-made case: a query that sees only itself and the unseen key."""
    onbits, win = [], []
    for _ in range(B):
        if P == 2:
            ob, w = [1 << 1, 1 << 0], [1, -1]
        else:
            raw = [int(x) for x in torch.randint(0, 1 << V, (P,), generator=g) & torch.randint(0, 1 << V, (P,), generator=g)]
            raw = [r & ~(1 << (V - 1)) for r in raw]
            raw[1] = 1 | (1 << (V - 1))                   # on view 0 and alone on view V-1
            raw[3] = raw[4] = 0                           # on no view
            raw[5] = raw[6] = 0b11 if V >= 3 else 1
            if V >= 3:
                raw = [r | 0b10 if r & 1 else r for r in raw]
            ob, w = _groups(raw, V)
            assert not any((o >> (V - 1)) & 1 for o in ob) and w[3] == w[4] == -1
            assert (V < 3 or (w[5] == 1 and ob[5] == 0b11 and 0 not in w))
            ob[2], w[2] = 1 << (V - 1), -1
        onbits += ob
        win += w
    return torch.tensor(onbits, dtype=torch.int32), torch.tensor(win, dtype=torch.int32)


def _masked_attn_grads(qkv, dout, onbits, win, B, P, dtype):
    """autograd of dense attention per sample and head under the mask (win[i] >= 0 and bit win[i] of onbits[j]); rows
    with win < 0 output 0 -> d qkv [B*P, 3C]."""
    x = qkv.to(dev(), dtype).requires_grad_(True)
    ob, w = onbits.to(dev()).long().view(B, P), win.to(dev()).long().view(B, P)
    live = w >= 0
    mask = ((ob[:, None, :] >> w.clamp(min=0)[:, :, None]) & 1).bool() & live[:, :, None]       # [B, i, j]
    with torch.enable_grad():
        qh, kh, vh = (x[:, i * C:(i + 1) * C].reshape(B, P, H, 16) for i in range(3))
        s = torch.einsum('bphd,bkhd->bhpk', qh, kh)
        s = s.masked_fill(~mask[:, None], float('-inf')).masked_fill(~live[:, None, :, None], 0.0)
        o = torch.einsum('bhpk,bkhd->bphd', s.softmax(-1), vh) * live[:, :, None, None]
        (o.reshape(B * P, C) * dout.to(dev(), dtype)).sum().backward()
    return x.grad


def _mha_bwd(qkv, dout, B, P, onbits=None, win=None):
    ops = _ops()
    qd = qkv.to(dev())
    m = () if onbits is None else (onbits.to(dev()), win.to(dev()))
    return ops.mha_small_bwd(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], dout.to(dev()), B, P, H, *m)


@pytest.mark.parametrize('V', [2, 6, 8])
@pytest.mark.parametrize('P', [2, 33, 200, 512])
@pytest.mark.parametrize('B', [1, 2])
def test_masked_mha_small_bwd_matches_float64_autograd(B, P, V):
    g = torch.Generator().manual_seed(B * 1000 + P * 10 + V)
    onbits, win = _mask_draw(B, P, V, g)
    qkv = torch.randn(B * P, 3 * C, generator=g)
    qkv[:, :C] *= 0.5
    dout = torch.randn(B * P, C, generator=g)
    got = _mha_bwd(qkv, dout, B, P, onbits, win)
    want = _masked_attn_grads(qkv, dout, onbits, win, B, P, torch.float64)
    f32 = _masked_attn_grads(qkv, dout, onbits, win, B, P, torch.float32)
    for n, name in enumerate(('dq', 'dk', 'dv')):
        sl = slice(n * C, (n + 1) * C)
        e, bar = _row_err(got[:, sl], want[:, sl]), max(1e-5, 5 * _row_err(f32[:, sl], want[:, sl]))
        print('%s %.1e (bar %.1e)' % (name, e, bar))
        assert e <= bar, (name, e, bar)
    dead = win < 0
    unseen = torch.zeros(B * P, dtype=torch.bool)
    for b in range(B):
        sl = slice(b * P, (b + 1) * P)
        w, ob = win[sl].long(), onbits[sl].long()
        seen = ((ob[:, None] >> w.clamp(min=0)[None, :]) & 1).bool() & (w >= 0)[None, :]          # [j, i]
        unseen[sl] = ~seen.any(1)
    assert bool(dead.any()) and bool((unseen & (onbits != 0)).any())
    gc = got.cpu()
    assert bool((gc[dead, :C] == 0).all()) and bool((gc[unseen, C:] == 0).all())
    assert same_bits(got, _mha_bwd(qkv, dout, B, P, onbits, win)), 'two calls differ'
    # a win < 0 query's q / k / v / dout rows are never read: NaN there changes no other bit
    bad = qkv.clone()
    bad[dead] = float('nan')
    dbad = dout.clone()
    dbad[dead] = float('nan')
    got_nan = _mha_bwd(bad, dbad, B, P, onbits, win).cpu()
    assert same_bits(got_nan, gc)


@pytest.mark.parametrize('B,P', [(1, 1), (2, 200), (1, 512)])
def test_mha_small_bwd_one_group_mask_is_the_unmasked_gradient(B, P):
    g = torch.Generator().manual_seed(P + 5)
    qkv = torch.randn(B * P, 3 * C, generator=g)
    dout = torch.randn(B * P, C, generator=g)
    ones, zeros = torch.ones(B * P, dtype=torch.int32), torch.zeros(B * P, dtype=torch.int32)
    assert same_bits(_mha_bwd(qkv, dout, B, P, ones, zeros), _mha_bwd(qkv, dout, B, P))


def test_mha_small_bwd_takes_both_masks_or_neither():
    ops = _ops()
    B, P = 1, 8
    qd = torch.randn(B * P, 3 * C, device=dev())
    m = torch.zeros(B * P, dtype=torch.int32, device=dev())
    for onbits, win in ((m, None), (None, m)):
        with pytest.raises(RuntimeError, match='go together'):
            ops.mha_small_bwd(qd[:, :C], qd[:, C:2 * C], qd[:, 2 * C:], qd[:, :C], B, P, H, onbits, win)


# ---------------------------------------------------------------------------------------------------------------------
# 2. the whole block
# ---------------------------------------------------------------------------------------------------------------------
def _decoder(base_shape, plusplus=False):
    from test_gpu_rcnn_backward import _decoder as build
    return build(base_shape, plusplus)


def _metas(V, in_hw, B):
    from deepinteraction_b200 import synth
    rig = synth.camera_rig(V, in_hw)
    return [dict(lidar2img=[r.astype(np.float32) for r in rig], input_shape=in_hw, img_shape=[(*in_hw, 3)] * V)
            for _ in range(B)]


def _az_ranges(V, b):
    """Azimuth intervals (degrees) of the query centres of sample b.  The rig's cameras look along k * 360 / V with a
    horizontal half field of view of atan(0.5 / 0.79) = 32.3 degrees; view V / 2 looks along 180 degrees and is kept
    empty (but for one query, _block_inputs).  2 views: view 0 and the blind sides, and in sample 1 also view 1.  6 views:
    the overlap of views 0 and 1 (the only queries on view 0, so its group has no winner), views 1, 2, 4, 5 and the
    overlaps of 1 / 2 and 4 / 5."""
    if V == 2:
        return [(-25, 25), (45, 135), (225, 315)] + ([(155, 205)] if b else [])
    return [(29.5, 30.5), (36, 85), (89.5, 90.5), (95, 140), (215, 265), (269.5, 270.5), (275, 320)]


def _block_inputs(m, B, seed):
    """query rows, prediction rows (centres at 30 - 50 m on the azimuths of _az_ranges, heights -1.5 - 0.5 m; every ninth
    at 60 m above the cameras, on no view; the first query alone on view V / 2; log-dims of 0.4 - 4.5 m; random heading),
    image maps and output gradient, and the frame's camera metadata."""
    g = torch.Generator().manual_seed(seed)
    P, V = m.num_proposals, m.num_views
    h, w = (112, 200) if V == 6 else (28, 50)
    tc = m.test_cfg
    cell, off = tc['out_size_factor'] * tc['voxel_size'][0], tc['pc_range'][0]
    az = torch.empty(B * P, dtype=torch.float64)
    for b in range(B):
        rng = torch.tensor(_az_ranges(V, b), dtype=torch.float64)
        pick = torch.randint(0, rng.shape[0], (P,), generator=g)
        az[b * P:(b + 1) * P] = rng[pick, 0] + torch.rand(P, generator=g, dtype=torch.float64) * (rng[pick, 1] - rng[pick, 0])
    az[0] = 180.0
    az = az * math.pi / 180
    r = 30 + 20 * torch.rand(B * P, generator=g, dtype=torch.float64)
    pred = torch.randn(B * P, m.NP, generator=g)
    pred[:, 0] = ((r * torch.cos(az) - off) / cell).float()
    pred[:, 1] = ((r * torch.sin(az) - off) / cell).float()
    pred[:, 2] = torch.rand(B * P, generator=g) * 2 - 1.5
    pred[torch.arange(B * P) % 9 == 4, 2] = 60.0
    pred[:, 3:6] = torch.rand(B * P, 3, generator=g) * 2.5 - 1.0
    return (torch.randn(B * P, C, generator=g), pred, torch.randn(B * V, h, w, C, generator=g),
            torch.randn(B * P, C, generator=g), _metas(V, (4 * h, 4 * w), B))


def _product_groups(m, pred, metas, B):
    """The product's RoIs, win and onbits (di_rcnn_rois_f32, image mode)."""
    from deepinteraction_b200 import geom
    ops = _ops()
    d = dev()
    proj, aux = (t.to(d) for t in m._camera_consts(metas))
    P, V = m.num_proposals, m.num_views
    rois, win, onbits = ops.rcnn_rois(pred.to(d), B, P, V, 0, m._roi_params(geom.input_hw(metas)), proj, aux)
    return rois.cpu(), win.cpu().long(), onbits.cpu().long()


def _coverage(win, onbits, B, P, V):
    """-> dict of the cases the draw covers: queries on 2+ live views, live groups in which no query wins, queries on no
    live view (a view with exactly one query is not live, so its query is one of them)."""
    multi = sum(bin(int(o)).count('1') >= 2 for o in onbits)
    idle = 0
    for b in range(B):
        sl = slice(b * P, (b + 1) * P)
        for v in range(V):
            if bool(((onbits[sl] >> v) & 1).any()) and not bool((win[sl] == v).any()):
                idle += 1
    return dict(multi_view=multi, idle_groups=idle, no_view=int((win < 0).sum()))


def _oracle_block_grads(m, li, query, rois, win, onbits, img, grad, dtype):
    """autograd through oracle.mmpi.ImageRCNNBlock._tail per (sample, live view) group {j : bit v of onbits[j]} in
    ascending order, with oracle.geometry.roi_align on view v's map at 1 / out_size_factor_img; the output is the rows
    whose win == v.  The product's rectangles serve for the winners; the others get a fixed finite one (their outputs are
    discarded).  Also -> 'reach': the image-map pixels the winners' RoIs sample (gradient of the RoI sums, weights >= 0)."""
    import oracle.mmpi as om
    from oracle.geometry import roi_align
    d = dev()
    BV, h, w, _ = img.shape
    V = m.num_views
    B = BV // V
    P = query.shape[0] // B
    blk = om.ImageRCNNBlock(V, P, m.out_size_factor_img, None, None, C, H, 0.1)
    blk.load_state_dict(m.decode_head[li].state_dict(), strict=True)
    blk = blk.to(device=d, dtype=dtype).eval()
    q = query.to(d, dtype).requires_grad_(True)
    fm = img.to(d, dtype).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    ones = torch.zeros_like(fm, requires_grad=True)
    scale = 1.0 / m.out_size_factor_img
    with torch.enable_grad():
        tot, reach = 0, 0
        for b in range(B):
            for v in range(V):
                grp = (((onbits >> v) & 1) == 1).nonzero().squeeze(1)
                grp = grp[(grp >= b * P) & (grp < (b + 1) * P)]
                if len(grp) == 0:
                    continue
                won = win[grp] == v
                rect = torch.where(won[:, None], rois[grp, 1:].double(), torch.tensor([1.0, 2.0, 30.0, 20.0], dtype=torch.float64))
                roi = roi_align(fm[b * V + v], rect.to(d, dtype), 7, scale, 2)
                out = blk._tail(q[grp.to(d)].unsqueeze(1), roi)
                sel = won.to(d)
                tot = tot + (out[sel] * grad[grp].to(d, dtype)[sel]).sum()
                if bool(won.any()):
                    reach = reach + roi_align(ones[b * V + v] + 1, rect[won].to(d, dtype), 7, scale, 2).sum()
        tot.backward()
        reach.backward()
    res = dict(d_query=q.grad, d_img=fm.grad.permute(0, 2, 3, 1))
    res.update({'grads.' + n: p.grad for n, p in blk.named_parameters()})
    return res, ones.grad.permute(0, 2, 3, 1)


def _relu_margin(m, li, query, pred, img, metas, win):
    """Smallest |pre-activation| of the block's ReLUs (DynamicConv LN1, LN2 and norm3) over the rows with win >= 0 (the
    others are written as 0 and take no gradient), evaluated in float64 from the product's own saved inputs of each.  A
    pre-activation within fp32 rounding of 0 may take the other side of the kink in float64, which moves that element's
    gradient by its full size: such inputs cannot be compared at 1e-4."""
    from deepinteraction_b200 import backward
    d = dev()
    P = m.num_proposals
    B = query.shape[0] // P
    bp, sv = m.pack()['blocks'][li], {}
    with backward._precise():
        backward._rcnn_forward(m, bp, query.to(d), pred.to(d), img.to(d), metas, B, P, saved=sv)
    live = (win >= 0).to(d)
    ln = lambda z, gb: F.layer_norm(z, (C,), gb[0].double(), gb[1].double(), 1e-5)
    Pm, roi = sv['params'][live].double(), sv['roi'][live].double()
    n = roi.shape[0]
    a1 = ln(torch.bmm(roi, Pm[:, :16384].view(n, C, C)), bp['dn1'])
    a2 = ln(torch.bmm(F.relu(a1), Pm[:, 16384:].view(n, C, C)), bp['dn2'])
    a3 = ln(sv['zd3'][live].double(), bp['dn3'])
    nz = lambda a: a.abs()[a != 0]
    return float(min(nz(a1).min(), nz(a2).min(), nz(a3).min()))


def _draw(m, li, B, seed):
    """The first input seed from `seed` on whose draw every ReLU pre-activation is at least 1e-6 from 0 (_relu_margin;
    typical draws have a few within 1e-7) -> (inputs, rois, win, onbits)."""
    P = m.num_proposals
    for s in range(seed, seed + 64):
        inp = _block_inputs(m, B, s)
        rois, win, onbits = _product_groups(m, inp[1], inp[4], B)
        if _relu_margin(m, li, inp[0], inp[1], inp[2], inp[4], win) > 1e-6:
            print('seed', s)
            return inp, rois, win, onbits
    raise AssertionError('no draw with every ReLU pre-activation 1e-6 from 0 in 64 seeds')


@pytest.mark.parametrize('li', [0, 2])
@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_image_rcnn_backward_matches_oracle_autograd(base_shape, li):
    from deepinteraction_b200 import backward
    d = dev()
    m = _decoder(base_shape)
    B, P, V = (1 if base_shape else 2), m.num_proposals, m.num_views
    (query, pred, img, grad, metas), rois, win, onbits = _draw(m, li, B, 300 + 20 * li + base_shape)
    cov = _coverage(win, onbits, B, P, V)
    print(cov)
    assert cov['no_view'] > 0
    assert int(win[0]) == -1 and not bool(((onbits[:P] >> (V // 2)) & 1).any())        # alone on view V / 2: not live
    if base_shape:
        # 2 back-to-back cameras of 64.6 degrees never share a query; the 6-view rig does at its overlaps
        assert cov['multi_view'] > 0 and cov['idle_groups'] > 0
    r = backward.image_rcnn_backward(m, li, query.to(d), pred.to(d), img.to(d), metas, grad.to(d))
    got = dict(d_query=r['d_query'], d_img=r['d_img'])
    got.update({'grads.' + n: t for n, t in r['grads'].items()})
    want, reach = _oracle_block_grads(m, li, query, rois, win, onbits, img, grad, torch.float64)
    f32, _ = _oracle_block_grads(m, li, query, rois.float(), win, onbits, img, grad, torch.float32)
    assert set(got) == set(want) and len(r['grads']) == 24
    sd = m.decode_head[li].state_dict()
    for k, w in want.items():
        if k.startswith('grads.'):
            assert got[k].shape == sd[k[6:]].shape, k
        bar = max(TOL, 5 * rel_err(f32[k].double(), w))
        e = rel_err(got[k].double(), w)
        print('%-45s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)
    dead = (win < 0).to(d)
    assert bool((r['d_query'][dead] == 0).all()), 'd_query of a query on no live view is not exactly 0'
    assert bool((reach > 0).any()) and bool((r['d_img'][reach == 0] == 0).all()), 'a pixel no RoI reaches is not exactly 0'
    # grad_out rows of queries on no live view are ignored
    loud = grad.clone()
    loud[win < 0] = 3e38
    r2 = backward.image_rcnn_backward(m, li, query.to(d), pred.to(d), img.to(d), metas, loud.to(d))
    assert same_bits(r2['d_query'], r['d_query']) and same_bits(r2['d_img'], r['d_img'])
    assert all(same_bits(r2['grads'][k], t) for k, t in r['grads'].items())


# ---------------------------------------------------------------------------------------------------------------------
# 3. autograd.Function, synchronisation, rejections
# ---------------------------------------------------------------------------------------------------------------------
def test_image_rcnn_function_forward_is_the_block_and_backward_matches():
    from deepinteraction_b200 import backward
    from tools.make_goldens import small_frame
    m = _decoder(False)
    gen = torch.Generator().manual_seed(1810)
    fr = small_frame(1810, aug=True, views=2, batch=2)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    pts, new_pts = nhwc(torch.randn(2, 128, 36, 36, generator=gen)), nhwc(torch.randn(2, 128, 36, 36, generator=gen))
    img = nhwc(torch.randn(4, 128, 28, 50, generator=gen))
    dbg = {}
    out = m.forward_rows(pts, new_pts, img, fr['img_metas'], debug=dbg)
    inputs = {0: (dbg['query_feat1'], dbg['first_res']), 2: (dbg['layer_query'][1], out['preds'][1])}
    for li, (q, pred) in inputs.items():
        q0 = q.clone().requires_grad_(True)
        i0 = img.clone().requires_grad_(True)
        with torch.enable_grad():
            y = backward.ImageRCNNFunction.apply(m, li, q0, pred, i0, fr['img_metas'])
            assert same_bits(y.detach(), dbg['layer_query'][li]), li
            grad = torch.randn(y.shape, generator=gen).to(dev())
            (y * grad).sum().backward()
        r = backward.image_rcnn_backward(m, li, q, pred, img, fr['img_metas'], grad)
        assert same_bits(q0.grad, r['d_query']) and same_bits(i0.grad, r['d_img']), li


def test_image_rcnn_backward_rejects_point_v2_and_unsupported_shapes():
    from deepinteraction_b200 import backward
    d = dev()
    m = _decoder(False)
    query, pred, img, grad, metas = _block_inputs(m, 2, 5)
    query, pred, img, grad = (t.to(d) for t in (query, pred, img, grad))
    cases = [(m, li, query, pred, grad) for li in (1, 3)]                                        # PointRCNNBlock
    cases += [(m, 0, query.repeat(13, 1), pred.repeat(13, 1), grad.repeat(13, 1)),               # P = 520
              (m, 0, query[:, :64].contiguous(), pred, grad[:, :64].contiguous())]               # C = 64
    mpp = _decoder(False, plusplus=True)
    cases += [(mpp, li, query, pred[:, :mpp.NP].contiguous(), grad) for li in (0, 2)]              # ImageRCNNBlockV2
    m.pack()
    mpp.pack()
    for dec, li, q, p, gr in cases:
        with record_calls() as calls:
            with pytest.raises(NotImplementedError, match='ImageRCNNBlock'):
                backward.image_rcnn_backward(dec, li, q, p, img, metas, gr)
            with pytest.raises(NotImplementedError, match='ImageRCNNBlock'):
                backward.ImageRCNNFunction.apply(dec, li, q, p, img, metas)
        assert calls == [], (li, calls)


def test_image_rcnn_backward_does_not_synchronise():
    from deepinteraction_b200 import backward
    m = _decoder(False)
    d = dev()
    query, pred, img, grad, metas = _block_inputs(m, 2, 6)
    args = (query.to(d), pred.to(d), img.to(d), metas, grad.to(d))
    backward.image_rcnn_backward(m, 0, *args)               # warm-up: builds the per-pack tensors
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = backward.image_rcnn_backward(m, 0, *args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(r['d_img']).all())
