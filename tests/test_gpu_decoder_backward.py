"""Gradient of the base decoder's losses: the loss-gradient kernel (di_mmpi_losses_bwd_f32), the query-init gradient
(di_query_init_bwd_f32), the prediction and heat-map head backwards and backward.decoder_backward / DecoderLossFunction.

Bars are per tensor, max(1e-4, 5x the error fp32 autograd makes) against float64 autograd, as for the block backwards.
The class-score gradient follows mmcv's closed form (FLT_MIN only inside the logs); where |logit| >= 87 the oracle's
clamp removes autograd's gradient, so those entries are compared with the closed form restated here in float64.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import record_calls, same_bits

pytestmark = pytest.mark.gpu

C = 128


def dev():
    return torch.device('cuda:0')


class _no_tf32:
    """fp32 references in true fp32: cuDNN convolutions default to TF32 on this GPU, whose error would make the bars
    meaningless."""

    def __enter__(self):
        self.saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *a):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.saved


def _bar(got, want, f32):
    return rel_err(got.double().cpu(), want.cpu()), max(1e-4, 5 * rel_err(f32.double().cpu(), want.cpu()))


# ---------------------------------------------------------------------------------------------------------------------
# 1. the loss gradient
# ---------------------------------------------------------------------------------------------------------------------
def _loss_head(P, code, Y):
    from deepinteraction_b200 import mmpi
    from tools import make_goldens as mg
    tc = dict(mg.DEC_TRAIN_CFG, grid_size=[Y * 8, Y * 8, 40], voxel_size=[108.0 / (Y * 8), 108.0 / (Y * 8), 0.2])
    heads = dict(center=(2, 2), height=(1, 2), dim=(3, 2), rot=(2, 2))
    if code == 10:
        heads['vel'] = (2, 2)
    else:
        tc['code_weights'] = tc['code_weights'][:8]
    coder = dict(mg.DEC_CODER, code_size=code, voxel_size=tc['voxel_size'][:2])
    test_cfg = dict(mg.DEC_TEST_CFG, grid_size=tc['grid_size'], voxel_size=tc['voxel_size'][:2])
    return mmpi.DeepInteractionDecoder(num_views=2, num_proposals=P, auxiliary=True, hidden_channel=128, num_classes=10,
                                       num_mmpi=4, num_heads=8, initialize_by_heatmap=True, nms_kernel_size=3,
                                       common_heads=heads, bbox_coder=coder, test_cfg=test_cfg, train_cfg=tc,
                                       **mg.DEC_LOSSES).to(dev()).eval()


def _loss_inputs(m, B, g, positives=True):
    from test_gpu_loss import _random_boxes
    P, L, K, Y = m.num_proposals, 4, 10, m.y_size
    LP = L * P
    code = m.bbox_coder.code_size
    gts = [_random_boxes(12 if positives else 0, g, 40.0)[:, :9 if code == 10 else 7] for _ in range(B)]
    gls = [torch.randint(0, K, (t.shape[0],), generator=g) for t in gts]
    cell = 108.0 / Y
    centre = torch.rand(B, 2, LP, generator=g) * (Y - 2) + 1
    for b in range(B):
        for l in range(L):
            n = gts[b].shape[0]
            centre[b, :, l * P:l * P + n] = ((gts[b][:, :2] + 54.0) / cell).T + 0.3 * torch.randn(2, n, generator=g)
    preds = dict(center=centre, height=torch.randn(B, 1, LP, generator=g) - 1, dim=torch.randn(B, 3, LP, generator=g) * 0.3 + 0.8,
                 rot=torch.randn(B, 2, LP, generator=g), heatmap=torch.randn(B, K, LP, generator=g) * 2,
                 dense_heatmap=torch.randn(B, K, Y, Y, generator=g) * 3 - 2, query_heatmap_score=torch.rand(B, K, P, generator=g))
    if code == 10:
        preds['vel'] = torch.randn(B, 2, LP, generator=g)
    # clip_sigmoid bounds: logits 1e-2 inside and outside p = 1e-4 and 1 - 1e-4 (p 1e-6 from the bound, > 10 fp32 ulp), and
    # the logits whose fp32 p is at each bound (_at_bound)
    x0 = math.log(1e-4 / (1 - 1e-4))
    edge = torch.tensor([x0 + 1e-2, x0 - 1e-2, -x0 - 1e-2, -x0 + 1e-2, _at_bound(x0, LO), _at_bound(-x0, HI)])
    preds['dense_heatmap'].view(-1)[:edge.numel()] = edge
    # saturated class logits (mmcv closed form), on rows the mask keeps (label weight 1)
    preds['heatmap'][0, 0, :4] = torch.tensor([90.0, -90.0, 88.0, -100.0])
    masks = [torch.rand(B, P, generator=g) > 0.25 for _ in range(2)]
    masks[0][0, :4] = True
    return gts, gls, preds, masks


LO = torch.tensor(1e-4, dtype=torch.float32)
HI = torch.tensor(1.0, dtype=torch.float32) - LO          # 1.f - 1e-4f, as the kernels and torch's fp32 clamp take it


def _p32(x):
    """The fp32 sigmoid as the loss kernels evaluate it, 1 / (1 + exp(-x)) (IEEE division, no fast math)."""
    x = x.to(dev(), torch.float32)
    return (1.0 / (1.0 + torch.exp(-x))).cpu()


def _at_bound(x0, bound):
    """The fp32 logit near x0 whose fp32 p equals the bound, or (no fp32 logit hits it exactly: near 1e-4 one logit ulp
    moves p by ~13 ulp) the one whose p is nearest to it."""
    x = torch.tensor(x0, dtype=torch.float32)
    cand = x + torch.arange(-4000, 4001, dtype=torch.float32) * torch.finfo(torch.float32).eps * abs(x0)
    p = _p32(cand)
    hit = (p == bound).nonzero()
    return float(cand[hit[0, 0]] if hit.numel() else cand[(p.double() - float(bound)).abs().argmin()])


def _masked(t, masks, B, P, L=4):
    """label / bbox weights and avg factors of the base decoder's loss, with the on-image mask applied here to the
    unmasked targets t (mask l / 2 on layers 0 and 2, deepinteraction_decoder.py:503-526), not by di_loss_targets_f32."""
    lw, bw = t['label_weights'].clone().double(), t['bbox_weights'].clone().double()
    pos = t['bbox_weights'][..., 0] > 0
    num_pos = []
    for l in range(L):
        sl = slice(l * P, (l + 1) * P)
        if l % 2 == 0:
            mk = masks[l // 2].to(lw.device).double()
            lw[:, sl] *= mk
            bw[:, sl] *= mk[..., None]
        num_pos.append(float((pos[:, sl].double() * (lw[:, sl] != 0).double()).sum()))
    return lw, bw, num_pos


def _oracle_loss_grads(m, preds, t, masks, w, dtype):
    """float64 / fp32 autograd of oracle.loss on the product's UNMASKED targets t (use_masks=False), the on-image masks
    applied by _masked -> (d dense [B, Y, X, K], d rows [L, B*P, NP]).  clip_sigmoid's clamp passes the gradient where the
    fp32 p (_p32, what the product clamps) lies in [1e-4, 1 - 1e-4], torch's inclusive rule; away from the bounds that is
    oracle.loss.clip_sigmoid's own decision."""
    import oracle.loss as ol
    from tools import make_goldens as mg
    d = dev()
    P, L = m.num_proposals, 4
    code = m.bbox_coder.code_size
    cw = torch.tensor(m.train_cfg['code_weights'], dtype=dtype, device=d)
    x = {k: v.to(d, dtype).requires_grad_(True) for k, v in preds.items() if k != 'query_heatmap_score'}
    lc, lb, lh = (mg.DEC_LOSSES[k] for k in ('loss_cls', 'loss_bbox', 'loss_heatmap'))
    fl = ol.FocalLoss(**{k: v for k, v in lc.items() if k != 'type'})
    l1 = ol.L1Loss(**{k: v for k, v in lb.items() if k != 'type'})
    gf = ol.GaussianFocalLoss(**{k: v for k, v in lh.items() if k != 'type'})
    B, K = x['heatmap'].shape[:2]
    heat_t = t['heatmap'].to(dtype)
    lw_all, bw_all, num_pos = _masked(t, masks, B, P, L)
    p32 = _p32(preds['dense_heatmap']).to(d)
    keep = (p32 >= LO.to(d)) & (p32 <= HI.to(d))
    with torch.enable_grad():
        p = x['dense_heatmap'].sigmoid()
        pc = torch.where(keep, p, ol.clip_sigmoid(x['dense_heatmap'].detach().clone()))
        inside = (p.detach() >= 1e-4) & (p.detach() <= 1 - 1e-4)
        assert float((keep == inside).double().mean()) > 0.999
        tot = w[0] * gf(pc, heat_t, avg_factor=max(float((heat_t == 1).sum()), 1.0))
        box = torch.cat([x[k] for k in ('center', 'height', 'dim', 'rot', 'vel') if k in x], 1)      # [B, code, LP]
        for l in range(L):
            sl = slice(l * P, (l + 1) * P)
            af = max(num_pos[l], 1.0)
            sc = x['heatmap'][:, :, sl].permute(0, 2, 1).reshape(-1, K)
            tot = tot + w[1 + 2 * l] * fl(sc, t['labels'][:, sl].reshape(-1), lw_all[:, sl].reshape(-1).to(dtype), avg_factor=af)
            bp = box[:, :, sl].permute(0, 2, 1).reshape(-1, code)
            bw = bw_all[:, sl].reshape(-1, code).to(dtype) * cw
            tot = tot + w[2 + 2 * l] * l1(bp, t['bbox_targets'][:, sl].reshape(-1, code).to(dtype), bw, avg_factor=af)
        tot.backward()
    d_dense = x['dense_heatmap'].grad.permute(0, 2, 3, 1)
    rows = torch.cat([x[k].grad for k in m.head_order], 1)                 # [B, NP, LP]
    d_rows = rows.view(B, -1, L, P).permute(2, 0, 3, 1).reshape(L, B * P, -1)
    return d_dense, d_rows


def _closed_form_cls(x, label, k, alpha=0.25, gamma=2.0):
    """mmcv sigmoid_focal_loss backward, float64, FLT_MIN inside the logs only."""
    p = torch.sigmoid(x.double())
    tiny = torch.finfo(torch.float32).tiny
    if label == k:
        return -alpha * (1 - p) ** gamma * (1 - p - gamma * p * torch.log(p.clamp(min=tiny)))
    return -(1 - alpha) * p ** gamma * (gamma * (1 - p) * torch.log((1 - p).clamp(min=tiny)) - p)


@pytest.mark.parametrize('code', [8, 10])
@pytest.mark.parametrize('P', [24, 200])
@pytest.mark.parametrize('B', [1, 2])
def test_loss_gradient_matches_float64_autograd(B, P, code):
    d = dev()
    Y = 36 if P == 24 else 180
    m = _loss_head(P, code, Y)
    g = torch.Generator().manual_seed(B * 100 + P + code)
    gts, gls, preds, masks = _loss_inputs(m, B, g)
    m.on_the_image_mask = [k.to(d) for k in masks]
    gd, ld, pd = [b.to(d) for b in gts], [l.to(d) for l in gls], {k: v.to(d) for k, v in preds.items()}
    m.loss(gd, ld, [[pd]])
    t = m._last_targets
    tu = m._targets(gd, ld, pd, use_masks=False)
    assert int((t['bbox_targets'][..., :1] != 0).sum()) > 0 and bool((t['label_weights'] == 0).any())
    w = torch.rand(2 + 2 * 4, generator=g) + 0.5
    d_heat, d_pred = m.loss_backward(w.to(d))
    K, NP = 10, m.NP
    assert d_heat.shape == (B, Y, Y, 32) and d_pred.shape == (4, B * P, NP)
    want_h, want_r = _oracle_loss_grads(m, preds, tu, masks, w.double(), torch.float64)
    f32_h, f32_r = _oracle_loss_grads(m, preds, tu, masks, w.float(), torch.float32)
    # saturated logits: the closed form, on rows of label weight 1
    af0 = max(_masked(tu, masks, B, P)[2][0], 1.0)
    for q in range(4):
        lab, lw = int(t['labels'][0, q]), float(t['label_weights'][0, q])
        assert lw == 1.0
        ref = torch.tensor([float(_closed_form_cls(preds['heatmap'][0, c, q], lab, c)) * lw * float(w[1]) / af0
                            for c in range(K)], dtype=torch.float64)
        want_r[0, q, code:] = ref.to(want_r.device)
        f32_r[0, q, code:] = ref.to(f32_r.device).float()
        assert float(ref.abs().max()) > 0
    e, bar = _bar(d_heat[..., :K], want_h, f32_h)
    print('d_dense %.1e (bar %.1e)' % (e, bar))
    assert e <= bar
    e, bar = _bar(d_pred, want_r, f32_r)
    print('d_pred %.1e (bar %.1e)' % (e, bar))
    assert e <= bar
    assert bool((d_heat[..., K:] == 0).all()), 'pad channels are not 0'
    flat = d_heat.permute(0, 3, 1, 2)[:, :K].reshape(-1)
    assert float(flat[1]) == 0 and float(flat[3]) == 0 and float(flat[0]) != 0 and float(flat[2]) != 0   # outside / inside
    p_at = _p32(flat.new_tensor([float(preds['dense_heatmap'].view(-1)[i]) for i in (4, 5)]))
    assert float(p_at[1]) == float(HI) and float(flat[5]) != 0        # exactly at 1 - 1e-4: torch's clamp passes it
    assert (float(flat[4]) != 0) == bool(p_at[0] >= LO)              # next to 1e-4: the side its fp32 p is on
    # zero-weight rows (masked or unassigned with weight 0) are exactly 0
    lw = t['label_weights'].view(B, 4, P).permute(1, 0, 2).reshape(4, B * P)
    bw = t['bbox_weights'].view(B, 4, P, code).permute(1, 0, 2, 3).reshape(4, B * P, code)
    assert bool((d_pred[..., code:][lw == 0] == 0).all()) and bool((lw == 0).any())
    assert bool((d_pred[..., :code][bw == 0] == 0).all())
    d2 = m.loss_backward(w.to(d))
    assert same_bits(d2[0], d_heat) and same_bits(d2[1], d_pred), 'two calls differ'


def test_loss_gradient_is_zero_at_equal_box_and_without_positives():
    d = dev()
    m = _loss_head(24, 10, 36)
    g = torch.Generator().manual_seed(77)
    gts, gls, preds, masks = _loss_inputs(m, 1, g, positives=False)
    m.on_the_image_mask = [k.to(d) for k in masks]
    gd, ld, pd = [b.to(d) for b in gts], [l.to(d) for l in gls], {k: v.to(d) for k, v in preds.items()}
    losses = m.loss(gd, ld, [[pd]])
    t = m._last_targets
    tu = m._targets(gd, ld, pd, use_masks=False)
    assert float(t['num_pos'].sum()) == 0 and float((t['heatmap'] == 1).sum()) == 0      # avg factors 1
    w = torch.ones(10)
    d_heat, d_pred = m.loss_backward(w.to(d))
    want_h, want_r = _oracle_loss_grads(m, preds, tu, masks, w.double(), torch.float64)
    f32_h, f32_r = _oracle_loss_grads(m, preds, tu, masks, w.float(), torch.float32)
    for q in range(4):
        lab, lw = int(t['labels'][0, q]), float(t['label_weights'][0, q])
        ref = torch.tensor([float(_closed_form_cls(preds['heatmap'][0, c, q], lab, c)) * lw for c in range(10)], dtype=torch.float64)
        want_r[0, q, 10:] = ref.to(d)
        f32_r[0, q, 10:] = ref.float().to(d)
    e, bar = _bar(d_heat[..., :10], want_h, f32_h)
    assert e <= bar
    e, bar = _bar(d_pred, want_r, f32_r)
    assert e <= bar and bool((d_pred[..., :10] == 0).all())
    assert float(losses['loss_heatmap']) > 0
    # pred == target: sign 0
    m2 = _loss_head(24, 8, 36)
    gts, gls, preds, masks = _loss_inputs(m2, 1, torch.Generator().manual_seed(5))
    m2.on_the_image_mask = [k.to(d) for k in masks]
    pd = {k: v.to(d) for k, v in preds.items()}
    m2.loss([b.to(d) for b in gts], [l.to(d) for l in gls], [[pd]])
    t = m2._last_targets
    pos = (t['bbox_weights'][0, :, 0] > 0).nonzero().squeeze(1)
    assert pos.numel() > 0
    j = int(pos[0])
    pd['height'][0, 0, j] = t['bbox_targets'][0, j, 2]
    m2.loss([b.to(d) for b in gts], [l.to(d) for l in gls], [[pd]])
    _, d_pred = m2.loss_backward(torch.ones(10, device=d))
    l, i = j // 24, j % 24
    assert float(d_pred[l, i, 2]) == 0 and float(d_pred[l, i, 0]) != 0


# ---------------------------------------------------------------------------------------------------------------------
# 2. query init
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,P,HW', [(1, 24, 36 * 36), (2, 200, 180 * 180), (2, 40, 9)])
def test_query_init_gradient_matches_index_add(B, P, HW):
    from deepinteraction_b200 import ops
    d = dev()
    K = 10
    g = torch.Generator().manual_seed(B + P)
    pix = torch.randint(0, HW, (B, P), generator=g)
    pix[0, 5] = pix[0, 2]                                  # one pixel selected for two classes
    cls = torch.randint(0, K, (B, P), generator=g)
    cls[0, 5] = (cls[0, 2] + 1) % K
    top = (cls * HW + pix).int()
    dq = torch.randn(B * P, C, generator=g)
    base = torch.randn(B, HW, C, generator=g)
    want = base.double().clone()
    for b in range(B):
        want[b].index_add_(0, pix[b], dq[b * P:(b + 1) * P].double())
    want_w = torch.zeros(C, K, dtype=torch.float64).index_add_(1, cls.reshape(-1), dq.double().t())
    # the kernel's order: per pixel the base row, then the proposals at that pixel in proposal order (fp32 adds)
    seq, seq_w = base.clone(), torch.zeros(C, K)
    for b in range(B):
        for j in range(P):
            seq[b, pix[b, j]] += dq[b * P + j]
            seq_w[:, cls[b, j]] += dq[b * P + j]
    seq_b = torch.zeros(C)
    for r_ in range(B * P):
        seq_b += dq[r_]
    sel = torch.zeros(B, HW, dtype=torch.bool)
    for b in range(B):
        sel[b, pix[b]] = True
    runs = []
    for _ in range(2):
        d_feat = base.to(d)
        d_w, d_b = ops.query_init_bwd(dq.to(d), top.to(d), cls.int().to(d), d_feat, K)
        runs.append((d_feat.cpu(), d_w.cpu(), d_b.cpu()))
    d_feat, d_w, d_b = runs[0]
    assert same_bits(d_feat[~sel], base[~sel]), 'an unselected row changed'
    assert rel_err(d_feat.double(), want) < 1e-6
    assert rel_err(d_w.double(), want_w) < 1e-5 and rel_err(d_b.double(), dq.double().sum(0)) < 1e-5
    assert same_bits(d_feat, seq) and same_bits(d_w, seq_w) and same_bits(d_b, seq_b), 'not summed in proposal order'
    assert all(same_bits(a, b) for a, b in zip(runs[0], runs[1])), 'two calls differ'


# ---------------------------------------------------------------------------------------------------------------------
# 3. prediction and heat-map heads
# ---------------------------------------------------------------------------------------------------------------------
def _decoder(base_shape):
    from test_gpu_rcnn_backward import _decoder as build
    return build(base_shape)


def _oracle_pred_grads(m, ffn, srcs, grad, dtype):
    import oracle.mmpi as om
    d = dev()
    o = om.PredictionFFN(sum(s.shape[1] for s in srcs), m.heads).to(d, dtype).eval()
    o.load_state_dict(ffn.state_dict(), strict=True)
    xs = [s.to(d, dtype).requires_grad_(True) for s in srcs]
    with torch.enable_grad():
        x = torch.cat(xs, 1).t().unsqueeze(0)                                 # [1, cin, M]
        out = o(x)
        y = torch.cat([out[h][0].t() for h in m.head_order], 1)             # [M, NP]
        (y * grad.to(d, dtype)).sum().backward()
    res = {'d%d' % i: x_.grad for i, x_ in enumerate(xs)}
    res.update({'grads.' + n: p.grad for n, p in o.named_parameters()})
    with torch.no_grad():
        margin = min(float(getattr(o, h)[0].bn(getattr(o, h)[0].conv(x)).abs().min()) for h in m.head_order)
    return res, margin


@pytest.mark.parametrize('li', [None, 0, 3])
def test_pred_head_backward_matches_oracle_autograd(li):
    from deepinteraction_b200 import backward
    m = _decoder(False)
    d = dev()
    ffn = m.prediction_heads[0] if li is None else m.pred_head[li]
    n = 1 if li is None else 2
    for seed in range(40):
        g = torch.Generator().manual_seed(600 + seed)
        srcs = [torch.randn(80, C, generator=g) for _ in range(n)]
        grad = torch.randn(80, m.NP, generator=g)
        want, margin = _oracle_pred_grads(m, ffn, srcs, grad, torch.float64)
        if margin > 1e-6:                                   # every ReLU pre-activation 1e-6 from 0 (_relu_margin)
            break
    with _no_tf32():
        f32, _ = _oracle_pred_grads(m, ffn, srcs, grad, torch.float32)
    r = backward.pred_head_backward(m, li, [s.to(d) for s in srcs], grad.to(d))
    got = {'d%d' % i: t for i, t in enumerate(r['d_srcs'])}
    got.update({'grads.' + k: v for k, v in r['grads'].items()})
    assert set(got) == set(want)
    sd = ffn.state_dict()
    for k, w in want.items():
        if k.startswith('grads.'):
            assert got[k].shape == sd[k[6:]].shape, k
        e, bar = _bar(got[k], w, f32[k])
        print('%-30s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)


@pytest.mark.parametrize('base_shape', [False, True], ids=['36x36', '180x180'])
def test_heatmap_head_backward_matches_oracle_autograd(base_shape):
    import oracle.mmpi as om
    from deepinteraction_b200 import backward
    m = _decoder(base_shape)
    d = dev()
    Y = m.y_size
    K = 10
    g = torch.Generator().manual_seed(700 + Y)
    x = torch.randn(1, Y, Y, C, generator=g)
    grad = torch.zeros(1, Y, Y, 32)
    grad[..., :K] = torch.randn(1, Y, Y, K, generator=g)

    def run(dtype):
        seq = torch.nn.Sequential(om.ConvModule2d(C, C), torch.nn.Conv2d(C, K, 3, padding=1)).to(d, dtype).eval()
        seq.load_state_dict(m.heatmap_head_img.state_dict(), strict=True)
        xi = x.permute(0, 3, 1, 2).to(d, dtype).requires_grad_(True)
        with torch.enable_grad():
            pre = seq[0].bn(seq[0].conv(xi))
            y = seq[1](F.relu(pre))
            (y * grad[..., :K].permute(0, 3, 1, 2).to(d, dtype)).sum().backward()
        res = {'d_new_pts': xi.grad.permute(0, 2, 3, 1)}
        res.update({'grads.' + n: p.grad for n, p in seq.named_parameters()})
        return res, float(pre.abs().min())
    want, margin = run(torch.float64)
    print('relu margin %.1e' % margin)
    with _no_tf32():
        f32, _ = run(torch.float32)
    r = backward.heatmap_head_backward(m, x.to(d), grad.to(d))
    got = dict(d_new_pts=r['d_new_pts'])
    got.update({'grads.' + k: v for k, v in r['grads'].items()})
    assert set(got) == set(want)
    sd = m.heatmap_head_img.state_dict()
    for k, w in want.items():
        if k.startswith('grads.'):
            assert got[k].shape == sd[k[6:]].shape, k
        e, bar = _bar(got[k], w, f32[k])
        print('%-20s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)


# ---------------------------------------------------------------------------------------------------------------------
# 4. the whole decoder
# ---------------------------------------------------------------------------------------------------------------------
def _frame(m, B, seed):
    from tools.make_goldens import small_frame, DEC_TRAIN_CFG
    from test_gpu_loss import _random_boxes
    d = dev()
    V = m.num_views
    Y = m.y_size
    h, w = (112, 200) if V == 6 else (28, 50)
    g = torch.Generator().manual_seed(seed)
    fr = small_frame(seed, aug=True, views=2, batch=B)
    metas = fr['img_metas']
    if V == 6:
        from test_gpu_image_rcnn_backward import _metas
        metas = _metas(6, (4 * h, 4 * w), B)
    nhwc = lambda t: t.contiguous().to(d)
    pts = nhwc(torch.randn(B, Y, Y, C, generator=g))
    new_pts = nhwc(torch.randn(B, Y, Y, C, generator=g))
    img = nhwc(torch.randn(B * V, h, w, C, generator=g))
    gts = [_random_boxes(15, g, 40.0).to(d) for _ in range(B)]
    gls = [torch.randint(0, 10, (15,), generator=g).to(d) for _ in range(B)]
    return pts, new_pts, img, metas, gts, gls


def _with_train_cfg(m, base_shape):
    from deepinteraction_b200 import loss as L
    from tools import make_goldens as mg
    tc = dict(mg.DEC_TRAIN_CFG)
    if base_shape:
        tc.update(grid_size=[1440, 1440, 40], voxel_size=[0.075, 0.075, 0.2])
    m.train_cfg = tc
    m.bbox_assigner = L._build(L.ASSIGNERS, tc['assigner'])
    m._loss_cfg['bbox'] = dict(mg.DEC_LOSSES['loss_bbox'])
    return m


@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_decoder_backward_losses_keys_and_determinism(base_shape):
    from deepinteraction_b200 import backward
    m = _with_train_cfg(_decoder(base_shape), base_shape)
    B = 1 if base_shape else 2
    pts, new_pts, img, metas, gts, gls = _frame(m, B, 910 + base_shape)
    w = (torch.rand(10, generator=torch.Generator().manual_seed(3)) + 0.5).to(dev())
    r = backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls, w)
    ref = m.loss(gts, gls, m.forward_nhwc(pts, new_pts, img, metas))
    assert set(ref) == set(r['losses']) and all(same_bits(r['losses'][k], ref[k]) for k in ref)
    sd = dict(m.named_parameters())
    want = {k for k in sd if not k.startswith('heatmap_head.')}
    assert set(r['grads']) == want
    for k, v in r['grads'].items():
        assert v.shape == sd[k].shape, k
        assert bool(torch.isfinite(v).all()), k
    assert all(bool((v == 0).all()) for k, v in r['grads'].items() if k.startswith('prediction_heads.0.'))
    for k in ('d_pts_conv', 'd_new_pts'):
        assert r[k].shape == pts.shape and bool(torch.isfinite(r[k]).all()) and float(r[k].abs().max()) > 0
    assert r['d_img'].shape == img.shape and float(r['d_img'].abs().max()) > 0
    nonzero = [k for k, v in r['grads'].items() if not k.startswith('prediction_heads.0.') and float(v.abs().max()) > 0]
    assert len(nonzero) > 0.9 * (len(want) - len(list(m.prediction_heads[0].parameters())))
    r2 = backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls, w)
    for k in ('d_pts_conv', 'd_new_pts', 'd_img'):
        assert same_bits(r2[k], r[k]), k
    assert all(same_bits(r2['grads'][k], v) for k, v in r['grads'].items()), 'two calls differ'


def test_decoder_backward_is_linear_in_the_upstream_weights():
    """Each loss term's gradient enters once: the gradient for weights w equals the w-weighted sum of the per-term ones."""
    from deepinteraction_b200 import backward
    m = _with_train_cfg(_decoder(False), False)
    pts, new_pts, img, metas, gts, gls = _frame(m, 2, 930)
    d = dev()
    eye = torch.eye(10, device=d)
    parts = [backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls, eye[i]) for i in range(9)]
    w = torch.tensor([0.7, 1.3, 0.4, 2.0, 0.9, 1.1, 0.6, 1.5, 0.8, 5.0], device=d)
    r = backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls, w)
    for k in ('d_pts_conv', 'd_new_pts', 'd_img'):
        want = sum(float(w[i]) * parts[i][k].double() for i in range(9))
        assert rel_err(r[k].double(), want) < 1e-5, k
    # the matched_ious entry takes no gradient
    z = backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls, eye[9])
    assert all(bool((z[k] == 0).all()) for k in ('d_pts_conv', 'd_new_pts', 'd_img'))


def test_decoder_loss_function_matches_decoder_backward():
    from deepinteraction_b200 import backward
    m = _with_train_cfg(_decoder(False), False)
    pts, new_pts, img, metas, gts, gls = _frame(m, 2, 940)
    xs = [t.clone().requires_grad_(True) for t in (pts, new_pts, img)]
    with torch.enable_grad():
        loss = backward.DecoderLossFunction.apply(m, *xs, metas, gts, gls)
        loss.backward()
    losses = m.loss(gts, gls, m.forward_nhwc(pts, new_pts, img, metas))
    assert same_bits(loss.detach(), torch.stack([v for k, v in losses.items() if 'loss' in k]).sum())
    r = backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls)
    for x, k in zip(xs, ('d_pts_conv', 'd_new_pts', 'd_img')):
        assert same_bits(x.grad, r[k]), k


def test_decoder_backward_does_not_synchronise():
    from deepinteraction_b200 import backward
    m = _with_train_cfg(_decoder(False), False)
    args = _frame(m, 2, 950)
    backward.decoder_backward(m, *args)                  # warm-up: builds the per-pack tensors
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = backward.decoder_backward(m, *args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(r['d_pts_conv']).all())


def test_decoder_backward_rejects_plusplus_before_any_launch():
    from deepinteraction_b200 import backward
    from test_gpu_rcnn_backward import _decoder as build
    mpp = build(False, True)
    pts, new_pts, img, metas, gts, gls = _frame(mpp, 2, 960)
    mpp.pack()
    with record_calls() as calls:
        with pytest.raises(NotImplementedError, match='base DeepInteractionDecoder'):
            backward.decoder_backward(mpp, pts, new_pts, img, metas, gts, gls)
        with pytest.raises(NotImplementedError, match='base DeepInteractionDecoder'):
            backward.DecoderLossFunction.apply(mpp, pts, new_pts, img, metas, gts, gls)
    assert calls == []
    # maps the block backwards would reject: a wrong view count, channel count or BEV size
    m = _with_train_cfg(_decoder(False), False)
    m.pack()
    bad = [(pts, new_pts, img[:3]), (pts, new_pts, img[..., :64].contiguous()), (pts[:, :20].contiguous(), new_pts, img),
           (pts, new_pts[..., :64].contiguous(), img)]
    with record_calls() as calls:
        for a, b, c in bad:
            with pytest.raises(NotImplementedError, match='pixel-major'):
                backward.decoder_backward(m, a, b, c, metas, gts, gls)
    assert calls == []


# ---------------------------------------------------------------------------------------------------------------------
# 5. the whole decoder against a float64 chain of the oracle's modules
# ---------------------------------------------------------------------------------------------------------------------
def _product_forward(m, pts, new_pts, img, metas, gts, gls):
    """The product's eager forward with its saved values, its outputs, the unmasked targets and the on-image masks."""
    from deepinteraction_b200 import geom
    d = dev()
    B = pts.shape[0]
    proj, aux = (t.to(d) for t in m._camera_consts(metas))
    sv = {}
    r = m._schedule(pts, new_pts, img, geom.input_hw(metas), proj, aux, sv)
    pd = m._outputs(r, B)[0][0]
    tu = m._targets(gts, gls, pd, use_masks=False)
    masks = [(w.view(B, -1) != -1) for w in r['wins']]
    return sv, r, pd, tu, masks


def _oracle_decoder_grads(m, pts, new_pts, img, metas, fw, w, dtype):
    """Gradient of the base decoder's loss as a chain of float64 (or fp32) autograd through the oracle's modules, each
    evaluated at the product's own saved activations and driven by its decisions (top-k, labels, RoI rectangles, win,
    onbits): oracle.loss on the unmasked targets with the masks applied here (_oracle_loss_grads), the fallback rows
    routed to prediction_heads[0] by selection, oracle.mmpi.PredictionFFN per head, the block drivers of
    test_gpu_rcnn_backward / test_gpu_image_rcnn_backward, the layer driver of test_gpu_decoder_layer_backward, the query
    init as an index_add and a one-hot product, and the heat-map head as ConvModule2d + Conv2d.
    -> (dict of d_pts_conv, d_new_pts, d_img and 'grads.<state_dict key>', reach of the image RoIs)."""
    import oracle.mmpi as om
    from test_gpu_decoder_layer_backward import _oracle_grads as layer_grads
    from test_gpu_image_rcnn_backward import _oracle_block_grads as image_grads, _product_groups
    from test_gpu_rcnn_backward import _oracle_block_grads as point_grads
    d = dev()
    sv, r, pd, tu, masks = fw
    B, Y, X, _ = pts.shape
    P, L, K = m.num_proposals, len(m.decode_head), m.num_classes_heat
    d_dense, d_rows = _oracle_loss_grads(m, pd, tu, masks, w.to(dtype), dtype)
    qs = [sv['query_feat1']] + sv['layer_query']
    out, wins = {}, list(r['wins'])
    put = lambda prefix, res: out.update({'grads.' + prefix + k[6:]: v for k, v in res.items() if k.startswith('grads.')})
    dq, d_first, d_img, d_new, reach = None, 0, 0, 0, 0
    acc = lambda a, b: b if a is None else a + b
    for li in reversed(range(L)):
        image = li % 2 == 0
        u = d_rows[li].to(dtype)
        if image:
            live = (wins[li // 2] >= 0).to(d)[:, None]
            d_first = d_first + torch.where(live, torch.zeros_like(u), u)
            u = torch.where(live, u, torch.zeros_like(u))
        ph, _ = _oracle_pred_grads(m, m.pred_head[li], [qs[li + 1], qs[li]], u, dtype)
        put('pred_head.%d.' % li, ph)
        d_out = acc(dq, ph['d0'])
        pred_in = r['preds'][li - 1] if li else sv['first_res']
        if image:
            rois, win, onbits = _product_groups(m, pred_in, metas, B)
            res, rc = image_grads(m, li, qs[li], rois, win, onbits, img, d_out, dtype)
            d_img, reach = d_img + res['d_img'], reach + rc
        else:
            res = point_grads(m, li, qs[li], sv['rois'][li][:, 1:].to(dtype), new_pts, d_out, dtype)
            d_new = d_new + res['d_bev']
        put('decode_head.%d.' % li, res)
        dq = res['d_query'] + ph['d1']
    pf, _ = _oracle_pred_grads(m, m.prediction_heads[0], [qs[0]], d_first, dtype)
    put('prediction_heads.0.', pf)
    dq = dq + pf['d0']
    rl = layer_grads(m, sv['query_feat0'], sv['query_pos0'], pts, dq, dtype, d)
    put('decoder.0.', rl)
    # query init: q0 = pts_conv[b, pix] + W[:, label] + bias
    top = sv['top'].long()
    pix, lab = top % (Y * X), top // (Y * X)
    dq0 = rl['d_query']
    d_pts = rl['d_bev'].reshape(B, Y * X, -1).clone()
    for b in range(B):
        d_pts[b].index_add_(0, pix[b].to(d), dq0[b * P:(b + 1) * P])
    onehot = F.one_hot(lab.reshape(-1), K).to(d, dtype)
    out['grads.class_encoding.weight'] = (dq0.t() @ onehot).unsqueeze(-1)
    out['grads.class_encoding.bias'] = dq0.sum(0)
    # heat-map head on new_pts.  Its ReLU has B*Y*X*C pre-activations (4.1 M at the base shape), several of which lie within
    # the product's 3xTF32 rounding of 0; the loss gradient concentrates on few pixels, so one such element taking the other
    # side of the kink moves the first convolution's weight gradient by ~1e-2.  The derivative at the kink is a decision
    # like the top-k: where the float64 pre-activation is within 1e-5 of 0 (relative to the largest), the side is the
    # product's (_heat_relu_side); everywhere else it is the oracle's own.
    seq = torch.nn.Sequential(om.ConvModule2d(C, C), torch.nn.Conv2d(C, K, 3, padding=1)).to(d, dtype).eval()
    seq.load_state_dict(m.heatmap_head_img.state_dict(), strict=True)
    xi = new_pts.to(d, dtype).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    with torch.enable_grad():
        z = seq[0].bn(seq[0].conv(xi))
        on = _heat_relu_side(m, new_pts, z.detach())
        (seq[1](z * on) * d_dense.to(dtype).permute(0, 3, 1, 2)).sum().backward()
    out.update({'grads.heatmap_head_img.' + n: p.grad for n, p in seq.named_parameters()})
    out.update(d_pts_conv=d_pts.view(B, Y, X, -1), d_new_pts=d_new + xi.grad.permute(0, 2, 3, 1), d_img=d_img)
    return out, reach


def _heat_relu_side(m, new_pts, z):
    """ReLU side of the heat-map head's pre-activations z [B, C, Y, X]: z > 0, but the product's side (its re-run of the
    first convolution) where |z| < 1e-5 max|z|.  Every disagreement must be such a near-kink element."""
    from deepinteraction_b200 import backward, ops
    pk = m.pack()
    w0, b0, _, _ = pk['heatmap_head_img']
    with backward._precise():
        h = ops.conv3x3(new_pts.contiguous(), w0, b0, C, True, False, ops.ACT_RELU).permute(0, 3, 1, 2)
    mine, theirs = z > 0, h > 0
    near = z.abs() < 1e-5 * float(z.abs().max())
    assert bool((near | (mine == theirs)).all()), 'the heat-map ReLU side differs away from the kink'
    print('heat-map ReLU: %d near-kink elements, %d on the other side' % (int(near.sum()), int((mine != theirs).sum())))
    return torch.where(near, theirs, mine).to(z.dtype)


@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_decoder_backward_matches_float64_oracle_chain(base_shape):
    from deepinteraction_b200 import backward
    m = _with_train_cfg(_decoder(base_shape), base_shape)
    B = 1 if base_shape else 2
    pts, new_pts, img, metas, gts, gls = _frame(m, B, 970 + base_shape)
    w = (torch.rand(10, generator=torch.Generator().manual_seed(11)) + 0.5).to(dev())
    r = backward.decoder_backward(m, pts, new_pts, img, metas, gts, gls, w)
    got = dict(d_pts_conv=r['d_pts_conv'], d_new_pts=r['d_new_pts'], d_img=r['d_img'])
    got.update({'grads.' + k: v for k, v in r['grads'].items()})
    fw = _product_forward(m, pts, new_pts, img, metas, gts, gls)
    assert int(sum((w_ < 0).sum() for w_ in fw[1]['wins'])) > 0, 'no fallback rows in the draw'
    want, reach = _oracle_decoder_grads(m, pts, new_pts, img, metas, fw, w, torch.float64)
    assert set(got) == set(want)
    # Fixed bars: the chain is evaluated at the product's own activations, so no forward error compounds.  At the base
    # shape a query whose RoI runs past its image map's edge makes the image blocks' gradient ill-conditioned (DESIGN
    # §4.10: up to 4.7e-2 in the block test, where fp32 autograd is as far off); 5e-2 covers it.
    tol = 5e-2 if base_shape else 1e-3
    errs = []
    for k, v in want.items():
        if float(v.abs().max()) == 0:                     # prediction_heads.0: the fallback rows carry weight 0
            assert bool((got[k] == 0).all()), k
            continue
        errs.append((rel_err(got[k].double().cpu(), v.cpu()), k))
    errs.sort()
    for e, k in errs[-6:]:
        print('%-60s %.1e (bar %.0e)' % (k, e, tol))
    assert errs[-1][0] <= tol, errs[-1]
    assert all(float(v.abs().max()) == 0 for k, v in want.items() if k.startswith('grads.prediction_heads.0.'))
    assert bool((reach > 0).any()) and bool((r['d_img'][reach == 0] == 0).all()), 'a pixel no RoI reaches is not exactly 0'
