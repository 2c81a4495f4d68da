"""Gradient of the ++ decoder's losses: backward.decoder_pp_backward and DecoderPPLossFunction, against a float64 chain of
the oracle's modules evaluated at the product's own saved activations and driven by its decisions (top-k, labels, RoI
rectangles, win, onbits, the per-layer masks keep_l), with the bars of the base decoder's chain test.
"""
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import record_calls, same_bits

pytestmark = pytest.mark.gpu

C = 128


def dev():
    return torch.device('cuda:0')


def _decoder(base_shape):
    from test_gpu_rcnn_backward import _decoder as build
    from test_gpu_decoder_backward import _with_train_cfg
    return _with_train_cfg(build(base_shape, True), base_shape)


def _frame(m, B, seed):
    from test_gpu_decoder_backward import _frame as frame
    return frame(m, B, seed)


def _masked_pp(t, masks, B, P, L=4):
    """label / bbox weights and avg factors of the ++ decoder's loss: every layer's weights multiplied by that layer's mask
    (deepinteractionplusplus_decoder.py:513-514), applied here to the unmasked targets t."""
    lw, bw = t['label_weights'].clone().double(), t['bbox_weights'].clone().double()
    pos = t['bbox_weights'][..., 0] > 0
    num_pos = []
    for l in range(L):
        sl = slice(l * P, (l + 1) * P)
        mk = masks[l].to(lw.device).double()
        lw[:, sl] *= mk
        bw[:, sl] *= mk[..., None]
        num_pos.append(float((pos[:, sl].double() * (lw[:, sl] != 0).double()).sum()))
    return lw, bw, num_pos


def _oracle_decoder_pp_grads(m, pts, new_pts, img, metas, fw, w, dtype, monkeypatch):
    """The ++ decoder's loss gradient as a chain of float64 (or fp32) autograd: oracle.loss on the unmasked targets with
    the ++ masks applied by _masked_pp, oracle.mmpi_pp's centre and fallback chain (test_gpu_rcnn_v2_backward), the
    oracle's prediction FFNs, its V2 blocks per group (test_gpu_rcnn_v2_backward), the layer, query init and heat-map
    head as in the base decoder's chain test.  -> dict of d_pts_conv, d_new_pts, d_img and 'grads.<state_dict key>'."""
    import oracle.mmpi as om
    import test_gpu_decoder_backward as tdb
    from test_gpu_decoder_layer_backward import _oracle_grads as layer_grads
    from test_gpu_image_rcnn_backward import _product_groups
    from test_gpu_rcnn_v2_backward import _oracle_v2_grads, _pp_chain_oracle, _saved
    d = dev()
    sv, r, pd, tu, masks = fw
    B, Y, X, _ = pts.shape
    P, L, K = m.num_proposals, len(m.decode_head), m.num_classes_heat
    monkeypatch.setattr(tdb, '_masked', _masked_pp)
    d_dense, d_rows = tdb._oracle_loss_grads(m, pd, tu, masks, w.to(dtype), dtype)
    qs = [sv['query_feat1']] + sv['layer_query']
    # the chain is linear in the head outputs, so their values do not enter its gradient
    raw = torch.zeros(L, B * P, m.NP)
    d_raw, d_first, keep = _pp_chain_oracle(m, raw, sv['first_res'], [w_ for w_ in r['wins']], d_rows, dtype)
    assert same_bits(keep, torch.stack(r['keeps'])), 'the oracle chain keeps other rows than the product'
    out = {}
    put = lambda prefix, res: out.update({'grads.' + prefix + k[6:]: v for k, v in res.items() if k.startswith('grads.')})
    dq, d_img, d_new = None, 0, 0
    for li in reversed(range(L)):
        image = li % 2 == 0
        ph, _ = tdb._oracle_pred_grads(m, m.pred_head[li], [qs[li + 1]], d_raw[li], dtype)
        put('pred_head.%d.' % li, ph)
        d_out = ph['d0'] if dq is None else dq + ph['d0']
        pred_in = r['preds'][li - 1] if li else sv['first_res']
        maps = img if image else new_pts
        bsv = _saved(m, li, qs[li], pred_in, maps, metas if image else None)
        if image:
            rois, win, onbits = _product_groups(m, pred_in, metas, B)
        else:
            rois, win, onbits = bsv['rois'].cpu(), bsv['win'].cpu().long(), bsv['onbits'].cpu().long()
        res, _ = _oracle_v2_grads(m, li, qs[li], rois.to(torch.float64 if dtype == torch.float64 else torch.float32), win,
                                  onbits, maps, d_out, bsv, dtype)
        if image:
            d_img = d_img + res['d_maps']
        else:
            d_new = d_new + res['d_maps']
        put('decode_head.%d.' % li, res)
        dq = res['d_query']
    pf, _ = tdb._oracle_pred_grads(m, m.prediction_heads[0], [qs[0]], d_first, dtype)
    put('prediction_heads.0.', pf)
    dq = dq + pf['d0']
    rl = layer_grads(m, sv['query_feat0'], sv['query_pos0'], pts, dq, dtype, d)
    put('decoder.0.', rl)
    top = sv['top'].long()
    pix, lab = top % (Y * X), top // (Y * X)
    dq0 = rl['d_query']
    d_pts = rl['d_bev'].reshape(B, Y * X, -1).clone()
    for b in range(B):
        d_pts[b].index_add_(0, pix[b].to(d), dq0[b * P:(b + 1) * P])
    onehot = F.one_hot(lab.reshape(-1), K).to(d, dtype)
    out['grads.class_encoding.weight'] = (dq0.t() @ onehot).unsqueeze(-1)
    out['grads.class_encoding.bias'] = dq0.sum(0)
    seq = torch.nn.Sequential(om.ConvModule2d(C, C), torch.nn.Conv2d(C, K, 3, padding=1)).to(d, dtype).eval()
    seq.load_state_dict(m.heatmap_head_img.state_dict(), strict=True)
    xi = new_pts.to(d, dtype).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    with torch.enable_grad():
        z = seq[0].bn(seq[0].conv(xi))
        on = tdb._heat_relu_side(m, new_pts, z.detach())
        (seq[1](z * on) * d_dense.to(dtype).permute(0, 3, 1, 2)).sum().backward()
    out.update({'grads.heatmap_head_img.' + n: p.grad for n, p in seq.named_parameters()})
    out.update(d_pts_conv=d_pts.view(B, Y, X, -1), d_new_pts=d_new + xi.grad.permute(0, 2, 3, 1), d_img=d_img)
    return out


def _product_forward(m, pts, new_pts, img, metas, gts, gls):
    from deepinteraction_b200 import geom
    d = dev()
    B = pts.shape[0]
    proj, aux = (t.to(d) for t in m._camera_consts(metas))
    sv = {}
    r = m._schedule(pts, new_pts, img, geom.input_hw(metas), proj, aux, sv)
    pd = m._outputs(r, B)[0][0]
    tu = m._targets(gts, gls, pd, use_masks=False)
    masks = [(k.view(B, -1) != 0) for k in r['keeps']]
    return sv, r, pd, tu, masks


@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_decoder_pp_backward_matches_float64_oracle_chain(base_shape, monkeypatch):
    from deepinteraction_b200 import backward
    m = _decoder(base_shape)
    B = 1 if base_shape else 2
    pts, new_pts, img, metas, gts, gls = _frame(m, B, 1970 + base_shape)
    w = (torch.rand(10, generator=torch.Generator().manual_seed(12)) + 0.5).to(dev())
    r = backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls, w)
    got = dict(d_pts_conv=r['d_pts_conv'], d_new_pts=r['d_new_pts'], d_img=r['d_img'])
    got.update({'grads.' + k: v for k, v in r['grads'].items()})
    fw = _product_forward(m, pts, new_pts, img, metas, gts, gls)
    assert int(sum((k == 0).sum() for k in fw[1]['keeps'])) > 0, 'no fallback rows in the draw'
    want = _oracle_decoder_pp_grads(m, pts, new_pts, img, metas, fw, w, torch.float64, monkeypatch)
    assert set(got) == set(want)
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


@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_decoder_pp_backward_losses_keys_and_determinism(base_shape):
    from deepinteraction_b200 import backward
    m = _decoder(base_shape)
    B = 1 if base_shape else 2
    pts, new_pts, img, metas, gts, gls = _frame(m, B, 1910 + base_shape)
    w = (torch.rand(10, generator=torch.Generator().manual_seed(3)) + 0.5).to(dev())
    r = backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls, w)
    ref = m.loss(gts, gls, m.forward_nhwc(pts, new_pts, img, metas))
    assert set(ref) == set(r['losses'])
    differ = [(k, float(r['losses'][k]), float(ref[k])) for k in ref if not same_bits(r['losses'][k], ref[k])]
    assert not differ, differ
    sd = dict(m.named_parameters())
    want = {k for k in sd if not k.startswith('heatmap_head.')}
    assert set(r['grads']) == want
    for k, v in r['grads'].items():
        assert v.shape == sd[k].shape, k
        assert bool(torch.isfinite(v).all()), k
    assert all(bool((v == 0).all()) for k, v in r['grads'].items() if k.startswith('prediction_heads.0.'))
    nonzero = [k for k, v in r['grads'].items() if not k.startswith('prediction_heads.0.') and float(v.abs().max()) > 0]
    assert len(nonzero) > 0.9 * (len(want) - len(list(m.prediction_heads[0].parameters())))
    r2 = backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls, w)
    for k in ('d_pts_conv', 'd_new_pts', 'd_img'):
        assert same_bits(r2[k], r[k]), k
    assert all(same_bits(r2['grads'][k], v) for k, v in r['grads'].items()), 'two calls differ'


def test_decoder_pp_backward_is_linear_in_the_upstream_weights():
    from deepinteraction_b200 import backward
    m = _decoder(False)
    pts, new_pts, img, metas, gts, gls = _frame(m, 2, 1930)
    d = dev()
    eye = torch.eye(10, device=d)
    parts = [backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls, eye[i]) for i in range(9)]
    w = torch.tensor([0.7, 1.3, 0.4, 2.0, 0.9, 1.1, 0.6, 1.5, 0.8, 5.0], device=d)
    r = backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls, w)
    # each part carries its own fp32 rounding, relative to its own scale (measured up to 2.4e-5 of the sum on d_pts_conv);
    # a term entering twice or not at all would be off by a part's full size
    for k in ('d_pts_conv', 'd_new_pts', 'd_img'):
        want = sum(float(w[i]) * parts[i][k].double() for i in range(9))
        e = rel_err(r[k].double(), want)
        print('%s %.1e' % (k, e))
        assert e < 1e-4, k
    z = backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls, eye[9])
    assert all(bool((z[k] == 0).all()) for k in ('d_pts_conv', 'd_new_pts', 'd_img'))


def test_decoder_pp_loss_function_matches_decoder_pp_backward():
    from deepinteraction_b200 import backward
    m = _decoder(False)
    pts, new_pts, img, metas, gts, gls = _frame(m, 2, 1940)
    xs = [t.clone().requires_grad_(True) for t in (pts, new_pts, img)]
    with torch.enable_grad():
        loss = backward.DecoderPPLossFunction.apply(m, *xs, metas, gts, gls)
        loss.backward()
    losses = m.loss(gts, gls, m.forward_nhwc(pts, new_pts, img, metas))
    assert same_bits(loss.detach(), torch.stack([v for k, v in losses.items() if 'loss' in k]).sum())
    r = backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls)
    for x, k in zip(xs, ('d_pts_conv', 'd_new_pts', 'd_img')):
        assert same_bits(x.grad, r[k]), k


def test_decoder_pp_backward_does_not_synchronise():
    from deepinteraction_b200 import backward
    m = _decoder(False)
    args = _frame(m, 2, 1950)
    backward.decoder_pp_backward(m, *args)               # warm-up: builds the per-pack tensors
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = backward.decoder_pp_backward(m, *args)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(r['d_pts_conv']).all())


def test_decoder_pp_backward_rejects_the_base_decoder_and_bad_maps_before_any_launch():
    from deepinteraction_b200 import backward
    from test_gpu_decoder_backward import _decoder as base, _with_train_cfg
    m = _with_train_cfg(base(False), False)
    pts, new_pts, img, metas, gts, gls = _frame(m, 2, 1960)
    m.pack()
    with record_calls() as calls:
        with pytest.raises(NotImplementedError, match='DeepInteractionPlusPlusDecoder only'):
            backward.decoder_pp_backward(m, pts, new_pts, img, metas, gts, gls)
        with pytest.raises(NotImplementedError, match='DeepInteractionPlusPlusDecoder only'):
            backward.DecoderPPLossFunction.apply(m, pts, new_pts, img, metas, gts, gls)
    assert calls == []
    mpp = _decoder(False)
    mpp.pack()
    bad = [(pts, new_pts, img[:3]), (pts, new_pts, img[..., :64].contiguous()), (pts[:, :20].contiguous(), new_pts, img),
           (pts, new_pts[..., :64].contiguous(), img)]
    with record_calls() as calls:
        for a, b, c in bad:
            with pytest.raises(NotImplementedError, match='pixel-major'):
                backward.decoder_pp_backward(mpp, a, b, c, metas, gts, gls)
    assert calls == []
