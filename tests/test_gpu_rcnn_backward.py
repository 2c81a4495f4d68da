"""Backward of the base decoder's PointRCNNBlock (backward.point_rcnn_backward) and its kernels di_roi_align_bwd_f32,
di_dynconv_bwd_f32 and di_gelu_bwd_f32 against float64 autograd.

The RoIAlign gradient is held to row_err <= 1e-5 per pixel (kernel_check.row_err; the scale of a pixel is the gradient
of the same sum with |d_out|, the bilinear weights being non-negative).  Pixels that no sample reaches must be exactly 0.
The DynamicConv gradient, whose LayerNorm backward amplifies rounding by 1 / std of each row, is held per query to
max(1e-5, 5x the error fp32 autograd through the same chain makes), like the whole block, which is compared with autograd
through oracle.mmpi.PointRCNNBlock at 1e-4 or 5x the fp32 error.  The oracle block is driven on the RoI rectangles the
product computes (di_rcnn_rois_f32), so that the rounding of the box corners is not under test.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from kernel_check import _capi, row_err, same_bits
from test_gpu_decoder_kernels import _edge_rois

pytestmark = pytest.mark.gpu

SENT = -1234.5
TOL = 1e-4


def dev():
    return torch.device('cuda:0')


def _ops():
    from deepinteraction_b200 import ops
    return ops


# ---------------------------------------------------------------------------------------------------------------------
# 1. RoIAlign gradient
# ---------------------------------------------------------------------------------------------------------------------
def _roi_align_bwd_ref(maps_shape, rois, d_out, scale):
    """float64 autograd of oracle.geometry.roi_align -> (d_maps [n_maps, H, W, C], the same with |d_out|).  RoIs with map
    index -1 or a NaN coordinate are left out: the forward skips all their samples, so they contribute nothing (the
    oracle's own gradient of such a RoI is NaN * 0)."""
    from oracle.geometry import roi_align
    n_maps, C, H, W = maps_shape
    d = dev()
    live = (rois[:, 0] >= 0) & ~torch.isnan(rois[:, 1:]).any(1)
    out = []
    for dd in (d_out, d_out.abs()):
        maps = torch.zeros(n_maps, C, H, W, dtype=torch.float64, device=d, requires_grad=True)
        with torch.enable_grad():
            tot = 0
            for m in range(n_maps):
                sel = ((rois[:, 0] == m) & live).nonzero().squeeze(1)
                for part in sel.split(64):
                    r = roi_align(maps[m], rois[part, 1:].double().to(d), 7, scale, 2)          # (R, C, 7, 7)
                    tot = tot + (r.flatten(2) * dd[part].double().to(d).transpose(1, 2)).sum()
            if torch.is_tensor(tot):
                tot.backward()
        g = maps.grad if maps.grad is not None else torch.zeros_like(maps)
        out.append(g.permute(0, 2, 3, 1).cpu())
    return out


def _run_roi_bwd(rois, d_out, n_maps, H, W, scale):
    """The C entry point into a sentinel-filled buffer."""
    ops = _ops()
    C = d_out.shape[2]
    dm = torch.full((n_maps, H, W, C), SENT, device=dev())
    _capi('di_roi_align_bwd_f32', ops._ptr(rois), ops._ptr(d_out), ops._ptr(dm), rois.shape[0], n_maps, H, W, C, float(scale))
    return dm


ROI_BWD_CASES = [  # n_maps, H, W, C, scale
    (2, 9, 13, 64, 1.0), (2, 9, 13, 128, 0.25), (3, 9, 13, 256, 1.0), (1, 5, 1, 64, 1.0), (1, 36, 36, 128, 1.0),
    (2, 180, 180, 128, 1.0),
]


@pytest.mark.parametrize('case', ROI_BWD_CASES, ids=lambda c: 'n%d_%dx%d_C%d_s%g' % c)
def test_roi_align_bwd_matches_float64_autograd(case):
    n_maps, H, W, C, scale = case
    g = torch.Generator().manual_seed(H * C + W + n_maps)
    edge = _edge_rois(n_maps, H, W, scale)                      # samples at -1, in [-1, 0), 0, H-1, H; zero-width, inverted
    rnd = torch.cat([torch.randint(0, n_maps, (64, 1), generator=g).float(),
                     (torch.randint(-8, 4 * max(H, W) + 8, (64, 2), generator=g).float() / 4 + 0.5) / scale], 1)
    ext = torch.randint(0, 6, (64, 2), generator=g).float()
    rnd = torch.cat([rnd, rnd[:, 1:3] + 7 * 2.0 ** (ext - 2) / scale], 1)
    nan = float('nan')
    # covers the whole map: pixel span [-1, -1 + 7 * 2^k] >= [-1, L], a dyadic bin size as every RoI here, so that the fp32
    # sample positions are exact and the float64 reference weighs the same points
    span = lambda L: 7.0 * 2.0 ** math.ceil(math.log2((L + 1) / 7.0))
    whole = [[m, -0.5 / scale, -0.5 / scale, (span(W) - 0.5) / scale, (span(H) - 0.5) / scale] for m in range(n_maps)]
    odd = torch.tensor(whole + [[-1.0, 0.0, 0.0, 8.0, 8.0], [0, nan, 1.0, 8.0, 8.0], [0, 1.0, nan, 8.0, 8.0],
                                [0, 1.0, 1.0, nan, 8.0], [0, 1.0, 1.0, 8.0, nan],
                                [0, -40.0 / scale, -40.0 / scale, -20.0 / scale, -20.0 / scale]])   # fully outside
    rois = torch.cat([edge, rnd, odd])
    rois = rois[torch.randperm(rois.shape[0], generator=g)].contiguous()
    d_out = torch.randn(rois.shape[0], 49, C, generator=g)
    rd, dd = rois.to(dev()), d_out.to(dev())
    got = _run_roi_bwd(rd, dd, n_maps, H, W, scale)
    want, mag = _roi_align_bwd_ref((n_maps, C, H, W), rois, d_out, scale)
    assert not bool((got == SENT).any()), 'a pixel was not written'
    e = row_err(got, want, mag)
    print('row_err %.1e' % e)
    assert e < 1e-5
    assert bool((got.cpu()[mag == 0] == 0).all()), 'a pixel no sample reaches is not exactly 0'
    assert bool((mag > 0).any())
    assert same_bits(got, _run_roi_bwd(rd, dd, n_maps, H, W, scale)), 'two calls differ'


def test_roi_align_bwd_without_rois_writes_zeros():
    dm = _run_roi_bwd(torch.zeros(0, 5, device=dev()), torch.zeros(0, 49, 64, device=dev()), 2, 7, 5, 1.0)
    assert bool((dm == 0).all())


# ---------------------------------------------------------------------------------------------------------------------
# 2. DynamicConv gradient
# ---------------------------------------------------------------------------------------------------------------------
def _dynconv_grads(roi, params, norms, d_out, dtype):
    """autograd of relu(LN2(relu(LN1(F P1)) P2)) flattened -> (d_roi, d_params, dg1, db1, dg2, db2)."""
    n = roi.shape[0]
    leaves = [t.to(dev(), dtype).detach().requires_grad_(True) for t in [roi, params] + list(norms)]
    F0, P, g1, b1, g2, b2 = leaves
    with torch.enable_grad():
        P1, P2 = P[:, :16384].view(n, 128, 128), P[:, 16384:].view(n, 128, 128)
        y = F.relu(F.layer_norm(torch.bmm(F0, P1), (128,), g1, b1, 1e-5))
        y = F.relu(F.layer_norm(torch.bmm(y, P2), (128,), g2, b2, 1e-5))
        (y.flatten(1) * d_out.to(dev(), dtype)).sum().backward()
    return [t.grad for t in leaves]


def _per_query_err(got, want):
    """max over queries of max|got - want| / max|want| on that query's values; a query whose reference is all zero must
    be exactly zero."""
    g, w = got.double().reshape(got.shape[0], -1), want.double().reshape(want.shape[0], -1)
    den = w.abs().amax(1)
    err = (g - w).abs().amax(1)
    return float(torch.where(den > 0, err / den.clamp_min(1e-300), err * 1e30).max())


@pytest.mark.parametrize('n', [1, 2, 200, 400])
def test_dynconv_bwd_matches_float64_autograd(n):
    ops = _ops()
    d = dev()
    g = torch.Generator().manual_seed(n + 17)
    roi = torch.randn(n, 49, 128, generator=g)
    params = torch.randn(n, 2 * 128 * 128, generator=g) / 11
    b1, b2 = torch.randn(128, generator=g) * 0.5, torch.randn(128, generator=g) * 0.5
    if n in (2, 400):
        # non-positive betas: a zero row of F has zero variance in LN1 (the eps path), ReLU then kills the whole row, and
        # the row is zero again, with zero variance, in LN2
        b1, b2 = -b1.abs(), -b2.abs()
    norms = [torch.rand(128, generator=g) + 0.5, b1, torch.rand(128, generator=g) + 0.5, b2]
    roi[0, :7] = 0.0                                                # zero-variance rows
    if n > 1:
        roi[1] = 64.0 + torch.randn(49, 128, generator=g) * 0.5   # large mean, small spread
        params[1, :16384] = 1.0 / 16 + params[1, :16384] / 8
        roi[n - 1] = 0.0                                          # a whole query of zero rows
    d_out = torch.randn(n, 49 * 128, generator=g)
    dv = lambda t: t.contiguous().to(d)
    args = (dv(roi), dv(params), *(dv(t) for t in norms))
    d_roi, d_params, d_norm = ops.dynconv_bwd(*args, dv(d_out))
    dn = ops.col_sum(d_norm).view(4, 128)
    got = [d_roi, d_params] + [t[None] for t in dn.unbind(0)]
    want = _dynconv_grads(roi, params, norms, d_out, torch.float64)
    f32 = _dynconv_grads(roi, params, norms, d_out, torch.float32)
    names = ['d_roi', 'd_params', 'dgamma1', 'dbeta1', 'dgamma2', 'dbeta2']
    for k, gt, w, f in zip(names, got, want, f32):
        w = w.reshape(gt.shape)
        e, bar = _per_query_err(gt, w), max(1e-5, 5 * _per_query_err(f.reshape(gt.shape), w))
        print('%-8s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)
    if n in (2, 400):
        assert bool((d_roi[n - 1] == 0).all()) and bool((d_params[n - 1] == 0).all()), 'a killed query must get exact zeros'
    again = ops.dynconv_bwd(*args, dv(d_out))
    assert all(same_bits(a, b) for a, b in zip((d_roi, d_params, d_norm), again)), 'two calls differ'


# ---------------------------------------------------------------------------------------------------------------------
# 3. GELU gradient
# ---------------------------------------------------------------------------------------------------------------------
def test_gelu_bwd_matches_float64():
    ops = _ops()
    g = torch.Generator().manual_seed(3)
    h = torch.cat([torch.randn(4096, generator=g) * 3, torch.tensor([0.0, -0.0, 1e-30, -1e-30, 5.0, -5.0, 9.0, -9.0,
                                                                      30.0, -30.0, 1e4, -1e4, 88.0, -88.0])])
    dy = torch.randn(h.shape, generator=g)
    got = ops.gelu_bwd(dy.to(dev()), h.to(dev())).cpu().double()
    h64 = h.double()
    phi = torch.exp(-0.5 * h64 * h64) / (2 * torch.pi) ** 0.5
    want = dy.double() * (0.5 * (1 + torch.erf(h64 / 2 ** 0.5)) + h64 * phi)
    # Phi is evaluated as 0.5 (1 + erf): its absolute error is a few units of 2^-24, whatever its size
    bar = 5e-7 * dy.double().abs() + 2e-6 * want.abs()
    assert bool(((got - want).abs() <= bar).all()), float(((got - want).abs() - bar).max())
    assert torch.equal(got[4096:4098], dy[4096:4098].double() * 0.5)          # h = 0: exactly dy / 2


# ---------------------------------------------------------------------------------------------------------------------
# 4. the whole block
# ---------------------------------------------------------------------------------------------------------------------
def _decoder(base_shape, plusplus=False):
    from test_gpu_decoder import _build
    if base_shape:
        test_cfg = dict(dataset='nuScenes', grid_size=[1440, 1440, 40], out_size_factor=8, pc_range=[-54.0, -54.0],
                        voxel_size=[0.075, 0.075], nms_type=None)
        coder = dict(type='TransFusionBBoxCoder', pc_range=[-54.0, -54.0], voxel_size=[0.075, 0.075], out_size_factor=8,
                     post_center_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], score_threshold=0.0, code_size=10)
        return _build(1800 + plusplus, 6, 200, test_cfg, coder, plusplus=plusplus)[1]
    return _build(1810 + plusplus, 2, 40, plusplus=plusplus)[1]


def _block_inputs(m, B, seed):
    """query rows, prediction rows (box centres in BEV cells, some beyond the map's edge; log-dims of 0.4 - 4.5 m; random
    heading), bev map and output gradient."""
    g = torch.Generator().manual_seed(seed)
    Y, X, C, P = m.y_size, m.x_size, 128, m.num_proposals
    pred = torch.randn(B * P, m.NP, generator=g)
    pred[:, 0] = torch.rand(B * P, generator=g) * (X + 4) - 2
    pred[:, 1] = torch.rand(B * P, generator=g) * (Y + 4) - 2
    pred[:, 3:6] = torch.rand(B * P, 3, generator=g) * 2.5 - 1.0
    return (torch.randn(B * P, C, generator=g), pred, torch.randn(B, Y, X, C, generator=g), torch.randn(B * P, C, generator=g))


def _oracle_block_grads(m, li, query, rects, bev, grad, dtype):
    """autograd through oracle.mmpi.PointRCNNBlock._tail with oracle.geometry.roi_align on the given RoI rectangles."""
    import oracle.mmpi as om
    from oracle.geometry import roi_align
    d = dev()
    B, Y, X, C = bev.shape
    P = query.shape[0] // B
    blk = om.PointRCNNBlock(C, 8, 0.1, None)
    blk.load_state_dict(m.decode_head[li].state_dict(), strict=True)
    blk = blk.to(device=d, dtype=dtype).eval()
    q = query.to(d, dtype).requires_grad_(True)
    fm = bev.to(d, dtype).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    with torch.enable_grad():
        outs = []
        for b in range(B):
            roi = roi_align(fm[b], rects[b * P:(b + 1) * P].to(d, dtype), 7, 1.0, 2)
            outs.append(blk._tail(q[b * P:(b + 1) * P].unsqueeze(1), roi))
        (torch.cat(outs) * grad.to(d, dtype)).sum().backward()
    res = dict(d_query=q.grad, d_bev=fm.grad.permute(0, 2, 3, 1))
    res.update({'grads.' + n: p.grad for n, p in blk.named_parameters()})
    return res


def _relu_margin(m, li, query, pred, bev):
    """Smallest |pre-activation| of the block's ReLUs (DynamicConv LN1, LN2 and norm3), evaluated in float64 from the
    product's own saved inputs of each.  A pre-activation within fp32 rounding of 0 may take the other side of the kink in
    float64, which moves that element's gradient by its full size: such inputs cannot be compared at 1e-4."""
    from deepinteraction_b200 import backward
    d = dev()
    B = bev.shape[0]
    bp, sv = m.pack()['blocks'][li], {}
    with backward._precise():
        m._rcnn_block(bp, query.to(d), pred.to(d), bev.to(d), None, B, query.shape[0] // B, backward._bev_roi_params(m),
                      None, None, saved=sv)
    ln = lambda z, gb: F.layer_norm(z, (128,), gb[0].double(), gb[1].double(), 1e-5)
    n = query.shape[0]
    P = sv['params'].double()
    a1 = ln(torch.bmm(sv['roi'].double(), P[:, :16384].view(n, 128, 128)), bp['dn1'])
    a2 = ln(torch.bmm(F.relu(a1), P[:, 16384:].view(n, 128, 128)), bp['dn2'])
    a3 = ln(sv['zd3'].double(), bp['dn3'])
    nz = lambda a: a.abs()[a != 0]                 # exact zeros: zero-variance rows with beta = 0 are not a rounding case
    return float(min(nz(a1).min(), nz(a2).min(), nz(a3).min()))


def _check_block(m, li, B, seed):
    from deepinteraction_b200 import backward, ops
    d = dev()
    query, pred, bev, grad = _block_inputs(m, B, seed)
    assert _relu_margin(m, li, query, pred, bev) > 1e-6, 'inputs with a ReLU pre-activation at fp32 rounding of 0'
    P = m.num_proposals
    r = backward.point_rcnn_backward(m, li, query.to(d), pred.to(d), bev.to(d), grad.to(d))
    rois = ops.rcnn_rois(pred.to(d), B, P, m.num_views, 1, backward._bev_roi_params(m))[0].cpu()
    assert bool((rois[:, 0] == torch.arange(B).repeat_interleave(P)).all())
    rects = rois[:, 1:].double()
    got = dict(d_query=r['d_query'], d_bev=r['d_bev'])
    got.update({'grads.' + n: t for n, t in r['grads'].items()})
    want = _oracle_block_grads(m, li, query, rects, bev, grad, torch.float64)
    f32 = _oracle_block_grads(m, li, query, rects.float(), bev, grad, torch.float32)
    assert set(got) == set(want) and len(r['grads']) == 24
    sd = m.decode_head[li].state_dict()
    for k, w in want.items():
        if k.startswith('grads.'):
            assert got[k].shape == sd[k[6:]].shape, k
        bar = max(TOL, 5 * rel_err(f32[k].double(), w))
        e = rel_err(got[k].double(), w)
        print('%-55s %.1e (bar %.1e)' % (k, e, bar))
        assert e <= bar, (k, e, bar)
    return r


# input seeds whose smallest ReLU pre-activation (about 600 000 of them per block) is at least 1e-6 from 0 (_relu_margin):
# typical draws have a few within 1e-7, where a float64 reference may take the other side of the kink
BLOCK_SEEDS = {(False, 1): 84, (False, 3): 80, (True, 1): 79, (True, 3): 89}


@pytest.mark.parametrize('li', [1, 3])
@pytest.mark.parametrize('base_shape', [False, True], ids=['small', 'base_shape'])
def test_point_rcnn_backward_matches_oracle_autograd(base_shape, li):
    m = _decoder(base_shape)
    _check_block(m, li, 1 if base_shape else 2, BLOCK_SEEDS[(base_shape, li)])


# ---------------------------------------------------------------------------------------------------------------------
# 5. autograd.Function, 6. synchronisation, limits
# ---------------------------------------------------------------------------------------------------------------------
def test_point_rcnn_function_forward_is_the_block_and_backward_matches():
    from deepinteraction_b200 import backward
    from tools.make_goldens import small_frame
    from test_gpu_decoder import _build
    _, m = _build(1620, 2, 24)
    gen = torch.Generator().manual_seed(1620)
    fr = small_frame(1620, aug=True, views=2, batch=2)
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(dev())
    pts, new_pts = nhwc(torch.randn(2, 128, 36, 36, generator=gen)), nhwc(torch.randn(2, 128, 36, 36, generator=gen))
    img = nhwc(torch.randn(4, 128, 28, 50, generator=gen))
    dbg = {}
    out = m.forward_rows(pts, new_pts, img, fr['img_metas'], debug=dbg)
    for li in (1, 3):
        q0 = dbg['layer_query'][li - 1].clone().requires_grad_(True)
        b0 = new_pts.clone().requires_grad_(True)
        pred = out['preds'][li - 1]
        with torch.enable_grad():
            y = backward.PointRCNNFunction.apply(m, li, q0, pred, b0)
            assert same_bits(y.detach(), dbg['layer_query'][li]), li
            grad = torch.randn(y.shape, generator=gen).to(dev())
            (y * grad).sum().backward()
        r = backward.point_rcnn_backward(m, li, dbg['layer_query'][li - 1], pred, new_pts, grad)
        assert same_bits(q0.grad, r['d_query']) and same_bits(b0.grad, r['d_bev']), li


def test_point_rcnn_backward_rejects_image_v2_and_unsupported_shapes():
    from deepinteraction_b200 import backward
    d = dev()
    m = _decoder(False)
    query, pred, bev, grad = (t.to(d) for t in _block_inputs(m, 2, 5))
    for li in (0, 2):                                           # ImageRCNNBlock
        with pytest.raises(NotImplementedError, match='PointRCNNBlock'):
            backward.point_rcnn_backward(m, li, query, pred, bev, grad)
        with pytest.raises(NotImplementedError, match='PointRCNNBlock'):
            backward.PointRCNNFunction.apply(m, li, query, pred, bev)
    with pytest.raises(NotImplementedError, match='P <= 512'):
        backward.point_rcnn_backward(m, 1, query.repeat(13, 1), pred.repeat(13, 1), bev, grad.repeat(13, 1))
    mpp = _decoder(False, plusplus=True)
    for li in (1, 3):                                           # PointRCNNBlockV2
        with pytest.raises(NotImplementedError, match='PointRCNNBlock'):
            backward.point_rcnn_backward(mpp, li, query, pred[:, :mpp.NP].contiguous(), bev, grad)


def test_point_rcnn_backward_does_not_synchronise():
    from deepinteraction_b200 import backward
    m = _decoder(False)
    d = dev()
    query, pred, bev, grad = (t.to(d) for t in _block_inputs(m, 2, 6))
    backward.point_rcnn_backward(m, 1, query, pred, bev, grad)        # warm-up: builds the per-pack tensors
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        r = backward.point_rcnn_backward(m, 1, query, pred, bev, grad)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(r['d_bev']).all())


def test_rcnn_backward_limits_are_rejected():
    ops = _ops()
    p = ops._ptr
    buf = torch.zeros(1 << 16, device=dev())
    for C in (6, 516):
        with pytest.raises(RuntimeError):
            _capi('di_roi_align_bwd_f32', p(buf), p(buf), p(buf), 1, 1, 2, 2, C, 1.0)
    with pytest.raises(RuntimeError):                              # n_maps > 0
        _capi('di_roi_align_bwd_f32', p(buf), p(buf), p(buf), 1, 0, 2, 2, 4, 1.0)
    import ctypes
    mis = ctypes.c_void_p(buf.data_ptr() + 4)
    for i in range(2):
        a = [p(buf)] * 10
        a[i] = mis                                                   # roi, params: 16-byte aligned
        with pytest.raises(RuntimeError):
            _capi('di_dynconv_bwd_f32', *a, 1, 1e-5)
