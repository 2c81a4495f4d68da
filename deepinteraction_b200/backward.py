"""Backward of LocalContextAttentionBlock on libdi_b200 (SURVEY.md 8(b) `di_lcab_backward`, the training side of the
hot module; forward: mmri.lcab_forward / di_lcab_forward_f32).

Reference: models/utils/encoder_utils.py:36-81 (autograd Functions around the window ops: similar_backward x 2,
weighting_backward_ori, weighting_backward_weight), :119-135 (the block), ops/locatt_ops kernels.cuh:44-119.

Scope: gradients of the block with BatchNorm in EVAL mode (running statistics, folded into the 1x1 convolutions -- the
form the forward kernels use): d/d target map, d/d source map, d/d folded weight and bias of the five Conv+BN layers.
The gradient of a folded weight maps to the convolution weight by the BN scale (dW_conv = dW_folded * gamma / sqrt(var +
eps)), and d beta = d bias_folded.  Train-mode BatchNorm (batch statistics with their own gradient) and dropout are not
covered.  The intermediates are recomputed in fp32 (q1, k1, q, k, v and the [P, 81] attention weights), the window
products run in the unfused kernels of csrc/lcab_bwd.cu, dense products on the wgmma / FFMA GEMMs.
"""
import torch

from . import fold, ops


class _precise:
    """Gradient products run on the 3xTF32 split (error ~1e-7 per product) rather than the bf16 split of the inference
    path (~1e-5): the backward chains a dozen products per layer."""

    def __enter__(self):
        self.saved = ops.TC_BF16[0]
        ops.TC_BF16[0] = False

    def __exit__(self, *a):
        ops.TC_BF16[0] = self.saved


def _bw_pack(pk):
    """Transposed weights for the dX products, built once per pack."""
    if '_bw' in pk:
        return pk['_bw']
    C = pk['C']
    dev = pk['b_self'].device
    w1, w2 = pk['w_self'].w.detach().cpu().double(), pk['w_2'].w.detach().cpu().double()
    wq1, wk1, wv = w1[:C], w1[C:2 * C], w1[2 * C:]
    wq2, wk2 = w2[:C], w2[C:]
    T = lambda m: fold.Weight(m.t().contiguous(), dev)
    pk['_bw'] = dict(q2=T(wq2), k2=T(wk2), q1=T(wq1), kv1=T(torch.cat([wk1, wv], 0)), self1=T(torch.cat([wq1, wk1, wv], 0)))
    return pk['_bw']


def _wgrad(dy, x):
    """dy [M, N], x [M, K] (contiguous rows) -> dy^T x [N, K]: both operands transposed to channel-major, then a split-K
    product over the M pixels with a fixed-order sum of the partials."""
    M = dy.shape[0]
    dyt = ops.nhwc_to_nchw(dy.view(1, M, 1, dy.shape[1])).view(dy.shape[1], M)
    xt = ops.nhwc_to_nchw(x.view(1, M, 1, x.shape[1])).view(x.shape[1], M)
    splits = max(1, min(256, M // 512))
    part = ops.linear([dyt], xt, splits=splits)
    return ops.rows_finish(part) if part.shape[0] > 1 else part[0]


def lcab_backward(pk, target, source, N, H, W, grad_out):
    """target / source / grad_out: [N*H*W, C] fp32 pixel-major rows (same tensor object for target and source = self
    attention).  -> dict(d_target, d_source (None for self attention: summed into d_target), and per layer name in
    (q1, q2, k1, k2, v) a pair (dW_folded [C, C], db_folded [C]))."""
    with _precise():
        return _lcab_backward(pk, target, source, N, H, W, grad_out)


def _lcab_backward(pk, target, source, N, H, W, grad_out):
    C, ks = pk['C'], pk['ks']
    M = N * H * W
    bw = _bw_pack(pk)
    self_attn = target is source
    x_t, x_s, dO = target.contiguous(), source.contiguous(), grad_out.contiguous()
    R = ops.ACT_RELU
    # forward intermediates in fp32 rows
    if self_attn:
        t = ops.linear([x_s], pk['w_self'], pk['b_self'], R)
        q1, k1, v = t[:, :C].contiguous(), t[:, C:2 * C].contiguous(), t[:, 2 * C:].contiguous()
    else:
        q1 = ops.linear([x_t], pk['w_q1'], pk['b_q1'], R)
        t = ops.linear([x_s], pk['w_kv1'], pk['b_kv1'], R)
        k1, v = t[:, :C].contiguous(), t[:, C:].contiguous()
    q = ops.linear([q1], pk['w_q2'], pk['b_q2'], R)
    k = ops.linear([k1], pk['w_k2'], pk['b_k2'], R)
    scale = 1.0 / float(C) ** 0.5
    A = ops.win_softmax(ops.win_dot(q, k, N, H, W, ks), scale)
    # window attention
    dA = ops.win_dot(dO, v, N, H, W, ks)
    dv = ops.win_scatter(A, dO, N, H, W, ks)
    dS = ops.win_softmax_bwd(A, dA, scale)
    dq = ops.win_gather(dS, k, N, H, W, ks)
    dk = ops.win_scatter(dS, q, N, H, W, ks)
    # projections: ReLU masks from the saved outputs, dX on the GEMM kernels, dW as split-K products, db as column sums
    g = {}
    dq = ops.relu_bwd(dq, q)
    dk = ops.relu_bwd(dk, k)
    dv = ops.relu_bwd(dv, v)
    g['q2'] = (_wgrad(dq, q1), ops.col_sum(dq))
    g['k2'] = (_wgrad(dk, k1), ops.col_sum(dk))
    dq1 = ops.relu_bwd(ops.linear([dq], bw['q2']), q1)
    dk1 = ops.relu_bwd(ops.linear([dk], bw['k2']), k1)
    g['q1'] = (_wgrad(dq1, x_t), ops.col_sum(dq1))
    g['k1'] = (_wgrad(dk1, x_s), ops.col_sum(dk1))
    g['v'] = (_wgrad(dv, x_s), ops.col_sum(dv))
    if self_attn:
        d_t, d_s = ops.linear([dq1, dk1, dv], bw['self1']), None
    else:
        d_t, d_s = ops.linear([dq1], bw['q1']), ops.linear([dk1, dv], bw['kv1'])
    return dict(d_target=d_t, d_source=d_s, **g)


def i2p_backward(i2p_pack, pts_nhwc, img_nhwc, pts_metas, proj, V, in_hw, grad_out, dropout=None):
    """Backward of the MMRI_I2P block as the product evaluates it (mmri.DeepInteractionEncoder.i2p; reference
    encoder_utils.py:216-320): rows = pts[coors]; qk = M1 rows + c1; s = attend(qk, image samples); o = M2 s + c2;
    out[coors] = o where a pillar saw >= 1 sample.  i2p_pack = (M1, c1, M2, c2) folded from nn.MultiheadAttention
    (fold.i2p_fold); proj: [B, V, 12] device camera rows (mmri.Geometry.proj).  grad_out [B, Y, X, C].
    -> dict(d_pts [B,Y,X,C], d_img [B*V,h,w,C], dM1, dc1, dM2, dc2); fold.i2p_unfold_grads maps the last four to the
    attention module's own parameters.  dropout = (p, seed): the training-mode attention dropout the forward used."""
    with _precise():
        return _i2p_backward(i2p_pack, pts_nhwc, img_nhwc, pts_metas, proj, V, in_hw, grad_out, dropout)


def _i2p_backward(i2p_pack, pts_nhwc, img_nhwc, pts_metas, proj, V, in_hw, grad_out, dropout=None):
    M1, c1, M2, c2 = i2p_pack
    coors = pts_metas['pillar_coors']
    pillars, npts = pts_metas['pillars'], pts_metas['pillars_num_points']
    d_pts = torch.zeros_like(pts_nhwc)
    d_img = torch.zeros_like(img_nhwc)
    if coors.shape[0] == 0:
        z = lambda t: torch.zeros_like(t.w if hasattr(t, 'w') else t)
        return dict(d_pts=d_pts, d_img=d_img, dM1=z(M1), dc1=z(c1), dM2=z(M2), dc2=z(c2))
    dev = pts_nhwc.device
    # a plain tensor (the [C, C + 4] output weight of the dropout form) stays on the FFMA path
    T_ = lambda Wt: (fold.Weight(Wt.w.detach().t().contiguous(), dev, lazy=True) if hasattr(Wt, 'w') else Wt.detach().t().contiguous())
    # forward intermediates
    rows = ops.gather_rows(pts_nhwc, coors)
    qk = ops.linear([rows], M1, c1)
    s, cnt = ops.i2p_attend(qk, pillars, npts, coors, proj, img_nhwc, V, in_hw, dropout=dropout)
    # out = scatter(M2 s + c2) at pillars with cnt > 0
    do = ops.gather_rows_masked(grad_out.contiguous(), cnt, coors)
    dM2, dc2 = _wgrad(do, s), ops.col_sum(do)
    ds = ops.linear([do], T_(M2))
    dqk = ops.i2p_attend_bwd(qk, ds, pillars, npts, coors, proj, img_nhwc, d_img, V, in_hw, dropout)
    dM1, dc1 = _wgrad(dqk, rows), ops.col_sum(dqk)
    drows = ops.linear([dqk], T_(M1))
    ones = torch.ones(coors.shape[0], device=dev, dtype=torch.int32)
    ops.scatter_rows(drows, ones, coors, d_pts)             # one pillar per BEV cell: a plain store
    return dict(d_pts=d_pts, d_img=d_img, dM1=dM1, dc1=dc1, dM2=dM2, dc2=dc2)


def _t_weight(W, device):
    return fold.Weight(W.w.detach().t().contiguous(), device, lazy=True)


def _conv3x3_transposed(w_packed, cin, device):
    """Packed forward weight [Cout, (ky*3+kx)*Cin + ci] -> packed weight of the input-gradient convolution
    [Cin, (ky*3+kx)*Cout + co] with the taps flipped (d x = conv3x3(d y, W^T flipped))."""
    w = w_packed.w.detach()                                        # stays on the device: no host round trip
    cout = w.shape[0]
    w4 = w.view(cout, 3, 3, cin)                                   # co, ky, kx, ci
    wt = w4.flip(1, 2).permute(3, 1, 2, 0).reshape(cin, 9 * cout)   # ci, ky', kx', co
    return fold.Weight(wt.contiguous(), device, lazy=True)


def conv3x3_wgrad(x_nchw, g_rows, cout):
    """dW [Cout, Cin, 3, 3] and db of a 3x3 convolution: per tap a split-K product of the output gradient with the shifted
    input (dW[co, ci, ky, kx] = sum_p dY[p, co] X[p + (ky - 1, kx - 1), ci])."""
    x_nhwc = ops.nchw_to_nhwc(x_nchw.contiguous())
    cin = x_nhwc.shape[-1]
    dw = torch.empty(cout, cin, 3, 3, device=x_nchw.device)
    for ky in range(3):
        for kx in range(3):
            xs = ops.shift_map(x_nhwc, ky - 1, kx - 1).view(-1, cin)
            dw[:, :, ky, kx] = _wgrad(g_rows, xs)
    return dw, ops.col_sum(g_rows)


def encoder_backward(enc, img_feats, pts_feats, img_metas, pts_metas, d_img, d_pts_conv, d_pts):
    """Backward of DeepInteractionEncoder.forward (base model, hidden width 128, BatchNorm in eval mode = the folded
    weights of the forward; reference deepinteraction_encoder.py:8-85).  img_feats (B*V, Ci, h, w), pts_feats
    (B, Cp, Y, X): the module's NCHW inputs on the GPU; pts_metas with pillars; d_img [B*V, h, w, C], d_pts_conv / d_pts
    [B, Y, X, C]: gradients of the three outputs (pixel-major; None = zero).
    -> dict(d_img_feats [B*V, h, w, Ci], d_pts_feats [B, Y, X, Cp] (pixel-major), layers = per encoder layer the folded
    parameter gradients: i2p (dM1, dc1, dM2, dc2), p_iml / p2i / i_iml (lcab_backward dicts), p_fuse / i_fuse (dW [C, 3C], db)).
    shared_conv = dict(img / pts -> (dW [C, Cin, 3, 3], db)).  The forward is re-run eagerly with its intermediates kept."""
    with _precise():
        return _encoder_backward(enc, img_feats, pts_feats, img_metas, pts_metas, d_img, d_pts_conv, d_pts)


def _encoder_backward(enc, img_feats, pts_feats, img_metas, pts_metas, d_img, d_pts_conv, d_pts):
    from . import mmri
    pk = enc.pack()
    dev = img_feats.device
    C = enc.hidden_channel
    BV, Ci, h, w = img_feats.shape
    B, Cp, Y, X = pts_feats.shape
    V = BV // B
    pm = enc._canon_pts_metas(pts_metas, dev)
    pm['pts'] = [p.to(dev) for p in pts_metas['pts']]
    g = mmri.Geometry(img_metas, pm, (h, w), (Y, X), dev)
    g.wait()
    # ---- forward with saved intermediates
    img = ops.conv3x3(img_feats.contiguous(), *pk['shared_conv_img'], cout=C, x_nhwc=False)
    pts = ops.conv3x3(pts_feats.contiguous(), *pk['shared_conv_pts'], cout=C, x_nhwc=False)
    saved = []
    for lp in pk['layers']:
        img_r, pts_r = img.view(-1, C), pts.view(-1, C)
        i2p = enc.i2p(lp, pts, img, pm, g)
        p2p = mmri.lcab_forward(lp['p_iml'], pts_r, pts_r, B, Y, X)
        new_pts = ops.linear([i2p.view(-1, C), p2p, pts_r], *lp['p_fuse']).view(B, Y, X, C)
        warped = ops.bev_sample(pts, g.grid, V)
        p2i = mmri.lcab_forward(lp['p2i'], img_r, warped.view(-1, C), BV, h, w)
        i2i = mmri.lcab_forward(lp['i_iml'], img_r, img_r, BV, h, w)
        new_img = ops.linear([p2i, i2i, img_r], *lp['i_fuse']).view(BV, h, w, C)
        saved.append(dict(img=img, pts=pts, i2p=i2p, p2p=p2p, warped=warped, p2i=p2i, i2i=i2i))
        img, pts = new_img, new_pts
    # ---- backward
    one = torch.ones(1, device=dev)
    add = lambda a, b: b if a is None else (a if b is None else ops.axpy(a.contiguous(), b.contiguous(), one))
    zeros_i = lambda: torch.zeros(BV * h * w, C, device=dev)
    zeros_p = lambda: torch.zeros(B * Y * X, C, device=dev)
    gi = d_img.reshape(-1, C).contiguous() if d_img is not None else zeros_i()
    gp = d_pts.reshape(-1, C).contiguous() if d_pts is not None else zeros_p()
    layer_grads = []
    for lp, sv in zip(reversed(pk['layers']), reversed(saved)):
        img_r, pts_r = sv['img'].view(-1, C), sv['pts'].view(-1, C)
        lg = {}
        # fuse convolutions: new = Wf [a | b | c] + bf
        wi, wp = lp['i_fuse'][0], lp['p_fuse'][0]
        di3 = ops.linear([gi], _t_weight(wi, dev))                     # [M_i, 3C] = d p2i | d i2i | d img (direct)
        dp3 = ops.linear([gp], _t_weight(wp, dev))                     # [M_p, 3C] = d i2p | d p2p | d pts (direct)
        lg['i_fuse'] = (torch.cat([_wgrad(gi, sv['p2i']), _wgrad(gi, sv['i2i']), _wgrad(gi, img_r.contiguous())], 1), ops.col_sum(gi))
        lg['p_fuse'] = (torch.cat([_wgrad(gp, sv['i2p'].view(-1, C)), _wgrad(gp, sv['p2p']), _wgrad(gp, pts_r.contiguous())], 1),
                        ops.col_sum(gp))
        d_p2i, d_i2i, d_img_dir = (di3[:, k * C:(k + 1) * C].contiguous() for k in range(3))
        d_i2p, d_p2p, d_pts_dir = (dp3[:, k * C:(k + 1) * C].contiguous() for k in range(3))
        # image side
        r_ii = lcab_backward(lp['i_iml'], img_r, img_r, BV, h, w, d_i2i)
        r_pi = lcab_backward(lp['p2i'], img_r, sv['warped'].view(-1, C), BV, h, w, d_p2i)
        r_ip = i2p_backward(lp['i2p'], sv['pts'], sv['img'], pm, g.proj, V, g.in_hw, d_i2p.view(B, Y, X, C))
        r_pp = lcab_backward(lp['p_iml'], pts_r, pts_r, B, Y, X, d_p2p)
        new_gi = add(add(add(d_img_dir, r_ii['d_target']), r_pi['d_target']), r_ip['d_img'].view(-1, C))
        d_bev = ops.bev_sample_bwd(r_pi['d_source'].view(BV, h, w, C).contiguous(), g.grid, V, (B, Y, X, C))
        new_gp = add(add(add(d_pts_dir, r_pp['d_target']), r_ip['d_pts'].view(-1, C)), d_bev.view(-1, C))
        lg.update(i_iml={k: v for k, v in r_ii.items() if not k.startswith('d_')},
                  p2i={k: v for k, v in r_pi.items() if not k.startswith('d_')},
                  p_iml={k: v for k, v in r_pp.items() if not k.startswith('d_')},
                  i2p=(r_ip['dM1'], r_ip['dc1'], r_ip['dM2'], r_ip['dc2']))
        layer_grads.append(lg)
        gi, gp = new_gi, new_gp
    layer_grads.reverse()
    if d_pts_conv is not None:
        gp = add(gp, d_pts_conv.reshape(-1, C).contiguous())
    # shared 3x3 convolutions: input gradients = convolution of the output gradient with the transposed, flipped kernels
    wti = _conv3x3_transposed(pk['shared_conv_img'][0], Ci, dev)
    wtp = _conv3x3_transposed(pk['shared_conv_pts'][0], Cp, dev)
    d_img_feats = ops.conv3x3(gi.view(BV, h, w, C), wti, None, cout=Ci, x_nhwc=True)
    d_pts_feats = ops.conv3x3(gp.view(B, Y, X, C), wtp, None, cout=Cp, x_nhwc=True)

    shared = dict(img=conv3x3_wgrad(img_feats, gi, C), pts=conv3x3_wgrad(pts_feats, gp, C))
    return dict(d_img_feats=d_img_feats, d_pts_feats=d_pts_feats, layers=layer_grads, shared_conv=shared)


class LCABFunction(torch.autograd.Function):
    """autograd wrapper: out = LCAB(target, source) with the inference kernels, input gradients through lcab_backward.
    (Parameter gradients are returned by lcab_backward for the caller's optimiser on the folded weights.)"""

    @staticmethod
    def forward(ctx, pk, target, source, N, H, W):
        from .mmri import lcab_forward
        ctx.pk, ctx.dims, ctx.same = pk, (N, H, W), target is source
        ctx.save_for_backward(target, source)
        return lcab_forward(pk, target, source, N, H, W)

    @staticmethod
    def backward(ctx, grad_out):
        target, source = ctx.saved_tensors
        r = lcab_backward(ctx.pk, target, target if ctx.same else source, *ctx.dims, grad_out)
        return None, r['d_target'], r['d_source'], None, None, None
