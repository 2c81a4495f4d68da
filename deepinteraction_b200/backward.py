"""Backward of LocalContextAttentionBlock, of the encoder and of the decoder's query x BEV transformer layer on libdi_b200 (SURVEY.md 8(b) `di_lcab_backward`, the training side of the
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
    if splits == 1:
        return ops.linear([dyt], xt)
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


# ---- decoder: TransformerDecoderLayer (query x BEV) ---------------------------------------------------------------------
def _dec_bw_pack(dec, pk):
    """Transposed weights of the layer's dX products and the constants of fold.decoder_layer_unfold, built once per pack."""
    if '_bw' in pk:
        return pk['_bw']
    layer = dec.decoder[0]
    dev = pk['bce'].device
    C = dec.hidden_channel
    T = lambda w: fold.Weight(fold._d(w).reshape(w.shape[0], -1).t().contiguous(), dev)
    s = float(C // dec.num_heads) ** -0.5
    w_in = fold._d(layer.self_attn.in_proj_weight).clone()
    w_in[:C] *= s
    w_x = fold._d(layer.multihead_attn.in_proj_weight).clone()
    w_x[:C] *= s
    Td = lambda w: fold.Weight(w.t().contiguous(), dev)
    pk['_bw'] = dict(ffn2=T(layer.linear2.weight), ffn1=T(layer.linear1.weight), cross_out=T(layer.multihead_attn.out_proj.weight),
                     self_out=T(layer.self_attn.out_proj.weight), cross_q=Td(w_x[:C]), kv=Td(w_x[C:]), self_in=Td(w_in),
                     spe2=T(layer.self_posembed.position_embedding_head[3].weight),
                     cpe2=T(layer.cross_posembed.position_embedding_head[3].weight),
                     unfold=fold.decoder_layer_unfold_consts(layer, dec.num_heads, dev), one=torch.ones(1, device=dev))
    return pk['_bw']


def decoder_layer_backward(dec, query, query_pos, bev, grad_out):
    """Backward of the decoder's TransformerDecoderLayer (reference models/utils/decoder_utils.py:35-113, 116-495; the call
    self.decoder[0](query_feat, lidar_feat_flatten, query_pos, bev_pos) of deepinteraction_decoder.py), shared by the base
    and the ++ decoder, with BatchNorm in eval mode (the folded weights of the forward) and dropout off.
    dec: DeepInteractionDecoder / DeepInteractionPlusPlusDecoder on the GPU; query [B*P, C] and query_pos [B*P, 2]: the rows
    the forward feeds the layer; bev [B, Y, X, C]: pts_conv (pixel-major); grad_out [B*P, C].
    -> dict(d_query [B*P, C], d_bev [B, Y, X, C] (through K and V), grads = {name: tensor} for the 30 parameters of
    dec.decoder[0], keyed and shaped as in its state_dict).  query_pos gets no gradient (a gather of the constant bev_pos).
    The layer is re-run eagerly with its intermediates kept; everything stays on the device, without host synchronisation
    after the first call of a pack."""
    with _precise():
        return _decoder_layer_backward(dec, query, query_pos, bev, grad_out)


def _decoder_layer_backward(dec, query, query_pos, bev, grad_out):
    pk = dec.pack()
    C, H = dec.hidden_channel, dec.num_heads
    B, Y, X, _ = bev.shape
    HW, M = Y * X, query.shape[0]
    P = M // B
    if H != 8 or C != 128 or P > 256 or P * B != M:
        raise NotImplementedError('decoder_layer_backward: the cross-attention gradient kernel takes 8 heads x 16 channels and '
                                  f'P <= 256 queries per sample (got heads={H}, C={C}, rows={M}, B={B})')
    bw = _dec_bw_pack(dec, pk)
    query, query_pos, bev = query.contiguous(), query_pos.contiguous(), bev.contiguous()
    sv = {}
    dec._layer(pk, query, query_pos, bev, B, P, saved=sv)
    add = lambda a, b: ops.axpy(a.contiguous(), b.contiguous(), bw['one'])
    R, F = {}, {}
    # norm3, FFN
    dz3, R['norm3.weight'], R['norm3.bias'] = ops.ln_bwd(grad_out.contiguous(), sv['z3'], pk['norm3'][0])
    R['linear2.weight'], R['linear2.bias'] = _wgrad(dz3, sv['f']), ops.col_sum(dz3)
    df = ops.relu_bwd(ops.linear([dz3], bw['ffn2']), sv['f'])
    R['linear1.weight'], R['linear1.bias'] = _wgrad(df, sv['q2']), ops.col_sum(df)
    dq2 = ops.linear([df], bw['ffn1'], res=dz3)
    # norm2, query x BEV cross attention
    dz2, R['norm2.weight'], R['norm2.bias'] = ops.ln_bwd(dq2, sv['z2'], pk['norm2'][0])
    R['multihead_attn.out_proj.weight'], R['multihead_attn.out_proj.bias'] = _wgrad(dz2, sv['a2']), ops.col_sum(dz2)
    da2 = ops.linear([dz2], bw['cross_out'])
    dqc, dkv = ops.xattn_bwd(sv['planes'], sv['a2'], sv['lse'], da2, B, P, HW, H)
    F['cross_q'] = (_wgrad(dqc, torch.cat([sv['q1'], sv['qpe']], 1)), ops.col_sum(dqc))
    F['cross_kv'] = (_wgrad(dkv, sv['kk']), ops.col_sum(dkv))
    tq = ops.linear([dqc], bw['cross_q'])               # the [Wq | Wq] pack: the same gradient for q1 and qpe
    d_bev = ops.linear([dkv], bw['kv'])                 # d kk [B*HW, C] = d bev
    # constant key positional embedding: d kpe = sum over the batch of d kk, back through its MLP over the grid positions
    dkpe = d_bev[:HW]
    for b in range(1, B):
        dkpe = add(dkpe, d_bev[b * HW:(b + 1) * HW])
    cpe = pk['cross_pe']
    dh = ops.relu_bwd(ops.linear([dkpe.contiguous()], bw['cpe2']), cpe['hidden'])
    F['cross_posembed'] = (_wgrad(dh, cpe['pos']), ops.col_sum(dh), _wgrad(dkpe.contiguous(), cpe['hidden']), ops.col_sum(dkpe))
    # norm1, self attention over the queries
    dz1, R['norm1.weight'], R['norm1.bias'] = ops.ln_bwd(add(dz2, tq), sv['z1'], pk['norm1'][0])
    R['self_attn.out_proj.weight'], R['self_attn.out_proj.bias'] = _wgrad(dz1, sv['a1']), ops.col_sum(dz1)
    da1 = ops.linear([dz1], bw['self_out'])
    qkv = sv['qkv']
    dqkv = ops.mha_small_bwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], da1, B, P, H)
    F['self_in'] = (_wgrad(dqkv, torch.cat([query, sv['qpe']], 1)), ops.col_sum(dqkv))
    ts = ops.linear([dqkv], bw['self_in'])              # the [W | W] pack: the same gradient for query and qpe
    d_query = add(dz1, ts)
    dqpe = add(tq, ts)
    # self positional MLP
    dhs = ops.relu_bwd(ops.linear([dqpe], bw['spe2']), sv['hs'])
    F['self_posembed'] = (_wgrad(dhs, query_pos), ops.col_sum(dhs), _wgrad(dqpe, sv['hs']), ops.col_sum(dqpe))
    R.update(fold.decoder_layer_unfold(bw['unfold'], F))
    return dict(d_query=d_query, d_bev=d_bev.view(B, Y, X, C), grads=R)


class DecoderLayerFunction(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = the decoder's TransformerDecoderLayer (the forward schedule's kernels, bit for bit);
    backward -> (d_query, d_bev) through decoder_layer_backward.  Parameter gradients are returned by decoder_layer_backward."""

    @staticmethod
    def forward(ctx, dec, query, query_pos, bev):
        ctx.dec = dec
        ctx.save_for_backward(query, query_pos, bev)
        with _precise():
            pk = dec.pack()
            B = bev.shape[0]
            return dec._layer(pk, query.contiguous(), query_pos.contiguous(), bev.contiguous(), B, query.shape[0] // B)

    @staticmethod
    def backward(ctx, grad_out):
        query, query_pos, bev = ctx.saved_tensors
        r = decoder_layer_backward(ctx.dec, query, query_pos, bev, grad_out)
        return None, r['d_query'], None, r['d_bev']


# ---- decoder: PointRCNNBlock (the BEV refinement block of the MMPI layers) -----------------------------------------------
def _rcnn_bw_pack(dec, bp, li):
    """Transposed weights of the block's dX products, built once per pack.  The DynamicConv generator's transpose
    [C, 2*128*128] stays a plain tensor: its dX product (K = 32768 over B*P rows) runs as a split-K FFMA product."""
    if '_bw' in bp:
        return bp['_bw']
    blk = dec.decode_head[li]
    g = lambda n: getattr(blk, n + blk.sfx)
    dev = bp['norm1'][0].device
    C = dec.hidden_channel
    T = lambda w: fold.Weight(fold._d(w).t().contiguous(), dev)
    s = float(C // dec.num_heads) ** -0.5
    mha, dyn = g('dyconv_pre_self_attn'), g('dyconv')
    w_in = fold._d(mha.in_proj_weight).clone()
    w_in[:C] *= s                                   # the q rows _pack_mha folds the head_dim^-0.5 into
    qscale = torch.cat([torch.full((C,), s, dtype=torch.float64), torch.ones(2 * C, dtype=torch.float64)])
    bp['_bw'] = dict(ffn2=T(g('linear2').weight), ffn1=T(g('linear1').weight), dout=T(dyn.out_layer.weight),
                     dyn=fold.dev(fold._d(dyn.dynamic_layer.weight).t(), dev), attn_out=T(mha.out_proj.weight),
                     attn_in=fold.Weight(w_in.t().contiguous(), dev), qscale=fold.dev(qscale, dev))
    return bp['_bw']


# the dX product of the DynamicConv generator: d q1 [B*P, C] = d params [B*P, 32768] W_dyn.  The tensor-core GEMM has no
# split-K, and at M ~ 200 - 400 rows and N = 128 it would run on 2 - 4 CTAs over the whole K; 64 splits of 512 give
# 128 - 256 CTAs of the FFMA kernel, reduced in a fixed order by di_rows_finish_f32 together with the residual gradient.
_DYN_SPLITS = 64


def _point_rcnn_block(dec, li, query, bev):
    """-> (block pack, B, P); NotImplementedError before any launch for what point_rcnn_backward does not cover."""
    bp = dec.pack()['blocks'][li]
    if bp['image'] or bp['v2']:
        raise NotImplementedError('point_rcnn_backward covers the V1 PointRCNNBlock only (decode_head[%d] is %s)'
                                  % (li, type(dec.decode_head[li]).__name__))
    C, M, B = dec.hidden_channel, query.shape[0], bev.shape[0]
    P = M // B
    if C != 128 or bev.shape[3] != C or query.shape[1] != C or P > 512 or P * B != M:
        raise NotImplementedError('point_rcnn_backward: C = 128 and P <= 512 queries per sample '
                                  f'(got C={query.shape[1]}, rows={M}, B={B})')
    return bp, B, P


def _bev_roi_params(dec):
    return dec._roi_params((0, 0))          # the image size enters the image-mode RoIs only


def point_rcnn_backward(dec, li, query, pred, bev, grad_out):
    """Backward of the base decoder's PointRCNNBlock (reference models/utils/decoder_utils.py:765-841; dec.decode_head[li],
    li = 1 or 3 in the base configuration), LayerNorms as they are, dropout off.
    dec: DeepInteractionDecoder on the GPU; query [B*P, C]: the rows the block reads; pred [B*P, NP]: the prediction rows its
    RoIs come from (di_rcnn_rois_f32, BEV mode); bev [B, Y, X, C]: new_pts (pixel-major); grad_out [B*P, C].
    -> dict(d_query [B*P, C], d_bev [B, Y, X, C] (through RoIAlign), grads = {name: tensor} for the 24 parameters of
    dec.decode_head[li], keyed and shaped as in its state_dict).  The RoIs are constants (the reference computes them
    from detached predictions), so pred gets no gradient.  The block is re-run eagerly with its intermediates kept;
    everything stays on the device, without host synchronisation after the first call of a pack."""
    bp, B, P = _point_rcnn_block(dec, li, query, bev)
    with _precise():
        return _point_rcnn_backward(dec, li, bp, query.contiguous(), pred.contiguous(), bev.contiguous(),
                                    grad_out.contiguous(), B, P)


def _point_rcnn_backward(dec, li, bp, query, pred, bev, grad_out, B, P):
    C, H = dec.hidden_channel, dec.num_heads
    _, Y, X, _ = bev.shape
    sv = {}
    dec._rcnn_block(bp, query, pred, bev, None, B, P, _bev_roi_params(dec), None, None, saved=sv)
    bw = _rcnn_bw_pack(dec, bp, li)
    R = {}
    # norm3, FFN (GELU)
    dz3, R['norm3_pts.weight'], R['norm3_pts.bias'] = ops.ln_bwd(grad_out, sv['z3'], bp['norm3'][0])
    R['linear2_pts.weight'], R['linear2_pts.bias'] = _wgrad(dz3, sv['f']), ops.col_sum(dz3)
    dh = ops.gelu_bwd(ops.linear([dz3], bw['ffn2']), sv['h'])
    R['linear1_pts.weight'], R['linear1_pts.bias'] = _wgrad(dh, sv['q2']), ops.col_sum(dh)
    dq2 = ops.linear([dh], bw['ffn1'], res=dz3)
    # norm2, DynamicConv: norm3 + ReLU, out_layer, the dynamic convolution, the parameter generator, RoIAlign
    dz2, R['norm2_pts.weight'], R['norm2_pts.bias'] = ops.ln_bwd(dq2, sv['z2'], bp['norm2'][0])
    D = 'dyconv_pts.'
    dzd3, R[D + 'norm3.weight'], R[D + 'norm3.bias'] = ops.ln_bwd(ops.relu_bwd(dz2, sv['t']), sv['zd3'], bp['dn3'][0])
    R[D + 'out_layer.weight'], R[D + 'out_layer.bias'] = _wgrad(dzd3, sv['flat']), ops.col_sum(dzd3)
    d_roi, d_params, d_norm = ops.dynconv_bwd(sv['roi'], sv['params'], *bp['dn1'], *bp['dn2'], ops.linear([dzd3], bw['dout']))
    dn = ops.col_sum(d_norm).view(4, C)
    R[D + 'norm1.weight'], R[D + 'norm1.bias'], R[D + 'norm2.weight'], R[D + 'norm2.bias'] = dn.unbind(0)
    R[D + 'dynamic_layer.weight'], R[D + 'dynamic_layer.bias'] = _wgrad(d_params, sv['q1']), ops.col_sum(d_params)
    dq1 = ops.rows_finish(ops.linear([d_params], bw['dyn'], splits=_DYN_SPLITS), res=dz2)
    d_bev = ops.roi_align_bwd(d_roi, sv['rois'], B, Y, X, 1.0)
    # norm1, self attention over the queries of a sample (BEV mode: one group, no masks)
    dz1, R['norm1_pts.weight'], R['norm1_pts.bias'] = ops.ln_bwd(dq1, sv['z1'], bp['norm1'][0])
    A = 'dyconv_pre_self_attn_pts.'
    R[A + 'out_proj.weight'], R[A + 'out_proj.bias'] = _wgrad(dz1, sv['a']), ops.col_sum(dz1)
    qkv = sv['qkv']
    dqkv = ops.mha_small_bwd(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ops.linear([dz1], bw['attn_out']), B, P, H)
    d_query = ops.linear([dqkv], bw['attn_in'], res=dz1)
    # dqkv is the gradient of the packed projection, whose q rows carry head_dim^-0.5
    R[A + 'in_proj_weight'] = _wgrad(dqkv, query) * bw['qscale'][:, None]
    R[A + 'in_proj_bias'] = ops.col_sum(dqkv) * bw['qscale']
    return dict(d_query=d_query, d_bev=d_bev, grads=R)


class PointRCNNFunction(torch.autograd.Function):
    """autograd wrapper: out [B*P, C] = dec.decode_head[li] (a V1 PointRCNNBlock) with the forward schedule's kernels, bit
    for bit; backward -> (d_query, d_bev) through point_rcnn_backward, no gradient for pred (the RoIs are constants).
    Parameter gradients are returned by point_rcnn_backward."""

    @staticmethod
    def forward(ctx, dec, li, query, pred, bev):
        bp, B, P = _point_rcnn_block(dec, li, query, bev)
        ctx.dec, ctx.li = dec, li
        ctx.save_for_backward(query, pred, bev)
        with _precise():
            return dec._rcnn_block(bp, query.contiguous(), pred.contiguous(), bev.contiguous(), None, B, P,
                                   _bev_roi_params(dec), None, None)[0]

    @staticmethod
    def backward(ctx, grad_out):
        query, pred, bev = ctx.saved_tensors
        r = point_rcnn_backward(ctx.dec, ctx.li, query, pred, bev, grad_out)
        return None, None, r['d_query'], None, r['d_bev']
